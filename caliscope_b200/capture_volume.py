"""Seam S2 (SURVEY.md 8b): a replacement for ``CaptureVolume.optimize`` and for the observation ->
world-point map that runs on every ``CaptureVolume`` construction, with the host preparation
vectorised (the reference's per-row Python loops cost ~30 s at 2 M observations and would otherwise
dwarf a GPU solve of a few milliseconds).

Mirrors /root/reference/src/caliscope/core/capture_volume.py:
  * ``fast_img_to_obj_map``  == ``_compute_img_to_obj_map`` (:119-139)
  * ``optimize``             == ``CaptureVolume.optimize``   (:322-444), same signature, same result type,
                                same errors (``CalibrationError`` iff ``strict`` and not converged).
  * ``reprojection_report``  == ``CaptureVolume.reprojection_report`` (:150-235): pixel errors from the engine,
                                per-camera / per-point RMSE by ``np.bincount`` instead of one boolean mask per key.
  * ``pose_uncertainty``     (no reference counterpart) per-camera position / orientation uncertainty at the current
                                state, from the arrays optimize() builds (DESIGN.md 4.6).

Everything except the solve itself is the reference's own classes (imported from ``caliscope`` at call
time); the solve goes to the CUDA engine through ``caliscope_b200.solver.solve_arrays``.
"""
from __future__ import annotations

import logging
from copy import deepcopy

import numpy as np
import pandas as pd

from . import solver
from .problem import blocks_to_arrays

logger = logging.getLogger(__name__)

_KEYS = ["sync_index", "object_id", "keypoint_id"]


def fast_img_to_obj_map(self) -> np.ndarray:
    """Row index into ``world_points.df`` for every image observation, -1 if unmatched.  Observations of
    static objects are looked up at ``STATIC_SYNC_INDEX`` (capture_volume.py:124-132).  A dict keeps the
    LAST row for a duplicated key; ``drop_duplicates(keep='last')`` reproduces that."""
    from caliscope.core.point_data import STATIC_SYNC_INDEX

    wdf = self.world_points.df
    # the reference maps to the frame's index LABELS (reset_index().rename(index -> world_idx), :121)
    world = wdf[_KEYS].reset_index(drop=True).assign(world_idx=np.asarray(wdf.index, dtype=np.int64))
    world = world.drop_duplicates(subset=_KEYS, keep="last")
    img = self.image_points.df[_KEYS].copy()
    static_ids = self.constraints.static_object_ids if self.constraints else frozenset()
    if static_ids:
        is_static = img["object_id"].astype(np.int64).isin([int(s) for s in static_ids]).to_numpy()
        img.loc[is_static, "sync_index"] = STATIC_SYNC_INDEX
    for c in _KEYS:
        img[c] = img[c].astype(np.int64)
        world[c] = world[c].astype(np.int64)
    merged = img.merge(world, on=_KEYS, how="left", sort=False)
    out = merged["world_idx"].fillna(-1).to_numpy().astype(np.int32)
    n_unmatched = int(np.sum(out == -1))
    if n_unmatched > 0:
        logger.info(f"{n_unmatched} of {len(out)} image observations have no world point")
    return out


def ba_arrays(self):
    """capture_volume.py:346-358 without the per-row ``posed_cam_id_to_index`` property calls."""
    cam_index = self.camera_array.posed_cam_id_to_index  # built once
    cam_ids = self.image_points.df["cam_id"].to_numpy()
    lut_keys = np.fromiter(cam_index.keys(), dtype=np.int64, count=len(cam_index))
    lut_vals = np.fromiter(cam_index.values(), dtype=np.int64, count=len(cam_index))
    order = np.argsort(lut_keys)
    lut_keys, lut_vals = lut_keys[order], lut_vals[order]
    pos = np.searchsorted(lut_keys, cam_ids)
    pos_c = np.clip(pos, 0, max(len(lut_keys) - 1, 0))
    posed = (lut_keys[pos_c] == cam_ids) if len(lut_keys) else np.zeros(len(cam_ids), bool)
    mask = (self.img_to_obj_map >= 0) & posed
    camera_indices = lut_vals[pos_c[mask]].astype(np.int16)
    image_coords = self.image_points.df[["img_loc_x", "img_loc_y"]].to_numpy(dtype=np.float64)[mask]
    return camera_indices, image_coords, self.img_to_obj_map[mask], mask


def _problem_arrays(self, use_constraints: bool, pixel_sigma: float, refine_intrinsics: bool):
    """The arrays optimize() hands to the solver (capture_volume.py:346-399): (parameterization, its camera array copy,
    cam_flags, cam_const, camera_indices, image_to_world_indices, image_coords, x0, constraints or None, f_median)."""
    from caliscope.core.bundle_parameterization import BundleParameterization

    constraints = None
    focal = [cam.matrix[0, 0] for cam in self.camera_array.posed_cameras.values() if cam.matrix is not None]
    f_median = float(np.median(focal)) if focal else float("nan")
    if use_constraints and self.constraints is not None:
        arrays = self._build_constraint_arrays()
        if arrays is not None:  # capture_volume.py:373-383
            groups_a, groups_b, distances, sigmas = arrays
            constraints = (groups_a, groups_b, distances, (pixel_sigma / f_median) / sigmas)
            logger.info(f"Adding {len(groups_a)} constraint rows (f_median={f_median:.0f}, pixel_sigma={pixel_sigma})")
    camera_indices, image_coords, image_to_world_indices, _ = ba_arrays(self)
    new_camera_array = deepcopy(self.camera_array)
    parameterization = BundleParameterization.from_camera_array(
        new_camera_array, n_points=len(self.world_points.points), refine_intrinsics=refine_intrinsics
    )
    x0 = parameterization.pack(new_camera_array, self.world_points.points)
    flags, const = blocks_to_arrays(parameterization.blocks)
    return (parameterization, new_camera_array, flags, const, camera_indices, image_to_world_indices, image_coords, x0,
            constraints, f_median)  # fmt: skip


def optimize(self, ftol: float = 1e-8, max_nfev: int | None = None, verbose: int = 0, strict: bool = True,
             use_constraints: bool = True, pixel_sigma: float = 1.0, *, refine_intrinsics: bool = False,
             loss: str = "linear", f_scale: float = 1.0):  # fmt: skip
    """Bundle adjustment via pixel-space residuals on the GPU (drop-in for CaptureVolume.optimize)."""
    from caliscope.core.capture_volume import _SCIPY_STATUS_REASONS, CaptureVolume, OptimizationStatus
    from caliscope.core.point_data import WorldPoints

    (parameterization, new_camera_array, flags, const, camera_indices, image_to_world_indices, image_coords, x0,
     constraints, _) = _problem_arrays(self, use_constraints, pixel_sigma, refine_intrinsics)  # fmt: skip
    logger.info(f"Beginning bundle adjustment on {len(image_coords)} observations")
    result = solver.solve_arrays(
        flags, const, parameterization.n_points, camera_indices, image_to_world_indices, image_coords, x0,
        use_bounds=True, constraints=constraints, ftol=ftol, max_nfev=max_nfev, loss=loss, f_scale=f_scale,
        verbose=verbose,
    )  # fmt: skip
    termination_reason = _SCIPY_STATUS_REASONS.get(result.status, f"unknown_{result.status}")
    converged = result.status in (1, 2, 3, 4)
    if strict and not converged:
        from caliscope.exceptions import CalibrationError

        raise CalibrationError(
            f"Bundle adjustment did not converge: {termination_reason}\n"
            f"Pass strict=False to suppress this error and inspect the result."
        )
    new_points_xyz = parameterization.unpack_into(new_camera_array, result.x)
    status = OptimizationStatus(
        converged=converged,
        termination_reason=termination_reason,
        iterations=int(result.nfev),
        final_cost=float(result.cost),
        bound_warnings=parameterization.bound_warnings(result.x),
    )
    new_world_df = self.world_points.df.copy()
    new_world_df[["x_coord", "y_coord", "z_coord"]] = new_points_xyz
    return CaptureVolume(
        camera_array=new_camera_array,
        image_points=self.image_points,
        world_points=WorldPoints(new_world_df),
        constraints=self.constraints,
        _optimization_status=status,
    )


def pose_uncertainty(self, *, refine_intrinsics: bool = False, use_constraints: bool = True, pixel_sigma: float = 1.0):
    """How well each posed camera is determined by this capture volume's observations, at its current state (normally
    the result of optimize()): {cam_id: uncertainty.PoseUncertainty, or None for a camera without observations}.
    Built from the same arrays as optimize(); the covariance is scaled for ``pixel_sigma`` px of image noise,
    s2 = (pixel_sigma / f_median)^2, and is relative to uncertainty.default_gauge (the first observed camera shows 0)."""
    from . import uncertainty
    from .problem import BAProblem

    (_, _, flags, const, camera_indices, image_to_world_indices, image_coords, x0, constraints,
     f_median) = _problem_arrays(self, use_constraints, pixel_sigma, refine_intrinsics)  # fmt: skip
    n_points = len(self.world_points.points)
    with BAProblem(flags, const, n_points, camera_indices, image_to_world_indices, image_coords,
                   constraints=constraints) as p:  # fmt: skip
        cov = p.covariance(x0, variance_factor=(pixel_sigma / f_median) ** 2, points=False)
        offsets = p.cam_offsets
    poses = uncertainty.camera_poses(x0, offsets, cov.cameras)
    return {cam_id: poses[i] for cam_id, i in self.camera_array.posed_cam_id_to_index.items()}


def _errors_px(camera_array, camera_indices, image_coords, world_coords) -> np.ndarray:
    """reprojection.py:35-72 on the engine (module-level so the host-logic tests can substitute it)."""
    from . import reprojection

    return reprojection.reprojection_errors(camera_array, camera_indices, image_coords, world_coords)


def reprojection_report(self):
    """Same ``ReprojectionReport`` as capture_volume.py:150-235 (pixel units, stored intrinsics)."""
    from caliscope.core.reprojection_report import ReprojectionReport

    camera_indices, image_coords, obj_indices, mask = ba_arrays(self)
    n_total = len(self.img_to_obj_map)
    n_matched = int(mask.sum())
    if n_matched == 0:
        raise ValueError("No matched observations for reprojection error calculation")
    df = self.image_points.df
    matched = df[mask]
    world_coords = self.world_points.points[obj_indices]
    errors_xy = _errors_px(self.camera_array, camera_indices, image_coords, world_coords)
    euclid = np.sqrt(np.sum(errors_xy**2, axis=1))
    raw_errors = pd.DataFrame(
        {
            "sync_index": matched["sync_index"].values,
            "cam_id": matched["cam_id"].values,
            "object_id": matched["object_id"].values,
            "keypoint_id": matched["keypoint_id"].values,
            "error_x": errors_xy[:, 0],
            "error_y": errors_xy[:, 1],
            "euclidean_error": euclid,
        }
    )
    sq = euclid**2
    overall_rmse = float(np.sqrt(np.mean(sq)))
    # per camera: camera_indices are positions in posed_cam_id_to_index
    cam_index = self.camera_array.posed_cam_id_to_index
    n_idx = (max(cam_index.values()) + 1) if cam_index else 0
    cnt = np.bincount(camera_indices.astype(np.int64), minlength=n_idx)
    tot = np.bincount(camera_indices.astype(np.int64), weights=sq, minlength=n_idx)
    by_camera = {}
    for cam_id in self.camera_array.posed_cameras.keys():
        i = cam_index[cam_id]
        by_camera[cam_id] = float(np.sqrt(tot[i] / cnt[i])) if cnt[i] > 0 else 0.0
    # per (object_id, keypoint_id)
    obj = matched["object_id"].to_numpy()
    kp = matched["keypoint_id"].to_numpy()
    pairs, inv = np.unique(np.stack([obj, kp], axis=1), axis=0, return_inverse=True)
    inv = np.asarray(inv).reshape(-1)
    pc = np.bincount(inv, minlength=len(pairs))
    pt = np.bincount(inv, weights=sq, minlength=len(pairs))
    by_point = {(o.item(), k.item()): float(np.sqrt(t / c)) for (o, k), t, c in zip(pairs, pt, pc)}
    # unmatched observations per camera (all cameras, capture_volume.py:213-218)
    all_cam = df["cam_id"].to_numpy()
    unmatched_by_camera = {}
    for cam_id in self.camera_array.cameras.keys():
        sel = all_cam == cam_id
        unmatched_by_camera[cam_id] = int(sel.sum() - (sel & mask).sum())
    n_unmatched = n_total - n_matched
    return ReprojectionReport(
        overall_rmse=overall_rmse,
        by_camera=by_camera,
        by_point=by_point,
        n_unmatched_observations=int(n_unmatched),
        unmatched_rate=n_unmatched / n_total if n_total > 0 else 0.0,
        unmatched_by_camera=unmatched_by_camera,
        raw_errors=raw_errors,
        n_observations_matched=int(n_matched),
        n_observations_total=int(n_total),
        n_cameras=len(self.camera_array.posed_cameras),
        n_points=len(self.world_points.points),
    )


# ---- filtering (capture_volume.py:607-753) -------------------------------------------------------------------
def _pack_columns(frames, cols):
    """One non-negative int64 per row of each frame, equal iff the ``cols`` tuples are equal (shared
    offsets/spans over all frames); ``None`` when the ranges do not fit 62 bits."""
    arrs = [[f[c].to_numpy().astype(np.int64) for c in cols] for f in frames]
    lo, span = [], []
    for j in range(len(cols)):
        vals = [a[j] for a in arrs if len(a[j])]
        if not vals:
            lo.append(0)
            span.append(1)
            continue
        mn = min(int(v.min()) for v in vals)
        mx = max(int(v.max()) for v in vals)
        lo.append(mn)
        span.append(mx - mn + 1)
    total = 1
    for s in span:
        total *= s
    if total >= 2**62:
        return None
    out = []
    for a in arrs:
        key = np.zeros(len(a[0]), dtype=np.int64)
        for j in range(len(cols)):
            key = key * span[j] + (a[j] - lo[j])
        out.append(key)
    return out


def filter_by_reprojection_thresholds(self, thresholds: dict, min_per_camera: int):
    """``CaptureVolume._filter_by_reprojection_thresholds`` (capture_volume.py:607-683) without the row-wise
    pandas work: keep mask by ``filtering.keep_mask`` (index-exact, tests/golden), kept image rows selected by
    position instead of a 4-key merge, orphaned world points pruned by packed-key membership.  Falls back to the
    reference implementation when image keys repeat (the merge would then multiply rows)."""
    from caliscope.core.capture_volume import CaptureVolume
    from caliscope.core.point_data import STATIC_SYNC_INDEX, ImagePoints, WorldPoints

    from .filtering import keep_mask

    img_df = self.image_points.df
    obs_keys = ["sync_index", "cam_id", "object_id", "keypoint_id"]
    if img_df.duplicated(subset=obs_keys).any():
        return _reference_filter(self, thresholds, min_per_camera)
    raw = self.reprojection_report.raw_errors
    _, _, _, mask = ba_arrays(self)  # raw_errors rows are image rows [mask], in order (capture_volume.py:157-170)
    cam_ids = raw["cam_id"].to_numpy()
    err = raw["euclidean_error"].to_numpy()
    uniq, inv = np.unique(cam_ids, return_inverse=True)
    thr = np.array([float(thresholds[int(c)]) if int(c) in thresholds else np.nan for c in uniq])
    inv = np.asarray(inv).reshape(-1)
    if len(err) == 0:
        keep = np.zeros(0, dtype=bool)
    elif min_per_camera >= 1:
        keep = keep_mask(err, inv, thr, int(min_per_camera))
    else:  # the private method does not validate; a floor below 1 never restores anything (:626-631)
        keep = err <= thr[inv]
    rows = np.flatnonzero(mask)[keep]
    filtered_img_df = img_df.iloc[rows].reset_index(drop=True)

    wdf = self.world_points.df
    pt_keys = ["sync_index", "object_id", "keypoint_id"]
    packed = _pack_columns([wdf, filtered_img_df], pt_keys)
    if packed is None:
        return _reference_filter(self, thresholds, min_per_camera)
    filtered_world_df = wdf[np.isin(packed[0], packed[1])].reset_index(drop=True)
    static_world_df = wdf[wdf["sync_index"] == STATIC_SYNC_INDEX]
    if not static_world_df.empty:
        ok = _pack_columns([static_world_df, filtered_img_df], ["object_id", "keypoint_id"])
        if ok is None:
            return _reference_filter(self, thresholds, min_per_camera)
        static_to_keep = static_world_df[np.isin(ok[0], ok[1])]
        if not static_to_keep.empty:
            filtered_world_df = pd.concat([filtered_world_df, static_to_keep], ignore_index=True)
    return CaptureVolume(
        camera_array=self.camera_array,
        image_points=ImagePoints(filtered_img_df),
        world_points=WorldPoints(filtered_world_df),
        constraints=self.constraints,
    )


def _reference_filter(self, thresholds, min_per_camera):
    from . import seam

    fn = seam._original_methods.get("_filter_by_reprojection_thresholds")
    if fn is None:
        from caliscope.core.capture_volume import CaptureVolume

        fn = CaptureVolume._filter_by_reprojection_thresholds
        if fn is filter_by_reprojection_thresholds:  # pragma: no cover - patched without the seam's bookkeeping
            raise RuntimeError("reference filter implementation is not reachable")
    return fn(self, thresholds, min_per_camera)


def filter_by_percentile_error(self, percentile: float, scope="per_camera", min_per_camera: int = 10):
    """``CaptureVolume.filter_by_percentile_error`` (capture_volume.py:709-753): the per-camera thresholds are
    ``np.percentile`` of each camera's errors, taken from one grouping pass instead of one boolean mask per camera."""
    if not (0 < percentile <= 100):
        raise ValueError(f"percentile must be between 0 and 100, got {percentile}")
    if min_per_camera < 1:
        raise ValueError(f"min_per_camera must be >= 1, got {min_per_camera}")
    raw = self.reprojection_report.raw_errors
    err = raw["euclidean_error"].to_numpy()
    keep_percentile = 100 - percentile
    posed = list(self.camera_array.posed_cameras.keys())
    if scope == "per_camera":
        cam_ids = raw["cam_id"].to_numpy()
        order = np.argsort(cam_ids, kind="stable")
        sorted_ids = cam_ids[order]
        thresholds = {}
        for cam_id in posed:
            b, e = np.searchsorted(sorted_ids, cam_id, "left"), np.searchsorted(sorted_ids, cam_id, "right")
            thresholds[cam_id] = float(np.percentile(err[order[b:e]], keep_percentile)) if e > b else float(np.inf)
    elif scope == "overall":
        g = float(np.percentile(err, keep_percentile))
        thresholds = {cam_id: g for cam_id in posed}
    else:
        raise ValueError(f"scope must be 'per_camera' or 'overall', got {scope}")
    return self._filter_by_reprojection_thresholds(thresholds, min_per_camera)
