"""GPU-backed mirrors of the step in front of bundle adjustment (SURVEY.md §8(f) rank 3).

``triangulate_image_points`` has the signature, return value and output ORDER of the reference
function (``caliscope/core/point_data.py:122-229``); ``undistort_points`` is
``CameraData.undistort_points`` (``caliscope/cameras/camera_array.py:135-174``) at array level, for
the observations of every camera in one launch.  Both go through the C ABI
(``cb_triangulate_dlt`` / ``cb_undistort_points``); there is no CPU path.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import _lib as L


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _empty():
    return (np.array([], dtype=np.int64), np.array([], dtype=np.int64), np.array([], dtype=np.int64), np.zeros((0, 3)))


def pack_keys(sync_indices, object_ids, keypoint_ids) -> np.ndarray:
    """Non-negative int64 key, order-isomorphic to the reference's lexsort on
    (sync_index, object_id, keypoint_id) (point_data.py:143).  Falls back to dense ranks when the
    value ranges do not fit 63 bits."""
    cols = [np.asarray(c).astype(np.int64, copy=False) for c in (sync_indices, object_ids, keypoint_ids)]
    lo = [int(c.min()) for c in cols]
    span = [int(c.max()) - l + 1 for c, l in zip(cols, lo)]
    if span[0] * span[1] * span[2] >= 2**62:
        cols = [np.unique(c, return_inverse=True)[1].astype(np.int64) for c in cols]
        lo = [0, 0, 0]
        span = [int(c.max()) + 1 for c in cols]
        if span[0] * span[1] * span[2] >= 2**62:
            raise ValueError("(sync_index, object_id, keypoint_id) key space exceeds 62 bits")
    return ((cols[0] - lo[0]) * span[1] + (cols[1] - lo[1])) * span[2] + (cols[2] - lo[2])


@dataclass
class TriangulationStats:
    group_ms: float = 0.0
    dlt_ms: float = 0.0
    total_ms: float = 0.0
    kernel_launches: int = 0
    n_groups: int = 0


def _camera_tables(matrices, distortions, fisheye):
    """(fisheye int32[n], k float64[n,5] = fx fy cx cy skew, dist float64[n,12]) for the C ABI."""
    mats = np.asarray(matrices, dtype=np.float64).reshape(-1, 3, 3)
    nc = len(mats)
    fish = np.ascontiguousarray(np.broadcast_to(np.asarray(fisheye, dtype=np.int32).ravel(), (nc,)))
    k = np.ascontiguousarray(np.stack([mats[:, 0, 0], mats[:, 1, 1], mats[:, 0, 2], mats[:, 1, 2], mats[:, 0, 1]], axis=1))
    dist = np.zeros((nc, 12))
    dl = [distortions] if nc == 1 and np.ndim(distortions[0]) == 0 else list(distortions)
    if len(dl) != nc:
        raise ValueError("one distortion vector per camera")
    for i, d in enumerate(dl):
        d = np.asarray(d, dtype=np.float64).ravel()
        if fish[i] and len(d) != 4:
            raise ValueError(f"fisheye camera needs 4 distortion coefficients, got {len(d)}")
        if len(d) > 12 and np.any(d[12:] != 0):
            raise ValueError("tilted-sensor coefficients (tau_x, tau_y) are not supported")
        dist[i, : min(len(d), 12)] = d[:12]
    return fish, k, dist


def triangulate_groups(proj: np.ndarray, obs_cam: np.ndarray, obs_key: np.ndarray, obs_xy: np.ndarray, *, device: int = 0,
                       stream: int = 0, stats: TriangulationStats | None = None, undistort=None):
    """Array-level call: ``proj`` (n_cams,3,4), camera ROW per observation, packed key, xy.
    ``undistort=(matrices, distortions, fisheye)``: ``obs_xy`` are raw pixels and are undistorted on
    the device first (``cb_undistort_triangulate``; nothing returns to the host in between).
    Returns per group in ascending key order: xyz (G,3), count (G,), rep_row (G,), camset_sig (G,2)."""
    lib = L.load()
    proj = np.ascontiguousarray(proj, dtype=np.float64).reshape(-1, 3, 4)
    cam = np.ascontiguousarray(obs_cam, dtype=np.int32)
    key = np.ascontiguousarray(obs_key, dtype=np.int64)
    xy = np.ascontiguousarray(obs_xy, dtype=np.float64).reshape(-1, 2)
    n = len(cam)
    if len(key) != n or len(xy) != n:
        raise ValueError("obs_cam, obs_key and obs_xy must have one row per observation")
    xyz = np.empty((max(n, 1), 3))
    count = np.empty(max(n, 1), dtype=np.int32)
    rep = np.empty(max(n, 1), dtype=np.int32)
    sig = np.empty((max(n, 1), 2), dtype=np.uint64)
    ng = C.c_int32(0)
    st = L.TriStats()
    tail = (n, _ptr(cam), _ptr(key), _ptr(xy), 0, n, C.byref(ng), _ptr(xyz), _ptr(count), _ptr(rep), _ptr(sig),
            C.byref(st), int(device), C.c_void_p(stream))  # fmt: skip
    if undistort is None:
        L.check(lib.cb_triangulate_dlt(len(proj), _ptr(proj), *tail), "triangulate_dlt")
    else:
        fish, k, dist = _camera_tables(*undistort)
        if len(fish) != len(proj):
            raise ValueError("one camera model per projection matrix")
        L.check(lib.cb_undistort_triangulate(len(proj), _ptr(fish), _ptr(k), _ptr(dist), _ptr(proj), *tail),
                "undistort_triangulate")  # fmt: skip
    g = ng.value
    if stats is not None:
        stats.group_ms, stats.dlt_ms, stats.total_ms = st.group_ms, st.dlt_ms, st.total_ms
        stats.kernel_launches, stats.n_groups = st.kernel_launches, g
    return xyz[:g], count[:g], rep[:g], sig[:g]


def triangulate_image_points(
    projection_matrices: dict,
    sync_indices: np.ndarray,
    camera_ids: np.ndarray,
    object_ids: np.ndarray,
    keypoint_ids: np.ndarray,
    img_xy: np.ndarray,
    *,
    device: int = 0,
    stats: TriangulationStats | None = None,
):
    """Drop-in for ``caliscope.core.point_data.triangulate_image_points`` (point_data.py:122-229):
    returns ``(sync_indices, object_ids, keypoint_ids, xyz)`` for every (sync, object, keypoint)
    seen by >= 2 rows, camera sets in order of first appearance, keys ascending inside a set."""
    sync_indices = np.asarray(sync_indices)
    camera_ids = np.asarray(camera_ids)
    object_ids = np.asarray(object_ids)
    keypoint_ids = np.asarray(keypoint_ids)
    n_obs = len(keypoint_ids)
    if n_obs < 2:
        return _empty()
    _, proj, row = _camera_rows(projection_matrices, camera_ids)
    key = pack_keys(sync_indices, object_ids, keypoint_ids)
    xyz, count, rep, sig = triangulate_groups(proj, row, key, img_xy, device=device, stats=stats)
    return _reference_order(sync_indices, object_ids, keypoint_ids, xyz, count, rep, sig)


def _camera_rows(projection_matrices: dict, camera_ids: np.ndarray):
    """Sorted camera ids, their stacked [R|t] and the row of every observation's camera (KeyError like the
    reference's dict lookup when a camera has no projection matrix)."""
    cam_ids = np.array(sorted(projection_matrices), dtype=np.int64)
    proj = np.stack([np.asarray(projection_matrices[int(c)], dtype=np.float64)[:3, :4] for c in cam_ids])
    row = np.searchsorted(cam_ids, camera_ids)
    if np.any(row >= len(cam_ids)) or np.any(cam_ids[np.minimum(row, len(cam_ids) - 1)] != camera_ids):
        missing = np.setdiff1d(camera_ids, cam_ids)
        raise KeyError(int(missing[0]))
    return cam_ids, proj, row


def _reference_order(sync_indices, object_ids, keypoint_ids, xyz, count, rep, sig):
    """Groups seen by >= 2 rows, camera sets in order of first appearance over the key-sorted groups (the
    reference's dict insertion order, point_data.py:164-172), keys ascending inside a set; the group size is
    part of a set's identity next to its 128-bit camera-multiset signature."""
    keep = np.flatnonzero(count >= 2)
    if len(keep) == 0:
        return _empty()
    ident = np.empty(len(keep), dtype=[("a", np.uint64), ("b", np.uint64), ("n", np.int64)])
    ident["a"], ident["b"], ident["n"] = sig[keep, 0], sig[keep, 1], count[keep]
    _, first, inverse = np.unique(ident, return_index=True, return_inverse=True)
    order = np.argsort(first[np.asarray(inverse).reshape(-1)], kind="stable")
    sel = keep[order]
    r = rep[sel]
    return (
        np.asarray(sync_indices)[r].astype(np.int64),
        np.asarray(object_ids)[r].astype(np.int64),
        np.asarray(keypoint_ids)[r].astype(np.int64),
        xyz[sel].copy(),
    )


def triangulate_pixels(projection_matrices: dict, camera_models: dict, sync_indices, camera_ids, object_ids, keypoint_ids,
                       img_px, *, device: int = 0, stats: TriangulationStats | None = None):
    """``_undistort_batch`` + ``triangulate_image_points`` (point_data.py:236-252, 122-229) in one device call:
    ``img_px`` are raw pixels, ``camera_models[cam_id] = (matrix 3x3, distortions, fisheye)``; the undistorted
    coordinates never come back to the host (``cb_undistort_triangulate``)."""
    sync_indices = np.asarray(sync_indices)
    camera_ids = np.asarray(camera_ids)
    object_ids = np.asarray(object_ids)
    keypoint_ids = np.asarray(keypoint_ids)
    if len(keypoint_ids) < 2:
        return _empty()
    cam_ids, proj, row = _camera_rows(projection_matrices, camera_ids)
    mats = np.stack([np.asarray(camera_models[int(c)][0], dtype=np.float64) for c in cam_ids])
    dists = [np.asarray(camera_models[int(c)][1], dtype=np.float64).ravel() for c in cam_ids]
    fish = np.array([1 if camera_models[int(c)][2] else 0 for c in cam_ids], dtype=np.int32)
    key = pack_keys(sync_indices, object_ids, keypoint_ids)
    xyz, count, rep, sig = triangulate_groups(proj, row, key, img_px, device=device, stats=stats, undistort=(mats, dists, fish))
    return _reference_order(sync_indices, object_ids, keypoint_ids, xyz, count, rep, sig)


def triangulate(self, camera_array, static_object_ids: frozenset = frozenset()):
    """Drop-in for ``ImagePoints.triangulate`` (point_data.py:416-559): same ``WorldPoints`` (rows, order, columns,
    frame times, static objects at ``STATIC_SYNC_INDEX``), with undistortion and DLT in one device call per part
    instead of a per-camera OpenCV loop followed by per-camera-set SVD batches."""
    import pandas as pd
    from caliscope.core.point_data import STATIC_SYNC_INDEX, WORLD_POINT_COLUMNS, WorldPoints

    def empty():
        return WorldPoints(pd.DataFrame(columns=list(WORLD_POINT_COLUMNS.keys())))

    xy_df = self.df
    if xy_df.empty:
        return empty()
    cam_ids_in_data = xy_df["cam_id"].unique()
    posed_cam_ids = list(camera_array.posed_cam_id_to_index.keys())
    valid_cam_ids = [c for c in cam_ids_in_data if c in posed_cam_ids]
    if not valid_cam_ids:
        return empty()
    pm = camera_array.normalized_projection_matrices
    # the reference undistorts every camera that has rows, posed or not, and fails on a missing calibration
    # (camera_array.py:152-153) before it filters to posed cameras
    for cam_id, camera in camera_array.cameras.items():
        if (camera.matrix is None or camera.distortions is None) and bool((xy_df["cam_id"] == cam_id).any()):
            raise ValueError(f"Camera {cam_id} lacks intrinsic calibration; cannot undistort points.")
    known = xy_df["cam_id"].isin(list(camera_array.cameras.keys()))
    valid_data = xy_df[known & xy_df["cam_id"].isin(valid_cam_ids)]
    if valid_data.empty:
        return empty()
    models = {int(c): (camera_array.cameras[c].matrix, camera_array.cameras[c].distortions, camera_array.cameras[c].fisheye)
              for c in pm}  # fmt: skip
    frame_times = xy_df.groupby("sync_index")["frame_time"].mean()
    if static_object_ids:
        static_mask = valid_data["object_id"].isin(static_object_ids)
        mobile_data, static_data = valid_data[~static_mask], valid_data[static_mask]
    else:
        mobile_data, static_data = valid_data, valid_data.iloc[0:0]

    def part(data, sync_arr):
        return triangulate_pixels(pm, models, sync_arr, data["cam_id"].to_numpy(), data["object_id"].to_numpy(),
                                  data["keypoint_id"].to_numpy(), data[["img_loc_x", "img_loc_y"]].to_numpy(np.float64))  # fmt: skip

    parts = []
    if not mobile_data.empty:
        s, o, k, xyz = part(mobile_data, mobile_data["sync_index"].to_numpy())
        if len(k) > 0:
            parts.append(pd.DataFrame({"sync_index": s, "object_id": o, "keypoint_id": k, "x_coord": xyz[:, 0],
                                       "y_coord": xyz[:, 1], "z_coord": xyz[:, 2],
                                       "frame_time": frame_times.reindex(s).to_numpy()}))  # fmt: skip
    if not static_data.empty:
        s, o, k, xyz = part(static_data, np.full(len(static_data), STATIC_SYNC_INDEX, dtype=np.int64))
        if len(k) > 0:
            parts.append(pd.DataFrame({"sync_index": s, "object_id": o, "keypoint_id": k, "x_coord": xyz[:, 0],
                                       "y_coord": xyz[:, 1], "z_coord": xyz[:, 2],
                                       "frame_time": np.full(len(k), np.nan)}))  # fmt: skip
    if not parts:
        return empty()
    return WorldPoints(pd.concat(parts, ignore_index=True))


@dataclass
class RefinedPoints:
    """``triangulate_refined``: per group in ascending key order.  status: 0 ok, 1 fewer than 2 rows, 2 not positive
    definite (xyz is the DLT point, cov NaN), 3 iteration limit, 4 behind a camera."""

    xyz: np.ndarray  # (G, 3)
    cov: np.ndarray  # (G, 3, 3)
    rmse_px: np.ndarray  # (G,)
    count: np.ndarray  # (G,) int32
    rep_row: np.ndarray  # (G,) int32
    status: np.ndarray  # (G,) int32


@dataclass
class RefineStats:
    group_ms: float = 0.0
    dlt_ms: float = 0.0
    refine_ms: float = 0.0
    cov_ms: float = 0.0
    total_ms: float = 0.0
    kernel_launches: int = 0
    n_groups: int = 0


def _check_device_tri_obs(obs_cam, obs_key, obs_px, device: int) -> int:
    """Device-resident observations, read in place (no conversion): CUDA tensors on ``device``, contiguous; obs_cam
    int32 (n,), obs_key int64 (n,), obs_px float64 (n, 2).  Returns n."""
    dtypes = {"obs_cam": "torch.int32", "obs_key": "torch.int64", "obs_px": "torch.float64"}
    arrays = {"obs_cam": obs_cam, "obs_key": obs_key, "obs_px": obs_px}
    for name, a in arrays.items():
        dev = getattr(a, "device", None)
        if getattr(dev, "type", None) != "cuda" or dev.index != device:
            raise ValueError(f"{name} must be a CUDA tensor on cuda:{device}, got device {dev}")
        if str(getattr(a, "dtype", None)) != dtypes[name]:
            raise ValueError(f"{name} must have dtype {dtypes[name]}, got {getattr(a, 'dtype', None)}")
        if not a.is_contiguous():
            raise ValueError(f"{name} must be contiguous")
    n = int(obs_cam.shape[0])
    if tuple(obs_cam.shape) != (n,) or tuple(obs_key.shape) != (n,):
        raise ValueError(f"obs_cam and obs_key must be 1-D of the same length, got {tuple(obs_cam.shape)}, "
                         f"{tuple(obs_key.shape)}")  # fmt: skip
    if tuple(obs_px.shape) != (n, 2):
        raise ValueError(f"obs_px must have shape ({n}, 2), got {tuple(obs_px.shape)}")
    return n


def _calibrated_inputs(cam_flags, cam_const, cam_x, camera_cov, obs_cam, obs_key, obs_px, device: int, obs_pt=None):
    """Cameras in the BA layout and observations (host arrays or CUDA tensors read in place) of the calibrated
    triangulation calls as the C ABI takes them: (n_cams, flags, const, cam_x, camera_cov or None, n, on_device,
    observation pointers, host arrays the pointers refer to).  With ``obs_pt`` (the point of each row, int32; resection)
    its pointer follows the other three."""
    flags = np.ascontiguousarray(cam_flags, dtype=np.int32).ravel()
    nc = len(flags)
    const = np.ascontiguousarray(cam_const, dtype=np.float64).reshape(nc, 9)
    ncp = int(np.where(flags & L.CB_CAM_FREE_INTRINSICS, 9, 6).sum())
    cx = np.ascontiguousarray(cam_x, dtype=np.float64).ravel()
    if len(cx) < ncp:
        raise ValueError(f"cam_x must hold the {ncp} camera parameters, got {len(cx)}")
    cx = np.ascontiguousarray(cx[:ncp])
    ccov = None
    if camera_cov is not None:
        ccov = np.ascontiguousarray(camera_cov, dtype=np.float64)
        if ccov.shape != (ncp, ncp):
            raise ValueError(f"camera_cov must be ({ncp}, {ncp}), got {ccov.shape}")
    on_dev = hasattr(obs_px, "data_ptr")
    if on_dev:
        n = _check_device_tri_obs(obs_cam, obs_key, obs_px, device)
        ptrs = tuple(C.c_void_p(t.data_ptr()) for t in (obs_cam, obs_key, obs_px))
        if obs_pt is not None:
            dev = getattr(obs_pt, "device", None)
            if getattr(dev, "type", None) != "cuda" or dev.index != device:
                raise ValueError(f"obs_pt must be a CUDA tensor on cuda:{device}, got device {dev}")
            if str(getattr(obs_pt, "dtype", None)) != "torch.int32" or not obs_pt.is_contiguous():
                raise ValueError(f"obs_pt must be a contiguous torch.int32 tensor, got {getattr(obs_pt, 'dtype', None)}")
            if tuple(obs_pt.shape) != (n,):
                raise ValueError(f"obs_pt must have shape ({n},), got {tuple(obs_pt.shape)}")
            ptrs += (C.c_void_p(obs_pt.data_ptr()),)
        return nc, flags, const, cx, ccov, n, True, ptrs, ()
    cam = np.ascontiguousarray(obs_cam, dtype=np.int32)
    key = np.ascontiguousarray(obs_key, dtype=np.int64)
    px = np.ascontiguousarray(obs_px, dtype=np.float64).reshape(-1, 2)
    n = len(cam)
    if len(key) != n or len(px) != n:
        raise ValueError("obs_cam, obs_key and obs_px must have one row per observation")
    keep = (cam, key, px)
    if obs_pt is not None:
        pt = np.ascontiguousarray(obs_pt, dtype=np.int32)
        if pt.shape != (n,):
            raise ValueError(f"obs_pt must have one entry per observation, got shape {pt.shape}")
        keep += (pt,)
    return nc, flags, const, cx, ccov, n, False, tuple(_ptr(a) for a in keep), keep


def triangulate_refined(cam_flags, cam_const, cam_x, obs_cam, obs_key, obs_px, *, pixel_sigma: float = 1.0,
                        camera_cov=None, max_iter: int = 20, xtol: float = 1e-12, device: int = 0, stream: int = 0,
                        stats: RefineStats | None = None) -> RefinedPoints:
    """Maximum-likelihood triangulation with calibrated cameras and a covariance per point (``cb_triangulate_refine``,
    DESIGN.md section 4.7).

    The cameras are ``BAProblem.cam_flags``, ``BAProblem.cam_const`` and ``x[:n_camera_params]`` of a solution;
    ``camera_cov`` is ``Covariance.cameras`` at that solution (None: pixel noise only).  Observations with equal
    ``obs_key`` are one point; ``obs_px`` are raw pixels.  They may be host arrays or CUDA tensors on ``device``
    (obs_cam int32, obs_key int64, obs_px float64 (n, 2)), read in place.  Each point starts at the DLT point and is
    refined to the least-squares reprojection optimum; ``cov = pixel_sigma^2 H^-1 + H^-1 G camera_cov G^T H^-1``.  This
    assumes the observations are independent of those the calibration used (for a point that was itself in the
    bundle adjustment, use ``Covariance.points``), and the camera term is relative to ``camera_cov``'s gauge."""
    lib = L.load()
    nc, flags, const, cx, ccov, n, on_dev, (cam_p, key_p, px_p), _keep = _calibrated_inputs(
        cam_flags, cam_const, cam_x, camera_cov, obs_cam, obs_key, obs_px, device)
    m = max(n, 1)
    xyz, cov, rmse = np.empty((m, 3)), np.empty((m, 3, 3)), np.empty(m)
    count, rep, status = np.empty(m, np.int32), np.empty(m, np.int32), np.empty(m, np.int32)
    ng = C.c_int32(0)
    st = L.TriRefineStats()
    L.check(
        lib.cb_triangulate_refine(nc, _ptr(flags), _ptr(const), _ptr(cx), None if ccov is None else _ptr(ccov), n, cam_p,
                                  key_p, px_p, 1 if on_dev else 0, float(pixel_sigma), int(max_iter), float(xtol), n,
                                  C.byref(ng), _ptr(xyz), _ptr(cov), _ptr(rmse), _ptr(count), _ptr(rep), _ptr(status),
                                  C.byref(st), int(device), C.c_void_p(stream)),
        "triangulate_refine",
    )  # fmt: skip
    g = ng.value
    if stats is not None:
        stats.group_ms, stats.dlt_ms, stats.refine_ms, stats.cov_ms = st.group_ms, st.dlt_ms, st.refine_ms, st.cov_ms
        stats.total_ms, stats.kernel_launches, stats.n_groups = st.total_ms, st.kernel_launches, g
    return RefinedPoints(xyz=xyz[:g], cov=cov[:g], rmse_px=rmse[:g], count=count[:g], rep_row=rep[:g],
                         status=status[:g])  # fmt: skip


@dataclass
class RobustPoints(RefinedPoints):
    """``triangulate_robust``: the ``RefinedPoints`` fields over each group's consensus rows (``count`` is still every
    row of the group), plus n_inliers per group and the caller-order inlier mask.  status 5: no consensus (xyz, cov and
    rmse NaN, n_inliers 0)."""

    n_inliers: np.ndarray = None  # (G,) int32
    inlier: np.ndarray = None  # (n_obs,) bool, caller order


@dataclass
class RobustStats:
    group_ms: float = 0.0
    consensus_ms: float = 0.0
    refine_ms: float = 0.0
    cov_ms: float = 0.0
    total_ms: float = 0.0
    kernel_launches: int = 0
    n_groups: int = 0


def triangulate_robust(cam_flags, cam_const, cam_x, obs_cam, obs_key, obs_px, *, threshold_px: float,
                       min_inliers: int = 2, max_pairs: int = 64, pixel_sigma: float = 1.0, camera_cov=None,
                       max_iter: int = 20, xtol: float = 1e-12, device: int = 0, stream: int = 0,
                       stats: RobustStats | None = None) -> RobustPoints:
    """``triangulate_refined`` on each point's agreeing views (``cb_triangulate_robust``, DESIGN.md section 4.8).

    Inputs as ``triangulate_refined``.  Inside each group the DLT points of up to ``max_pairs`` view pairs (every pair,
    or an evenly spaced deterministic subset of the lexicographically ranked pairs) are scored by MSAC over all rows of
    the group, sum min(e^2, threshold_px^2) in raw pixels; the lowest score wins (the lowest rank on a tie).  The rows
    within ``threshold_px`` of the winner, in front of their camera, are the consensus set; the point is refined on them
    alone from the winner and gets its covariance from them.  Fewer than ``min_inliers`` consensus rows, or no valid
    pair (every row from one camera, for example), gives status 5.  There is one consensus round (rows are not
    re-classified at the refined point), and in a two-view group an error along the epipolar line cannot be seen."""
    if not (np.isfinite(threshold_px) and threshold_px > 0):
        raise ValueError(f"threshold_px must be finite and > 0, got {threshold_px}")
    if int(min_inliers) < 2:
        raise ValueError(f"min_inliers must be >= 2, got {min_inliers}")
    if int(max_pairs) < 1:
        raise ValueError(f"max_pairs must be >= 1, got {max_pairs}")
    lib = L.load()
    nc, flags, const, cx, ccov, n, on_dev, (cam_p, key_p, px_p), _keep = _calibrated_inputs(
        cam_flags, cam_const, cam_x, camera_cov, obs_cam, obs_key, obs_px, device)
    m = max(n, 1)
    xyz, cov, rmse = np.empty((m, 3)), np.empty((m, 3, 3)), np.empty(m)
    count, nin, rep, status = (np.empty(m, np.int32) for _ in range(4))
    inlier = np.zeros(m, np.uint8)
    ng = C.c_int32(0)
    st = L.TriRobustStats()
    L.check(
        lib.cb_triangulate_robust(nc, _ptr(flags), _ptr(const), _ptr(cx), None if ccov is None else _ptr(ccov), n, cam_p,
                                  key_p, px_p, 1 if on_dev else 0, float(threshold_px), int(min_inliers), int(max_pairs),
                                  float(pixel_sigma), int(max_iter), float(xtol), n, C.byref(ng), _ptr(xyz), _ptr(cov),
                                  _ptr(rmse), _ptr(count), _ptr(nin), _ptr(rep), _ptr(status), _ptr(inlier), C.byref(st),
                                  int(device), C.c_void_p(stream)),
        "triangulate_robust",
    )  # fmt: skip
    g = ng.value
    if stats is not None:
        stats.group_ms, stats.consensus_ms, stats.refine_ms = st.group_ms, st.consensus_ms, st.refine_ms
        stats.cov_ms, stats.total_ms, stats.kernel_launches, stats.n_groups = st.cov_ms, st.total_ms, st.kernel_launches, g
    return RobustPoints(xyz=xyz[:g], cov=cov[:g], rmse_px=rmse[:g], count=count[:g], rep_row=rep[:g], status=status[:g],
                        n_inliers=nin[:g], inlier=inlier[:n].astype(bool))  # fmt: skip


def undistort_points(points, cam_rows, matrices, distortions, fisheye, *, output: str = "normalized", device: int = 0,
                     stream: int = 0) -> np.ndarray:
    """``CameraData.undistort_points`` for many cameras at once.

    points (N,2); cam_rows (N,) row into ``matrices`` (n_cams,3,3) / ``distortions`` (list of
    coefficient vectors, <= 12 each) / ``fisheye`` (n_cams,) — or ``None`` with one camera.
    Returns (N,2) float32, like the reference (values produced in double, rounded once)."""
    if output not in ("normalized", "pixels"):
        raise ValueError("output must be 'normalized' or 'pixels'")
    lib = L.load()
    fish, k, dist = _camera_tables(matrices, distortions, fisheye)
    nc = len(fish)
    pts = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 2)
    rows = None if cam_rows is None else np.ascontiguousarray(cam_rows, dtype=np.int32)
    if rows is not None and len(rows) != len(pts):
        raise ValueError("one camera row per point")
    out = np.empty_like(pts)
    L.check(
        lib.cb_undistort_points(nc, _ptr(fish), _ptr(k), _ptr(dist), len(pts), None if rows is None else _ptr(rows),
                                _ptr(pts), 0, 1 if output == "pixels" else 0, _ptr(out), int(device), C.c_void_p(stream)),
        "undistort_points",
    )  # fmt: skip
    return out.astype(np.float32)
