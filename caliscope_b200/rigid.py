"""Robust pose of a rigid body seen by a calibrated rig: hypotheses from triangulated model points, refinement on every
camera's rows and a covariance with the rig's uncertainty, on the GPU (``cb_rigid_pose_robust``, DESIGN.md section
4.14)."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import _lib as L
from .triangulation import _calibrated_inputs, _ptr
from .uncertainty import PoseUncertainty, pose_from_body


@dataclass
class RigidPoses:
    """Per group in ascending key order.  pose = (r, t) with X_w = R(r) M + t for the model points M.  status: 0 ok,
    1 fewer than 4 rows, 2 not positive definite (pose is the winning hypothesis, cov NaN), 3 iteration limit, 4 a
    consensus row behind its camera at the solution, 5 no consensus (pose, cov, rmse NaN), 6 (gP3P only) ambiguous: a
    gP3P winner whose consensus rows hold fewer than four distinct markers, which can fit two poses exactly (pose and
    rmse of the refined winner, cov NaN)."""

    pose: np.ndarray  # (G, 6)
    cov: np.ndarray  # (G, 6, 6)
    rmse_px: np.ndarray  # (G,) over the consensus rows
    count: np.ndarray  # (G,) int32, every row of the group
    n_inliers: np.ndarray  # (G,) int32
    n_points: np.ndarray  # (G,) int32, model points with a triangulated hypothesis
    rep_row: np.ndarray  # (G,) int32
    status: np.ndarray  # (G,) int32
    inlier: np.ndarray  # (n_obs,) bool, caller order
    key: np.ndarray  # (G,) int64, the group's obs_key

    def uncertainty(self) -> list[PoseUncertainty | None]:
        """Position and orientation uncertainty of each group's pose (``uncertainty.pose_from_body``), None where the
        covariance is NaN."""
        return [None if not np.isfinite(c).all() else pose_from_body(p[:3], p[3:], c) for p, c in zip(self.pose, self.cov)]


@dataclass
class RigidStats:
    group_ms: float = 0.0
    points_ms: float = 0.0
    consensus_ms: float = 0.0
    refine_ms: float = 0.0
    cov_ms: float = 0.0
    total_ms: float = 0.0
    kernel_launches: int = 0
    n_groups: int = 0


def pose_rigid_robust(cam_flags, cam_const, cam_x, model_xyz, obs_cam, obs_key, obs_pt, obs_px, *, threshold_px: float,
                      min_inliers: int = 6, max_pairs: int = 16, max_samples: int = 64, prior=None,
                      pixel_sigma: float = 1.0, camera_cov=None, max_iter: int = 20, xtol: float = 1e-12,
                      gp3p_samples: int = 0, device: int = 0, stream: int = 0,
                      stats: RigidStats | None = None) -> RigidPoses:
    """Robust pose of a rigid body seen by several calibrated cameras at once (``cb_rigid_pose_robust``, DESIGN.md
    section 4.14).

    The cameras are ``BAProblem.cam_flags``, ``BAProblem.cam_const`` and ``x[:n_camera_params]``; ``camera_cov`` is
    ``Covariance.cameras`` at that solution (None: pixel noise only).  ``model_xyz`` (n_model, 3) is the body's marker
    layout in its own frame and ``obs_pt`` the model point of each row; rows with equal ``obs_key`` are one body at one
    moment (key = frame, or (body, frame) with the bodies on disjoint ranges of the model table), from any cameras.
    ``obs_px`` are raw pixels.  The observations may be host arrays or CUDA tensors on ``device`` (obs_cam and obs_pt
    int32, obs_key int64, obs_px float64 (n, 2)), read in place.

    Each model point with rows in a group is triangulated by view-pair consensus (``triangulate_robust``'s rule); Horn
    poses of up to ``max_samples`` triples of those points and the group's prior pose are scored by MSAC over all the
    group's rows, sum min(e^2, threshold_px^2) in raw pixels; the lowest score wins.  The rows within ``threshold_px``
    of the winner are the consensus set (fewer than ``min_inliers``: status 5), markers seen by one camera included; the
    pose is refined on them and ``cov = pixel_sigma^2 H^-1 + H^-1 G camera_cov G^T H^-1``.

    ``prior`` is ``(keys, poses)``: a pose (n, 6) per key, e.g. the previous frame's ``RigidPoses.key`` and ``pose``.
    Rows that are not finite are dropped, so a tracking loop can pass the last output unchanged.

    ``gp3p_samples`` (0: off, else 1..4096) poses groups with fewer than three triangulated markers, e.g. markers each
    seen by one camera, without a prior: up to that many triples of the group's rows from any cameras go through a
    generalized-camera three-point solver (gP3P), whose poses join the prior in the same consensus.  Groups with three
    or more triangulated markers give the same outputs, bit for bit, as with ``gp3p_samples=0``.  A group that gP3P
    poses from fewer than four distinct markers is status 6 (no covariance): with two triangulated markers and a third
    seen by one camera, two poses can fit every row."""
    if not (np.isfinite(threshold_px) and threshold_px > 0):
        raise ValueError(f"threshold_px must be finite and > 0, got {threshold_px}")
    if int(min_inliers) < 4:
        raise ValueError(f"min_inliers must be >= 4, got {min_inliers}")
    if int(max_pairs) < 1:
        raise ValueError(f"max_pairs must be >= 1, got {max_pairs}")
    if not 1 <= int(max_samples) <= 4096:
        raise ValueError(f"max_samples must be in 1..4096, got {max_samples}")
    if not 0 <= int(gp3p_samples) <= 4096:
        raise ValueError(f"gp3p_samples must be in 0..4096, got {gp3p_samples}")
    if not (np.isfinite(pixel_sigma) and pixel_sigma >= 0):
        raise ValueError(f"pixel_sigma must be finite and >= 0, got {pixel_sigma}")
    if int(max_iter) < 1:
        raise ValueError(f"max_iter must be >= 1, got {max_iter}")
    if not (np.isfinite(xtol) and xtol >= 0):
        raise ValueError(f"xtol must be finite and >= 0, got {xtol}")
    model = np.ascontiguousarray(model_xyz, dtype=np.float64)
    if model.ndim != 2 or model.shape[1] != 3 or len(model) == 0:
        raise ValueError(f"model_xyz must be (n_model, 3) with n_model >= 1, got {model.shape}")
    pkey, ppose = np.zeros(0, np.int64), np.zeros((0, 6))
    if prior is not None:
        pkey = np.asarray(prior[0], dtype=np.int64).ravel()
        ppose = np.asarray(prior[1], dtype=np.float64).reshape(-1, 6)
        if len(pkey) != len(ppose):
            raise ValueError(f"prior keys and poses differ in length: {len(pkey)} and {len(ppose)}")
        keep = np.isfinite(ppose).all(axis=1)
        pkey, ppose = pkey[keep], ppose[keep]
        if len(pkey) > 1 and not (np.diff(pkey) > 0).all():
            raise ValueError("prior keys must be strictly ascending")
    pkey, ppose = np.ascontiguousarray(pkey), np.ascontiguousarray(ppose)
    lib = L.load()
    nc, flags, const, cx, ccov, n, on_dev, (cam_p, key_p, px_p, pt_p), _keep = _calibrated_inputs(
        cam_flags, cam_const, cam_x, camera_cov, obs_cam, obs_key, obs_px, device, obs_pt=obs_pt)
    m = max(n, 1)
    pose, cov, rmse = np.empty((m, 6)), np.empty((m, 6, 6)), np.empty(m)
    count, nin, npts, rep, status = (np.empty(m, np.int32) for _ in range(5))
    inlier = np.zeros(m, np.uint8)
    ng = C.c_int32(0)
    st = L.RigidStats()
    L.check(
        lib.cb_rigid_pose_robust_gp3p(nc, _ptr(flags), _ptr(const), _ptr(cx), None if ccov is None else _ptr(ccov),
                                      len(model), _ptr(model), n, cam_p, key_p, pt_p, px_p, 1 if on_dev else 0,
                                      float(threshold_px), int(min_inliers), int(max_pairs), int(max_samples),
                                      int(gp3p_samples), len(pkey), _ptr(pkey), _ptr(ppose), float(pixel_sigma),
                                      int(max_iter), float(xtol), n, C.byref(ng), _ptr(pose), _ptr(cov), _ptr(rmse),
                                      _ptr(count), _ptr(nin), _ptr(npts), _ptr(rep), _ptr(status), _ptr(inlier),
                                      C.byref(st), int(device), C.c_void_p(stream)),
        "pose_rigid_robust",
    )  # fmt: skip
    g = ng.value
    if stats is not None:
        stats.group_ms, stats.points_ms, stats.consensus_ms = st.group_ms, st.points_ms, st.consensus_ms
        stats.refine_ms, stats.cov_ms, stats.total_ms = st.refine_ms, st.cov_ms, st.total_ms
        stats.kernel_launches, stats.n_groups = st.kernel_launches, g
    rep = rep[:g]
    if on_dev:
        import torch

        keys = obs_key[torch.from_numpy(rep.astype(np.int64)).to(obs_key.device)].cpu().numpy()
    else:
        keys = _keep[1][rep]
    return RigidPoses(pose=pose[:g], cov=cov[:g], rmse_px=rmse[:g], count=count[:g], n_inliers=nin[:g],
                      n_points=npts[:g], rep_row=rep, status=status[:g], inlier=inlier[:n].astype(bool),
                      key=np.asarray(keys, np.int64))  # fmt: skip


@dataclass
class RigidModel:
    """Refined marker layouts (``refine_rigid_model``).  Per body: status 0 ok, 1 not solved (no used frame, or a marker
    without a row in a used frame: layout and poses are the start, cov NaN), 2 not positive definite at the start or
    at the solution (layout and poses are the start, cov and rmse NaN), 3 iteration limit, 4 a row behind its camera at
    the solution.  Per frame in ascending key order; a frame's status is 1 when it takes no part (no finite start pose,
    fewer than 4 rows or fewer than 3 markers) or its body has status 1, else its body's status."""

    model: np.ndarray  # (n_model, 3)
    cov: list  # per body, (3K, 3K)
    status: np.ndarray  # (n_bodies,) int32
    iterations: np.ndarray
    rmse_px: np.ndarray  # over the body's rows in used frames
    n_frames: np.ndarray  # used frames
    n_rows: np.ndarray
    key: np.ndarray  # (F,) int64
    pose: np.ndarray  # (F, 6) refined (r, t), X_w = R(r) M + t
    frame_rmse_px: np.ndarray
    count: np.ndarray  # every row of the key
    frame_status: np.ndarray


@dataclass
class RigidModelStats:
    group_ms: float = 0.0
    solve_ms: float = 0.0
    cov_ms: float = 0.0
    total_ms: float = 0.0
    kernel_launches: int = 0


def refine_rigid_model(cam_flags, cam_const, cam_x, model_xyz, obs_cam, obs_key, obs_pt, obs_px, start, *, bodies=None,
                       pixel_sigma: float = 1.0, camera_cov=None, max_iter: int = 100, xtol: float = 1e-12,
                       device: int = 0, stream: int = 0, stats: RigidModelStats | None = None) -> RigidModel:  # fmt: skip
    """Refine rigid-body marker layouts from tracked frames (``cb_rigid_model_refine``, DESIGN.md section 4.15).

    The rig, ``model_xyz`` (the start layout, e.g. a nominal CAD layout) and the observations follow
    ``pose_rigid_robust``; pass the rows to use, typically those ``RigidPoses.inlier`` marks.  ``start`` is
    ``(keys, poses)``, one start pose per key (e.g. ``RigidPoses.key`` and ``pose``); non-finite rows are dropped.
    ``bodies`` is ``body_start`` (n_bodies + 1, from 0 to n_model): model points body_start[b] .. body_start[b+1]-1 are
    body b, with 3 to 32 markers; None is one body.  Every frame's rows must belong to one body, and every
    ``obs_key`` must be non-negative (``EngineError`` otherwise).

    One Levenberg-Marquardt per body over its layout and every frame pose, the frames eliminated, with the gauge held
    by inner constraints on the start layout: the result keeps the start's centroid and has no net rotation against
    it.  ``cov`` is ``pixel_sigma^2 P + P G camera_cov G^T P`` with ``P = N (N^T S N)^-1 N^T``: the pixel term, which
    shrinks as frames are added, and the rig's term through the Schur-reduced cross term G to the camera parameters,
    which does not.  ``camera_cov`` is ``Covariance.cameras`` of the rig (None: the pixel term alone)."""
    model = np.ascontiguousarray(model_xyz, dtype=np.float64)
    if model.ndim != 2 or model.shape[1] != 3 or len(model) == 0:
        raise ValueError(f"model_xyz must be (n_model, 3) with n_model >= 1, got {model.shape}")
    bs = np.ascontiguousarray([0, len(model)] if bodies is None else np.asarray(bodies).ravel(), dtype=np.int32)
    skey = np.asarray(start[0], dtype=np.int64).ravel()
    spose = np.asarray(start[1], dtype=np.float64).reshape(-1, 6)
    if len(skey) != len(spose):
        raise ValueError(f"start keys and poses differ in length: {len(skey)} and {len(spose)}")
    keep = np.isfinite(spose).all(axis=1)
    skey, spose = np.ascontiguousarray(skey[keep]), np.ascontiguousarray(spose[keep])
    lib = L.load()
    nc, flags, const, cx, ccov, n, on_dev, (cam_p, key_p, px_p, pt_p), _keep = _calibrated_inputs(
        cam_flags, cam_const, cam_x, camera_cov, obs_cam, obs_key, obs_px, device, obs_pt=obs_pt)
    nb = len(bs) - 1
    m = max(n, 1)
    sizes = 3 * np.diff(bs.astype(np.int64)) if nb > 0 else np.zeros(0, np.int64)
    out_model = np.empty_like(model)
    cov = np.empty(max(int((sizes * sizes).sum()), 1))
    status, iters, nfr, nrows = (np.zeros(max(nb, 1), np.int32) for _ in range(4))
    rmse = np.empty(max(nb, 1))
    key, pose, frmse = np.empty(m, np.int64), np.empty((m, 6)), np.empty(m)
    count, fstatus = np.empty(m, np.int32), np.empty(m, np.int32)
    nf = C.c_int32(0)
    st = L.RigidModelStats()
    L.check(
        lib.cb_rigid_model_refine(nc, _ptr(flags), _ptr(const), _ptr(cx), None if ccov is None else _ptr(ccov), len(model), _ptr(model), nb, _ptr(bs), n,
                                  cam_p, key_p, pt_p, px_p, 1 if on_dev else 0, len(skey), _ptr(skey), _ptr(spose),
                                  float(pixel_sigma), int(max_iter), float(xtol), n, C.byref(nf), _ptr(out_model),
                                  _ptr(cov), _ptr(status), _ptr(iters), _ptr(rmse), _ptr(nfr), _ptr(nrows), _ptr(key),
                                  _ptr(pose), _ptr(frmse), _ptr(count), _ptr(fstatus), C.byref(st), int(device),
                                  C.c_void_p(stream)),
        "refine_rigid_model",
    )  # fmt: skip
    if stats is not None:
        stats.group_ms, stats.solve_ms, stats.cov_ms = st.group_ms, st.solve_ms, st.cov_ms
        stats.total_ms, stats.kernel_launches = st.total_ms, st.kernel_launches
    offs = np.concatenate([[0], np.cumsum(sizes * sizes)])
    covs = [cov[offs[b] : offs[b + 1]].reshape(sizes[b], sizes[b]).copy() for b in range(nb)]
    f = nf.value
    return RigidModel(model=out_model, cov=covs, status=status[:nb], iterations=iters[:nb], rmse_px=rmse[:nb],
                      n_frames=nfr[:nb], n_rows=nrows[:nb], key=key[:f], pose=pose[:f], frame_rmse_px=frmse[:f],
                      count=count[:f], frame_status=fstatus[:f])  # fmt: skip
