"""Robust resection with calibrated cameras: the pose of a camera from 2-D detections of points whose 3-D positions are
known, chosen by P3P consensus, refined to the reprojection optimum and given a covariance on the GPU
(``cb_resect_robust``, DESIGN.md section 4.9)."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import _lib as L
from .triangulation import _calibrated_inputs, _ptr
from .uncertainty import PoseUncertainty, pose_from_extrinsics


@dataclass
class ResectedPoses:
    """Per group in ascending key order.  pose = (r, t) in x's camera layout, ready to be written into x at the camera's
    offset.  status: 0 ok, 1 fewer than 4 rows, 2 not positive definite (pose is the winning hypothesis, cov NaN),
    3 iteration limit, 4 a consensus row behind the camera at the solution, 5 no consensus (pose, cov, rmse NaN),
    6 rows from more than one camera."""

    cam: np.ndarray  # (G,) int32 camera slot
    pose: np.ndarray  # (G, 6)
    cov: np.ndarray  # (G, 6, 6)
    rmse_px: np.ndarray  # (G,) over the consensus rows
    count: np.ndarray  # (G,) int32, every row of the group
    n_inliers: np.ndarray  # (G,) int32
    rep_row: np.ndarray  # (G,) int32
    status: np.ndarray  # (G,) int32
    inlier: np.ndarray  # (n_obs,) bool, caller order

    def uncertainty(self) -> list[PoseUncertainty | None]:
        """Position and orientation uncertainty of each group's pose (``uncertainty.pose_from_extrinsics``), None where
        the covariance is NaN."""
        out: list[PoseUncertainty | None] = []
        for p, c in zip(self.pose, self.cov):
            out.append(None if not np.isfinite(c).all() else pose_from_extrinsics(p[:3], p[3:], c))
        return out


@dataclass
class ResectStats:
    group_ms: float = 0.0
    consensus_ms: float = 0.0
    refine_ms: float = 0.0
    cov_ms: float = 0.0
    total_ms: float = 0.0
    kernel_launches: int = 0
    n_groups: int = 0


def resect_robust(cam_flags, cam_const, cam_x, pts_xyz, obs_cam, obs_key, obs_pt, obs_px, *, threshold_px: float,
                  min_inliers: int = 6, max_samples: int = 64, use_prior: bool = True, pixel_sigma: float = 1.0,
                  points_cov=None, max_iter: int = 20, xtol: float = 1e-12, device: int = 0, stream: int = 0,
                  stats: ResectStats | None = None) -> ResectedPoses:
    """Robust pose of a camera from detections of known points (``cb_resect_robust``, DESIGN.md section 4.9).

    The cameras are ``BAProblem.cam_flags``, ``BAProblem.cam_const`` and ``x[:n_camera_params]``; each camera's
    intrinsics stay fixed.  ``pts_xyz`` (n_pts, 3) are the known points and ``obs_pt`` the point of each row; rows with
    equal ``obs_key`` are one pose of one camera (key = camera, or (camera, frame)).  ``obs_px`` are raw pixels.  The
    observations may be host arrays or CUDA tensors on ``device`` (obs_cam and obs_pt int32, obs_key int64, obs_px
    float64 (n, 2)), read in place.

    Inside each group, the P3P poses of up to ``max_samples`` row triples (every triple, or a deterministic hashed subset)
    and, with ``use_prior``, the camera's pose in ``cam_x`` are scored by MSAC over all rows, sum
    min(e^2, threshold_px^2) in raw pixels; the lowest score wins.  The rows within ``threshold_px`` of the winner are the
    consensus set (fewer than ``min_inliers``: status 5); the pose is refined on them alone and
    ``cov = pixel_sigma^2 H^-1 + H^-1 M H^-1`` with M the points' term from ``points_cov`` (n_pts, 3, 3).  That term
    assumes the points are independent of each other and of this camera's observations: triangulate them without the
    resected camera's rows (``triangulation.triangulate_robust`` on the other cameras)."""
    if not (np.isfinite(threshold_px) and threshold_px > 0):
        raise ValueError(f"threshold_px must be finite and > 0, got {threshold_px}")
    if int(min_inliers) < 4:
        raise ValueError(f"min_inliers must be >= 4, got {min_inliers}")
    if not 1 <= int(max_samples) <= 4096:
        raise ValueError(f"max_samples must be in 1..4096, got {max_samples}")
    if not (np.isfinite(pixel_sigma) and pixel_sigma >= 0):
        raise ValueError(f"pixel_sigma must be finite and >= 0, got {pixel_sigma}")
    if int(max_iter) < 1:
        raise ValueError(f"max_iter must be >= 1, got {max_iter}")
    if not (np.isfinite(xtol) and xtol >= 0):
        raise ValueError(f"xtol must be finite and >= 0, got {xtol}")
    pts = np.ascontiguousarray(pts_xyz, dtype=np.float64)
    if pts.ndim != 2 or pts.shape[1] != 3:
        raise ValueError(f"pts_xyz must be (n_pts, 3), got {pts.shape}")
    pcov = None
    if points_cov is not None:
        pcov = np.ascontiguousarray(points_cov, dtype=np.float64)
        if pcov.shape != (len(pts), 3, 3):
            raise ValueError(f"points_cov must be ({len(pts)}, 3, 3), got {pcov.shape}")
    lib = L.load()
    nc, flags, const, cx, _, n, on_dev, (cam_p, key_p, px_p, pt_p), _keep = _calibrated_inputs(
        cam_flags, cam_const, cam_x, None, obs_cam, obs_key, obs_px, device, obs_pt=obs_pt)
    m = max(n, 1)
    pose, cov, rmse = np.empty((m, 6)), np.empty((m, 6, 6)), np.empty(m)
    cam, count, nin, rep, status = (np.empty(m, np.int32) for _ in range(5))
    inlier = np.zeros(m, np.uint8)
    ng = C.c_int32(0)
    st = L.ResectStats()
    L.check(
        lib.cb_resect_robust(nc, _ptr(flags), _ptr(const), _ptr(cx), len(pts), _ptr(pts),
                             None if pcov is None else _ptr(pcov), n, cam_p, key_p, pt_p, px_p, 1 if on_dev else 0,
                             float(threshold_px), int(min_inliers), int(max_samples), 1 if use_prior else 0,
                             float(pixel_sigma), int(max_iter), float(xtol), n, C.byref(ng), _ptr(cam), _ptr(pose),
                             _ptr(cov), _ptr(rmse), _ptr(count), _ptr(nin), _ptr(rep), _ptr(status), _ptr(inlier),
                             C.byref(st), int(device), C.c_void_p(stream)),
        "resect_robust",
    )  # fmt: skip
    g = ng.value
    if stats is not None:
        stats.group_ms, stats.consensus_ms, stats.refine_ms = st.group_ms, st.consensus_ms, st.refine_ms
        stats.cov_ms, stats.total_ms, stats.kernel_launches, stats.n_groups = st.cov_ms, st.total_ms, st.kernel_launches, g
    return ResectedPoses(cam=cam[:g], pose=pose[:g], cov=cov[:g], rmse_px=rmse[:g], count=count[:g], n_inliers=nin[:g],
                         rep_row=rep[:g], status=status[:g], inlier=inlier[:n].astype(bool))  # fmt: skip
