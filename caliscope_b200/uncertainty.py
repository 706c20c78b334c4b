"""Gauge choice and camera-pose uncertainty from ``BAProblem.covariance`` (DESIGN.md section 4.6).

Reprojection residuals are invariant under a similarity transform of the world and the cameras, so J^T J has a 7-dim
null space (6 with rigid-distance constraint rows, which fix the scale).  A covariance needs a gauge: parameters held
fixed to remove that null space.  Every number derived here is relative to the gauge: the reference camera's pose is
exactly known by construction and shows zero.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np


def rodrigues(r: np.ndarray) -> np.ndarray:
    """Rotation vector (3,) -> matrix (cv2.Rodrigues convention)."""
    r = np.asarray(r, dtype=np.float64)
    th = float(np.linalg.norm(r))
    K = _skew(r)
    if th < 1e-12:
        return np.eye(3) + K
    return np.eye(3) + np.sin(th) / th * K + (1 - np.cos(th)) / th**2 * (K @ K)


def _skew(v) -> np.ndarray:
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def so3_right_jacobian(r: np.ndarray) -> np.ndarray:
    """Jr(r) with R(r + d) = R(r) exp([Jr(r) d]x) to first order, i.e. d(R(r) X)/dr = -R [X]x Jr(r)."""
    r = np.asarray(r, dtype=np.float64)
    th2 = float(r @ r)
    th = np.sqrt(th2)
    if th < 1e-4:
        B = 0.5 - th2 / 24.0 + th2 * th2 / 720.0
        C = 1.0 / 6.0 - th2 / 120.0 + th2 * th2 / 5040.0
    else:
        B = (1 - np.cos(th)) / th2
        C = (th - np.sin(th)) / th**3
    K = _skew(r)
    return np.eye(3) - B * K + C * (K @ K)


def camera_centers(x, cam_offsets) -> np.ndarray:
    """World-frame camera centres C = -R^T t, (n_cams, 3)."""
    out = np.empty((len(cam_offsets) - 1, 3))
    for c in range(len(out)):
        o = int(cam_offsets[c])
        out[c] = -rodrigues(x[o : o + 3]).T @ x[o + 3 : o + 6]
    return out


def default_gauge(x, cam_offsets, observed, has_constraints: bool) -> np.ndarray:
    """The usual gauge: the 6 extrinsics of the first observed camera c0 and, without constraint rows, one translation
    component of the observed camera c1 farthest from c0.  Scaling the world about C_c0 moves t_c1 along
    R_c1 (C_c0 - C_c1), so fixing its largest component k fixes the scale to first order.  Indices into x."""
    x = np.asarray(x, dtype=np.float64)
    cams = np.nonzero(np.asarray(observed, bool))[0]
    if len(cams) == 0:
        raise ValueError("no camera has observations")
    c0 = int(cams[0])
    o0 = int(cam_offsets[c0])
    fixed = list(range(o0, o0 + 6))
    if not has_constraints:
        if len(cams) < 2:
            raise ValueError("the scale gauge needs a second observed camera")
        C = camera_centers(x, cam_offsets)
        c1 = int(cams[1:][np.argmax(np.linalg.norm(C[cams[1:]] - C[c0], axis=1))])
        o1 = int(cam_offsets[c1])
        d = rodrigues(x[o1 : o1 + 3]) @ (C[c0] - C[c1])
        fixed.append(o1 + 3 + int(np.argmax(np.abs(d))))
    return np.asarray(fixed, np.int32)


@dataclass
class PoseUncertainty:
    """A pose's uncertainty, in one of two conventions.  A camera's (``pose_from_extrinsics``, X_cam = R X_w + t,
    relative to the gauge): position_cov is the world-frame covariance of the centre C = -R^T t.  A rigid body's
    (``pose_from_body``, X_w = R M + t): position_cov is the world-frame covariance of the body origin t.  In both,
    orientation_cov is the covariance of the rotation error on the right (R_true = R exp([e]x)), rad^2."""

    position_cov: np.ndarray
    orientation_cov: np.ndarray

    @property
    def position_std(self) -> float:
        """RMS position error (square root of the trace), in the world's length unit."""
        return float(np.sqrt(max(np.trace(self.position_cov), 0.0)))

    @property
    def orientation_std_deg(self) -> float:
        """RMS rotation angle (square root of the trace), degrees."""
        return float(np.degrees(np.sqrt(max(np.trace(self.orientation_cov), 0.0))))


def pose_from_extrinsics(rvec, tvec, cov6) -> PoseUncertainty:
    """First-order propagation of the 6x6 (rvec, tvec) covariance block of one camera:
    dC/dt = -R^T, dC/dr = -R^T [t]x Jr(-r) (R^T = R(-r)), and the body-frame rotation error e = Jr(r) dr."""
    r = np.asarray(rvec, dtype=np.float64)
    t = np.asarray(tvec, dtype=np.float64)
    Rt = rodrigues(r).T
    G = np.hstack([-Rt @ _skew(t) @ so3_right_jacobian(-r), -Rt])
    Jr = so3_right_jacobian(r)
    cov6 = np.asarray(cov6, dtype=np.float64)
    return PoseUncertainty(position_cov=G @ cov6 @ G.T, orientation_cov=Jr @ cov6[:3, :3] @ Jr.T)


def pose_from_body(rvec, tvec, cov6) -> PoseUncertainty:
    """First-order uncertainty of a rigid body's pose X_w = R(r) M + t from its 6x6 (r, t) covariance: the body origin
    is t, so position_cov = cov[3:, 3:]; the rotation error e = Jr(r) dr.  ``tvec`` is unused and kept for the
    signature of ``pose_from_extrinsics``."""
    del tvec
    Jr = so3_right_jacobian(np.asarray(rvec, dtype=np.float64))
    cov6 = np.asarray(cov6, dtype=np.float64)
    return PoseUncertainty(position_cov=cov6[3:, 3:].copy(), orientation_cov=Jr @ cov6[:3, :3] @ Jr.T)


def camera_poses(x, cam_offsets, cam_cov) -> list[PoseUncertainty | None]:
    """Per camera (caller order) the pose uncertainty from the camera block of a covariance; None for cameras whose
    block is NaN (no observations)."""
    out = []
    for c in range(len(cam_offsets) - 1):
        o = int(cam_offsets[c])
        blk = cam_cov[o : o + 6, o : o + 6]
        out.append(None if np.isnan(blk).any() else pose_from_extrinsics(x[o : o + 3], x[o + 3 : o + 6], blk))
    return out


def prior_information(cov, pixel_sigma: float, fx: float) -> np.ndarray:
    """Information matrix of a Gaussian prior (``BAProblem``'s ``camera_priors`` / ``point_priors``, DESIGN.md section
    4.13) from a physical covariance ``cov`` (k, k): ``(pixel_sigma / fx) ** 2 * inv(cov)``, in the objective's units
    (reprojection rows are pixels / fx_initial; exact when the cameras share one focal length).

    A row and column whose variance is ``inf`` is unconstrained: its information is zero, and the rest is the inverse of
    the remaining block.  A zero variance, or a finite block that is singular, would be an exactly known direction:
    refused (ValueError), since that is ``fixed_cam_params`` / ``fixed_points``.  So is a ``cov`` that is not symmetric
    to 1e-12 relative.

    Intrinsics example.  x holds ``s`` with ``fx = s * fx_initial``, so from ``intrinsics.calibrate_cameras``' standard
    deviations ``std`` (fx first) ``sigma_s = std[0] / fx_initial``; with ``k1``, ``k2`` from the same row and the pose
    free (infinite variance)::

        var = np.full(9, np.inf)
        var[6:] = (std[0] / fx_initial) ** 2, std[4] ** 2, std[5] ** 2
        info = prior_information(np.diag(var), pixel_sigma, fx_initial)   # (9, 9), zero outside s, k1, k2
    """
    cov = np.asarray(cov, dtype=np.float64)
    if cov.ndim != 2 or cov.shape[0] != cov.shape[1]:
        raise ValueError(f"cov must be square, got shape {cov.shape}")
    if not (pixel_sigma > 0 and fx != 0 and np.isfinite(pixel_sigma) and np.isfinite(fx)):
        raise ValueError("pixel_sigma must be positive and fx non-zero, both finite")
    var = np.diag(cov)
    if np.isnan(cov).any() or (var < 0).any() or (var == -np.inf).any():
        raise ValueError("cov has NaN entries or negative variances")
    if (var == 0).any():
        raise ValueError("a zero variance is an exactly known parameter: use fixed_cam_params / fixed_points instead")
    free = np.isfinite(var)
    info = np.zeros_like(cov)
    if not free.any():
        return info
    sub = cov[np.ix_(free, free)]
    if not np.isfinite(sub).all():
        raise ValueError("cov has an infinite entry outside the rows and columns of infinite variance")
    scale = np.abs(sub).max()
    if np.abs(sub - sub.T).max() > 1e-12 * scale:
        raise ValueError("cov is not symmetric")
    ev = np.linalg.eigvalsh(0.5 * (sub + sub.T))
    if ev[0] <= 1e-12 * ev[-1]:
        raise ValueError("cov is singular (or not positive definite) on its finite rows: an exactly known direction is "
                         "a fixed parameter, not a prior")  # fmt: skip
    inv = np.linalg.inv(0.5 * (sub + sub.T))
    info[np.ix_(free, free)] = (pixel_sigma / fx) ** 2 * 0.5 * (inv + inv.T)
    return info
