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
    """One camera's pose uncertainty relative to the gauge.  position_cov: world-frame covariance of the centre
    C = -R^T t; orientation_cov: covariance of the body-frame rotation error (R_true = R exp([e]x)), rad^2."""

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


def camera_poses(x, cam_offsets, cam_cov) -> list[PoseUncertainty | None]:
    """Per camera (caller order) the pose uncertainty from the camera block of a covariance; None for cameras whose
    block is NaN (no observations)."""
    out = []
    for c in range(len(cam_offsets) - 1):
        o = int(cam_offsets[c])
        blk = cam_cov[o : o + 6, o : o + 6]
        out.append(None if np.isnan(blk).any() else pose_from_extrinsics(x[o : o + 3], x[o + 3 : o + 6], blk))
    return out
