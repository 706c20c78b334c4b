"""Intrinsic calibration of every camera from planar-board views on the GPU (``cb_calibrate_intrinsics``, DESIGN.md
section 4.10): pinhole + Brown-Conrady (k1 k2 p1 p2 k3), the model and the optimum of ``cv2.calibrateCamera``, with its
standard deviations, for all views of all cameras in one call."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import _lib as L
from .triangulation import _check_device_tri_obs, _ptr

PARAM_NAMES = ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2", "k3")
CB_CAM_FISHEYE = L.CB_CAM_FISHEYE
CB_INTR_USE_GUESS = 0x100  # include/caliscope_b200.h

# OpenCV's calib3d flag values (checked against cv2 in tests/test_intrinsics_cpu.py; this module does not import cv2)
CALIB_USE_INTRINSIC_GUESS = 0x00001
CALIB_FIX_ASPECT_RATIO = 0x00002
CALIB_FIX_PRINCIPAL_POINT = 0x00004
CALIB_ZERO_TANGENT_DIST = 0x00008
CALIB_FIX_FOCAL_LENGTH = 0x00010
CALIB_FIX_K1 = 0x00020
CALIB_FIX_K2 = 0x00040
CALIB_FIX_K3 = 0x00080
CALIB_FIX_K4 = 0x00800
CALIB_FIX_K5 = 0x01000
CALIB_FIX_K6 = 0x02000
CALIB_RATIONAL_MODEL = 0x04000
CALIB_THIN_PRISM_MODEL = 0x08000
CALIB_FIX_S1_S2_S3_S4 = 0x10000
CALIB_TILTED_MODEL = 0x40000
CALIB_FIX_TAUX_TAUY = 0x80000
_SUPPORTED = (CALIB_USE_INTRINSIC_GUESS | CALIB_FIX_PRINCIPAL_POINT | CALIB_ZERO_TANGENT_DIST | CALIB_FIX_FOCAL_LENGTH |
              CALIB_FIX_K1 | CALIB_FIX_K2 | CALIB_FIX_K3)  # fmt: skip
# flags that only fix coefficients the 5-coefficient model does not have: accepted, nothing to do
_NO_OP = CALIB_FIX_K4 | CALIB_FIX_K5 | CALIB_FIX_K6 | CALIB_FIX_S1_S2_S3_S4 | CALIB_FIX_TAUX_TAUY


@dataclass
class IntrinsicCalibration:
    """Per camera: params (C, 9) = (fx, fy, cx, cy, k1, k2, p1, p2, k3), std (C, 9) (0 at fixed parameters), cov
    (C, 9, 9), rms (cv2's return value), sigma2, n_views (used), n_rows, iterations, status (0 ok, 1 fewer than
    min_views usable views, 2 no Zhang start, 3 not positive definite at the solution, 4 iteration limit).
    Per view in key order: cam, pose (V, 6) = (r, t) of the board in the camera, std (V, 6), rmse_px (cv2's
    perViewErrors), count, rep_row, status (0 used, 1 too few rows, 2 non-planar, 5 degenerate, 6 several cameras)."""

    params: np.ndarray
    std: np.ndarray
    cov: np.ndarray
    rms: np.ndarray
    sigma2: np.ndarray
    n_views: np.ndarray
    n_rows: np.ndarray
    iterations: np.ndarray
    status: np.ndarray
    view_cam: np.ndarray
    view_pose: np.ndarray
    view_std: np.ndarray
    view_rmse: np.ndarray
    view_count: np.ndarray
    view_rep: np.ndarray
    view_status: np.ndarray

    def camera_matrix(self, c: int) -> np.ndarray:
        fx, fy, cx, cy = self.params[c, :4]
        return np.array([[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]])


@dataclass
class IntrinsicsStats:
    group_ms: float = 0.0
    start_ms: float = 0.0
    lm_ms: float = 0.0
    cov_ms: float = 0.0
    total_ms: float = 0.0
    iterations: int = 0
    kernel_launches: int = 0


def calibrate_cameras(obs_cam, obs_key, obs_obj, obs_px, image_size, *, fixed=None, guess=None, min_points: int = 4,
                      min_views: int = 2, max_iter: int = 100, xtol: float = 1e-12, with_cov: bool = True,
                      device: int = 0, stream: int = 0, stats: IntrinsicsStats | None = None) -> IntrinsicCalibration:
    """Calibrate every camera's intrinsics from its board views (``cb_calibrate_intrinsics``, DESIGN.md section 4.10).

    Rows with equal ``obs_key`` (int64 >= 0) are one view of one camera ``obs_cam``; ``obs_obj`` (n, 3) are the board
    coordinates (planar, constant z) and ``obs_px`` (n, 2) the raw pixels.  The rows may be host arrays or CUDA tensors
    on ``device`` (obs_cam int32, obs_key int64, obs_obj float64 (n, 3), obs_px float64 (n, 2)), read in place.
    ``image_size`` (C, 2) = (w, h) per camera.  ``fixed`` (C, 9) bool (or (C,) int bit masks over PARAM_NAMES) keeps
    parameters at their start value; ``guess`` (C, 9), with NaN rows for cameras without one, is the start of the others
    (else Zhang's closed form)."""
    isize = np.ascontiguousarray(image_size, dtype=np.int32).reshape(-1, 2)
    nc = len(isize)
    if fixed is None:
        fixed_bits = np.zeros(nc, np.int32)
    else:
        fx = np.asarray(fixed)
        if fx.dtype == bool or fx.ndim == 2:
            fx = np.asarray(fx, bool).reshape(nc, 9)
            fixed_bits = (fx * (1 << np.arange(9))).sum(1).astype(np.int32)
        else:
            fixed_bits = np.ascontiguousarray(fx, dtype=np.int32).reshape(nc)
        if (fixed_bits & ~0x1FF).any():
            raise ValueError("fixed bit masks cover the 9 parameters only")
    flags = np.zeros(nc, np.int32)
    g = None
    if guess is not None:
        g = np.ascontiguousarray(guess, dtype=np.float64).reshape(nc, 9).copy()
        has = np.isfinite(g).all(1)
        flags = np.where(has, CB_INTR_USE_GUESS, 0).astype(np.int32)
        g[~has] = 0.0
    if int(min_points) < 4 or int(min_views) < 2 or int(max_iter) < 1 or not (np.isfinite(xtol) and xtol >= 0):
        raise ValueError("min_points >= 4, min_views >= 2, max_iter >= 1 and a finite xtol >= 0 are required")
    on_dev = hasattr(obs_px, "data_ptr")
    if on_dev:
        n = _check_device_tri_obs(obs_cam, obs_key, obs_px, device)
        o = obs_obj
        if getattr(getattr(o, "device", None), "type", None) != "cuda" or str(o.dtype) != "torch.float64" \
                or tuple(o.shape) != (n, 3) or not o.is_contiguous():
            raise ValueError(f"obs_obj must be a contiguous float64 CUDA tensor of shape ({n}, 3)")
        ptrs = tuple(C.c_void_p(t.data_ptr()) for t in (obs_cam, obs_key, obs_obj, obs_px))
        keep = ()
    else:
        cam = np.ascontiguousarray(obs_cam, dtype=np.int32)
        key = np.ascontiguousarray(obs_key, dtype=np.int64)
        obj = np.ascontiguousarray(obs_obj, dtype=np.float64).reshape(-1, 3)
        px = np.ascontiguousarray(obs_px, dtype=np.float64).reshape(-1, 2)
        n = len(cam)
        if len(key) != n or len(obj) != n or len(px) != n:
            raise ValueError("obs_cam, obs_key, obs_obj and obs_px must have one row per observation")
        keep = (cam, key, obj, px)
        ptrs = tuple(_ptr(a) for a in keep)
    lib = L.load()
    m = max(n, 1)
    params, std, rms, sig2 = np.empty((nc, 9)), np.empty((nc, 9)), np.empty(nc), np.empty(nc)
    cov = np.empty((nc, 9, 9)) if with_cov else None
    nv, nr, its, st = (np.empty(nc, np.int32) for _ in range(4))
    vcam, vcount, vrep, vstatus = (np.empty(m, np.int32) for _ in range(4))
    vpose, vstd, vrmse = np.empty((m, 6)), np.empty((m, 6)), np.empty(m)
    nviews = C.c_int32(0)
    cst = L.IntrinsicsStats()
    L.check(
        lib.cb_calibrate_intrinsics(nc, _ptr(isize), _ptr(flags), _ptr(fixed_bits), None if g is None else _ptr(g), n,
                                    *ptrs,
                                    1 if on_dev else 0, int(min_points), int(min_views), int(max_iter), float(xtol), n,
                                    C.byref(nviews), _ptr(params), _ptr(std), None if cov is None else _ptr(cov),
                                    _ptr(rms), _ptr(sig2), _ptr(nv), _ptr(nr), _ptr(its), _ptr(st), _ptr(vcam),
                                    _ptr(vpose), _ptr(vstd), _ptr(vrmse), _ptr(vcount), _ptr(vrep), _ptr(vstatus),
                                    C.byref(cst), int(device), C.c_void_p(stream)),
        "calibrate_intrinsics",
    )  # fmt: skip
    del keep
    V = nviews.value
    if stats is not None:
        for f in ("group_ms", "start_ms", "lm_ms", "cov_ms", "total_ms", "iterations", "kernel_launches"):
            setattr(stats, f, getattr(cst, f))
    return IntrinsicCalibration(params, std, cov, rms, sig2, nv, nr, its, st, vcam[:V], vpose[:V], vstd[:V], vrmse[:V],
                                vcount[:V], vrep[:V], vstatus[:V])  # fmt: skip


def flags_to_fixed(flags: int) -> tuple[np.ndarray, bool, bool]:
    """cv2 CALIB_* flags -> (fixed (9,) bool, use_guess, zero_tangent); NotImplementedError for what this call lacks."""
    bad = int(flags) & ~(_SUPPORTED | _NO_OP)
    if bad:
        raise NotImplementedError(f"calibration flags 0x{bad:x} are not implemented (fisheye, rational, thin-prism and "
                                  "tilted models and CALIB_FIX_ASPECT_RATIO are out of scope)")  # fmt: skip
    fixed = np.zeros(9, bool)
    if flags & CALIB_FIX_FOCAL_LENGTH:
        fixed[[0, 1]] = True
    if flags & CALIB_FIX_PRINCIPAL_POINT:
        fixed[[2, 3]] = True
    for bit, k in ((CALIB_FIX_K1, 4), (CALIB_FIX_K2, 5), (CALIB_FIX_K3, 8)):
        if flags & bit:
            fixed[k] = True
    if flags & CALIB_ZERO_TANGENT_DIST:
        fixed[[6, 7]] = True
    return fixed, bool(flags & CALIB_USE_INTRINSIC_GUESS), bool(flags & CALIB_ZERO_TANGENT_DIST)


def calibrate_camera(objectPoints, imagePoints, imageSize, cameraMatrix=None, distCoeffs=None, flags: int = 0, *,
                     max_iter: int = 100, xtol: float = 1e-12, device: int = 0):
    """``cv2.calibrateCameraExtended``'s arguments and return tuple, computed by ``calibrate_cameras``:
    (rms, cameraMatrix, distCoeffs (1, 5), rvecs, tvecs, stdDeviationsIntrinsics (18, 1), stdDeviationsExtrinsics
    (6 V, 1), perViewErrors (V, 1)).  Every view must be planar and usable; a view or a camera the call cannot use
    raises ValueError."""
    fixed, use_guess, zero_tan = flags_to_fixed(flags)
    objs = [np.asarray(o, np.float64).reshape(-1, 3) for o in objectPoints]
    imgs = [np.asarray(p, np.float64).reshape(-1, 2) for p in imagePoints]
    if len(objs) != len(imgs) or any(len(o) != len(p) for o, p in zip(objs, imgs)):
        raise ValueError("objectPoints and imagePoints must hold the same views with the same point counts")
    if any(not np.ptp(o[:, 2]) < 1e-6 for o in objs):
        raise NotImplementedError("non-planar calibration rigs are not implemented")
    guess = None
    if use_guess:
        if cameraMatrix is None:
            raise ValueError("CALIB_USE_INTRINSIC_GUESS needs a cameraMatrix")
        K = np.asarray(cameraMatrix, np.float64).reshape(3, 3)
        d = np.zeros(5)
        if distCoeffs is not None:
            dd = np.asarray(distCoeffs, np.float64).ravel()
            if (dd[5:] != 0).any():
                raise NotImplementedError("distortion coefficients beyond k1 k2 p1 p2 k3 are not implemented")
            d[: min(5, len(dd))] = dd[:5]
        guess = np.array([[K[0, 0], K[1, 1], K[0, 2], K[1, 2], *d]])
    if zero_tan and guess is not None:
        guess[0, 6:8] = 0.0
    cnt = np.array([len(o) for o in objs])
    n = int(cnt.sum())
    key = np.repeat(np.arange(len(objs), dtype=np.int64), cnt)
    res = calibrate_cameras(np.zeros(n, np.int32), key, np.concatenate(objs), np.concatenate(imgs),
                            [tuple(int(v) for v in imageSize)], fixed=fixed[None], guess=guess, max_iter=max_iter,
                            xtol=xtol, device=device)  # fmt: skip
    if (res.view_status != 0).any():
        raise ValueError(f"views {np.flatnonzero(res.view_status != 0).tolist()} cannot be used "
                         f"(statuses {res.view_status[res.view_status != 0].tolist()})")  # fmt: skip
    if res.status[0] not in (0, 4):
        raise ValueError(f"calibration failed with status {int(res.status[0])}")
    sdi = np.zeros((18, 1))
    sdi[:9, 0] = res.std[0]
    rv = tuple(p[:3].reshape(3, 1) for p in res.view_pose)
    tv = tuple(p[3:].reshape(3, 1) for p in res.view_pose)
    return (float(res.rms[0]), res.camera_matrix(0), res.params[0, 4:].reshape(1, 5), rv, tv, sdi,
            res.view_std.reshape(-1, 1), res.view_rmse.reshape(-1, 1))  # fmt: skip
