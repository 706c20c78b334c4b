"""NumPy statement of cb_calibrate_intrinsics' rule (DESIGN.md section 4.10): pinhole + Brown-Conrady (k1 k2 p1 p2 k3)
intrinsic calibration of every camera from its planar-board views, the reference the GPU tests compare against.

    1. views: ascending key order, rows in caller order within a key; status 6 rows from more than one camera, 1 fewer
       than min_points rows, 2 z spread >= 1e-6, 5 degenerate homography or a non-finite start pose.
    2. start: the guess, or Zhang's closed form (principal point at the image centre, distortion 0, a = 1/fx^2 and
       b = 1/fy^2 from cv2.initIntrinsicParams2D's two constraints per view, summed in view order); the pose of each view
       by IPPE on the pixels undistorted with the start.
    3. fixed parameters keep their start value and leave the system.
    4. Levenberg-Marquardt over the free intrinsics and every used view's (r, t) in Schur form.
    5. covariance at the solution: sigma^2 = SSE / (2N - p), cov_theta = sigma^2 S^-1, cov_q = sigma^2 (V^-1 + V^-1 W^T
       S^-1 W V^-1).
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from . import ippe
from .resection_robust import rot_log
from .triangulation import undistort_points

NAMES = ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2", "k3")
USE_GUESS = 1 << 9
LAMBDA0 = 1e-3
PD_RTOL = 1e-12
VIEW_OK, VIEW_TOO_FEW, VIEW_NON_PLANAR, VIEW_DEGENERATE, VIEW_MULTI_CAM = 0, 1, 2, 5, 6
CAM_OK, CAM_TOO_FEW_VIEWS, CAM_NO_START, CAM_NOT_PD, CAM_MAX_ITER = 0, 1, 2, 3, 4


def rodrigues_jr(r):
    """R(r) and the SO(3) right Jacobian Jr (d(R X)/dr = -R [X]x Jr), as the engine's cam_prep_rot."""
    r0, r1, r2 = r
    th2 = r0 * r0 + r1 * r1 + r2 * r2
    th = np.sqrt(th2)
    Km = np.array([[0, -r2, r1], [r2, 0, -r0], [-r1, r0, 0]])
    if th < 1e-12:
        R = np.eye(3) + Km
    else:
        k = np.asarray(r) / th
        Kn = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
        R = np.cos(th) * np.eye(3) + (1 - np.cos(th)) * np.outer(k, k) + np.sin(th) * Kn
    if th < 1e-4:
        B = 0.5 - th2 / 24.0 + th2 * th2 / 720.0
        C = 1.0 / 6.0 - th2 / 120.0 + th2 * th2 / 5040.0
    else:
        B = (1.0 - np.cos(th)) / th2
        C = (th - np.sin(th)) / (th2 * th)
    return R, np.eye(3) - B * Km + C * (Km @ Km)


def project(theta, q, X, jac: bool = False):
    """Pixels of board points X (n, 3) in a view with pose q = (r, t) and intrinsics theta; with jac also d/dtheta
    (2n, 9) and d/dq (2n, 6), rows u_0..u_{n-1}, v_0..v_{n-1}."""
    fx, fy, cx, cy, k1, k2, p1, p2, k3 = theta
    R, Jr = rodrigues_jr(q[:3])
    Xc = X @ R.T + q[3:]
    iz = 1.0 / Xc[:, 2]
    a, b = Xc[:, 0] * iz, Xc[:, 1] * iz
    r2 = a * a + b * b
    cd = 1.0 + r2 * (k1 + r2 * (k2 + r2 * k3))
    xd = a * cd + 2.0 * p1 * a * b + p2 * (r2 + 2.0 * a * a)
    yd = b * cd + p1 * (r2 + 2.0 * b * b) + 2.0 * p2 * a * b
    uv = np.stack([fx * xd + cx, fy * yd + cy], axis=1)
    if not jac:
        return uv
    n = len(X)
    z, o = np.zeros(n), np.ones(n)
    Ju = np.stack([xd, z, o, z, fx * a * r2, fx * a * r2**2, fx * 2 * a * b, fx * (r2 + 2 * a * a), fx * a * r2**3], 1)
    Jv = np.stack([z, yd, z, o, fy * b * r2, fy * b * r2**2, fy * (r2 + 2 * b * b), fy * 2 * a * b, fy * b * r2**3], 1)
    dcd = k1 + r2 * (2.0 * k2 + 3.0 * k3 * r2)
    xa = cd + 2.0 * a * a * dcd + 2.0 * p1 * b + 6.0 * p2 * a
    xb = 2.0 * a * b * dcd + 2.0 * p1 * a + 2.0 * p2 * b
    yb = cd + 2.0 * b * b * dcd + 6.0 * p1 * b + 2.0 * p2 * a
    Jt = np.concatenate([np.stack([fx * iz * xa, fx * iz * xb, -fx * iz * (xa * a + xb * b)], 1),
                         np.stack([fy * iz * xb, fy * iz * yb, -fy * iz * (xb * a + yb * b)], 1)])  # fmt: skip
    JX = Jt @ R
    XX = np.concatenate([X, X])
    Jq = np.concatenate([-np.cross(JX, XX) @ Jr, Jt], 1)
    return uv, np.concatenate([Ju, Jv]), Jq


def homography(obj2, px):
    """Harker-O'Leary homography px ~ H (X, Y, 1) (H[2,2] = 1), or None when degenerate."""
    A = obj2 - obj2.mean(1, keepdims=True)
    AAt = A @ A.T
    if not abs(np.linalg.det(AAt)) > 1e-12 * np.trace(AAt) ** 2 or not np.ptp(px, axis=1).max() > 0:
        return None
    with np.errstate(all="ignore"):
        try:
            H = ippe.homography_ho(obj2, px)
        except np.linalg.LinAlgError:
            return None
    return H if np.isfinite(H).all() else None


def zhang(Hs, w, h):
    """fx, fy from the homographies in view order (cv2.initIntrinsicParams2D without an aspect ratio), or None."""
    c = np.array([(w - 1) * 0.5, (h - 1) * 0.5])
    AtA, Atb = np.zeros((2, 2)), np.zeros(2)
    for H in Hs:
        H = H.copy()
        H[0] -= H[2] * c[0]
        H[1] -= H[2] * c[1]
        hh, vv = H[:, 0], H[:, 1]
        d1, d2 = (hh + vv) * 0.5, (hh - vv) * 0.5
        hh, vv, d1, d2 = (x / np.sqrt(x @ x) for x in (hh, vv, d1, d2))
        A = np.array([[hh[0] * vv[0], hh[1] * vv[1]], [d1[0] * d2[0], d1[1] * d2[1]]])
        b = np.array([-hh[2] * vv[2], -d1[2] * d2[2]])
        AtA += A.T @ A
        Atb += A.T @ b
    with np.errstate(all="ignore"):
        f = np.linalg.solve(AtA, Atb) if np.isfinite(AtA).all() and np.linalg.det(AtA) != 0 else np.full(2, np.nan)
    if not (np.isfinite(f).all() and f[0] > 0 and f[1] > 0):
        return None
    return np.array([np.sqrt(1 / f[0]), np.sqrt(1 / f[1]), c[0], c[1], 0, 0, 0, 0, 0.0])


def chol_pd(S, scaled_rtol=None):
    """Cholesky factor, or None when a pivot is <= 0 (or, with scaled_rtol, <= that of the Jacobi-scaled matrix)."""
    if scaled_rtol is not None:
        d = 1.0 / np.sqrt(np.diag(S))
        Ss = S * d[:, None] * d[None, :]
    else:
        Ss = S
    n = len(S)
    L = np.zeros_like(S)
    thr = 0.0 if scaled_rtol is None else scaled_rtol
    for j in range(n):
        v = Ss[j, j] - L[j, :j] @ L[j, :j]
        if not v > thr:
            return None
        L[j, j] = np.sqrt(v)
        L[j + 1:, j] = (Ss[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
    return L


class _Camera:
    """Normal equations of one camera in Schur form: the view blocks of its used views."""

    def __init__(self, X, px, free):
        self.X, self.px, self.free = X, px, free

    def linearize(self, theta, q):
        self.U, self.gt, self.W, self.V, self.gq, self.cost_v = np.zeros((9, 9)), np.zeros(9), [], [], [], []
        for X, px, qv in zip(self.X, self.px, q):
            uv, Jt, Jq = project(theta, qv, X, jac=True)
            r = np.concatenate([uv[:, 0] - px[:, 0], uv[:, 1] - px[:, 1]])
            self.U += Jt.T @ Jt
            self.gt += Jt.T @ r
            self.W.append(Jt.T @ Jq)
            self.V.append(Jq.T @ Jq)
            self.gq.append(Jq.T @ r)
            self.cost_v.append(r @ r)
        return float(np.sum(self.cost_v))

    def step(self, lam):
        """(dtheta (9, zero at fixed), dq (V, 6)), or None when a damped block is not positive definite."""
        f = self.free
        S = self.U + lam * np.diag(np.diag(self.U))
        rhs = self.gt.copy()
        Vl = []
        for W, V, gq in zip(self.W, self.V, self.gq):
            Vd = V + lam * np.diag(np.diag(V))
            if chol_pd(Vd) is None:
                return None
            Y = np.linalg.solve(Vd, W.T).T
            S -= Y @ W.T
            rhs -= Y @ gq
            Vl.append(Vd)
        dth = np.zeros(9)
        if f.any():
            Sf = S[np.ix_(f, f)]
            if chol_pd(Sf) is None:
                return None
            dth[f] = -np.linalg.solve(Sf, rhs[f])
        dq = np.array([-np.linalg.solve(Vd, gq + W.T @ dth) for Vd, W, gq in zip(Vl, self.W, self.gq)])
        return dth, dq

    def cost(self, theta, q):
        c = 0.0
        for X, px, qv in zip(self.X, self.px, q):
            e = project(theta, qv, X) - px
            c += float(np.sum(e * e))
        return c


@dataclass
class IntrinsicsResult:
    params: np.ndarray  # (C, 9)
    std: np.ndarray  # (C, 9), 0 at fixed parameters
    cov: np.ndarray  # (C, 9, 9)
    rms: np.ndarray  # (C,)
    sigma2: np.ndarray
    n_views: np.ndarray  # used views
    n_rows: np.ndarray
    iterations: np.ndarray
    status: np.ndarray
    view_key: np.ndarray  # (V,) ascending
    view_cam: np.ndarray
    view_pose: np.ndarray  # (V, 6) = (r, t)
    view_std: np.ndarray
    view_rmse: np.ndarray
    view_count: np.ndarray
    view_rep: np.ndarray
    view_status: np.ndarray


def views(obs_cam, obs_key, obs_obj, min_points):
    keys, inv = np.unique(obs_key, return_inverse=True)
    out = []
    for v in range(len(keys)):
        rows = np.flatnonzero(inv == v)
        cams = obs_cam[rows]
        z = obs_obj[rows, 2]
        if (cams != cams[0]).any():
            st = VIEW_MULTI_CAM
        elif len(rows) < min_points:
            st = VIEW_TOO_FEW
        elif not np.ptp(z) < 1e-6:
            st = VIEW_NON_PLANAR
        else:
            st = VIEW_OK
        out.append((int(keys[v]), rows, int(cams[0]), st))
    return out


def calibrate(obs_cam, obs_key, obs_obj, obs_px, image_size, cam_flags, guess=None, *, min_points=4, min_views=2,
              max_iter=100, xtol=1e-12) -> IntrinsicsResult:
    """The rule of cb_calibrate_intrinsics.  cam_flags: bits 0-8 fix (fx fy cx cy k1 k2 p1 p2 k3), bit 9 starts from
    guess[c]."""
    obs_cam = np.asarray(obs_cam, np.int64)
    obs_obj = np.asarray(obs_obj, np.float64)
    obs_px = np.asarray(obs_px, np.float64)
    C = len(image_size)
    vl = views(obs_cam, np.asarray(obs_key, np.int64), obs_obj, min_points)
    V = len(vl)
    nan = np.nan
    res = IntrinsicsResult(np.full((C, 9), nan), np.full((C, 9), nan), np.full((C, 9, 9), nan), np.full(C, nan),
                           np.full(C, nan), np.zeros(C, np.int32), np.zeros(C, np.int32), np.zeros(C, np.int32),
                           np.zeros(C, np.int32), np.array([v[0] for v in vl], np.int64),
                           np.array([v[2] for v in vl], np.int32), np.full((V, 6), nan), np.full((V, 6), nan),
                           np.full(V, nan), np.array([len(v[1]) for v in vl], np.int32),
                           np.array([v[1][0] for v in vl], np.int32), np.array([v[3] for v in vl], np.int32))  # fmt: skip
    Hs = {}
    for i, (_, rows, _, st) in enumerate(vl):
        if st == VIEW_OK:
            H = homography(obs_obj[rows, :2].T, obs_px[rows].T)
            if H is None:
                res.view_status[i] = VIEW_DEGENERATE
            else:
                Hs[i] = H
    for c in range(C):
        flags = int(cam_flags[c])
        mine = [i for i in range(V) if vl[i][2] == c and res.view_status[i] == VIEW_OK]
        if flags & USE_GUESS:
            theta = np.asarray(guess[c], np.float64).copy()
        else:
            theta = zhang([Hs[i] for i in mine], *image_size[c])
        if theta is not None:
            res.params[c] = theta
            K = np.array([[theta[0], 0, theta[2]], [0, theta[1], theta[3]], [0, 0, 1.0]])
            for i in mine:
                rows = vl[i][1]
                norm = undistort_points(obs_px[rows], K, theta[4:9], False, "normalized")
                R, t, _ = ippe.solve_pnp_planar(obs_obj[rows], norm)
                if np.isfinite(R).all() and np.isfinite(t).all():
                    res.view_pose[i] = np.concatenate([rot_log(R), t])
                else:
                    res.view_status[i] = VIEW_DEGENERATE
        used = [i for i in mine if res.view_status[i] == VIEW_OK]
        if len(used) < min_views:
            res.status[c] = CAM_TOO_FEW_VIEWS
            res.view_pose[used] = nan
            continue
        if theta is None:
            res.status[c] = CAM_NO_START
            continue
        res.n_views[c] = len(used)
        res.n_rows[c] = sum(len(vl[i][1]) for i in used)
        _solve_camera(res, c, flags, theta, used, [obs_obj[vl[i][1]] for i in used], [obs_px[vl[i][1]] for i in used],
                      max_iter, xtol)  # fmt: skip
    return res


def _solve_camera(res, c, flags, theta, used, X, px, max_iter, xtol):
    free = np.array([not (flags >> k) & 1 for k in range(9)])
    cam = _Camera(X, px, free)
    q = res.view_pose[used].copy()
    lam, it, st = LAMBDA0, 0, CAM_OK
    cost = cam.linearize(theta, q)
    while True:
        if it == max_iter:
            st = CAM_MAX_ITER
            break
        s = cam.step(lam)
        it += 1
        if s is None:
            lam *= 10.0
            continue
        dth, dq = s
        tt, qt = theta + dth, q + dq
        dn = np.sqrt(np.sum(dth[free] ** 2) + np.sum(dq * dq))
        xn = np.sqrt(np.sum(theta[free] ** 2) + np.sum(q * q))
        if cam.cost(tt, qt) < cost:
            theta, q = tt, qt
            cost = cam.linearize(theta, q)
            lam *= 0.1
        else:
            lam *= 10.0
        if dn <= xtol * (xn + xtol):
            break
    res.params[c] = theta
    res.view_pose[used] = q
    res.iterations[c] = it
    N = res.n_rows[c]
    res.rms[c] = np.sqrt(cost / N)
    for j, i in enumerate(used):
        res.view_rmse[i] = np.sqrt(cam.cost_v[j] / len(X[j]))
    cov, view_std, sig2 = covariance(cam, free)
    res.sigma2[c] = sig2
    if cov is None:
        res.status[c] = CAM_NOT_PD
        return
    res.status[c] = st
    res.cov[c] = cov
    res.std[c] = np.sqrt(np.diag(cov))
    res.view_std[used] = view_std


def covariance(cam: _Camera, free):
    """(cov_theta (9, 9), per-view std (V, 6), sigma^2) at the point cam was last linearised at, lambda = 0; cov_theta
    None when S is not positive definite."""
    cost = float(np.sum(cam.cost_v))
    N = sum(len(X) for X in cam.X)
    p = int(free.sum()) + 6 * len(cam.X)
    sig2 = cost / (2 * N - p) if 2 * N > p else np.nan
    S = cam.U.copy()
    Vi = [np.linalg.inv(V) for V in cam.V]
    for W, Vinv in zip(cam.W, Vi):
        S -= W @ Vinv @ W.T
    Sf = S[np.ix_(free, free)]
    if free.any() and chol_pd(Sf, PD_RTOL) is None:
        return None, None, sig2
    Si = np.zeros((9, 9))
    if free.any():
        Si[np.ix_(free, free)] = np.linalg.inv(Sf)
    view_std = np.array([np.sqrt(np.diag(sig2 * (Vinv + (Vinv @ W.T) @ Si @ (Vinv @ W.T).T))) for W, Vinv in zip(cam.W, Vi)])
    return sig2 * Si, view_std, sig2


def standard_deviations(theta, poses, X, px, free):
    """cv2.calibrateCameraExtended's stdDeviationsIntrinsics[:9] and stdDeviationsExtrinsics (V, 6) evaluated at any
    point (theta, poses) of one camera: sqrt(diag((J^T J)^-1) SSE / (2N - p)) with J the full pixel Jacobian."""
    cam = _Camera(X, px, np.asarray(free, bool))
    cam.linearize(np.asarray(theta, np.float64), np.asarray(poses, np.float64))
    cov, view_std, _ = covariance(cam, np.asarray(free, bool))
    return np.sqrt(np.diag(cov)), view_std
