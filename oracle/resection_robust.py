"""CPU oracle of robust resection with calibrated cameras: P3P consensus, then refinement of the pose and its covariance
on the consensus rows (``cb_resect_robust``, DESIGN.md section 4.9).

TEST INFRASTRUCTURE ONLY — the product (caliscope_b200/) never imports this module.

Cameras in the bundle-adjustment layout (cam_flags, cam_const, the camera section of x); points pts_xyz (n_pts, 3) and
an optional pts_cov (n_pts, 3, 3); observations obs_cam, obs_key, obs_pt, obs_px (raw pixels).  A group is the rows of
one obs_key, k rows key-sorted and in caller order within a key, positions 0..k-1.
  1. Rows from more than one obs_cam: status 6.   2. k < 4: status 1.
  3. A row whose point is not finite is unusable: it scores tau^2, is in no sample's solution set, is never an inlier.
  4. Candidate samples, T = C(k, 3): every triple i < j < l in lexicographic order when T <= max_samples; else sample
     m = 0..max_samples-1 draws positions splitmix64(m 2^32 + t) mod k for t = 0, 1, ..., keeps the first three
     distinct (sorted) and gives up after 16 draws.  splitmix64(x): z = x + 0x9e3779b97f4a7c15, then the standard
     finaliser, in exact unsigned 64-bit arithmetic.
  5. Hypotheses of a sample of three usable rows: ``p3p`` (Lambda Twist) on the bearings of the float32-rounded
     undistorted normalised coordinates, up to 4 in the solver's order; a solution that is not finite or puts one of
     its three points at Xc.z <= 0 is none.  With use_prior the pose of the group's camera in cam_x is one more
     hypothesis, ranked before every sample.  Slot of a hypothesis: 0 for the prior, 1 + 4 m + c for candidate c of
     sample m.
  6. Score (MSAC): sum over all k rows of min(e_r^2, tau^2), e_r = |pi(X_r; R, t, intrinsics) - u_r| in raw pixels with
     the engine's projection and the hypothesis's R; a row with Xc.z <= 0, a non-finite e_r or an unusable point adds
     tau^2.  The lowest score wins, the lowest slot on a tie.
  7. Consensus set: the usable rows with Xc.z > 0 and e_r^2 <= tau^2 at the winner.  No hypothesis, or fewer than
     min_inliers rows: status 5 (pose, cov, rmse NaN, n_inliers 0, no inlier).
  8. Levenberg-Marquardt over q = (r, t) on the consensus rows, intrinsics fixed, from ``rot_log`` of the winner's R:
     H = sum J^T J, g = sum J^T r in pixels (J = d pi / d q); solve (H + lam diag H) d = -g, lam0 = 1e-3; accept when
     the cost drops (lam /= 10) else lam *= 10; q += d; stop when |d| <= xtol (|q| + xtol) (|q| before the step) or
     after max_iter steps.
  9. Covariance at q*: pixel_sigma^2 H^-1 + H^-1 M H^-1, M = sum_p G_p Sigma_p G_p^T, G_p = sum over the consensus rows
     of point p of J_q^T J_X (6 x 3, pixels), Sigma_p = pts_cov[p]; without pts_cov the first term alone.  It assumes
     the points are independent of each other and of the group's own observations, and uses each point's marginal.
 10. Status, first match wins: 6, 1, 5, 2 (H fails ``pd6`` at the start or at the solution; pose = the hypothesis, cov
     NaN), 3 (max_iter reached), 4 (a consensus row has Xc.z <= 0 at q*), 0.
"""
from __future__ import annotations

from dataclasses import dataclass
from math import acos, sqrt

import numpy as np

from oracle.triangulation_refine import PD_RTOL, REFINE_LAMBDA0, group_rows
from oracle.triangulation_robust import undistorted_coordinates

STATUS_OK, STATUS_FEW_ROWS, STATUS_NOT_PD, STATUS_MAX_ITER, STATUS_BEHIND, STATUS_NO_CONSENSUS, STATUS_MULTI_CAM = range(7)
DRAWS = 16
_MASK = (1 << 64) - 1


def splitmix64(x: int) -> int:
    z = (x + 0x9E3779B97F4A7C15) & _MASK
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _MASK
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _MASK
    return z ^ (z >> 31)


def candidate_samples(k: int, max_samples: int) -> list:
    """Positions (i, j, l) of every candidate sample of a group of k rows, in order (None: the hashed draw gave up)."""
    T = k * (k - 1) * (k - 2) // 6
    if T <= max_samples:
        return [(i, j, l) for i in range(k) for j in range(i + 1, k) for l in range(j + 1, k)]
    out = []
    for m in range(max_samples):
        got: list[int] = []
        for t in range(DRAWS):
            v = splitmix64((m << 32) + t) % k
            if v not in got:
                got.append(v)
                if len(got) == 3:
                    break
        out.append(tuple(sorted(got)) if len(got) == 3 else None)
    return out


# ---- Lambda Twist P3P (Persson & Nordberg, ECCV 2018), the kernel's arithmetic --------------------------------------
def _root2(b, c):
    v = b * b - 4.0 * c
    if not v >= 0.0:
        return None
    y = sqrt(v)
    q = 0.5 * (-b + y) if b < 0.0 else 0.5 * (-b - y)
    return q, _safe_div(c, q)


def _cubic_root(b, c, d):
    if b * b >= 3.0 * c:
        v = sqrt(b * b - 3.0 * c)
        t1 = (-b - v) / 3.0
        k = ((t1 + b) * t1 + c) * t1 + d
        if k > 0.0:
            r0 = t1 - _sqrt(_safe_div(-k, 3.0 * t1 + b))
        else:
            t2 = (-b + v) / 3.0
            k = ((t2 + b) * t2 + c) * t2 + d
            r0 = t2 + _sqrt(_safe_div(-k, 3.0 * t2 + b))
    else:
        r0 = -b / 3.0
        if abs((3.0 * r0 + 2.0 * b) * r0 + c) < 1e-4:
            r0 += 1.0
    for it in range(50):
        fx = ((r0 + b) * r0 + c) * r0 + d
        if it >= 7 and not abs(fx) > 2.220446049250313e-16:
            break
        r0 -= _safe_div(fx, (3.0 * r0 + 2.0 * b) * r0 + c)
    return r0


def _safe_div(a, b):
    with np.errstate(divide="ignore", invalid="ignore"):
        return float(np.float64(a) / np.float64(b))


def _sqrt(v):
    return sqrt(v) if v >= 0.0 else float("nan")


def p3p(y, x) -> list:
    """Lambda Twist on unit bearings y (3, 3) (rows) and world points x (3, 3): 4 candidates in the solver's order, each
    (R, t) with y_i ~ R x_i + t, or None.  A candidate is none when its quadratic has no real root, tau <= 0, its depth
    is not positive, l1 < 0, its pose is not finite or a point has Xc.z <= 0."""
    y = np.asarray(y, np.float64)
    x = np.asarray(x, np.float64)
    b12, b13, b23 = (-2.0 * float(y[i] @ y[j]) for i, j in ((0, 1), (0, 2), (1, 2)))
    d12, d13, d23 = x[0] - x[1], x[0] - x[2], x[1] - x[2]
    a12, a13, a23 = float(d12 @ d12), float(d13 @ d13), float(d23 @ d23)
    c31, c23, c12 = -0.5 * b13, -0.5 * b23, -0.5 * b12
    blob = c12 * c23 * c31 - 1.0
    s31, s23, s12 = 1.0 - c31 * c31, 1.0 - c23 * c23, 1.0 - c12 * c12
    p3 = a13 * (a23 * s31 - a13 * s23)
    p2 = 2.0 * blob * a23 * a13 + a13 * (2.0 * a12 + a13) * s23 + a23 * (a23 - a12) * s31
    p1 = a23 * (a13 - a23) * s12 - a12 * a12 * s23 - 2.0 * a12 * (blob * a23 + a13 * s23)
    p0 = a12 * (a12 * s23 - a23 * s12)
    p3 = _safe_div(1.0, p3)
    p2, p1, p0 = p2 * p3, p1 * p3, p0 * p3
    out = [None] * 4
    if not all(np.isfinite([p2, p1, p0])):
        return out
    g = _cubic_root(p2, p1, p0)
    A00, A01, A02 = a23 * (1.0 - g), (a23 * b12) * 0.5, (a23 * b13 * g) * (-0.5)
    A11, A12, A22 = a23 - a12 + a13 * g, b23 * (a13 * g - a12) * 0.5, g * (a13 - a23) - a12
    eb = -A00 - A11 - A22
    ec = -A01 * A01 - A02 * A02 - A12 * A12 + A00 * (A11 + A22) + A11 * A22
    ee = _root2(eb, ec)
    if ee is None:
        return out
    e1, e2 = ee
    if abs(e1) < abs(e2):
        e1, e2 = e2, e1
    mx0011 = -A00 * A11
    prec0, prec1 = A01 * A12 - A02 * A11, A01 * A02 - A00 * A12
    V = np.empty((3, 2))
    for q, e in enumerate((e1, e2)):
        tmp = _safe_div(1.0, e * (A00 + A11) + mx0011 - e * e + A01 * A01)
        v0, v1 = -(e * A02 + prec0) * tmp, -(e * A12 + prec1) * tmp
        rn = _safe_div(1.0, _sqrt(v0 * v0 + v1 * v1 + 1.0))
        V[:, q] = (v0 * rn, v1 * rn, rn)
    v = _sqrt(max(0.0, _safe_div(-e2, e1)))
    Ls = [None] * 4
    for sgn in range(2):
        s = -v if sgn else v
        w2 = _safe_div(1.0, s * V[0, 1] - V[0, 0])
        w0, w1 = (V[1, 0] - s * V[1, 1]) * w2, (V[2, 0] - s * V[2, 1]) * w2
        a = _safe_div(1.0, (a13 - a12) * w1 * w1 - a12 * b13 * w1 - a12)
        bq = (a13 * b12 * w1 - a12 * b13 * w0 - 2.0 * w0 * w1 * (a12 - a13)) * a
        cq = ((a13 - a12) * w0 * w0 + a13 * b12 * w0 + a13) * a
        taus = _root2(bq, cq) if np.isfinite(bq) and np.isfinite(cq) else None
        if taus is None:
            continue
        for r, tq in enumerate(taus):
            d = _safe_div(a23, tq * (b23 + tq) + 1.0)
            l2 = _sqrt(d)
            l3 = tq * l2
            l1 = w0 * l2 + w1 * l3
            if tq > 0.0 and d > 0.0 and l1 >= 0.0:
                Ls[2 * sgn + r] = [l1, l2, l3]
    # Gauss-Newton polish of the depths
    for c in range(4):
        if Ls[c] is None:
            continue
        l1, l2, l3 = Ls[c]
        for _ in range(5):
            r1 = l1 * l1 + l2 * l2 + b12 * l1 * l2 - a12
            r2 = l1 * l1 + l3 * l3 + b13 * l1 * l3 - a13
            r3 = l2 * l2 + l3 * l3 + b23 * l2 * l3 - a23
            rs = abs(r1) + abs(r2) + abs(r3)
            if rs < 1e-10:
                break
            v0, v1 = 2.0 * l1 + b12 * l2, 2.0 * l2 + b12 * l1
            v3, v5 = 2.0 * l1 + b13 * l3, 2.0 * l3 + b13 * l1
            v7, v8 = 2.0 * l2 + b23 * l3, 2.0 * l3 + b23 * l2
            det = _safe_div(1.0, -v0 * v5 * v7 - v1 * v3 * v8)
            n1 = l1 - det * (-v5 * v7 * r1 - v1 * v8 * r2 + v1 * v5 * r3)
            n2 = l2 - det * (-v3 * v8 * r1 + v0 * v8 * r2 - v0 * v5 * r3)
            n3 = l3 - det * (v3 * v7 * r1 - v0 * v7 * r2 - v1 * v3 * r3)
            q1 = n1 * n1 + n2 * n2 + b12 * n1 * n2 - a12
            q2 = n1 * n1 + n3 * n3 + b13 * n1 * n3 - a13
            q3 = n2 * n2 + n3 * n3 + b23 * n2 * n3 - a23
            if abs(q1) + abs(q2) + abs(q3) > rs:
                break
            l1, l2, l3 = n1, n2, n3
        Ls[c] = [l1, l2, l3]
    Xm = np.stack([d12, d13, np.cross(d12, d13)], axis=1)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        try:
            Xi = np.linalg.inv(Xm)
        except np.linalg.LinAlgError:
            return out
        for c in range(4):
            if Ls[c] is None:
                continue
            p = y * np.asarray(Ls[c])[:, None]
            u, w = p[0] - p[1], p[0] - p[2]
            R = np.stack([u, w, np.cross(u, w)], axis=1) @ Xi
            t = p[0] - R @ x[0]
            if not (np.isfinite(R).all() and np.isfinite(t).all()):
                continue
            if not ((x @ R[2] + t[2]) > 0).all():
                continue
            out[c] = (R, t)
    return out


def rot_log(R) -> np.ndarray:
    """Rotation vector of R with theta in [0, pi]: cv2.Rodrigues' matrix-to-vector branch without its SVD
    re-orthonormalisation."""
    R = np.asarray(R, np.float64)
    rx, ry, rz = R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]
    s = sqrt((rx * rx + ry * ry + rz * rz) * 0.25)
    c = min(1.0, max(-1.0, (R[0, 0] + R[1, 1] + R[2, 2] - 1.0) * 0.5))
    th = acos(c)
    if s < 1e-5:
        if c > 0:
            return np.zeros(3)
        rx = sqrt(max((R[0, 0] + 1.0) * 0.5, 0.0))
        ry = sqrt(max((R[1, 1] + 1.0) * 0.5, 0.0)) * (-1.0 if R[0, 1] < 0 else 1.0)
        rz = sqrt(max((R[2, 2] + 1.0) * 0.5, 0.0)) * (-1.0 if R[0, 2] < 0 else 1.0)
        if abs(rx) < abs(ry) and abs(rx) < abs(rz) and ((R[1, 2] > 0) != (ry * rz > 0)):
            rz = -rz
        return np.array([rx, ry, rz]) * (th / sqrt(rx * rx + ry * ry + rz * rz))
    return np.array([rx, ry, rz]) * (th / (2.0 * s))


# ---- cameras and the projection ----------------------------------------------------------------------------------------
@dataclass
class Cam:
    flags: int
    const: np.ndarray  # (9,)
    q: np.ndarray  # the camera's block of x: r t (s k1 k2)
    fx: float
    fy: float
    cx: float
    cy: float
    d: np.ndarray  # (5,) Brown-Conrady k1 k2 p1 p2 k3 | fisheye k1 k2 k3 k4 -


def cameras(cam_flags, cam_const, cam_x) -> list[Cam]:
    flags = np.asarray(cam_flags, np.int32).ravel()
    const = np.asarray(cam_const, np.float64).reshape(-1, 9)
    cam_x = np.asarray(cam_x, np.float64)
    out, o = [], 0
    for c, f in enumerate(flags):
        w = 9 if f & 1 else 6
        q = cam_x[o : o + w].copy()
        o += w
        s, k1, k2 = (q[6], q[7], q[8]) if f & 1 else (1.0, const[c, 4], const[c, 5])
        k = const[c]
        out.append(Cam(int(f), k, q, s * k[0], s * k[1], k[2], k[3], np.array([k1, k2, k[6], k[7], k[8]])))
    return out


def project(cam: Cam, R, t, X):
    """pi(X; R, t, intrinsics of cam) (..., 2) and Xc.z (...); R (..., 3, 3), t (..., 3), X (..., 3) broadcast."""
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        Xc = np.einsum("...ij,...j->...i", R, X) + t
        z = Xc[..., 2]
        iz = np.where(z != 0.0, 1.0 / np.where(z != 0.0, z, 1.0), 1.0)
        a, b = Xc[..., 0] * iz, Xc[..., 1] * iz
        r2 = a * a + b * b
        d = cam.d
        if cam.flags & 2:
            rr = np.sqrt(r2)
            th = np.arctan(rr)
            th2 = th * th
            thd = th * (1 + th2 * (d[0] + th2 * (d[1] + th2 * (d[2] + th2 * d[3]))))
            big = rr > 1e-8
            cdist = np.where(big, thd / np.where(big, rr, 1.0), 1.0)
            xd, yd = a * cdist, b * cdist
        else:
            cd = 1.0 + r2 * (d[0] + r2 * (d[1] + r2 * d[4]))
            xd = a * cd + 2.0 * d[2] * a * b + d[3] * (r2 + 2.0 * a * a)
            yd = b * cd + d[2] * (r2 + 2.0 * b * b) + 2.0 * d[3] * a * b
        return np.stack([cam.fx * xd + cam.cx, cam.fy * yd + cam.cy], axis=-1), z


def pose_jacobians(cam: Cam, q, X, px):
    """Residuals pi - u (n, 2), d pi / d (r, t) (n, 2, 6) and d pi / d X (n, 2, 3) in pixels at pose q, the BA
    projection's derivatives (``ba_oracle._project`` with this camera alone)."""
    from oracle.ba_oracle import Rig, _project

    X = np.asarray(X, np.float64).reshape(-1, 3)
    n = len(X)
    rig = Rig(np.array([cam.flags]), cam.const[None], n, np.zeros(n, np.int32), np.arange(n, dtype=np.int32),
              np.asarray(px, np.float64).reshape(-1, 2))  # fmt: skip
    xc = cam.q.copy()
    xc[:6] = q
    x = np.concatenate([xc, X.ravel()])
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        uv, (Jrv, Jt, _, _, _, JX) = _project(x, rig, True)
    return uv - rig.obs_xy, np.concatenate([Jrv, Jt], axis=2), JX


def pd6(H) -> bool:
    """Every Cholesky pivot of the Jacobi-scaled D^-1/2 H D^-1/2 above PD_RTOL (NaN fails)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        s = 1.0 / np.sqrt(np.diag(H))
        A = H * s[:, None] * s[None, :]
        L = np.zeros((6, 6))
        for j in range(6):
            d = A[j, j] - L[j, :j] @ L[j, :j]
            if not d > PD_RTOL:
                return False
            L[j, j] = sqrt(d)
            for i in range(j + 1, 6):
                L[i, j] = (A[i, j] - L[i, :j] @ L[j, :j]) / L[j, j]
    return True


def _normal_eq(cam, q, X, px):
    r, J, _ = pose_jacobians(cam, q, X, px)
    H = np.einsum("nki,nkj->ij", J, J)
    g = np.einsum("nki,nk->i", J, r)
    return float((r * r).sum()), H, g


def refine_pose(cam: Cam, q0, X, px, *, max_iter=20, xtol=1e-12):
    """Step 8 on one group's consensus rows: (q, rmse, status in {0, 2, 3, 4})."""
    q0 = np.asarray(q0, np.float64)
    q = q0.copy()
    cost, H, g = _normal_eq(cam, q, X, px)
    cost0 = cost
    n = len(X)
    if not pd6(H):
        return q0, sqrt(cost0 / n), STATUS_NOT_PD
    status = STATUS_OK
    lam = REFINE_LAMBDA0
    it = 0
    while True:
        if it == max_iter:
            status = STATUS_MAX_ITER
            break
        A = H + lam * np.diag(np.diag(H))
        d = np.linalg.solve(A, -g)
        ct, Ht, gt = _normal_eq(cam, q + d, X, px)
        it += 1
        conv = np.linalg.norm(d) <= xtol * (np.linalg.norm(q) + xtol)
        if ct < cost:
            q, cost, H, g = q + d, ct, Ht, gt
            lam /= 10.0
        else:
            lam *= 10.0
        if conv:
            break
    if not pd6(H):
        return q0, sqrt(cost0 / n), STATUS_NOT_PD
    from oracle.ba_oracle import rodrigues

    R = rodrigues(q[:3])[0]
    if status == STATUS_OK and not ((X @ R[2] + q[5]) > 0).all():
        status = STATUS_BEHIND
    return q, sqrt(cost / n), status


def pose_covariance(cam: Cam, q, X, px, pt, pixel_sigma, pts_cov=None):
    """Step 9 at q on one group's consensus rows (points pt)."""
    _, J, JX = pose_jacobians(cam, q, X, px)
    H = np.einsum("nki,nkj->ij", J, J)
    Hi = np.linalg.inv(H)
    cov = pixel_sigma**2 * Hi
    if pts_cov is not None:
        Gr = np.einsum("nki,nkj->nij", J, JX)  # (n, 6, 3)
        M = np.zeros((6, 6))
        for p in np.unique(pt):
            Gp = Gr[pt == p].sum(axis=0)
            M += Gp @ pts_cov[p] @ Gp.T
        cov = cov + Hi @ M @ Hi
    return 0.5 * (cov + cov.T)


@dataclass
class ResectResult:
    cam: np.ndarray
    pose: np.ndarray  # (G, 6)
    cov: np.ndarray  # (G, 6, 6)
    rmse_px: np.ndarray
    count: np.ndarray
    n_inliers: np.ndarray
    rep_row: np.ndarray
    status: np.ndarray
    inlier: np.ndarray  # (n,) caller order
    hyp: np.ndarray  # (G, 12) the winner (R row-major, t), NaN without consensus
    slot: np.ndarray  # (G,) the winner's slot, -1 without a hypothesis
    best: np.ndarray  # (G,) lowest score (+inf: no hypothesis)
    second: np.ndarray  # (G,) second-lowest score (+inf: none)


def bearings(norm) -> np.ndarray:
    norm = np.asarray(norm, np.float64).reshape(-1, 2)
    inv = 1.0 / np.sqrt(norm[:, 0] ** 2 + norm[:, 1] ** 2 + 1.0)
    return np.stack([norm[:, 0] * inv, norm[:, 1] * inv, inv], axis=1)


def resect_robust(cam_flags, cam_const, cam_x, pts_xyz, obs_cam, obs_key, obs_pt, obs_px, *, threshold_px,
                  min_inliers=6, max_samples=64, use_prior=True, pixel_sigma=1.0, points_cov=None, max_iter=20,
                  xtol=1e-12) -> ResectResult:  # fmt: skip
    """Steps 1-10 for every group."""
    from oracle.ba_oracle import rodrigues

    cams = cameras(cam_flags, cam_const, cam_x)
    obs_cam = np.asarray(obs_cam, np.int64)
    obs_pt = np.asarray(obs_pt, np.int64)
    obs_px = np.asarray(obs_px, np.float64).reshape(-1, 2)
    pts = np.asarray(pts_xyz, np.float64).reshape(-1, 3)
    pcov = None if points_cov is None else np.asarray(points_cov, np.float64).reshape(-1, 3, 3)
    tau2 = threshold_px * threshold_px
    grp, G = group_rows(obs_key)
    order = np.argsort(grp, kind="stable")
    bounds = np.searchsorted(grp[order], np.arange(G + 1))
    norm = undistorted_coordinates(cam_flags, cam_const, cam_x, obs_cam, obs_px)
    nan = np.nan
    res = ResectResult(cam=np.zeros(G, np.int32), pose=np.full((G, 6), nan), cov=np.full((G, 6, 6), nan),
                       rmse_px=np.full(G, nan), count=np.diff(bounds).astype(np.int32), n_inliers=np.zeros(G, np.int32),
                       rep_row=order[bounds[:-1]].astype(np.int32), status=np.zeros(G, np.int32),
                       inlier=np.zeros(len(obs_cam), bool), hyp=np.full((G, 12), nan), slot=np.full(G, -1),
                       best=np.full(G, np.inf), second=np.full(G, np.inf))  # fmt: skip
    for g in range(G):
        rows = order[bounds[g] : bounds[g + 1]]
        k = len(rows)
        c0 = int(obs_cam[rows[0]])
        res.cam[g] = c0
        if (obs_cam[rows] != c0).any():
            res.status[g] = STATUS_MULTI_CAM
            continue
        if k < 4:
            res.status[g] = STATUS_FEW_ROWS
            continue
        cam = cams[c0]
        X = pts[obs_pt[rows]]
        usable = np.isfinite(X).all(axis=1)
        slots, Rs, ts = [], [], []
        if use_prior:
            slots.append(0)
            Rs.append(rodrigues(cam.q[:3])[0])
            ts.append(cam.q[3:6])
        y_all = bearings(norm[rows])
        for m, smp in enumerate(candidate_samples(k, max_samples)):
            if smp is None or not usable[list(smp)].all():
                continue
            for c, sol in enumerate(p3p(y_all[list(smp)], X[list(smp)])):
                if sol is not None:
                    slots.append(1 + 4 * m + c)
                    Rs.append(sol[0])
                    ts.append(sol[1])
        if not slots:
            res.status[g] = STATUS_NO_CONSENSUS
            continue
        Rs, ts, slots = np.array(Rs), np.array(ts), np.array(slots)
        uv, z = project(cam, Rs[:, None], ts[:, None], X[None])
        with np.errstate(invalid="ignore", over="ignore"):
            d = uv - obs_px[rows][None]
            e2 = d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]
            inl = usable[None] & (z > 0) & (e2 <= tau2)
        score = np.where(inl, e2, tau2).sum(axis=1)
        srt = np.lexsort((slots, score))
        w = srt[0]
        res.best[g], res.slot[g] = score[w], slots[w]
        if len(srt) > 1:
            res.second[g] = score[srt[1]]
        cons = inl[w]
        if cons.sum() < min_inliers:
            res.status[g] = STATUS_NO_CONSENSUS
            continue
        res.inlier[rows[cons]] = True
        res.n_inliers[g] = int(cons.sum())
        res.hyp[g] = np.concatenate([Rs[w].ravel(), ts[w]])
        crow = rows[cons]
        q0 = np.concatenate([rot_log(Rs[w]), ts[w]])
        q, rmse, st = refine_pose(cam, q0, pts[obs_pt[crow]], obs_px[crow], max_iter=max_iter, xtol=xtol)
        res.pose[g], res.rmse_px[g], res.status[g] = q, rmse, st
        if st != STATUS_NOT_PD:
            res.cov[g] = pose_covariance(cam, q, pts[obs_pt[crow]], obs_px[crow], obs_pt[crow], pixel_sigma, pcov)
    return res
