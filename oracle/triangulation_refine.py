"""CPU oracle of triangulation with calibrated cameras to the pixel reprojection optimum, and of the first-order
covariance of each point (``cb_triangulate_refine``, DESIGN.md section 4.7).

TEST INFRASTRUCTURE ONLY — the product (caliscope_b200/) never imports this module.

Cameras are given in the bundle-adjustment layout (cam_flags, cam_const, the camera section of x).  The projection and
its derivatives are ``ba_oracle``'s, on a ``Rig`` in which every group is one point; the DLT start reuses
``oracle.triangulation.undistort_points``.
"""
from __future__ import annotations

import numpy as np

from oracle.triangulation import undistort_points
REFINE_LAMBDA0 = 1e-3
PD_RTOL = 1e-12
STATUS_OK, STATUS_FEW_ROWS, STATUS_NOT_PD, STATUS_MAX_ITER, STATUS_BEHIND = 0, 1, 2, 3, 4


def _group_rig(cam_flags, cam_const, obs_cam, obs_px, group, n_groups):
    from oracle.ba_oracle import Rig

    return Rig(cam_flags, cam_const, n_groups, obs_cam, np.asarray(group, np.int32), obs_px)


def pixel_jacobians(cam_flags, cam_const, cam_x, obs_cam, obs_px, group, xyz):
    """Per row at the points ``xyz`` (one per group): residual pi(X; c) - u (n,2), d pi / d X (n,2,3) and d pi / d c
    (n,2,9; columns r t s k1 k2, the last three zero for locked cameras), all in pixels."""
    from oracle.ba_oracle import jacobian_blocks, _project

    xyz = np.asarray(xyz, dtype=np.float64).reshape(-1, 3)
    rig = _group_rig(cam_flags, cam_const, obs_cam, obs_px, group, len(xyz))
    x = np.concatenate([np.asarray(cam_x, np.float64)[: rig.n_camera_params], xyz.ravel()])
    uv, _ = _project(x, rig, False)
    Jc, JX = jacobian_blocks(x, rig)
    fx0 = rig.cam_const[rig.obs_cam, 0][:, None, None]
    return uv - rig.obs_xy, JX * fx0, Jc * fx0


def _normal_eq(cam_flags, cam_const, cam_x, obs_cam, obs_px, group, xyz):
    r, JX, _ = pixel_jacobians(cam_flags, cam_const, cam_x, obs_cam, obs_px, group, xyz)
    G = len(xyz)
    H = np.zeros((G, 3, 3))
    g = np.zeros((G, 3))
    np.add.at(H, group, np.einsum("nki,nkj->nij", JX, JX))
    np.add.at(g, group, np.einsum("nki,nk->ni", JX, r))
    cost = np.bincount(group, weights=(r * r).sum(axis=1), minlength=G)
    return cost, H, g


def chol_pd(H):
    """The positive-definiteness rule of the kernel: every Cholesky pivot of H above PD_RTOL times H's largest diagonal
    entry (NaN fails)."""
    d = np.fmax(np.fmax(H[:, 0, 0], H[:, 1, 1]), H[:, 2, 2])
    thr = PD_RTOL * d
    with np.errstate(invalid="ignore", divide="ignore"):
        p0 = H[:, 0, 0]
        l0 = np.sqrt(p0)
        l1, l2 = H[:, 0, 1] / l0, H[:, 0, 2] / l0
        p1 = H[:, 1, 1] - l1 * l1
        l4 = (H[:, 1, 2] - l2 * l1) / np.sqrt(p1)
        p2 = H[:, 2, 2] - l2 * l2 - l4 * l4
    return (p0 > thr) & (p1 > thr) & (p2 > thr)


def group_rows(obs_key):
    """(group index per row, number of groups), groups in ascending key order."""
    keys, group = np.unique(np.asarray(obs_key, np.int64), return_inverse=True)
    return group.astype(np.int64).ravel(), len(keys)


def dlt_camera_models(cam_flags, cam_const, cam_x):
    """The DLT start's inputs derived from the BA layout: normalised [R|t] (n,3,4), camera matrices (n,3,3) with
    f = s fx0, distortion vectors and fisheye flags (the ``undistort=`` argument of ``triangulate_groups``)."""
    from oracle.ba_oracle import rodrigues

    flags = np.asarray(cam_flags, np.int32)
    const = np.asarray(cam_const, np.float64).reshape(-1, 9)
    cam_x = np.asarray(cam_x, np.float64)
    proj, mats, dists = [], [], []
    o = 0
    for c in range(len(flags)):
        free = bool(flags[c] & 1)
        q = cam_x[o : o + (9 if free else 6)]
        o += 9 if free else 6
        s, k1, k2 = (q[6], q[7], q[8]) if free else (1.0, const[c, 4], const[c, 5])
        proj.append(np.hstack([rodrigues(q[:3])[0], q[3:6, None]]))
        mats.append(np.array([[s * const[c, 0], 0.0, const[c, 2]], [0.0, s * const[c, 1], const[c, 3]], [0.0, 0.0, 1.0]]))
        fish = bool(flags[c] & 2)
        dists.append(np.array([k1, k2, const[c, 6], const[c, 7]] if fish else [k1, k2, const[c, 6], const[c, 7], const[c, 8]]))
    return np.array(proj), np.array(mats), dists, (flags & 2 != 0).astype(np.int32)


def dlt_start(cam_flags, cam_const, cam_x, obs_cam, obs_px, group, n_groups):
    """The DLT point of every group (NaN with fewer than 2 rows) from float32-rounded undistorted coordinates."""
    proj, mats, dists, fish = dlt_camera_models(cam_flags, cam_const, cam_x)
    obs_cam = np.asarray(obs_cam)
    norm = np.empty((len(obs_cam), 2))
    for c in np.unique(obs_cam):
        m = obs_cam == c
        norm[m] = undistort_points(np.asarray(obs_px)[m], mats[c], dists[c], bool(fish[c]))
    out = np.full((n_groups, 3), np.nan)
    order = np.argsort(group, kind="stable")
    bounds = np.searchsorted(group[order], np.arange(n_groups + 1))
    for gi in range(n_groups):
        rows = order[bounds[gi] : bounds[gi + 1]]
        if len(rows) < 2:
            continue
        A = np.empty((2 * len(rows), 4))
        for j, r in enumerate(rows):
            P = proj[obs_cam[r]]
            A[2 * j] = norm[r, 0] * P[2] - P[0]
            A[2 * j + 1] = norm[r, 1] * P[2] - P[1]
        w = np.linalg.svd(A)[2][-1]
        out[gi] = w[:3] / w[3]
    return out


def refine_points(cam_flags, cam_const, cam_x, obs_cam, obs_px, group, x_start, *, max_iter=20, xtol=1e-12):
    """Per group, Levenberg-Marquardt on sum_i |pi(X; c_i) - u_i|^2 (pixels) from x_start, the rule of tri_refine_kernel:
      H, g, cost at the start; status 1 with < 2 rows, else 2 when H fails chol_pd.  lam = REFINE_LAMBDA0.  Repeat:
      if max_iter steps were taken, status 3 and stop; solve (H + lam diag H) d = -g; evaluate at X + d; accept when the
      cost is lower (lam /= 10; H, g, cost from X + d), else lam *= 10; stop when |d| <= xtol (|X| + xtol), |X| before
      the step.  At the end status 2 when H (at the solution) fails chol_pd (xyz = the start), else 4 (from 0) when some
      row has Xc.z <= 0.  Returns xyz, rmse_px (sqrt(cost / rows); at the start for status 2, NaN for 1), status and
      the number of steps."""
    from oracle.ba_oracle import rodrigues

    group = np.asarray(group, np.int64)
    X0 = np.asarray(x_start, np.float64).reshape(-1, 3)
    G = len(X0)
    args = (cam_flags, cam_const, cam_x, obs_cam, obs_px, group)
    count = np.bincount(group, minlength=G)
    X = np.where((count >= 2)[:, None], X0, 0.0)
    cost, H, g = _normal_eq(*args, X)
    cost0 = cost.copy()
    status = np.where(count < 2, STATUS_FEW_ROWS, STATUS_OK)
    status[(status == STATUS_OK) & ~chol_pd(H)] = STATUS_NOT_PD
    active = status == STATUS_OK
    lam = np.full(G, REFINE_LAMBDA0)
    it = np.zeros(G, np.int64)
    eye = np.eye(3)[None]
    while active.any():
        hit = active & (it == max_iter)
        status[hit] = STATUS_MAX_ITER
        active &= ~hit
        if not active.any():
            break
        A = H + lam[:, None, None] * (H * eye)
        d = np.zeros((G, 3))
        d[active] = np.linalg.solve(A[active], -g[active][:, :, None])[:, :, 0]
        Xt = X + d
        ct, Ht, gt = _normal_eq(*args, Xt)
        it[active] += 1
        acc = active & (ct < cost)
        rej = active & ~acc
        conv = active & (np.linalg.norm(d, axis=1) <= xtol * (np.linalg.norm(X, axis=1) + xtol))
        X[acc], cost[acc], H[acc], g[acc] = Xt[acc], ct[acc], Ht[acc], gt[acc]
        lam[acc] /= 10.0
        lam[rej] *= 10.0
        active &= ~conv
    fin = (status == STATUS_OK) | (status == STATUS_MAX_ITER)
    status[fin & ~chol_pd(H)] = STATUS_NOT_PD
    at_start = (status == STATUS_FEW_ROWS) | (status == STATUS_NOT_PD)
    xyz = np.where(at_start[:, None], X0, X)
    # behind a camera at the solution
    flags = np.asarray(cam_flags, np.int32)
    offs = np.concatenate([[0], np.cumsum(np.where(flags & 1, 9, 6))])
    cam_x = np.asarray(cam_x, np.float64)
    R = rodrigues(np.stack([cam_x[o : o + 3] for o in offs[:-1]]))
    t = np.stack([cam_x[o + 3 : o + 6] for o in offs[:-1]])
    oc = np.asarray(obs_cam)
    z = np.einsum("nj,nj->n", R[oc, 2], X[group]) + t[oc, 2]
    behind = np.bincount(group, weights=(~(z > 0)).astype(np.float64), minlength=G) > 0
    status[(status == STATUS_OK) & behind] = STATUS_BEHIND
    with np.errstate(invalid="ignore", divide="ignore"):
        rmse = np.sqrt(np.where(at_start, cost0, cost) / count)
    rmse[status == STATUS_FEW_ROWS] = np.nan
    return xyz, rmse, status, it


def point_covariance(cam_flags, cam_const, cam_x, obs_cam, obs_px, group, xyz, status, pixel_sigma, cam_cov=None):
    """First-order covariance of each refined point: pixel_sigma^2 H^-1 + H^-1 G cam_cov G^T H^-1 with H = sum J_X^T J_X
    and G = sum J_X^T J_c (3 x n_camera_params, pixels); cam_cov in x's camera layout.  NaN for status 1 and 2."""
    xyz = np.asarray(xyz, np.float64).reshape(-1, 3)
    G_ = len(xyz)
    ok = (status != STATUS_FEW_ROWS) & (status != STATUS_NOT_PD)
    Xe = np.where(ok[:, None], xyz, 0.0)
    _, JX, Jc = pixel_jacobians(cam_flags, cam_const, cam_x, obs_cam, obs_px, group, Xe)
    H = np.zeros((G_, 3, 3))
    np.add.at(H, group, np.einsum("nki,nkj->nij", JX, JX))
    out = np.full((G_, 3, 3), np.nan)
    Hi = np.linalg.inv(H[ok])
    cov = pixel_sigma**2 * Hi
    if cam_cov is not None:
        flags = np.asarray(cam_flags, np.int32)
        widths = np.where(flags & 1, 9, 6)
        offs = np.concatenate([[0], np.cumsum(widths)])
        ncp = int(offs[-1])
        Gm = np.zeros((G_, 3, ncp))
        B = np.einsum("nki,nkj->nij", JX, Jc)  # (n, 3, 9)
        oc = np.asarray(obs_cam)
        for q in range(9):
            m = q < widths[oc]
            np.add.at(Gm, (group[m], slice(None), offs[oc[m]] + q), B[m, :, q])
        Gk = Gm[ok]
        cov = cov + Hi @ Gk @ np.asarray(cam_cov, np.float64) @ np.transpose(Gk, (0, 2, 1)) @ Hi
    out[ok] = 0.5 * (cov + np.transpose(cov, (0, 2, 1)))
    return out
