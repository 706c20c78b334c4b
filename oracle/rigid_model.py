"""CPU oracle of the refinement of a rigid body's marker layout from tracked frames: one Levenberg-Marquardt over the
layout and every frame pose with the frames eliminated, and the layout's covariance (``cb_rigid_model_refine``,
DESIGN.md section 4.15).

TEST INFRASTRUCTURE ONLY — the product (caliscope_b200/) never imports this module.

Cameras in the bundle-adjustment layout (cam_flags, cam_const, the camera section of x), an optional camera_cov
(n_camera_params^2); the start layout model_xyz (n_model, 3), X_w = R(r_f) M_k + t_f; observations obs_cam, obs_key,
obs_pt (the model point of the row), obs_px (raw pixels); keys are non-negative (the engine refuses a negative
obs_key, as every call that groups rows by key does; this oracle does not check it); start poses (keys strictly
ascending, poses (n, 6) finite); body_start (n_bodies + 1): model points body_start[b] .. body_start[b+1]-1 are
body b, 3 <= K <= 32.  A frame is the rows of one obs_key; all its rows belong to one body.
  1. Frames.  A frame is used when it has a finite start pose, at least 4 rows and at least 3 distinct markers among
     them; otherwise its status is 1 and its rows take no part.  A body's status is 1 when it has no used frame, or
     when one of its markers has no row in a used frame; its layout is then the start, its cov NaN and its frames'
     poses the start.
  2. Residuals.  Over body b's rows in used frames: the projection of R(r_f) M_k + t_f with the row's own camera, minus
     the raw pixel, in pixels (the engine's projection, as in section 4.14).
  3. Gauge.  The layout is fixed up to a rigid motion, which the frame poses absorb; calibrated cameras fix the scale,
     so the gauge has 6 dof.  It is held by inner constraints on the start layout M0:
     sum_k (M_k - M0_k) = 0 and sum_k (M0_k - mean M0) x (M_k - M0_k) = 0, i.e. steps dM lie in the null space of
     C^T, C (3K x 6) = [I_3 | [M0_k - mean M0]x] per marker.  The result keeps the start's centroid and has no net
     rotation against it (the first-order conditions of a Kabsch fit of the result onto the start).
  4. Step.  The damped normal equations in the original parameters, H_MM + lam diag(H_MM) and H_ff + lam diag(H_ff) per
     frame; every frame eliminated into S_lam = H_MM,lam - sum_f H_Mf H_ff,lam^-1 H_fM; the layout step is the
     constrained minimiser dM = -N (N^T S_lam N)^-1 N^T b for a basis N of null(C^T) (the result does not depend on
     the choice of N); each frame's step by back-substitution.  Acceptance and stopping as intr_lm_kernel: lam0 = 1e-3,
     / 10 on a lower cost, * 10 otherwise; stop when |d| <= xtol (|x| + xtol) with d and x over the layout and every
     frame pose of the body (x before the step); max_iter steps at most; a damped block that is not positive definite
     is a rejected step.
  5. Covariance at the solution (lam = 0), P = N (N^T S N)^-1 N^T: cov = pixel_sigma^2 P + P G Sigma_c G^T P, with
     G = sum_f (G_M,f - H_Mf H_ff^-1 G_f) the Schur-reduced cross term to the camera parameters and G_.,f = sum over the
     frame's rows of J_.^T J_c in pixels; without camera_cov the first term alone.  Cross-body correlation through the
     cameras is not given.
  6. Status, first match wins: 1 (step 1); 2 (N^T S N fails the Jacobi-scaled Cholesky pivot test, pivots > 1e-12, at
     the start or at the solution: layout and poses are the start, cov and rmse NaN); 3 (max_iter reached); 4 (a row
     behind its camera at the solution); 0.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from oracle.rigid_pose_robust import body_jacobians
from oracle.triangulation_robust import row_errors

LAMBDA0 = 1e-3
PD_RTOL = 1e-12
KMIN, KMAX = 3, 32
STATUS_OK, STATUS_UNUSED, STATUS_NOT_PD, STATUS_MAX_ITER, STATUS_BEHIND = 0, 1, 2, 3, 4
__all__ = ["gauge_constraints", "gauge_basis", "model_covariance", "frame_table", "refine_body_model", "rigid_model_refine", "RigidModelResult"]


def _skew(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def gauge_constraints(M0):
    """C (3K x 6) of step 3."""
    M0 = np.asarray(M0, np.float64).reshape(-1, 3)
    d = M0 - M0.mean(axis=0)
    return np.concatenate([np.concatenate([np.eye(3), _skew(dk)], axis=1) for dk in d], axis=0)


def gauge_basis(M0):
    """An orthonormal basis N (3K x (3K - 6)) of null(C^T)."""
    C = gauge_constraints(M0)
    Q, _ = np.linalg.qr(C, mode="complete")
    return Q[:, 6:]


def frame_table(obs_key, obs_pt, start_key, start_pose):
    """Step 1's frame test: (keys ascending, rows per key (list of arrays, caller order), start pose or NaN, used)."""
    obs_key = np.asarray(obs_key, np.int64)
    keys, inv = np.unique(obs_key, return_inverse=True)
    order = np.argsort(inv, kind="stable")
    bounds = np.searchsorted(inv[order], np.arange(len(keys) + 1))
    rows = [order[bounds[i] : bounds[i + 1]] for i in range(len(keys))]
    sk = np.asarray(start_key, np.int64)
    sp = np.asarray(start_pose, np.float64).reshape(-1, 6)
    pose = np.full((len(keys), 6), np.nan)
    i = np.searchsorted(sk, keys)
    hit = (i < len(sk)) & (sk[np.minimum(i, len(sk) - 1)] == keys) if len(sk) else np.zeros(len(keys), bool)
    pose[hit] = sp[i[hit]]
    pts = np.asarray(obs_pt, np.int64)
    used = np.array([np.isfinite(pose[f]).all() and len(r) >= 4 and len(np.unique(pts[r])) >= 3
                     for f, r in enumerate(rows)], bool)  # fmt: skip
    return keys, rows, pose, used


def _frame_blocks(cams, oc, px, M_rows, k_rows, K, q):
    """One frame's residual (n, 2) and blocks: J_M scattered to the layout (n, 2, 3K), J_q (n, 2, 6), J_c."""
    from oracle.ba_oracle import rodrigues

    r, Jq, Jc = body_jacobians(*cams, oc, px, M_rows, q)
    R = rodrigues(q[:3])[0]
    JM = Jq[:, :, 3:6] @ R  # d pi / d M = J_X R
    JMf = np.zeros((len(r), 2, 3 * K))
    for i, k in enumerate(k_rows):
        JMf[i, :, 3 * k : 3 * k + 3] = JM[i]
    return r, JMf, Jq, Jc


def _normal(cams, frames, M, poses, K):
    """Per frame (cost, H_MM (3K^2), H_Mf (3K x 6), H_ff, b_M, b_f)."""
    out = []
    for f, (oc, px, k_rows) in enumerate(frames):
        r, JM, Jq, _ = _frame_blocks(cams, oc, px, M[k_rows], k_rows, K, poses[f])
        out.append((float((r * r).sum()), np.einsum("nki,nkj->ij", JM, JM), np.einsum("nki,nkj->ij", JM, Jq),
                    np.einsum("nki,nkj->ij", Jq, Jq), np.einsum("nki,nk->i", JM, r), np.einsum("nki,nk->i", Jq, r)))
    return out


def _schur(blocks, lam, K):
    """(S_lam, b reduced, ok): the frames eliminated at damping lam."""
    S = np.zeros((3 * K, 3 * K))
    b = np.zeros(3 * K)
    for _, Hmm, Hmf, Hff, bm, bf in blocks:
        S += Hmm + lam * np.diag(np.diag(Hmm))
        V = Hff + lam * np.diag(np.diag(Hff))
        try:
            L = np.linalg.cholesky(V)
        except np.linalg.LinAlgError:
            return S, b, False
        X = np.linalg.solve(L.T, np.linalg.solve(L, Hmf.T))  # V^-1 H_fM
        S -= Hmf @ X
        b += bm - X.T @ bf
    return S, b, True


def pd_scaled(A) -> bool:
    """Every Cholesky pivot of the Jacobi-scaled D^-1/2 A D^-1/2 above PD_RTOL (NaN fails)."""
    A = np.asarray(A, np.float64)
    n = len(A)
    with np.errstate(divide="ignore", invalid="ignore"):
        s = 1.0 / np.sqrt(np.diag(A))
        A = A * s[:, None] * s[None, :]
        L = np.zeros((n, n))
        for j in range(n):
            d = A[j, j] - L[j, :j] @ L[j, :j]
            if not d > PD_RTOL:
                return False
            L[j, j] = np.sqrt(d)
            L[j + 1 :, j] = (A[j + 1 :, j] - L[j + 1 :, :j] @ L[j, :j]) / L[j, j]
    return True


def _chol_ok(A):
    try:
        np.linalg.cholesky(A)
        return bool(np.isfinite(A).all())
    except np.linalg.LinAlgError:
        return False


def refine_body_model(cams, frames, M0, poses0, *, max_iter=100, xtol=1e-12):
    """Steps 3, 4 and the status-2/3 tests of step 6 for one body.  frames: per used frame (obs_cam, obs_px, marker
    index in the body per row).  Returns (M, poses, iterations, status in {0, 2, 3}, N, blocks at the result)."""
    K = len(M0)
    N = gauge_basis(M0)
    M, poses = M0.copy(), poses0.copy()
    blocks = _normal(cams, frames, M, poses, K)
    S0, _, ok0 = _schur(blocks, 0.0, K)
    if not (ok0 and pd_scaled(N.T @ S0 @ N)):
        return M0, poses0, 0, STATUS_NOT_PD, N, blocks
    cost = sum(bl[0] for bl in blocks)
    lam, it, status = LAMBDA0, 0, STATUS_OK
    while True:
        S, b, ok = _schur(blocks, lam, K)
        R = N.T @ S @ N
        if not (ok and _chol_ok(R)):
            it += 1
            lam *= 10.0
            if it == max_iter:
                status = STATUS_MAX_ITER
                break
            continue
        dM = -N @ np.linalg.solve(R, N.T @ b)
        dq = np.empty_like(poses)
        for f, (_, Hmm, Hmf, Hff, bm, bf) in enumerate(blocks):
            V = Hff + lam * np.diag(np.diag(Hff))
            dq[f] = -np.linalg.solve(V, bf + Hmf.T @ dM.ravel())
        Mt, pt = M + dM.reshape(-1, 3), poses + dq
        bt = _normal(cams, frames, Mt, pt, K)
        ct = sum(bl[0] for bl in bt)
        it += 1
        dn = np.sqrt((dM * dM).sum() + (dq * dq).sum())
        xn = np.sqrt((M * M).sum() + (poses * poses).sum())
        lower = ct < cost
        done = dn <= xtol * (xn + xtol)
        if not done and it == max_iter:
            status, done = STATUS_MAX_ITER, True
        if lower:
            M, poses, cost, blocks = Mt, pt, ct, bt
            lam *= 0.1
        else:
            lam *= 10.0
        if done:
            break
    S, _, ok = _schur(blocks, 0.0, K)
    if not (ok and pd_scaled(N.T @ S @ N)):
        return M0, poses0, it, STATUS_NOT_PD, N, _normal(cams, frames, M0, poses0, K)
    return M, poses, it, status, N, blocks


def model_covariance(cams, frames, M, poses, N, blocks, pixel_sigma, camera_cov=None):
    """Step 5 for one body at its solution."""
    K = len(M)
    S, _, _ = _schur(blocks, 0.0, K)
    P = N @ np.linalg.inv(N.T @ S @ N) @ N.T
    cov = pixel_sigma**2 * P
    if camera_cov is not None:
        flags = np.asarray(cams[0], np.int32)
        widths = np.where(flags & 1, 9, 6)
        offs = np.concatenate([[0], np.cumsum(widths)])
        G = np.zeros((3 * K, int(offs[-1])))
        for f, (oc, px, k_rows) in enumerate(frames):
            _, JM, Jq, Jc = _frame_blocks(cams, oc, px, M[k_rows], k_rows, K, poses[f])
            Hmf, Hff = blocks[f][2], blocks[f][3]
            X = Hmf @ np.linalg.inv(Hff)
            for i, c in enumerate(oc):
                w = widths[c]
                G[:, offs[c] : offs[c] + w] += (JM[i].T - X @ Jq[i].T) @ Jc[i, :, :w]
        cov = cov + P @ G @ np.asarray(camera_cov, np.float64) @ G.T @ P
    return 0.5 * (cov + cov.T)


@dataclass
class RigidModelResult:
    model: np.ndarray  # (n_model, 3)
    cov: list  # per body (3K, 3K)
    status: np.ndarray  # per body
    iterations: np.ndarray
    rmse_px: np.ndarray
    n_frames: np.ndarray
    n_rows: np.ndarray
    key: np.ndarray  # per frame, ascending
    pose: np.ndarray  # (F, 6)
    frame_rmse_px: np.ndarray
    count: np.ndarray
    frame_status: np.ndarray


def rigid_model_refine(cam_flags, cam_const, cam_x, model_xyz, obs_cam, obs_key, obs_pt, obs_px, start, *,
                       body_start=None, pixel_sigma=1.0, camera_cov=None, max_iter=100,
                       xtol=1e-12) -> RigidModelResult:  # fmt: skip
    """Steps 1-6 for every body.  start: (keys, poses)."""
    cams = (cam_flags, cam_const, cam_x)
    model = np.asarray(model_xyz, np.float64).reshape(-1, 3)
    bs = np.array([0, len(model)]) if body_start is None else np.asarray(body_start, np.int64)
    obs_cam = np.asarray(obs_cam, np.int64)
    obs_pt = np.asarray(obs_pt, np.int64)
    obs_px = np.asarray(obs_px, np.float64).reshape(-1, 2)
    keys, rows, pose0, used = frame_table(obs_key, obs_pt, start[0], start[1])
    F, B = len(keys), len(bs) - 1
    fbody = np.array([np.searchsorted(bs, obs_pt[r[0]], side="right") - 1 for r in rows], np.int64)
    nan = np.nan
    res = RigidModelResult(model=model.copy(), cov=[np.full((3 * (bs[b + 1] - bs[b]),) * 2, nan) for b in range(B)],
                           status=np.full(B, STATUS_UNUSED, np.int32), iterations=np.zeros(B, np.int32),
                           rmse_px=np.full(B, nan), n_frames=np.zeros(B, np.int32), n_rows=np.zeros(B, np.int32),
                           key=keys, pose=pose0.copy(), frame_rmse_px=np.full(F, nan),
                           count=np.array([len(r) for r in rows], np.int32),
                           frame_status=np.full(F, STATUS_UNUSED, np.int32))  # fmt: skip
    for b in range(B):
        lo, K = int(bs[b]), int(bs[b + 1] - bs[b])
        fs = [f for f in range(F) if used[f] and fbody[f] == b]
        res.n_frames[b] = len(fs)
        res.n_rows[b] = sum(len(rows[f]) for f in fs)
        seen = np.zeros(K, bool)
        for f in fs:
            seen[obs_pt[rows[f]] - lo] = True
        if not fs or not seen.all():
            continue
        frames = [(obs_cam[rows[f]], obs_px[rows[f]], obs_pt[rows[f]] - lo) for f in fs]
        M0 = model[lo : lo + K]
        M, poses, it, st, N, blocks = refine_body_model(cams, frames, M0, pose0[fs], max_iter=max_iter, xtol=xtol)
        if st != STATUS_NOT_PD:
            from oracle.ba_oracle import rodrigues

            for f, q in zip(fs, poses):
                Xw = M[obs_pt[rows[f]] - lo] @ rodrigues(q[:3])[0].T + q[3:]
                if not (row_errors(*cams, obs_cam, obs_px, rows[f], Xw)[1] > 0).all():
                    st = STATUS_BEHIND if st == STATUS_OK else st
            res.cov[b] = model_covariance(cams, frames, M, poses, N, blocks, pixel_sigma, camera_cov)
        res.model[lo : lo + K] = M
        res.pose[fs] = poses
        if st != STATUS_NOT_PD:
            costs = np.array([bl[0] for bl in blocks])
            res.frame_rmse_px[fs] = np.sqrt(costs / res.count[fs])
            res.rmse_px[b] = np.sqrt(costs.sum() / res.n_rows[b])
        res.status[b], res.iterations[b] = st, it
        res.frame_status[fs] = st
    return res
