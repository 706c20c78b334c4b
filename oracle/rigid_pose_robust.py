"""CPU oracle of the robust pose of a rigid body seen by a calibrated rig: Horn poses of triangulated model points chosen
by consensus, then refinement of the body pose and its covariance on the consensus rows (``cb_rigid_pose_robust``,
DESIGN.md section 4.14).

TEST INFRASTRUCTURE ONLY — the product (caliscope_b200/) never imports this module.

Cameras in the bundle-adjustment layout (cam_flags, cam_const, the camera section of x), an optional camera_cov
(n_camera_params^2); the body's model model_xyz (n_model, 3) in its own frame, X_w = R(r) M + t; observations obs_cam,
obs_key, obs_pt (the model point of the row), obs_px (raw pixels); optional priors (prior_key strictly ascending,
prior_pose (n_prior, 6) finite).  A group is the rows of one obs_key: one body at one moment, k rows key-sorted and in
caller order within a key.
  1. k < 4: status 1.  A row whose model point is not finite is unusable: it scores tau^2 and is never an inlier.
  2. Point hypotheses: each model point p with rows in the group gets the section 4.8 consensus on those rows (the same
     tau, min_inliers 2, max_pairs): the DLT point of the best view pair, or none (rows all from one camera, or views
     that do not agree; such rows still take part in scoring and refinement).  The qualified points are the points with
     a point hypothesis, positions 0..n_q-1 in ascending model index.
  3. Samples, T = C(n_q, 3): every triple in lexicographic order when T <= max_samples, else section 4.9's splitmix64
     draw.
  4. Pose hypothesis of a sample: Horn's closed-form absolute orientation (JOSA A 4(4), 1987) without scale of the three
     model points against their point hypotheses: q the eigenvector of the largest eigenvalue of Horn's 4 x 4 N,
     R = R(q), t = mean(X) - R mean(M).  None when the model triangle is degenerate,
     |(M_j - M_i) x (M_l - M_i)| <= 1e-9 |M_j - M_i| |M_l - M_i|, or R or t is not finite.  The group's prior, if it
     has one, is slot 0; sample m is slot 1 + m.
  5. Score (MSAC): sum over all k rows of min(e_r^2, tau^2), e_r = |pi(R M_r + t; c_r) - u_r| in raw pixels with each
     row's own camera; a row behind its camera, with a non-finite error or an unusable point adds tau^2.  The lowest
     score wins, the lowest slot on a tie.
  6. Consensus: the usable rows in front of their camera with e_r^2 <= tau^2 at the winner.  No hypothesis, or fewer
     than min_inliers rows: status 5 (pose, cov, rmse NaN, no inlier).  One consensus round.
  7. Levenberg-Marquardt over q = (r, t) on the consensus rows from ``rot_log`` of the winner's R: section 4.9's loop
     (lambda0 1e-3, / 10, * 10, |d| <= xtol (|q| + xtol) with |q| before the step, max_iter), with
     J_q = J_X [d(R(r) M)/dr | I] per row, d(R(r) M)/dr = -R [M]x Jr(r).
  8. Covariance at q*: pixel_sigma^2 H^-1 + H^-1 G camera_cov G^T H^-1, G = sum over the consensus rows of J_q^T J_c
     (6 x n_camera_params, pixels); without camera_cov the first term alone.  It assumes the body's observations are
     independent of those that calibrated the rig, and takes the model as exact.
  9. Status, first match wins: 1, 5, 2 (H fails ``pd6`` at the start or at the solution; pose = the hypothesis, cov NaN),
     3 (max_iter reached), 4 (a consensus row is behind its camera at q*), 0.
"""
from __future__ import annotations

from dataclasses import dataclass
from math import sqrt

import numpy as np

from oracle.resection_robust import STATUS_NO_CONSENSUS, candidate_samples, pd6, rot_log
from oracle.triangulation_refine import (PD_RTOL, REFINE_LAMBDA0, STATUS_BEHIND, STATUS_FEW_ROWS, STATUS_MAX_ITER,
                                         STATUS_NOT_PD, STATUS_OK, group_rows, pixel_jacobians)  # fmt: skip
from oracle.triangulation_robust import consensus, row_errors

DEGENERATE = 1e-9
__all__ = ["PD_RTOL", "STATUS_OK", "STATUS_FEW_ROWS", "STATUS_NOT_PD", "STATUS_MAX_ITER", "STATUS_BEHIND",
           "STATUS_NO_CONSENSUS", "horn", "point_hypotheses", "body_jacobians", "refine_body", "body_covariance",
           "rigid_pose_robust", "RigidResult"]  # fmt: skip


def horn(M, X):
    """Step 4 on model points M (3, 3) and world points X (3, 3): (R, t) or None."""
    M = np.asarray(M, np.float64)
    X = np.asarray(X, np.float64)
    u, v = M[1] - M[0], M[2] - M[0]
    with np.errstate(invalid="ignore", over="ignore"):
        c = np.cross(u, v)
        if not sqrt(c @ c) > DEGENERATE * sqrt(u @ u) * sqrt(v @ v):
            return None
        mb, xb = M.mean(axis=0), X.mean(axis=0)
        S = (M - mb).T @ (X - xb)
        if not np.isfinite(S).all():
            return None
    N = np.array([
        [S[0, 0] + S[1, 1] + S[2, 2], S[1, 2] - S[2, 1], S[2, 0] - S[0, 2], S[0, 1] - S[1, 0]],
        [S[1, 2] - S[2, 1], S[0, 0] - S[1, 1] - S[2, 2], S[0, 1] + S[1, 0], S[2, 0] + S[0, 2]],
        [S[2, 0] - S[0, 2], S[0, 1] + S[1, 0], -S[0, 0] + S[1, 1] - S[2, 2], S[1, 2] + S[2, 1]],
        [S[0, 1] - S[1, 0], S[2, 0] + S[0, 2], S[1, 2] + S[2, 1], -S[0, 0] - S[1, 1] + S[2, 2]],
    ])  # fmt: skip
    w, x, y, z = np.linalg.eigh(N)[1][:, -1]
    R = np.array([
        [w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y)],
        [2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x)],
        [2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z],
    ])  # fmt: skip
    t = xb - R @ mb
    if not (np.isfinite(R).all() and np.isfinite(t).all()):
        return None
    return R, t


def point_hypotheses(cam_flags, cam_const, cam_x, obs_cam, obs_px, grp, obs_pt, n_model, *, threshold_px, max_pairs):
    """Step 2 for every (group, model point) sub-group: (group, point, hypothesis (3,)) of each qualified point, in
    (group, point) order."""
    sub = np.asarray(grp, np.int64) * int(n_model) + np.asarray(obs_pt, np.int64)
    cs = consensus(cam_flags, cam_const, cam_x, obs_cam, obs_px, sub, threshold_px=threshold_px, min_inliers=2,
                   max_pairs=max_pairs)  # fmt: skip
    keys = np.unique(sub)
    ok = cs.status == STATUS_OK
    return keys[ok] // n_model, keys[ok] % n_model, cs.hyp[ok]


def body_jacobians(cam_flags, cam_const, cam_x, obs_cam, obs_px, M, q):
    """Per row at body pose q: residual pi - u (n, 2), J_q (n, 2, 6), J_c (n, 2, 9; columns r t s k1 k2) in pixels."""
    from oracle.ba_oracle import _skew, rodrigues, so3_right_jacobian

    M = np.asarray(M, np.float64).reshape(-1, 3)
    q = np.asarray(q, np.float64)
    R = rodrigues(q[:3])[0]
    Xw = M @ R.T + q[3:]
    n = len(M)
    r, JX, Jc = pixel_jacobians(cam_flags, cam_const, cam_x, obs_cam, obs_px, np.arange(n), Xw)
    dXdr = -R[None] @ _skew(M) @ so3_right_jacobian(q[:3])  # (n, 3, 3)
    return r, np.concatenate([JX @ dXdr, JX], axis=2), Jc


def _normal_eq(cams, obs_cam, obs_px, M, q):
    r, J, _ = body_jacobians(*cams, obs_cam, obs_px, M, q)
    return float((r * r).sum()), np.einsum("nki,nkj->ij", J, J), np.einsum("nki,nk->i", J, r)


def _depths(cams, obs_cam, obs_px, M, q):
    from oracle.ba_oracle import rodrigues

    R = rodrigues(q[:3])[0]
    return row_errors(*cams, obs_cam, obs_px, np.arange(len(M)), np.asarray(M) @ R.T + q[3:])


def refine_body(cam_flags, cam_const, cam_x, obs_cam, obs_px, M, q0, *, max_iter=20, xtol=1e-12):
    """Step 7 on one group's consensus rows: (q, rmse, status in {0, 2, 3, 4})."""
    cams = (cam_flags, cam_const, cam_x)
    q0 = np.asarray(q0, np.float64)
    q = q0.copy()
    cost, H, g = _normal_eq(cams, obs_cam, obs_px, M, q)
    cost0, n = cost, len(M)
    if not pd6(H):
        return q0, sqrt(cost0 / n), STATUS_NOT_PD
    status, lam, it = STATUS_OK, REFINE_LAMBDA0, 0
    while True:
        if it == max_iter:
            status = STATUS_MAX_ITER
            break
        d = np.linalg.solve(H + lam * np.diag(np.diag(H)), -g)
        ct, Ht, gt = _normal_eq(cams, obs_cam, obs_px, M, q + d)
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
    if status == STATUS_OK and not (_depths(cams, obs_cam, obs_px, M, q)[1] > 0).all():
        status = STATUS_BEHIND
    return q, sqrt(cost / n), status


def body_covariance(cam_flags, cam_const, cam_x, obs_cam, obs_px, M, q, pixel_sigma, camera_cov=None):
    """Step 8 at q on one group's consensus rows."""
    _, J, Jc = body_jacobians(cam_flags, cam_const, cam_x, obs_cam, obs_px, M, q)
    Hi = np.linalg.inv(np.einsum("nki,nkj->ij", J, J))
    cov = pixel_sigma**2 * Hi
    if camera_cov is not None:
        widths = np.where(np.asarray(cam_flags, np.int32) & 1, 9, 6)
        offs = np.concatenate([[0], np.cumsum(widths)])
        G = np.zeros((6, int(offs[-1])))
        B = np.einsum("nki,nkj->nij", J, Jc)  # (n, 6, 9)
        oc = np.asarray(obs_cam)
        for i, c in enumerate(oc):
            G[:, offs[c] : offs[c] + widths[c]] += B[i, :, : widths[c]]
        cov = cov + Hi @ G @ np.asarray(camera_cov, np.float64) @ G.T @ Hi
    return 0.5 * (cov + cov.T)


@dataclass
class RigidResult:
    pose: np.ndarray  # (G, 6)
    cov: np.ndarray  # (G, 6, 6)
    rmse_px: np.ndarray
    count: np.ndarray
    n_inliers: np.ndarray
    n_points: np.ndarray
    rep_row: np.ndarray
    status: np.ndarray
    inlier: np.ndarray  # (n,) caller order
    hyp: np.ndarray  # (G, 12) the winner (R row-major, t), NaN without consensus
    slot: np.ndarray  # (G,) the winner's slot, -1 without a hypothesis
    best: np.ndarray  # (G,) lowest score (+inf: no hypothesis)
    second: np.ndarray  # (G,) second-lowest score (+inf: none)


def rigid_pose_robust(cam_flags, cam_const, cam_x, model_xyz, obs_cam, obs_key, obs_pt, obs_px, *, threshold_px,
                      min_inliers=6, max_pairs=16, max_samples=64, prior=None, pixel_sigma=1.0, camera_cov=None,
                      max_iter=20, xtol=1e-12) -> RigidResult:  # fmt: skip
    """Steps 1-9 for every group.  prior: (keys, poses) or None."""
    from oracle.ba_oracle import rodrigues

    cams = (cam_flags, cam_const, cam_x)
    obs_cam = np.asarray(obs_cam, np.int64)
    obs_pt = np.asarray(obs_pt, np.int64)
    obs_key = np.asarray(obs_key, np.int64)
    obs_px = np.asarray(obs_px, np.float64).reshape(-1, 2)
    model = np.asarray(model_xyz, np.float64).reshape(-1, 3)
    tau2 = threshold_px * threshold_px
    grp, G = group_rows(obs_key)
    order = np.argsort(grp, kind="stable")
    bounds = np.searchsorted(grp[order], np.arange(G + 1))
    qg, qm, qx = point_hypotheses(*cams, obs_cam, obs_px, grp, obs_pt, len(model), threshold_px=threshold_px,
                                  max_pairs=max_pairs)  # fmt: skip
    qb = np.searchsorted(qg, np.arange(G + 1))
    pk = np.zeros(0, np.int64) if prior is None else np.asarray(prior[0], np.int64)
    pp = np.zeros((0, 6)) if prior is None else np.asarray(prior[1], np.float64).reshape(-1, 6)
    nan = np.nan
    res = RigidResult(pose=np.full((G, 6), nan), cov=np.full((G, 6, 6), nan), rmse_px=np.full(G, nan),
                      count=np.diff(bounds).astype(np.int32), n_inliers=np.zeros(G, np.int32),
                      n_points=np.diff(qb).astype(np.int32), rep_row=order[bounds[:-1]].astype(np.int32),
                      status=np.zeros(G, np.int32), inlier=np.zeros(len(obs_cam), bool), hyp=np.full((G, 12), nan),
                      slot=np.full(G, -1), best=np.full(G, np.inf), second=np.full(G, np.inf))  # fmt: skip
    for g in range(G):
        rows = order[bounds[g] : bounds[g + 1]]
        k = len(rows)
        if k < 4:
            res.status[g] = STATUS_FEW_ROWS
            continue
        M = model[obs_pt[rows]]
        usable = np.isfinite(M).all(axis=1)
        slots, Rs, ts = [], [], []
        key = obs_key[rows[0]]
        i = np.searchsorted(pk, key)
        if i < len(pk) and pk[i] == key:
            slots.append(0)
            Rs.append(rodrigues(pp[i, :3])[0])
            ts.append(pp[i, 3:])
        QM, QX = model[qm[qb[g] : qb[g + 1]]], qx[qb[g] : qb[g + 1]]
        for m, smp in enumerate(candidate_samples(len(QM), max_samples)):
            if smp is None:
                continue
            sol = horn(QM[list(smp)], QX[list(smp)])
            if sol is not None:
                slots.append(1 + m)
                Rs.append(sol[0])
                ts.append(sol[1])
        if not slots:
            res.status[g] = STATUS_NO_CONSENSUS
            continue
        score, inl = np.empty(len(slots)), np.empty((len(slots), k), bool)
        for h, (R, t) in enumerate(zip(Rs, ts)):
            with np.errstate(invalid="ignore", over="ignore"):
                e2, z = row_errors(*cams, obs_cam, obs_px, rows, M @ R.T + t)
                inl[h] = usable & (z > 0) & (e2 <= tau2)
            score[h] = np.where(inl[h], e2, tau2).sum()
        slots = np.array(slots)
        srt = np.lexsort((slots, score))
        w = srt[0]
        res.best[g], res.slot[g] = score[w], slots[w]
        if len(srt) > 1:
            res.second[g] = score[srt[1]]
        cons = inl[w]
        if cons.sum() < min_inliers:
            res.status[g] = STATUS_NO_CONSENSUS
            continue
        crow = rows[cons]
        res.inlier[crow] = True
        res.n_inliers[g] = int(cons.sum())
        res.hyp[g] = np.concatenate([Rs[w].ravel(), ts[w]])
        q0 = np.concatenate([rot_log(Rs[w]), ts[w]])
        Mc = model[obs_pt[crow]]
        q, rmse, st = refine_body(*cams, obs_cam[crow], obs_px[crow], Mc, q0, max_iter=max_iter, xtol=xtol)
        res.pose[g], res.rmse_px[g], res.status[g] = q, rmse, st
        if st != STATUS_NOT_PD:
            res.cov[g] = body_covariance(*cams, obs_cam[crow], obs_px[crow], Mc, q, pixel_sigma, camera_cov)
    return res
