"""CPU oracle of robust triangulation with calibrated cameras: view-pair consensus, then refinement and covariance on the
consensus rows (``cb_triangulate_robust``, DESIGN.md section 4.8).

TEST INFRASTRUCTURE ONLY — the product (caliscope_b200/) never imports this module.

Inside a group of k rows (key-sorted, caller order within a key, positions 0..k-1):
  1. k < 2: status 1.
  2. Candidate pairs: the pairs i < j ranked lexicographically, rank(i, j) = i k - i (i + 1) / 2 + (j - i - 1),
     T = k (k - 1) / 2.  Every rank when T <= max_pairs, else floor(m T / max_pairs) for m = 0..max_pairs-1 (exact
     integers; no random sampling).
  3. Hypothesis of a pair: none when both rows come from one camera; else the DLT point of the two rows (normal matrix on
     the float32-rounded undistorted coordinates, its smallest eigenvector, de-homogenised); none when that is not
     finite or has Xc.z <= 0 in either of the pair's cameras.
  4. Score (MSAC): sum over all k rows of min(e_r^2, tau^2), e_r = |pi(X; c_r) - u_r| in raw pixels; a row with
     Xc.z <= 0 or a non-finite e_r adds tau^2; no hypothesis scores +inf.
  5. Selection: the lowest score, the lowest rank on a tie.
  6. Consensus set: the rows with Xc.z > 0 and e_r <= tau (compared as e_r^2 <= tau^2) at the selected hypothesis.  No
     hypothesis, or fewer than min_inliers rows: status 5 (xyz, cov, rmse NaN, n_inliers 0, no row inlier).
  7. ``refine_points`` and ``point_covariance`` on the consensus rows, from the selected hypothesis; statuses 2, 3, 4 keep
     their meaning (for 2, xyz is the hypothesis).  One consensus round: rows are not re-classified at the refined
     point.  In a two-view group an error along the epipolar line cannot be seen.
Status, first match wins: 1, 5, 2, 3, 4, 0.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from oracle.triangulation import undistort_points
from oracle.triangulation_refine import (STATUS_FEW_ROWS, _group_rig, dlt_camera_models, group_rows, point_covariance,
                                         refine_points)  # fmt: skip

STATUS_NO_CONSENSUS = 5


def candidate_pairs(k: int, max_pairs: int) -> np.ndarray:
    """Ranks of the candidate pairs of a group of k rows, ascending (int64)."""
    T = k * (k - 1) // 2
    if T <= max_pairs:
        return np.arange(T, dtype=np.int64)
    return np.array([m * T // max_pairs for m in range(max_pairs)], dtype=np.int64)  # Python ints: exact


def pair_rank(i, j, k):
    i, j = np.asarray(i, np.int64), np.asarray(j, np.int64)
    return i * k - i * (i + 1) // 2 + (j - i - 1)


def unrank_pair(r, k):
    """Positions (i, j) of lexicographic ranks r in a group of k rows."""
    r = np.asarray(r, np.int64)
    base = pair_rank(np.arange(max(k - 1, 1)), np.arange(max(k - 1, 1)) + 1, k)  # rank of (i, i + 1)
    i = np.searchsorted(base, r, side="right") - 1
    return i, r - base[i] + i + 1


def _camera_poses(cam_flags, cam_x):
    from oracle.ba_oracle import rodrigues

    flags = np.asarray(cam_flags, np.int32)
    offs = np.concatenate([[0], np.cumsum(np.where(flags & 1, 9, 6))])
    cam_x = np.asarray(cam_x, np.float64)
    R = rodrigues(np.stack([cam_x[o : o + 3] for o in offs[:-1]]))
    t = np.stack([cam_x[o + 3 : o + 6] for o in offs[:-1]])
    return R, t


def undistorted_coordinates(cam_flags, cam_const, cam_x, obs_cam, obs_px):
    """Float32-rounded normalised coordinates of every row, as ``dlt_start`` forms them."""
    _, mats, dists, fish = dlt_camera_models(cam_flags, cam_const, cam_x)
    obs_cam = np.asarray(obs_cam)
    norm = np.empty((len(obs_cam), 2))
    for c in np.unique(obs_cam):
        m = obs_cam == c
        norm[m] = undistort_points(np.asarray(obs_px)[m], mats[c], dists[c], bool(fish[c]))
    return norm


def pair_hypotheses(cam_flags, cam_const, cam_x, obs_cam, norm, row_i, row_j):
    """DLT points (m, 3) of the row pairs (row_i, row_j) and whether each is a hypothesis (distinct cameras, finite, in
    front of both cameras)."""
    proj = dlt_camera_models(cam_flags, cam_const, cam_x)[0]
    obs_cam = np.asarray(obs_cam)
    M = np.zeros((len(row_i), 4, 4))
    for r in (row_i, row_j):
        P = proj[obs_cam[r]]
        a = norm[r, 0, None] * P[:, 2] - P[:, 0]
        b = norm[r, 1, None] * P[:, 2] - P[:, 1]
        M += a[:, :, None] * a[:, None, :] + b[:, :, None] * b[:, None, :]
    with np.errstate(invalid="ignore", divide="ignore"):
        w = np.linalg.eigh(M)[1][:, :, 0]
        X = w[:, :3] / w[:, 3:4]
    R, t = _camera_poses(cam_flags, cam_x)
    ok = (obs_cam[row_i] != obs_cam[row_j]) & np.isfinite(X).all(axis=1)
    Xs = np.where(ok[:, None], X, 0.0)
    for r in (row_i, row_j):
        z = np.einsum("nj,nj->n", R[obs_cam[r], 2], Xs) + t[obs_cam[r], 2]
        ok &= z > 0
    return X, ok


def row_errors(cam_flags, cam_const, cam_x, obs_cam, obs_px, rows, X):
    """Squared pixel error e^2 and Xc.z of each row of ``rows`` at the point X of the same index."""
    from oracle.ba_oracle import _project

    rows = np.asarray(rows, np.int64)
    X = np.asarray(X, np.float64).reshape(-1, 3)
    cams = np.asarray(obs_cam)[rows]
    rig = _group_rig(cam_flags, cam_const, cams, np.asarray(obs_px, np.float64)[rows], np.arange(len(rows)), len(rows))
    x = np.concatenate([np.asarray(cam_x, np.float64)[: rig.n_camera_params], X.ravel()])
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        uv, _ = _project(x, rig, False)
        d = uv - rig.obs_xy
        e2 = d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]
    R, t = _camera_poses(cam_flags, cam_x)
    z = np.einsum("nj,nj->n", R[cams, 2], X) + t[cams, 2]
    return e2, z


def msac_cost(e2, z, tau):
    """Per row: e^2 for an inlier (Xc.z > 0 and e^2 <= tau^2), tau^2 otherwise."""
    tau2 = tau * tau
    inl = (z > 0) & (e2 <= tau2)
    return np.where(inl, e2, tau2), inl


@dataclass
class Consensus:
    hyp: np.ndarray  # (G, 3) selected hypothesis (NaN without consensus)
    best: np.ndarray  # (G,) lowest score (+inf: no hypothesis)
    second: np.ndarray  # (G,) second-lowest score (+inf when there is none)
    rank: np.ndarray  # (G,) rank of the selected pair (-1: none)
    n_hyp: np.ndarray  # (G,) number of candidate pairs
    inlier: np.ndarray  # (n,) bool, caller order
    n_inliers: np.ndarray  # (G,)
    status: np.ndarray  # (G,) 0, 1 or 5
    count: np.ndarray  # (G,)


def consensus(cam_flags, cam_const, cam_x, obs_cam, obs_px, obs_key, *, threshold_px, min_inliers=2, max_pairs=64):
    """Steps 1-6 for every group."""
    obs_cam = np.asarray(obs_cam)
    obs_px = np.asarray(obs_px, np.float64).reshape(-1, 2)
    grp, G = group_rows(obs_key)
    order = np.argsort(grp, kind="stable")  # key-sorted rows, caller order within a key
    bounds = np.searchsorted(grp[order], np.arange(G + 1))
    count = np.diff(bounds)
    norm = undistorted_coordinates(cam_flags, cam_const, cam_x, obs_cam, obs_px)
    # every candidate pair of every group: group, rank, caller rows
    hg, hr, ri, rj = [], [], [], []
    for g in range(G):
        k = int(count[g])
        r = candidate_pairs(k, max_pairs)
        if len(r) == 0:
            continue
        i, j = unrank_pair(r, k)
        hg.append(np.full(len(r), g))
        hr.append(r)
        ri.append(order[bounds[g] + i])
        rj.append(order[bounds[g] + j])
    n_hyp = np.zeros(G, np.int64)
    best = np.full(G, np.inf)
    second = np.full(G, np.inf)
    rank = np.full(G, -1, np.int64)
    hyp = np.full((G, 3), np.nan)
    if hg:
        hg, hr, ri, rj = (np.concatenate(v) for v in (hg, hr, ri, rj))
        n_hyp = np.bincount(hg, minlength=G)
        X, ok = pair_hypotheses(cam_flags, cam_const, cam_x, obs_cam, norm, ri, rj)
        score = np.full(len(hg), np.inf)
        v = np.flatnonzero(ok)
        # every (valid hypothesis, row of its group) evaluation
        k_v = count[hg[v]]
        ev_h = np.repeat(v, k_v)
        first = np.repeat(bounds[hg[v]], k_v)
        ev_pos = first + (np.arange(len(ev_h)) - np.repeat(np.cumsum(k_v) - k_v, k_v))
        e2, z = row_errors(cam_flags, cam_const, cam_x, obs_cam, obs_px, order[ev_pos], X[ev_h])
        cost, _ = msac_cost(e2, z, threshold_px)
        score[v] = np.bincount(np.searchsorted(v, ev_h), weights=cost, minlength=len(v))
        srt = np.lexsort((hr, score, hg))  # by group, score, rank
        gs = hg[srt]
        head = np.flatnonzero(np.r_[True, gs[1:] != gs[:-1]])
        bi = srt[head]
        best[hg[bi]] = score[bi]
        rank[hg[bi]] = hr[bi]
        hyp[hg[bi]] = X[bi]
        nxt = head + 1
        has2 = (nxt < len(srt)) & (gs[np.minimum(nxt, len(srt) - 1)] == gs[head])
        second[gs[head[has2]]] = score[srt[nxt[has2]]]
    found = np.isfinite(best)
    # classification at the selected hypothesis
    inlier = np.zeros(len(obs_cam), bool)
    rows_f = np.flatnonzero(found[grp])
    if len(rows_f):
        e2, z = row_errors(cam_flags, cam_const, cam_x, obs_cam, obs_px, rows_f, hyp[grp[rows_f]])
        inlier[rows_f] = msac_cost(e2, z, threshold_px)[1]
    n_in = np.bincount(grp, weights=inlier, minlength=G).astype(np.int64)
    ok_g = found & (n_in >= min_inliers)
    inlier &= ok_g[grp]
    n_in[~ok_g] = 0
    hyp[~ok_g] = np.nan
    status = np.where(count < 2, STATUS_FEW_ROWS, np.where(ok_g, 0, STATUS_NO_CONSENSUS))
    return Consensus(hyp=hyp, best=best, second=second, rank=rank, n_hyp=n_hyp, inlier=inlier, n_inliers=n_in,
                     status=status, count=count)  # fmt: skip


@dataclass
class RobustResult:
    xyz: np.ndarray
    cov: np.ndarray
    rmse_px: np.ndarray
    status: np.ndarray
    consensus: Consensus


def robust_points(cam_flags, cam_const, cam_x, obs_cam, obs_px, obs_key, *, threshold_px, min_inliers=2, max_pairs=64,
                  pixel_sigma=1.0, cam_cov=None, max_iter=20, xtol=1e-12):
    """Steps 1-7: consensus, then ``refine_points`` and ``point_covariance`` on the consensus rows from the selected
    hypothesis, with the status rule 1, 5, 2, 3, 4, 0."""
    obs_cam = np.asarray(obs_cam)
    obs_px = np.asarray(obs_px, np.float64).reshape(-1, 2)
    cs = consensus(cam_flags, cam_const, cam_x, obs_cam, obs_px, obs_key, threshold_px=threshold_px,
                   min_inliers=min_inliers, max_pairs=max_pairs)  # fmt: skip
    grp, G = group_rows(obs_key)
    rows = np.flatnonzero(cs.inlier)
    args = (cam_flags, cam_const, cam_x, obs_cam[rows], obs_px[rows], grp[rows])
    xyz, rmse, st_r, _ = refine_points(*args, cs.hyp, max_iter=max_iter, xtol=xtol)
    cov = point_covariance(*args, xyz, st_r, pixel_sigma, cam_cov)
    status = np.where(cs.status == STATUS_NO_CONSENSUS, STATUS_NO_CONSENSUS, st_r)
    return RobustResult(xyz=xyz, cov=cov, rmse_px=rmse, status=status, consensus=cs)
