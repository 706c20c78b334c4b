"""CPU oracle of the robust rigid-body pose with gP3P hypotheses (``cb_rigid_pose_robust_gp3p``, DESIGN.md section
4.14): ``oracle.rigid_pose_robust``'s rule, whose steps 3-4 gain a second sample source in groups with fewer than three
qualified points.

TEST INFRASTRUCTURE ONLY — the product (caliscope_b200/) never imports this module.

Steps 1-2 and 5-9 are ``oracle/rigid_pose_robust.py``'s.  Steps 3-4 there, and in addition:
  3-4 with gp3p_samples > 0 (1..4096), in a group with k >= 4 rows and n_q < 3 (every other group as above):
     samples of three row positions 0..k-1, every triple in lexicographic order when C(k, 3) <= gp3p_samples, else
     section 4.9's splitmix64 draw of gp3p_samples.  A sample gives no hypothesis when two of its rows share a model
     point, a row is unusable (model point not finite, or undistorted coordinate not finite or the fisheye failure
     sentinel), the model triangle is degenerate or the rays are parallel; else oracle/gp3p.py's gp3p on the rows'
     camera centres c_i = -R_i^T t_i, unit rays d_i = R_i^T (x_i, y_i, 1) / |.| of the undistorted normalised
     coordinates and model points: the real roots of the octic in the first depth, each back-substituted, polished by
     Newton on the three distance equations and posed by Horn.  Hypothesis c of sample m is slot 1 + 8 m + c.
     Constants: rays parallel when det(sum (I - d_i d_i^T)) <= 1e-12; Delta_j >= -1e-8 (1 + p_j^2) clamped to 0,
     below it no hypothesis; roots with |u_1| <= 1e9; at most 3 Newton steps.
  9 in a group that gP3P reaches, with status 6 added: a group whose consensus winner is a gP3P hypothesis (slot >= 1)
     and whose consensus rows hold fewer than four distinct model points is ambiguous, status 6: refinement runs as
     for status 0, pose and rmse are reported, cov is NaN.  First match wins: 1, 5, 6, 2, 3, 4, 0.  Three markers of
     which fewer than three are triangulated fix the pose only up to a branch: two triangulated markers leave a
     rotation about their axis, the third marker lies on a circle and its ray meets that circle twice, and both poses
     fit the rows exactly.  A group won by its prior (slot 0) keeps step 9's statuses: the prior chooses the branch.

A group with n_q >= 3 (or k < 4) has no gP3P sample, so its outputs are ``rigid_pose_robust``'s own: this oracle takes
them from there and restates steps 3-9 only for the groups that gP3P reaches.
"""
from __future__ import annotations

import numpy as np

from oracle.gp3p import GP3P_MAX, gp3p
from oracle.resection_robust import STATUS_NO_CONSENSUS, candidate_samples, rot_log
from oracle.rigid_pose_robust import (STATUS_FEW_ROWS, STATUS_NOT_PD, RigidResult, body_covariance, refine_body,
                                      rigid_pose_robust)  # fmt: skip
from oracle.triangulation_refine import group_rows
from oracle.triangulation_robust import row_errors

STATUS_AMBIGUOUS = 6
__all__ = ["STATUS_AMBIGUOUS", "rigid_pose_gp3p", "rays"]


def rays(cam_flags, cam_const, cam_x, obs_cam, obs_px):
    """Every row's camera centre c = -R^T t and unit ray d = R^T (x, y, 1) / |.| (NaN where the row's undistorted
    coordinate is unusable)."""
    from oracle.relative_pose import usable_coordinates
    from oracle.triangulation_robust import _camera_poses

    obs_cam = np.asarray(obs_cam, np.int64)
    Rc, tc = _camera_poses(cam_flags, cam_x)
    centre = -np.einsum("cji,cj->ci", Rc, tc)
    norm = usable_coordinates(cam_flags, cam_const, cam_x, obs_cam, obs_px)
    ray = np.einsum("nji,nj->ni", Rc[obs_cam], np.concatenate([norm, np.ones((len(norm), 1))], axis=1))
    ray /= np.linalg.norm(ray, axis=1)[:, None]
    return centre[obs_cam], ray


def rigid_pose_gp3p(cam_flags, cam_const, cam_x, model_xyz, obs_cam, obs_key, obs_pt, obs_px, *, threshold_px,
                    min_inliers=6, max_pairs=16, max_samples=64, prior=None, pixel_sigma=1.0, camera_cov=None,
                    max_iter=20, xtol=1e-12, gp3p_samples=0) -> RigidResult:  # fmt: skip
    """Steps 1-9 with gP3P hypotheses for every group.  gp3p_samples = 0 is ``rigid_pose_robust``."""
    from oracle.ba_oracle import rodrigues

    res = rigid_pose_robust(cam_flags, cam_const, cam_x, model_xyz, obs_cam, obs_key, obs_pt, obs_px,
                            threshold_px=threshold_px, min_inliers=min_inliers, max_pairs=max_pairs,
                            max_samples=max_samples, prior=prior, pixel_sigma=pixel_sigma, camera_cov=camera_cov,
                            max_iter=max_iter, xtol=xtol)  # fmt: skip
    reach = (res.status != STATUS_FEW_ROWS) & (res.n_points < 3)
    if not gp3p_samples or not reach.any():
        return res
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
    centre, ray = rays(cam_flags, cam_const, cam_x, obs_cam, obs_px)
    pk = np.zeros(0, np.int64) if prior is None else np.asarray(prior[0], np.int64)
    pp = np.zeros((0, 6)) if prior is None else np.asarray(prior[1], np.float64).reshape(-1, 6)
    nan = np.nan
    for g in np.flatnonzero(reach):
        rows = order[bounds[g] : bounds[g + 1]]
        k = len(rows)
        M = model[obs_pt[rows]]
        usable = np.isfinite(M).all(axis=1)
        res.inlier[rows] = False
        res.pose[g], res.cov[g], res.rmse_px[g], res.hyp[g] = nan, nan, nan, nan
        res.n_inliers[g], res.slot[g], res.best[g], res.second[g] = 0, -1, np.inf, np.inf
        # steps 3-4: the prior (slot 0) and the gP3P samples
        slots, Rs, ts = [], [], []
        i = np.searchsorted(pk, obs_key[rows[0]])
        if i < len(pk) and pk[i] == obs_key[rows[0]]:
            slots.append(0)
            Rs.append(rodrigues(pp[i, :3])[0])
            ts.append(pp[i, 3:])
        ok = usable & np.isfinite(ray[rows]).all(axis=1)
        for m, smp in enumerate(candidate_samples(k, gp3p_samples)):
            if smp is None or not ok[list(smp)].all() or len(set(obs_pt[rows[list(smp)]])) < 3:
                continue
            r3 = rows[list(smp)]
            for c, (R, t) in enumerate(gp3p(centre[r3], ray[r3], model[obs_pt[r3]])):
                slots.append(1 + GP3P_MAX * m + c)
                Rs.append(R)
                ts.append(t)
        if not slots:
            res.status[g] = STATUS_NO_CONSENSUS
            continue
        # steps 5-9 as rigid_pose_robust states them
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
        if slots[w] >= 1 and len(np.unique(obs_pt[crow])) < 4:
            st = STATUS_AMBIGUOUS
        res.pose[g], res.rmse_px[g], res.status[g] = q, rmse, st
        if st not in (STATUS_NOT_PD, STATUS_AMBIGUOUS):
            res.cov[g] = body_covariance(*cams, obs_cam[crow], obs_px[crow], Mc, q, pixel_sigma, camera_cov)
    return res
