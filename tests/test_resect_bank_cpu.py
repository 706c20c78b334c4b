"""The resection bank's design claims (tests/_resect_bank.py), checked with the oracle alone: the decisive-row groups win by
about one tau^2 at the intended rows and flip to pose B without any one of them, both poses are among their sampled
hypotheses, the status recipes reach their statuses, the per-group oracle equals the whole-call oracle, and the shape
rule picks the shapes the device tests claim."""
from __future__ import annotations

import numpy as np
import pytest

from oracle.ba_oracle import rodrigues
from oracle.resection_robust import bearings, candidate_samples, cameras, p3p, project, resect_robust
from oracle.triangulation_robust import undistorted_coordinates
from tests._resect_bank import TAU, chunks, is_long, lanes, make_bank, make_group, oracle_bank, relabelled, tiles


def _alone(g, **kw):
    k = len(g.cam)
    return resect_robust(np.array(g.flags, np.int32), np.stack(g.const), np.concatenate(g.x), g.pts, g.cam,
                         np.zeros(k, np.int64), g.pt, g.px, threshold_px=TAU, **kw)  # fmt: skip


def _score(g, R, t, drop=None):
    cam = cameras(np.array(g.flags, np.int32), np.stack(g.const), np.concatenate(g.x))[0]
    uv, z = project(cam, R, t, g.pts[g.pt])
    e2 = ((uv - g.px) ** 2).sum(axis=1)
    c = np.where((z > 0) & (e2 <= TAU * TAU), e2, TAU * TAU)
    if drop is not None:
        c = np.delete(c, drop)
    return c.sum()


@pytest.mark.parametrize("k,at", [(12, (0, 11)), (513, (0, 511, 512)), (1025, (1023, 1024))])
def test_decisive_groups_win_by_one_tau2_at_the_intended_rows(k, at):
    g = make_group(dict(family="decisive", k=k, at=at), 7)
    assert all(g.role[a] == "A" for a in at)
    n_a = int((g.role == "A").sum())
    assert n_a == int((g.role == "B").sum()) + 1
    r = _alone(g, max_samples=64)
    assert r.status[0] == 0 and r.n_inliers[0] == n_a
    np.testing.assert_array_equal(r.inlier, g.role == "A")
    # A's best hypothesis wins by tau^2 less A's residual sum; B (the prior, exact) scores (n_a) tau^2
    margin = _score(g, g.RB, g.tB) - r.best[0]
    assert 0.8 * TAU * TAU < margin < TAU * TAU, margin
    assert r.second[0] - r.best[0] > 1e-6  # not a near-tie
    # without one of A's rows at an intended position, B (slot 0) wins
    for a in at:
        keep = np.arange(k) != a
        from dataclasses import replace

        h = replace(g, cam=g.cam[keep], pt=g.pt[keep], px=g.px[keep])
        s = _alone(h, max_samples=64)
        assert s.slot[0] == 0 and s.n_inliers[0] == (n_a - 1 if n_a - 1 >= 6 else 0), (a, s.slot[0], s.n_inliers[0])


@pytest.mark.parametrize("k", [12, 513])
def test_decisive_groups_sample_both_poses(k):
    g = make_group(dict(family="decisive", k=k, at=(0, k - 1)), 3)
    norm = undistorted_coordinates(np.array(g.flags, np.int32), np.stack(g.const), np.concatenate(g.x), g.cam, g.px)
    y = bearings(norm)
    near_a = near_b = False
    for smp in candidate_samples(k, 64):
        if smp is None:
            continue
        for sol in p3p(y[list(smp)], g.pts[g.pt[list(smp)]]):
            if sol is None:
                continue
            near_a |= np.abs(sol[0] - g.R).max() < 1e-3 and np.abs(sol[1] - g.t).max() < 1e-3
            near_b |= np.abs(sol[0] - g.RB).max() < 1e-6 and np.abs(sol[1] - g.tB).max() < 1e-6
    assert near_a and near_b


def test_status_recipes():
    assert _alone(make_group(dict(family="pad", k=3), 1)).status[0] == 1
    assert _alone(make_group(dict(family="far_px", k=10), 1)).status[0] == 5
    assert _alone(make_group(dict(family="two_cams", k=10, noise_px=0.3), 1)).status[0] == 6
    for fam in ("collinear", "near_collinear"):
        r = _alone(make_group(dict(family=fam), 1))
        assert r.status[0] == 2 and np.isnan(r.cov[0]).all() and np.isfinite(r.pose[0]).all()
    r = _alone(make_group(dict(family="general", k=40, noise_px=0.3), 1), max_iter=1)
    assert r.status[0] == 3
    g = make_group(dict(family="behind_axis"), 1)
    r = resect_robust(np.array(g.flags, np.int32), np.stack(g.const), np.concatenate(g.x), g.pts, g.cam,
                      np.zeros(len(g.cam), np.int64), g.pt, g.px, threshold_px=50.0, max_samples=1)  # fmt: skip
    assert r.slot[0] == 0 and r.status[0] == 4


def test_families_reach_their_edges():
    """identity and down groups with 0.001 px of noise start the refinement from rot_log's s < 1e-5 branch: the winning
    hypothesis is within 1e-6 of R, yet its score is not a near-tie with the others'."""
    from oracle.resection_robust import rot_log

    for sp in (dict(family="identity", k=20, noise_px=1e-3),
               dict(family="down", k=20, noise_px=1e-3, lens="free"),
               dict(family="down", k=20, noise_px=1e-3, tilted=True)):  # fmt: skip
        g = make_group(sp, 5)
        r = _alone(g)
        assert r.status[0] == 0 and r.second[0] - r.best[0] > 1e-9 * max(1.0, r.best[0])
        R = r.hyp[0, :9].reshape(3, 3)
        rx, ry, rz = R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]
        assert np.sqrt((rx * rx + ry * ry + rz * rz) * 0.25) < 1e-5
        assert np.abs(rodrigues(rot_log(R))[0] - g.R).max() < 1e-5
    g = make_group(dict(family="wide", k=20, lens="fisheye"), 2)
    Xc = g.pts @ g.R.T + g.t
    assert np.degrees(np.arctan2(np.linalg.norm(Xc[:, :2], axis=1), Xc[:, 2])).max() > 79.9
    g = make_group(dict(family="behind", k=20, noise_px=0.3), 2)
    assert ((g.pts @ g.R.T + g.t)[:, 2] < 0).sum() == 4


def test_per_group_oracle_equals_whole_call_oracle():
    specs = [dict(family=f, k=k, noise_px=0.3, lens=L, repeat=2 if k > 8 else 0)
             for f, k, L in (("general", 8, "pinhole"), ("planar", 12, "free"), ("wide", 20, "fisheye"), ("pad", 2, "pinhole"),
                             ("two_cams", 10, "pinhole"), ("behind", 12, "free"))]  # fmt: skip
    bank = make_bank(specs, 4, nan_cov=[(1, 0)])
    kw = dict(threshold_px=TAU, points_cov=bank.pts_cov)
    whole = resect_robust(*bank.args(), **kw)
    per = oracle_bank(bank, threshold_px=TAU, with_cov=True, workers=2)
    for f in ("cam", "pose", "cov", "rmse_px", "count", "n_inliers", "rep_row", "status", "inlier", "best", "slot"):
        np.testing.assert_array_equal(getattr(whole, f), getattr(per, f), err_msg=f)
    # a relabelled bank is the same groups in another order
    nb, src = relabelled(bank, 9)
    again = resect_robust(*nb.args(), **kw)
    for f in ("pose", "cov", "status", "n_inliers", "count"):
        np.testing.assert_array_equal(getattr(again, f), getattr(whole, f)[src], err_msg=f)


def test_shape_rule():
    assert is_long([513] * 682, 4096) and not is_long([513] * 683, 4096) and lanes([513] * 683, 4096) == 32
    assert not is_long([512] * 4, 64) and is_long([513] * 4, 64)
    assert lanes([98, 96], 64) == 32 and lanes([96, 96], 64) == 8
    assert chunks([511, 512, 513, 1024, 1025, 3000, 3]) == 1 + 1 + 2 + 2 + 3 + 6 + 1
    assert [tiles(m) for m in (31, 32, 4096)] == [1, 2, 129]
