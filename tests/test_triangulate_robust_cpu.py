"""The NumPy oracle of robust triangulation (oracle/triangulation_robust.py): candidate pairs, rejection of planted
outliers, agreement with plain refinement on clean data, and each status code."""
import numpy as np
import pytest

from caliscope_b200 import synthetic
from oracle import triangulation_refine as T
from oracle import triangulation_robust as R


def _ncp(flags):
    return int(np.where(np.asarray(flags) & 1, 9, 6).sum())


@pytest.mark.parametrize("k,max_pairs", [(2, 64), (5, 10), (12, 66), (12, 200)])
def test_candidate_pairs_all_when_they_fit(k, max_pairs):
    r = R.candidate_pairs(k, max_pairs)
    i, j = R.unrank_pair(r, k)
    assert list(zip(i.tolist(), j.tolist())) == [(a, b) for a in range(k) for b in range(a + 1, k)]


@pytest.mark.parametrize("k,max_pairs", [(5, 9), (12, 65), (40, 64), (300, 64), (300, 1), (100_000, 64)])
def test_candidate_pairs_sampled(k, max_pairs):
    r = R.candidate_pairs(k, max_pairs)
    T_ = k * (k - 1) // 2
    assert len(r) == max_pairs == len(np.unique(r)) and r[0] == 0 and r[-1] < T_
    assert np.all(np.diff(r) > 0)
    i, j = R.unrank_pair(r, k)
    assert np.all((0 <= i) & (i < j) & (j < k))
    assert np.array_equal(R.pair_rank(i, j, k), r)


def test_unranking_round_trips():
    for k in (2, 3, 7, 64):
        i, j = np.triu_indices(k, 1)
        r = R.pair_rank(i, j, k)
        assert np.array_equal(r, np.arange(k * (k - 1) // 2))
        ii, jj = R.unrank_pair(r, k)
        assert np.array_equal(ii, i) and np.array_equal(jj, j)


def _clean_projection(rig, ncp):
    from oracle import ba_oracle as O

    orc = O.Rig(rig.cam_flags, rig.cam_const, rig.n_pts, rig.obs_cam, rig.obs_pt, rig.obs_xy)
    return O._project(np.concatenate([rig.x_true[:ncp], rig.x_true[ncp:]]), orc, False)[0]


def test_planted_outliers_are_rejected():
    tau = 4.0
    rig = synthetic.make_rig(8, 2000, 10_000, cams_per_point=8, outlier_frac=0.1, outlier_px=300, noise_px=0.5, seed=11)
    ncp = _ncp(rig.cam_flags)
    cx = rig.x_true[:ncp]
    key = rig.obs_pt.astype(np.int64)
    out = R.robust_points(rig.cam_flags, rig.cam_const, cx, rig.obs_cam, rig.obs_xy, key, threshold_px=tau)
    cs = out.consensus
    offset = np.linalg.norm(rig.obs_xy - _clean_projection(rig, ncp), axis=1)
    clean = ~rig.outlier_mask
    grp, G = T.group_rows(key)
    n_clean_cams = np.array([len(np.unique(rig.obs_cam[(grp == g) & clean])) for g in range(G)])
    eligible = (cs.count >= 3) & (n_clean_cams >= 2)
    rows = eligible[grp]
    far = rows & (offset > 2 * tau)
    assert far.sum() > 500
    assert (~cs.inlier[far]).mean() >= 0.999
    assert cs.inlier[rows & clean].mean() >= 0.995
    # where the consensus set is the clean set, the point is the refinement of the clean rows alone
    same = eligible & np.array([np.array_equal(cs.inlier[grp == g], clean[grp == g]) for g in range(G)])
    assert same.mean() > 0.95
    cr = np.flatnonzero(clean)
    args = (rig.cam_flags, rig.cam_const, cx, rig.obs_cam[cr], rig.obs_xy[cr], grp[cr])
    x0 = T.dlt_start(*args, G)
    xyz_c, _, st_c, _ = T.refine_points(*args, x0)
    m = same & (st_c == 0) & (out.status == 0)
    assert m.sum() > 0.9 * same.sum()
    rel = np.linalg.norm(out.xyz[m] - xyz_c[m], axis=1) / np.linalg.norm(xyz_c[m], axis=1)
    assert rel.max() < 1e-9


def test_clean_data_with_a_huge_threshold_keeps_every_row():
    rig = synthetic.make_rig(8, 1500, 7500, cams_per_point=8, noise_px=0.5, seed=12)
    ncp = _ncp(rig.cam_flags)
    cx = rig.x_true[:ncp]
    key = rig.obs_pt.astype(np.int64)
    out = R.robust_points(rig.cam_flags, rig.cam_const, cx, rig.obs_cam, rig.obs_xy, key, threshold_px=1e6)
    grp, G = T.group_rows(key)
    n_cams = np.array([len(np.unique(rig.obs_cam[grp == g])) for g in range(G)])
    live = (out.consensus.count >= 2) & (n_cams >= 2)
    assert np.all(out.status[~live & (out.consensus.count >= 2)] == R.STATUS_NO_CONSENSUS)
    assert np.all(out.status[live] != R.STATUS_NO_CONSENSUS)
    assert out.consensus.inlier[live[grp]].all()
    args = (rig.cam_flags, rig.cam_const, cx, rig.obs_cam, rig.obs_xy, grp)
    xyz, _, st, _ = T.refine_points(*args, T.dlt_start(*args, G))
    m = (st == 0) & (out.status == 0)
    assert m.sum() > 0.9 * live.sum()
    rel = np.linalg.norm(out.xyz[m] - xyz[m], axis=1) / np.linalg.norm(xyz[m], axis=1)
    assert rel.max() < 1e-8


def _pinhole(centres, f=1000.0):
    """Identity-rotation cameras at `centres`: (flags, const, cam_x)."""
    n = len(centres)
    const = np.tile([f, f, 640.0, 480.0, 0, 0, 0, 0, 0], (n, 1)).astype(float)
    x = np.concatenate([np.r_[0.0, 0.0, 0.0, -np.asarray(c, float)] for c in centres])
    return np.zeros(n, np.int32), const, x


def _px(X, c, f=1000.0):
    d = np.asarray(X, float) - np.asarray(c, float)
    return [f * d[0] / d[2] + 640.0, f * d[1] / d[2] + 480.0]


def status_cases():
    """Hand-built groups (cameras along the x axis, so a vertical pixel offset is off the epipolar line) and their
    statuses at tau = 4 px: (flags, const, cam_x, obs_cam, obs_key, obs_px, expected status per group)."""
    X = np.array([0.3, 0.1, 3.0])
    cen = [(0, 0, 0), (1, 0, 0), (0.5, 0, 0), (-0.5, 0, 0)]
    flags, const, cx = _pinhole(cen)

    def at(c, dy=0.0):
        u, v = _px(X, cen[c])
        return [u, v + dy]

    groups = [
        (1, [(0, at(0))]),  # one row
        (5, [(0, at(0)), (1, at(1, 30.0)), (2, at(2, -30.0))]),  # three views disagreeing pairwise by more than tau
        (5, [(0, at(0)), (1, at(1, 30.0))]),  # two views, off the epipolar line
        (5, [(0, at(0)), (0, at(0, 0.5)), (0, at(0, -0.5))]),  # every row from one camera
        (0, [(0, at(0)), (1, at(1)), (2, at(2)), (3, at(3, 80.0))]),  # three agreeing views and one outlier
        (0, [(0, at(0)), (1, at(1, 0.3)), (0, at(0)), (1, at(1, 0.3))]),  # repeated rows: tied pairs, ranks 0, 2 and 5
    ]
    cam, key, px, expect = [], [], [], []
    for g, (s, obs) in enumerate(groups):
        expect.append(s)
        for c, p in obs:
            cam.append(c)
            key.append(g)
            px.append(p)
    return flags, const, cx, np.array(cam, np.int32), np.array(key, np.int64), np.array(px), expect


def test_status_codes():
    flags, const, cx, cam, key, px, expect = status_cases()
    out = R.robust_points(flags, const, cx, cam, px, key, threshold_px=4.0)
    cs = out.consensus
    assert out.status.tolist() == expect
    bad = out.status != 0
    assert np.isnan(out.xyz[bad]).all() and np.isnan(out.cov[bad]).all() and np.isnan(out.rmse_px[bad]).all()
    assert np.all(cs.n_inliers[bad] == 0) and not cs.inlier[np.isin(key, np.flatnonzero(bad))].any()
    assert cs.inlier[key == 4].tolist() == [True, True, True, False] and cs.n_inliers[4] == 3
    assert np.abs(out.xyz[4] - [0.3, 0.1, 3.0]).max() < 1e-9
    # an exact tie between the pairs (0, 1), (0, 3) and (2, 3) of identical rows resolves to the lowest rank
    assert cs.second[5] == cs.best[5] and cs.rank[5] == 0
    assert cs.inlier[key == 5].all()
    # a stricter min_inliers turns the three-view group into no consensus
    out4 = R.robust_points(flags, const, cx, cam, px, key, threshold_px=4.0, min_inliers=4)
    assert out4.status[4] == R.STATUS_NO_CONSENSUS and out4.status[5] == 0
