"""The extrinsic bootstrap's three device calls (cb_pnp_ippe, cb_relative_pose_network, cb_stereo_rmse) at rig scale, on
the cases of tests/_bootstrap_cases.py: PnP groups of more than 32 rows on both sides of every warp stride, frames with
20+ cameras, 1 000+ camera pairs, the 32-lane stereo kernel, fisheye lenses, several boards per frame, ignored cameras,
a camera without intrinsics, degenerate groups and the bench session itself.

References: OpenCV's own calls on the device's normalised coordinates (oracle.bootstrap.pnp_cv2 / stereo_rmse_cv2, pinned
to the unmodified reference in tests/test_bootstrap_cases_cpu.py), the oracle's IPPE and its fallback, the host array
pose network (pinned in tests/test_bootstrap_host.py) and the dict-based oracle chain."""
from __future__ import annotations

import functools

import numpy as np
import pytest

from oracle import bootstrap as OB
from tests import _bootstrap_cases as BC

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")

CASES = sorted(BC.BUILDERS)
BENCH = "bench_full"  # the O(groups x rows) oracle and the dict chain are skipped there


@functools.lru_cache(maxsize=None)
def _run(name):
    """Case, device normalised coordinates, device PnP, cv2 PnP on the calibrated rows, oracle PnP (not on the bench
    session) and its fallback keys."""
    from caliscope_b200 import bootstrap as B
    from caliscope_b200.triangulation import undistort_points

    c = BC.BUILDERS[name]()
    tab = c.tab
    mats = np.zeros((len(tab.cam_ids), 3, 3))
    mats[:, 0, 0], mats[:, 1, 1], mats[:, 0, 2], mats[:, 1, 2], mats[:, 0, 1] = tab.k.T
    mats[:, 2, 2] = 1.0
    dists = [d[:4] if f else d for d, f in zip(tab.dist, tab.fisheye)]
    known = np.isin(c.cam_id, tab.cam_ids)
    slot = np.array([tab.index_of.get(int(v), 0) for v in c.cam_id], np.int32)
    norm = np.full((c.n_obs, 2), np.nan, np.float32)
    norm[known] = undistort_points(c.img_xy[known], slot[known], mats, dists, tab.fisheye, output="normalized")
    res = B.pnp_arrays(tab, c.cam_id, c.sync_index, c.object_id, c.img_xy, c.obj_xyz)
    cal = c.calibrated()
    cv = OB.pnp_cv2(norm[cal], c.cam_id[cal], c.sync_index[cal], c.object_id[cal], c.obj_xyz[cal])
    orc, fb = None, []
    if name != BENCH:
        orc = OB.pnp_poses(tab.cam_ids[tab.has_intrinsics], norm[cal].astype(np.float64), c.sync_index[cal], c.cam_id[cal],
                           c.object_id[cal], c.obj_xyz[cal], fallback_keys=fb)  # fmt: skip
    return c, norm, res, cv, orc, set(fb)


@functools.lru_cache(maxsize=None)
def _chain(name):
    """Device network on the device's PnP poses: (pairs, R, t, kept count)."""
    from caliscope_b200 import bootstrap as B

    c, _, res, *_ = _run(name)
    live = res.status != B.PNP_TOO_FEW
    pairs, R, t, cnt, _, _ = B.pose_network_arrays(res.keys[live], res.R[live], res.t[live], c.tab, 1.5)
    return pairs, R, t, cnt


def _tuples(keys):
    return [tuple(int(v) for v in k) for k in keys]


@pytest.mark.parametrize("name", CASES)
def test_pnp_matches_cv2_and_oracle(name):
    """Same groups, order and status as cv2.solvePnP; IPPE poses to 1e-6 and the float32 RMSE to 1e-4 relative; the
    fallback set is the oracle's, each fallback pose within 1e-6 of the oracle's and at least as good as cv2 ITERATIVE's;
    degenerate groups NaN."""
    from caliscope_b200 import bootstrap as B

    c, _, res, (ck, cR, ct, crm, cst), orc, fb = _run(name)
    assert res.keys.tolist() == ck.tolist()
    assert res.status.tolist() == cst.tolist()
    ok = res.status == B.PNP_OK
    assert np.abs(res.R[ok] - cR[ok]).max() <= 1e-6 and np.abs(res.t[ok] - ct[ok]).max() <= 1e-6
    assert np.all(np.abs(res.rmse[ok] - crm[ok]) <= 1e-4 * crm[ok] + 1e-8)
    deg = res.status == B.PNP_DEGENERATE
    assert np.isnan(res.R[deg]).all() and np.isnan(res.t[deg]).all()
    f = res.status == B.PNP_OK_FALLBACK
    assert np.all(res.rmse[f] <= crm[f] * (1 + 1e-3) + 1e-12)
    if orc is not None:
        assert {k for k, s in zip(_tuples(res.keys), res.status) if s == B.PNP_OK_FALLBACK} == fb
        for i in np.flatnonzero(f | ok):
            Ro, to, rmo = orc[tuple(int(v) for v in res.keys[i])]
            assert np.abs(res.R[i] - Ro).max() <= 1e-6 and np.abs(res.t[i] - to).max() <= 1e-6, res.keys[i]
    if name == "planted":
        assert f.sum() >= 1 and deg.sum() >= 1 and (res.count[f] > 32).all()
    assert (res.count[res.status != B.PNP_TOO_FEW] >= 4).all() and (res.count[res.status == B.PNP_TOO_FEW] < 4).all()


@pytest.mark.parametrize("name", CASES)
def test_pose_network_matches_host_and_oracle_chain(name):
    """cb_relative_pose_network on the device's PnP poses == relative_pose_arrays + filter_and_aggregate (pairs, counts,
    keep mask row for row, R and t to 1e-12) with the default multipliers and with (0.5, 3.0); on cv2's poses == the
    dict-based oracle chain (pairs, kept counts, R and t to 1e-9)."""
    from caliscope_b200 import bootstrap as B

    c, _, res, (ck, cR, ct, _, cst), _, _ = _run(name)
    live = res.status != B.PNP_TOO_FEW
    keys, R, t = res.keys[live], res.R[live], res.t[live]
    rel = B.relative_pose_arrays(keys, R, t, c.tab)
    for mults in ((None, None), (0.5, 3.0)):
        ph, kh, Rh, th, nh = B.filter_and_aggregate(rel, 1.5, *mults)
        p, Rd, td, n, k, st = B.pose_network_arrays(keys, R, t, c.tab, 1.5, *mults, want_keep=True)
        assert p.tolist() == ph.tolist() and n.tolist() == nh.tolist()
        assert len(k) == len(kh) and np.array_equal(k, kh)
        assert np.abs(Rd - Rh).max() <= 1e-12 and np.abs(td - th).max() <= 1e-12
        assert st.kernel_launches > 0
    if name == "ring64_outliers":
        n_t, n_r = BC.iqr_rejections(c, keys, R, t)
        assert n_t > 0 and n_r > 0
    if name == BENCH:
        return
    cl = cst != B.PNP_TOO_FEW
    poses = {k: (cR[i], ct[i], 0.0) for i, k in zip(np.flatnonzero(cl), _tuples(ck[cl]))}
    filt = OB.reject_outliers(OB.relative_poses(poses, c.tab.cam_ids, c.tab.ignore), 1.5)
    agg = OB.aggregate(filt)
    p, Rd, td, n, _, _ = B.pose_network_arrays(ck[cl], cR[cl], ct[cl], c.tab, 1.5)
    assert _tuples(p) == sorted(agg)
    for i, pr in enumerate(_tuples(p)):
        assert n[i] == len(filt[pr])
        assert np.abs(Rd[i] - agg[pr][0]).max() <= 1e-9 and np.abs(td[i] - agg[pr][1]).max() <= 1e-9, pr


def _quirk_pairs(c, n=12):
    """Pairs the reference never finds common observations for: cameras in (b, a) dict order, or an ignored camera."""
    pos = {int(v): i for i, v in enumerate(c.tab.cam_ids)}
    ids = sorted(pos)
    out = [(a, b) for a in ids for b in ids if a < b and pos[a] > pos[b]][:n]
    out += [(a, b) for a in ids for b in ids if a < b and (c.tab.ignore[pos[a]] or c.tab.ignore[pos[b]])][:n]
    return np.array(out, np.int64).reshape(-1, 2)


def _stereo_check(rm, cnt, rc, cc):
    assert np.array_equal(cnt, cc)
    assert np.array_equal(np.isnan(rm), np.isnan(rc))
    has = ~np.isnan(rc)
    assert np.all(np.abs(rm[has] - rc[has]) <= 2e-5 * rc[has]), np.max(np.abs(rm[has] - rc[has]) / rc[has])


@pytest.mark.parametrize("name", CASES)
def test_stereo_rmse_matches_cv2(name):
    """stereo_rmse_arrays on the device chain's pairs and poses (plus pairs the dict-order / ignore quirk blanks) ==
    cv2.triangulatePoints + projectPoints per pair: counts equal, RMSE to 2e-5 relative, NaN exactly where the reference
    has none.  Also on subsets of exactly 1 and 1 024 pairs.  On the bench session cv2 runs on every 8th pair and the
    counts of all pairs are checked against a vectorised count."""
    from caliscope_b200 import bootstrap as B

    c, norm, *_ = _run(name)
    pairs, R, t, _ = _chain(name)
    q = _quirk_pairs(c)
    if len(q):
        pairs = np.concatenate([pairs, q])
        R = np.concatenate([R, np.repeat(np.eye(3)[None], len(q), 0)])
        t = np.concatenate([t, np.tile([0.3, 0.0, 0.0], (len(q), 1))])
    rm, cnt = B.stereo_rmse_arrays(c.tab, pairs, R, t, c.cam_id, c.sync_index, c.object_id, c.keypoint_id, c.img_xy)
    args = (c.tab.cam_ids, c.tab.ignore, norm, c.cam_id, c.sync_index, c.object_id, c.keypoint_id)
    sel = np.arange(0, len(pairs), 8) if name == BENCH else np.arange(len(pairs))
    rc, cc = OB.stereo_rmse_cv2(pairs[sel], R[sel], t[sel], *args)
    _stereo_check(rm[sel], cnt[sel], rc, cc)
    assert (~np.isnan(rc)).sum() > 0.5 * len(sel)
    if name == BENCH:
        assert np.array_equal(cnt[: len(pairs) - len(q)], BC.common_counts(c, pairs[: len(pairs) - len(q)]))
    if name == "planted":
        i = {p: k for k, p in enumerate(_tuples(pairs))}
        assert cnt[i[(8, 9)]] == 3 and np.isnan(rm[i[(8, 9)]]) and cnt[i[(10, 11)]] == 4 and np.isfinite(rm[i[(10, 11)]])
    if name == "ring64":
        assert len(pairs) > 1024
        for sub in (np.array([7]), np.arange(1024)):
            r1, c1 = B.stereo_rmse_arrays(c.tab, pairs[sub], R[sub], t[sub], c.cam_id, c.sync_index, c.object_id, c.keypoint_id,
                                          c.img_xy)  # fmt: skip
            _stereo_check(r1, c1, rc[sub], cc[sub])


@pytest.mark.parametrize("name, min_kept", [("ring64", 12), (BENCH, 5)])
def test_device_chain_recovers_the_rig(name, min_kept):
    """PnP -> network -> stereo on the device: aggregated relative poses of pairs with >= min_kept kept samples are the
    generator's cameras (R 5e-3, t 2e-2 m at 0.3 px noise), every stereo RMSE finite.  The 60 frames of ring64 leave many
    pairs with 5-11 samples, whose average carries the estimator's own error: OpenCV's chain on the same data is 8.8e-3 off
    in R at 5 samples and 3.6e-3 at 12; agreement with that chain is what the tests above check."""
    from caliscope_b200 import bootstrap as B

    c, *_ = _run(name)
    pairs, R, t, cnt = _chain(name)
    worst_R = worst_t = 0.0
    for k, (a, b) in enumerate(_tuples(pairs)):
        if cnt[k] < min_kept:
            continue
        (RA, tA), (RB, tB) = c.truth[a], c.truth[b]
        worst_R = max(worst_R, np.abs(R[k] - RB @ RA.T).max())
        worst_t = max(worst_t, np.abs(t[k] - (tB - RB @ RA.T @ tA)).max())
    assert (cnt >= min_kept).sum() > 200
    assert worst_R < 5e-3 and worst_t < 2e-2, (worst_R, worst_t)
    rm, _ = B.stereo_rmse_arrays(c.tab, pairs, R, t, c.cam_id, c.sync_index, c.object_id, c.keypoint_id, c.img_xy)
    assert np.isfinite(rm).all()


def test_bootstrap_calls_are_bit_reproducible():
    """DESIGN.md 4.3: fixed-order sums, no atomics -- two calls give the same bits (ring64)."""
    from caliscope_b200 import bootstrap as B

    c, *_ = _run("ring64")
    a = [B.pnp_arrays(c.tab, c.cam_id, c.sync_index, c.object_id, c.img_xy, c.obj_xyz) for _ in range(2)]
    for f in ("keys", "R", "t", "rmse", "status", "count"):
        assert np.array_equal(getattr(a[0], f), getattr(a[1], f), equal_nan=f not in ("keys", "status", "count")), f
    live = a[0].status != B.PNP_TOO_FEW
    n = [B.pose_network_arrays(a[0].keys[live], a[0].R[live], a[0].t[live], c.tab, 1.5, want_keep=True) for _ in range(2)]
    for x, y in zip(n[0][:5], n[1][:5]):
        assert np.array_equal(x, y)
    pairs, R, t = n[0][0], n[0][1], n[0][2]
    s = [B.stereo_rmse_arrays(c.tab, pairs, R, t, c.cam_id, c.sync_index, c.object_id, c.keypoint_id, c.img_xy) for _ in range(2)]
    assert np.array_equal(s[0][0], s[1][0], equal_nan=True) and np.array_equal(s[0][1], s[1][1])
