"""cb_rigid_pose_robust(_gp3p) on the GPU against its oracles at its edges: every status in one call with gP3P off and
on under both lane counts (and status 3 from max_iter = 1), the constructed ambiguous three-marker group (status 6),
the lane switch at 96 and 97 mean rows per group, group counts at block boundaries, the (group, point) key's pt_bits
step at 64 and 65 model points, keys up to 2^63 - 1 with priors on them (negative keys refused), max_groups at the
key count and one below, the winner's owning lane (a decisive sample at task LANES - 1, LANES, LANES + 1 and the last
task, on the Horn and the gP3P path, there as hypothesis c >= 1), groups of 65 537 and 100 000 rows, a 5 000-row group
among small groups and alone, and the camera term with one camera's run, all 160 cameras of a rig in one group,
one-row runs beside long runs and eight-lane groups sharing a warp, at P = 6 and P = 9.  Every test prints the path it
reaches (lanes, groups per block, camera table side and P derived from the inputs by the engine's own rules) and
asserts the lane count."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from caliscope_b200 import _lib as L
from caliscope_b200.rigid import RigidStats, pose_rigid_robust
from oracle.rigid_pose_gp3p import STATUS_AMBIGUOUS, rigid_pose_gp3p
from tests._gp3p_cases import ambiguous_three, branches, mixed
from tests._rigid_cases import camera_cov, make_bodies, plant_outliers
from tests._rigid_edges import decisive_gp3p, decisive_horn, huge, status_scene
from tests.test_gpu_rigid_pose import _check, _inliers_agree

pytestmark = pytest.mark.gpu

TRI_THREADS = 256
CAM_SMEM_MAX = 40 * 1024 // (8 * 37)  # 138: cameras whose table fits tri_camtab_smem's 40 KiB (CT_SMEM = 37 doubles)


def _lanes(n_rows, n_groups):
    return 32 if n_rows // max(n_groups, 1) > 96 else 8


def _path(name, b, dev, gp3p, cov=False):
    n, g = len(b.obs_cam), len(dev.status)
    lanes = _lanes(n, g)
    n_cams = len(b.flags)
    P = 9 if (np.asarray(b.flags) & 1).any() else 6
    print(f"{name}: {g} groups, {n} rows, lanes {lanes}, groups per block {TRI_THREADS // lanes}, "
          f"gP3P {'on' if gp3p else 'off'}, camera table {'shared' if n_cams <= CAM_SMEM_MAX else 'global'} "
          f"({n_cams} cameras), P {P if cov else '-'}, statuses {np.bincount(dev.status, minlength=7).tolist()}")
    return lanes


def _both(b, obs=None, **kw):
    obs = b.obs() if obs is None else obs
    kw.setdefault("threshold_px", 4.0)
    st = RigidStats()
    dev = pose_rigid_robust(*b.rig(), b.model, *obs, stats=st, **kw)
    orc = rigid_pose_gp3p(*b.rig(), b.model, *obs, **kw)
    return dev, orc, st


def _conventions(r):
    """The outputs each status promises: 5 NaN pose, cov, rmse; 2 and 6 finite pose and rmse, NaN cov; 0, 3 and 4
    finite pose, rmse and cov; 1 NaN everything."""
    for s in (1, 5):
        m = r.status == s
        assert np.isnan(r.pose[m]).all() and np.isnan(r.cov[m]).all() and np.isnan(r.rmse_px[m]).all(), s
    for s in (2, 6):
        m = r.status == s
        assert np.isfinite(r.pose[m]).all() and np.isfinite(r.rmse_px[m]).all() and np.isnan(r.cov[m]).all(), s
    m = np.isin(r.status, (0, 3, 4))
    assert np.isfinite(r.pose[m]).all() and np.isfinite(r.rmse_px[m]).all() and np.isfinite(r.cov[m]).all()


# ---- every status ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("with_cov", [False, True])
@pytest.mark.parametrize("lanes", [8, 32])
@pytest.mark.parametrize("gp3p", [0, 64])
def test_every_status(gp3p, lanes, with_cov):
    """tests/_rigid_edges.status_scene: statuses 0, 1, 2, 4, 5 (and 6 with gP3P) in one call, then 3 from max_iter = 1;
    a filler group of 200 markers in every camera moves the mean past 96 rows for 32 lanes.  The near-collinear group
    (key 3) is compared on status and pose only: its H is positive definite by a margin of 1e-14, so its covariance is
    conditioned no better than that on either side.  Covariances are compared at _check's cov_rtol = 1e-7, except that
    a group whose H has a condition number above 1e6 is allowed 1e-13 cond(H): the behind group (key 4) sees every
    row from camera 0, so its depth is weakly held (cond(H) 5.7e6), and H^-1 G Sigma_c G^T H^-1 takes that factor
    from the rounding of H's Cholesky factor on either side."""
    s, prior = status_scene(gp3p, filler=200 if lanes == 32 else 0)
    kw = dict(threshold_px=50.0, min_inliers=4, prior=prior, gp3p_samples=gp3p)
    if with_cov:
        kw.update(camera_cov=camera_cov(s.flags), pixel_sigma=0.3)
    want = {0, 1, 2, 4, 5} | ({STATUS_AMBIGUOUS} if gp3p else set())
    for max_iter in (20, 1):
        dev, orc, _ = _both(s, max_iter=max_iter, **kw)
        assert _path(f"statuses max_iter={max_iter}", s, dev, gp3p, with_cov) == lanes
        np.testing.assert_array_equal(dev.status, orc.status)
        reached = set(dev.status.tolist())
        assert reached >= (want if max_iter == 20 else {1, 3, 5}), reached
        keys = np.unique(s.obs_key)
        near = keys == 3
        cmp = ~near & (dev.status != STATUS_AMBIGUOUS)
        # cond(H) per group from the oracle's pixel-only covariance, sigma^2 H^-1
        pix = rigid_pose_gp3p(*s.rig(), s.model, *s.obs(), max_iter=max_iter,
                              **{k: v for k, v in kw.items() if k != "camera_cov"}) if with_cov else orc  # fmt: skip
        cond = np.array([np.linalg.cond(c) if np.isfinite(c).all() else 0.0 for c in pix.cov])
        weak = cond > 1e6
        sub = lambda r, m: type(r)(**{f: (getattr(r, f)[m] if f != "inlier" else r.inlier)  # noqa: E731
                                      for f in r.__dataclass_fields__})
        ok = _check(sub(dev, cmp & ~weak), sub(orc, cmp & ~weak))
        assert ok.all()
        for g in np.flatnonzero(cmp & weak):
            print(f"  key {keys[g]}: cond(H) {cond[g]:.2e}, cov_rtol {1e-13 * cond[g]:.2e}")
            ok = _check(sub(dev, np.arange(len(cmp)) == g), sub(orc, np.arange(len(cmp)) == g), cov_rtol=1e-13 * cond[g])
            assert ok.all()
        np.testing.assert_array_equal(dev.inlier, orc.inlier)
        np.testing.assert_allclose(dev.pose[near], orc.pose[near], rtol=0, atol=1e-8)
        two = orc.status == 2  # the pose is the winner, the prior here
        np.testing.assert_allclose(dev.pose[two], orc.pose[two], rtol=0, atol=1e-12)
        _conventions(dev)
        _conventions(orc)
        if gp3p:
            six = dev.status == STATUS_AMBIGUOUS
            assert six.sum() == 1 and np.isfinite(dev.pose[six]).all() and dev.rmse_px[six][0] < 1e-6


# ---- status 6 constructed -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lanes", [8, 32])
def test_ambiguous_three_markers(lanes):
    """tests/_gp3p_cases.ambiguous_three: two exact branches, status 6 on the device and in the oracle with NaN cov;
    a prior on either branch gives status 0 there, and a fourth marker in one view status 0 at the truth.  The two
    branches tie to rounding, so the device and the oracle may each report either; both must be one of them.  32 lanes:
    a filler group of 200 markers in every camera in the same call."""
    filler = 200 if lanes == 32 else 0
    b, model, obs, truth = ambiguous_three()
    kw = dict(threshold_px=3.0, gp3p_samples=64, camera_cov=camera_cov(b.flags), pixel_sigma=0.5)
    if filler:
        s, _ = status_scene(64, filler=filler)
        fsel = s.obs_key == 7
        off = len(model)
        b2 = type(b)(b.flags, b.const, b.cam_x, np.r_[model, s.model], None,
                     np.r_[obs[0], s.obs_cam[fsel]], np.r_[obs[1], s.obs_key[fsel]],
                     np.r_[obs[2], s.obs_pt[fsel] + off], np.r_[obs[3], s.obs_px[fsel]])  # fmt: skip
    else:
        b2 = type(b)(b.flags, b.const, b.cam_x, model, None, *obs)
    dev, orc, _ = _both(b2, **kw)
    assert _path("ambiguous", b2, dev, True, True) == lanes
    assert dev.status[0] == STATUS_AMBIGUOUS and orc.status[0] == STATUS_AMBIGUOUS
    assert np.isnan(dev.cov[0]).all() and np.isnan(orc.cov[0]).all()
    assert dev.n_inliers[0] == orc.n_inliers[0] == 7 and dev.n_points[0] == 2 and dev.rmse_px[0] < 1e-6
    fit = branches(b, model, obs)  # the two exact poses
    assert len(fit) == 2 and np.abs(fit[0] - fit[1]).max() > 0.1
    assert min(np.abs(dev.pose[0] - q).max() for q in fit) < 1e-8
    assert min(np.abs(orc.pose[0] - q).max() for q in fit) < 1e-8
    for q in fit:
        dp, op, _ = _both(b2, prior=([0], q[None]), **kw)
        assert dp.status[0] == 0 and op.status[0] == 0 and np.isfinite(dp.cov[0]).all()
        np.testing.assert_allclose(dp.pose[0], q, atol=1e-8)
        ok = _check(dp, op)
        assert ok.all()
    b4, model4, obs4, truth4 = ambiguous_three(fourth=True)
    b4 = type(b4)(b4.flags, b4.const, b4.cam_x, model4, None, *obs4)
    d4, o4, _ = _both(b4, **kw)
    assert d4.status[0] == 0 and o4.status[0] == 0
    np.testing.assert_allclose(d4.pose[0], truth4, atol=1e-8)
    np.testing.assert_allclose(o4.pose[0], truth4, atol=1e-8)
    # noise-free, every exact hypothesis ties to rounding: the covariance at the common pose, not _check's tie rule
    assert np.abs(d4.cov[0] - o4.cov[0]).max() <= 1e-7 * np.abs(o4.cov[0]).max()
    assert d4.n_inliers[0] == o4.n_inliers[0] == 8 and d4.inlier.all()


# ---- shape edges ----------------------------------------------------------------------------------------------------------
def _trimmed(seed, n_groups, per_group, n_cams=20, n_model=12, gp3p=False):
    """n_groups groups of exactly per_group rows (make_bodies rows cut to length), keys 0..n_groups-1."""
    b = make_bodies(seed, n_cams=n_cams, n_frames=n_groups, n_model=n_model, noise=0.4, visible=1.0)
    if gp3p:
        b = mixed(b, seed, np.arange(0, n_groups, 2), 1.0)
    rank = np.arange(len(b.obs_key)) - np.searchsorted(b.obs_key, b.obs_key)
    keep = rank < per_group
    assert (np.bincount(b.obs_key[keep]) == per_group).all() if not gp3p else True
    return type(b)(b.flags, b.const, b.cam_x, b.model, b.truth, *(a[keep] for a in b.obs()))


@pytest.mark.parametrize("per_group", [96, 97])
def test_lane_switch(per_group):
    """Mean rows per group 96 and 97: n / n_groups > 96 by integer division picks 32 lanes only at 97 (and at 96 plus
    a remainder below n_groups, here 96 * 12 + 11 rows)."""
    b = _trimmed(61, 12, per_group)
    if per_group == 96:  # 11 more rows on the last group: the mean is still 96 by integer division
        extra = make_bodies(61, n_cams=20, n_frames=12, n_model=12, noise=0.4, visible=1.0)
        last = extra.obs_key == 11
        idx = np.flatnonzero(last)[96:107]
        b = type(b)(b.flags, b.const, b.cam_x, b.model, b.truth, *(np.r_[a, e[idx]] for a, e in zip(b.obs(), extra.obs())))
    b.obs_px, _ = plant_outliers(62, b.obs_px, 0.05)
    dev, orc, _ = _both(b, prior=(np.arange(0, 12, 3), b.truth[::3] + 0.01), camera_cov=camera_cov(b.flags))
    assert _path(f"lane switch {per_group}", b, dev, False, True) == (32 if per_group == 97 else 8)
    ok = _check(dev, orc)
    _inliers_agree(dev, orc, b, ok)
    assert (dev.status == 0).mean() >= 0.9


@pytest.mark.parametrize("lanes, n_groups", [(8, 31), (8, 32), (8, 33), (32, 7), (32, 8), (32, 9)])
def test_block_boundaries(lanes, n_groups):
    """32 groups per 256-thread block at 8 lanes, 8 at 32 lanes: one group short of, at and one past a block, gP3P on
    (even keys seen as one_view sees them)."""
    per, n_model = (40, 8) if lanes == 8 else (240, 12)
    b = make_bodies(63 + n_groups, n_cams=12 if lanes == 8 else 20, n_frames=n_groups, n_model=n_model, noise=0.4,
                    visible=1.0)  # fmt: skip
    b = mixed(b, 64, np.arange(0, n_groups, 2), 1.0)
    rank = np.arange(len(b.obs_key)) - np.searchsorted(b.obs_key, b.obs_key)
    keep = rank < per
    b = type(b)(b.flags, b.const, b.cam_x, b.model, b.truth, *(a[keep] for a in b.obs()))
    dev, orc, _ = _both(b, gp3p_samples=64, camera_cov=camera_cov(b.flags))
    assert _path(f"block {n_groups}", b, dev, True, True) == lanes
    print(f"  blocks {-(-n_groups * lanes // TRI_THREADS)}, groups in the last block "
          f"{n_groups - (TRI_THREADS // lanes) * ((n_groups - 1) // (TRI_THREADS // lanes))}")
    ok = _check(dev, orc)
    _inliers_agree(dev, orc, b, ok)
    assert (dev.status == 0).mean() >= 0.8


@pytest.mark.parametrize("n_model", [64, 65])
def test_point_bits_step(n_model):
    """pt_bits = bits(n_model - 1): 6 at 64 model points, 7 at 65; the top model index in every group."""
    b = make_bodies(65, n_cams=8, n_frames=6, n_model=n_model, noise=0.4, visible=0.5)
    top = b.obs_pt == n_model - 1
    assert len(np.unique(b.obs_key[top])) == 6
    for gp in (0, 64):
        dev, orc, _ = _both(b, gp3p_samples=gp)
        _path(f"n_model {n_model} pt_bits {max(1, int(n_model - 1).bit_length())}", b, dev, gp)
        ok = _check(dev, orc)
        _inliers_agree(dev, orc, b, ok)
        assert (dev.status == 0).all()


def test_extreme_keys_with_priors():
    """Keys 0, 1, 2^31, 2^62, 2^63 - 2 and 2^63 - 1: groups come back in ascending key order, and priors on some of them
    (one-view groups, where the prior is the only hypothesis without gP3P) are found by the key search.  A negative
    key is refused."""
    keys = np.array([0, 1, 2**31, 2**62, 2**63 - 2, 2**63 - 1], np.int64)
    b = make_bodies(66, n_cams=6, n_frames=6, n_model=10, noise=0.0, visible=1.0)
    single = b.obs_cam == (b.obs_pt % 6)
    b = type(b)(b.flags, b.const, b.cam_x, b.model, b.truth, *(a[single] for a in b.obs()))
    b.obs_key = keys[b.obs_key]
    pk = keys[[0, 2, 3, 5]]
    prior = (pk, b.truth[[0, 2, 3, 5]] + 0.002)
    dev, orc, _ = _both(b, prior=prior)
    _path("extreme keys", b, dev, False)
    np.testing.assert_array_equal(dev.key, keys)
    want = np.where(np.isin(keys, pk), 0, 5)
    np.testing.assert_array_equal(dev.status, want)
    ok = _check(dev, orc)
    _inliers_agree(dev, orc, b, ok)
    np.testing.assert_allclose(dev.pose[want == 0], b.truth[[0, 2, 3, 5]], atol=1e-8)
    neg = b.obs_key.copy()
    neg[b.obs_key == keys[0]] = -(2**62)
    with pytest.raises(L.EngineError, match="negative group key"):
        pose_rigid_robust(*b.rig(), b.model, b.obs_cam, neg, b.obs_pt, b.obs_px, threshold_px=4.0)


def _raw_groups(b, max_groups):
    lib = L.load()
    n = len(b.obs_cam)
    flags = np.ascontiguousarray(b.flags, np.int32)
    const, cx, model = (np.ascontiguousarray(a) for a in (b.const, b.cam_x, b.model))
    cam, key = np.ascontiguousarray(b.obs_cam, np.int32), np.ascontiguousarray(b.obs_key, np.int64)
    pt, px = np.ascontiguousarray(b.obs_pt, np.int32), np.ascontiguousarray(b.obs_px)
    m = max(max_groups, 1)
    outs = [np.zeros((m, 6)), np.zeros((m, 36)), np.zeros(m)] + [np.zeros(m, np.int32) for _ in range(5)]
    inl = np.zeros(n, np.uint8)
    ng = C.c_int32(0)
    st = L.RigidStats()
    p = lambda x: x.ctypes.data_as(C.c_void_p)  # noqa: E731
    e = np.zeros(0, np.int64)
    code = lib.cb_rigid_pose_robust_gp3p(len(flags), p(flags), p(const), p(cx), None, len(model), p(model), n, p(cam),
                                         p(key), p(pt), p(px), 0, 4.0, 6, 16, 64, 64, 0, p(e), p(np.zeros(0)), 1.0, 20,
                                         1e-12, max_groups, C.byref(ng), *(p(o) for o in outs), p(inl), C.byref(st), 0,
                                         None)  # fmt: skip
    return code, ng.value, st, (lib.cb_ba_last_error() or b"").decode(), outs


def test_max_groups():
    """max_groups equal to the key count is accepted; one less is refused once the grouping stage has counted the
    keys: CB_E_INVALID, n_groups_out the key count and the outputs untouched.  The call fills its stats only on success,
    so they stay zero here; the launch counter is not exposed, so this does not show which kernels ran before the
    refusal (the validation and grouping kernels do)."""
    b = make_bodies(67, n_cams=6, n_frames=9, noise=0.3)
    code, ng, st, _, outs = _raw_groups(b, 9)
    assert code == 0 and ng == 9 and st.kernel_launches > 0 and (outs[7] == 0).sum() >= 8
    code, ng, st, err, outs = _raw_groups(b, 8)
    print(f"max_groups 8 of 9: code {code}, n_groups {ng}, launches {st.kernel_launches}, error {err!r}")
    assert code == -1 and ng == 9 and "9 groups but room for 8" in err
    assert st.kernel_launches == 0 and st.total_ms == 0.0
    assert all((o == 0).all() for o in outs)


# ---- camera-term edges ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", [6, 9])
def test_camera_term_runs(P):
    """With camera_cov: a group with one camera's run (every row in camera 0), a group with one row from each of all
    160 cameras (the camera table in global memory), a group whose runs are one row in most cameras beside 120 rows
    in two (the first two groups have no triangulated marker: their priors are their only hypotheses), and eight-lane groups with different run counts packed four to a warp.
    The covariance against the oracle's at the existing cov_rtol."""
    free = (3, 70) if P == 9 else ()
    b = make_bodies(68, n_cams=160, n_frames=8, n_model=300, noise=0.3, visible=1.0, radius=4.0, free=free)
    k, c, p = b.obs_key, b.obs_cam, b.obs_pt
    sel = np.zeros(len(k), bool)
    sel |= (k == 0) & (c == 0) & (p < 20)  # one camera's run of 20 rows (nh = 1)
    sel |= (k == 1) & (p == c)  # all 160 cameras, a run of one row each
    sel |= (k == 2) & (c < 2) & (p < 120) | (k == 2) & (c >= 2) & (c < 40) & (p == c)  # two runs of 120, 38 of one
    for g in range(3, 8):  # four to a warp at 8 lanes: 2, 5, 9, 13, 17 cameras, 6 markers each
        sel |= (k == g) & (c < [2, 5, 9, 13, 17][g - 3]) & (p < 6)
    b = type(b)(b.flags, b.const, b.cam_x, b.model, b.truth, *(a[sel] for a in b.obs()))
    cc = camera_cov(b.flags)
    prior = (np.array([0, 1]), b.truth[:2] + 0.001)
    dev, orc, _ = _both(b, prior=prior, camera_cov=cc, pixel_sigma=0.3)
    lanes = _path(f"camera term P={P}", b, dev, False, True)
    assert lanes == 8
    runs = [len(np.unique(b.obs_cam[b.obs_key == g])) for g in range(8)]
    print(f"  runs per group {runs}")
    assert runs[0] == 1 and runs[1] == 160 and runs[2] == 40
    ok = _check(dev, orc)
    assert ok.all() and (dev.status == 0).all()
    _inliers_agree(dev, orc, b, ok)


# ---- the winner's owning lane -------------------------------------------------------------------------------------------
def _only_truth(hyps, q, which):
    """Of every hypothesis (slot, R, t), only `which` is the true pose (to 1e-4: the point hypotheses come from the
    float32-rounded undistorted coordinates), every other one at least 1e-2 from it, so a wrong owner lane broadcasts a
    pose 1e6 times farther than the 1e-8 the refined pose is held to."""
    from oracle.ba_oracle import rodrigues

    R0 = rodrigues(q[:3])[0]
    dist = {sl: max(np.abs(R - R0).max(), np.abs(t - q[3:]).max()) for sl, R, t in hyps}
    assert [sl for sl, d in dist.items() if d < 1e-4] == [which], (which, sorted(dist.values())[:3])
    assert min(d for sl, d in dist.items() if sl != which) > 1e-2


@pytest.mark.parametrize("lanes", [8, 32])
def test_winner_owner_horn(lanes):
    """tests/_rigid_edges.decisive_horn: seven triangulated markers, C(7, 3) = 35 samples in lexicographic order, and in
    each group exactly one sample (task LANES - 1, LANES, LANES + 1 or 35, the last) whose Horn pose is the truth.  The
    lane that owns task t is t % LANES; the winner, its consensus and the refined pose are right only if that lane's
    pose is the one broadcast."""
    from oracle.rigid_pose_robust import horn

    tasks = [lanes - 1, lanes, lanes + 1, 35]
    s, q, good = decisive_horn(6 if lanes == 8 else 20, tasks)
    dev, orc, _ = _both(s, threshold_px=3.0, min_inliers=4)
    assert _path("owner horn", s, dev, False) == lanes
    print(f"  decisive tasks {tasks}, owner lanes {[t % lanes for t in tasks]}")
    np.testing.assert_array_equal(orc.slot, tasks)
    # every sample's Horn pose from the oracle's point hypotheses
    from oracle.rigid_pose_robust import point_hypotheses
    from oracle.triangulation_refine import group_rows

    grp, _ = group_rows(s.obs_key)
    qg, qm, qx = point_hypotheses(*s.rig(), s.obs_cam, s.obs_px, grp, s.obs_pt, len(s.model), threshold_px=3.0,
                                  max_pairs=16)  # fmt: skip
    for key, t in enumerate(tasks):
        sel = qg == key
        QM, QX = s.model[qm[sel]], qx[sel]
        hyps = []
        for m, trip in enumerate([(i, j, l) for i in range(7) for j in range(i + 1, 7) for l in range(j + 1, 7)]):
            sol = horn(QM[list(trip)], QX[list(trip)])
            if sol is not None:
                hyps.append((1 + m, sol[0], sol[1]))
        _only_truth(hyps, q, t)
    ok = _check(dev, orc)
    assert ok.all() and (dev.status == 0).all()
    _inliers_agree(dev, orc, s, ok)
    np.testing.assert_allclose(dev.pose, np.tile(q, (len(tasks), 1)), rtol=0, atol=1e-8)


@pytest.mark.parametrize("lanes", [8, 32])
def test_winner_owner_gp3p(lanes):
    """tests/_rigid_edges.decisive_gp3p: 12 rows without a triangulated triple, the hashed draw of 40 gP3P samples, and
    in each group exactly one sample (task LANES - 1, LANES, LANES + 1 or 40, the last) with the true pose among its
    hypotheses, there as hypothesis c >= 1, so its slot 1 + 8 m + c names neither the task nor the lane by itself: the
    owner is task 1 + (slot - 1) / 8, lane task % LANES.  32 lanes: a filler group of 80 markers in every camera."""
    from oracle.gp3p import gp3p
    from oracle.resection_robust import candidate_samples
    from oracle.rigid_pose_gp3p import rays

    g = 40
    tasks = [lanes - 1, lanes, lanes + 1, g]
    s, q, which = decisive_gp3p(tasks, gp3p_samples=g, filler=80 if lanes == 32 else 0)
    dev, orc, _ = _both(s, threshold_px=3.0, min_inliers=4, gp3p_samples=g)
    assert _path("owner gp3p", s, dev, True) == lanes
    slots = [1 + 8 * m + c for m, c in which]
    print(f"  decisive tasks {tasks}, (sample, hypothesis) {which}, slots {slots}, owner lanes "
          f"{[t % lanes for t in tasks]}")  # fmt: skip
    assert all(c >= 1 for _, c in which)
    np.testing.assert_array_equal(orc.slot[: len(tasks)], slots)
    cen, ray = rays(*s.rig(), s.obs_cam, s.obs_px)
    cs = candidate_samples(12, g)
    for key, sl in enumerate(slots):
        rows = np.flatnonzero(s.obs_key == key)
        hyps = []
        for m, smp in enumerate(cs):
            r3 = rows[list(smp)]
            if len(set(s.obs_pt[r3])) < 3:
                continue
            for c, (R, t) in enumerate(gp3p(cen[r3], ray[r3], s.model[s.obs_pt[r3]])):
                hyps.append((1 + 8 * m + c, R, t))
        _only_truth(hyps, q, sl)
    ok = _check(dev, orc)
    assert ok.all() and (dev.status == 0).all() and (dev.n_points[: len(tasks)] == 1).all()
    _inliers_agree(dev, orc, s, ok)
    assert (dev.n_inliers[: len(tasks)] == 5).all()
    np.testing.assert_allclose(dev.pose[: len(tasks)], np.tile(q, (len(tasks), 1)), rtol=0, atol=1e-8)


# ---- huge groups ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_rows", [65537, 100000])
@pytest.mark.parametrize("kind", ["horn", "gp3p", "ambiguous"])
def test_huge_group(kind, n_rows):
    """One group of 65 537 or 100 000 rows (tests/_rigid_edges.huge) with gP3P on, max_iter = 1 (status 3 where it
    converges no further): the Horn path (8 triangulated markers), the gP3P path (10 markers each in one camera) and the
    ambiguous three-marker rows, where lane 0 reads every consensus flag looking for a fourth marker (status 6 on both
    sides; the branches tie to rounding, so each side's pose is one of the two)."""
    b = huge(n_rows, kind)
    kw = dict(threshold_px=3.0, gp3p_samples=64, max_iter=1, pixel_sigma=0.3)
    dev, orc, _ = _both(b, **kw)
    assert _path(f"huge {kind}", b, dev, True) == 32
    assert dev.count[0] == n_rows
    if kind == "ambiguous":
        fit = branches(*ambiguous_three()[:3])
        assert dev.status[0] == STATUS_AMBIGUOUS and orc.status[0] == STATUS_AMBIGUOUS
        assert dev.n_inliers[0] == orc.n_inliers[0] == n_rows and np.isnan(dev.cov).all()
        # one Levenberg-Marquardt step from a gP3P hypothesis (3e-5 px from exact) lands within 1e-6 of a branch
        assert min(np.abs(dev.pose[0] - f).max() for f in fit) < 1e-6
        assert min(np.abs(orc.pose[0] - f).max() for f in fit) < 1e-6
        return
    ok = _check(dev, orc)
    assert ok.all() and dev.status[0] == orc.status[0] in (0, 3)
    assert dev.n_points[0] == (8 if kind == "horn" else 0)
    _inliers_agree(dev, orc, b, ok)


def test_5000_row_group_among_small_and_alone():
    """A 5 000-row group (tests/_rigid_edges.huge's Horn rows) among 100 groups of about 25 rows is posed under 8 lanes,
    alone under 32; both calls match the oracle and give the group the same status, consensus and pose."""
    big = huge(5000, "horn")
    small = make_bodies(91, n_cams=8, n_frames=101, n_model=8, noise=0.3, visible=0.4)
    keep = small.obs_key >= 1
    b = type(big)(big.flags, big.const, big.cam_x, big.model, None, *(np.r_[a, s[keep]] for a, s in zip(big.obs(),
                                                                                                      small.obs())))
    kw = dict(threshold_px=3.0, gp3p_samples=64, camera_cov=camera_cov(big.flags), pixel_sigma=0.3)
    dev, orc, _ = _both(b, **kw)
    assert _path("5000 among small", b, dev, True, True) == 8
    ok = _check(dev, orc)
    _inliers_agree(dev, orc, b, ok)
    one, orc1, _ = _both(big, **kw)
    assert _path("5000 alone", big, one, True, True) == 32
    ok1 = _check(one, orc1)
    _inliers_agree(one, orc1, big, ok1)
    assert ok[0] and ok1[0] and dev.status[0] == one.status[0] == 0 and dev.n_inliers[0] == one.n_inliers[0]
    np.testing.assert_array_equal(dev.inlier[:5000], one.inlier)
    np.testing.assert_allclose(dev.pose[0], one.pose[0], rtol=0, atol=1e-9)
