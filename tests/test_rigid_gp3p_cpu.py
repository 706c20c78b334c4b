"""The gP3P oracle (oracle/gp3p.py) and the rigid-body pose oracle with it (oracle/rigid_pose_gp3p.py, DESIGN.md
section 4.14): the truth among its poses on generalized and near-central rays, P3P's poses on central rays, no
hypothesis from degenerate samples, groups with three or more triangulated markers untouched, the groups it newly
poses, its sample rule on both sides of C(k, 3) = gp3p_samples, the chi-square calibration of the covariance on a
sparse scene, and status 6 for three-marker groups whose pose has two exact branches."""
import numpy as np
import pytest

from oracle.ba_oracle import rodrigues
from oracle.gp3p import GP3P_MAX, gp3p
from oracle.resection_robust import candidate_samples, p3p
from oracle.rigid_pose_gp3p import STATUS_AMBIGUOUS, rigid_pose_gp3p
from oracle.rigid_pose_robust import STATUS_NO_CONSENSUS, STATUS_OK, rigid_pose_robust
from oracle.triangulation_robust import row_errors
from tests._gp3p_cases import ambiguous_three, branches, on_rays, one_view, ray_case, sparse_bodies
from tests._rigid_cases import camera_cov, make_bodies, perturb, plant_outliers

FIELDS = ("pose", "cov", "rmse_px", "count", "n_inliers", "n_points", "rep_row", "status", "hyp", "slot", "best",
          "second")  # fmt: skip


@pytest.mark.parametrize("kind", ["wide", "near"])
def test_generalized_rays_recover_the_truth(kind):
    """Every returned pose puts the three model points on their rays and keeps the model's distances; the true pose is
    among them to 1e-9."""
    rng = np.random.default_rng({"wide": 1, "near": 2}[kind])
    for _ in range(200):
        c, d, M, R, t = ray_case(rng, kind)
        sols = gp3p(c, d, M)
        assert 1 <= len(sols) <= GP3P_MAX
        assert any(np.abs(Rs - R).max() <= 1e-9 and np.abs(ts - t).max() <= 1e-9 for Rs, ts in sols)
        for Rs, ts in sols:
            assert on_rays(c, d, M, Rs, ts) <= 1e-9
            X = M @ Rs.T + ts
            for i, j in ((0, 1), (0, 2), (1, 2)):
                Dm = np.linalg.norm(M[i] - M[j])
                assert abs(np.linalg.norm(X[i] - X[j]) - Dm) <= 1e-9 * Dm


def test_central_rays_give_the_p3p_poses():
    """Three rays from one centre: gP3P is P3P, so its poses are Lambda Twist's poses with positive depth, turned from
    the camera's frame into the body's (R_b = R_c^T R_p, t_b = R_c^T (t_p - t_c)).  To 1e-7: a pair of nearby roots is
    conditioned no better than that in either solver."""
    rng = np.random.default_rng(3)
    for _ in range(200):
        c, d, M, R, t = ray_case(rng, "central")
        z = d.mean(axis=0) / np.linalg.norm(d.mean(axis=0))  # the camera looks along the rays
        x = np.cross(rng.normal(size=3), z)
        x /= np.linalg.norm(x)
        Rc = np.stack([x, np.cross(z, x), z])
        tc = -Rc @ c[0]
        y = d @ Rc.T  # bearings in the camera's frame
        ref = [(Rc.T @ Rp, Rc.T @ (tp - tc)) for Rp, tp in (s for s in p3p(y, M) if s is not None)]
        ref = [(Rb, tb) for Rb, tb in ref if ((M @ Rb.T + tb - c[0]) @ d.T).diagonal().min() > 0]
        got = gp3p(c, d, M)
        match = lambda a, b: np.abs(a[0] - b[0]).max() <= 1e-7 and np.abs(a[1] - b[1]).max() <= 1e-7  # noqa: E731
        assert all(any(match(g, r) for r in ref) for g in got)
        assert all(any(match(g, r) for g in got) for r in ref)


def test_degenerate_samples_give_no_hypothesis():
    rng = np.random.default_rng(4)
    c, d, M, _, _ = ray_case(rng, "wide")
    assert gp3p(c, d, M[[0, 0, 1]]) == []  # a repeated marker
    assert gp3p(c, d, np.array([M[0], M[1], 2 * M[1] - M[0]])) == []  # collinear markers
    par = np.tile(d[0], (3, 1))
    assert gp3p(c, par, M) == []  # parallel rays
    # a group whose rows hold two markers: every sample repeats a model point
    b = one_view(make_bodies(5, n_cams=6, n_frames=1, n_model=8, noise=0.0, visible=1.0), 0)
    b2 = make_bodies(5, n_cams=6, n_frames=1, n_model=8, noise=0.0, visible=1.0)
    sel = b2.obs_pt < 2
    r = rigid_pose_gp3p(*b2.rig(), b2.model, *(a[sel] for a in b2.obs()), threshold_px=4.0, gp3p_samples=64)
    assert r.n_points[0] == 2 and r.status[0] == STATUS_NO_CONSENSUS and r.slot[0] == -1
    r = rigid_pose_gp3p(*b.rig(), b.model, *b.obs(), threshold_px=4.0, gp3p_samples=64)
    assert r.status[0] == STATUS_OK


def _mixed(seed, noise=0.4):
    """Frames 0..5 with every marker in one random camera (no qualified point), frames 6..11 as seen by all cameras."""
    b = make_bodies(seed, n_cams=6, n_frames=12, n_model=10, noise=noise, visible=1.0)
    return one_view(b, seed, keys=np.arange(6))


def test_groups_with_three_qualified_points_are_untouched():
    b = _mixed(9)
    r0 = rigid_pose_robust(*b.rig(), b.model, *b.obs(), threshold_px=4.0)
    for g in (1, 64, 4096):
        r = rigid_pose_gp3p(*b.rig(), b.model, *b.obs(), threshold_px=4.0, gp3p_samples=g)
        keep = r0.n_points >= 3
        assert keep.sum() == 6 and (r0.n_points[~keep] == 0).all()
        for f in FIELDS:
            np.testing.assert_array_equal(getattr(r, f)[keep], getattr(r0, f)[keep], err_msg=f)
        keys = np.unique(b.obs_key)
        rows = keep[np.searchsorted(keys, b.obs_key)]
        np.testing.assert_array_equal(r.inlier[rows], r0.inlier[rows])


def test_single_view_groups_are_newly_posed():
    """The frames of test_gpu_rigid_pose's case with every marker seen by one camera and no prior: status 5 without
    gP3P, status 0 with it, and the truth to 1e-9 without noise."""
    for noise in (0.3, 0.0):
        b = make_bodies(14, n_cams=6, n_frames=10, n_model=10, noise=noise, visible=1.0)
        single = b.obs_cam == (b.obs_pt % 6)
        keep = np.where(b.obs_key < 5, single, single | (b.obs_pt < 5))
        obs = [a[keep] for a in b.obs()]
        r0 = rigid_pose_robust(*b.rig(), b.model, *obs, threshold_px=4.0)
        r = rigid_pose_gp3p(*b.rig(), b.model, *obs, threshold_px=4.0, gp3p_samples=64)
        assert (r0.status[:5] == STATUS_NO_CONSENSUS).all() and (r0.n_points[:5] == 0).all()
        assert (r.status == STATUS_OK).all()
        assert ((r.slot[:5] - 1) // GP3P_MAX < 64).all() and (r.slot[:5] >= 1).all()
        if noise == 0.0:
            assert np.abs(r.pose - b.truth).max() <= 1e-9
        else:
            assert np.abs(r.pose[:5, 3:] - b.truth[:5, 3:]).max() < 0.05


@pytest.mark.parametrize("g", [20, 19])
def test_sample_rule_around_gp3p_samples(g):
    """A group of k = 6 rows: C(6, 3) = 20 <= 20 takes every triple in lexicographic order, 19 the hashed draw.  The
    winner is the lowest score over exactly those candidates' gP3P poses, found here by scoring them directly."""
    b = make_bodies(21, n_cams=6, n_frames=1, n_model=6, noise=0.8, visible=1.0)
    b = one_view(b, 3)
    assert len(b.obs_cam) == 6
    r = rigid_pose_gp3p(*b.rig(), b.model, *b.obs(), threshold_px=3.0, gp3p_samples=g)
    smp = candidate_samples(6, g)
    assert len(smp) == g
    lex = [(i, j, l) for i in range(6) for j in range(i + 1, 6) for l in range(j + 1, 6)]
    assert (smp == lex) == (g == 20)
    from oracle.relative_pose import usable_coordinates
    from oracle.triangulation_robust import _camera_poses

    Rc, tc = _camera_poses(b.flags, b.cam_x)
    norm = usable_coordinates(*b.rig(), b.obs_cam, b.obs_px)
    ray = np.einsum("nji,nj->ni", Rc[b.obs_cam], np.c_[norm, np.ones(6)])
    ray /= np.linalg.norm(ray, axis=1)[:, None]
    cen = -np.einsum("cji,cj->ci", Rc, tc)
    rows = np.arange(6)
    best, slot = np.inf, -1
    for m, s in enumerate(smp):
        if s is None:
            continue
        s = list(s)
        for c, (R, t) in enumerate(gp3p(cen[b.obs_cam[s]], ray[s], b.model[b.obs_pt[s]])):
            e2, z = row_errors(*b.rig(), b.obs_cam, b.obs_px, rows, b.model[b.obs_pt] @ R.T + t)
            sc = np.where((z > 0) & (e2 <= 9.0), e2, 9.0).sum()
            if sc < best:
                best, slot = sc, 1 + GP3P_MAX * m + c
    assert r.slot[0] == slot and r.best[0] == best


def _chi2(r, truth):
    ok = r.status == STATUS_OK
    e = r.pose[ok] - truth[ok]
    return np.array([ei @ np.linalg.solve(c, ei) for ei, c in zip(e, r.cov[ok])]), ok


def test_covariance_is_calibrated_on_a_sparse_scene():
    """Every marker seen by one camera, no prior: the groups gP3P poses carry a calibrated covariance."""
    b = one_view(make_bodies(22, n_cams=6, n_frames=150, n_model=10, noise=0.5, visible=1.0), 5)
    r = rigid_pose_gp3p(*b.rig(), b.model, *b.obs(), threshold_px=3.0, pixel_sigma=0.5, gp3p_samples=32)
    assert (r.n_points == 0).all()
    d, ok = _chi2(r, b.truth)
    assert ok.mean() > 0.97
    assert abs(d.mean() - 6.0) < 4 * np.sqrt(12 / len(d)), d.mean()


def test_covariance_is_calibrated_on_a_sparse_scene_with_camera_cov():
    """As test_rigid_pose_cpu's camera-covariance case: each trial draws its own calibration error from camera_cov."""
    base = one_view(make_bodies(23, n_cams=6, n_frames=60, n_model=10, noise=0.3, visible=1.0, free=(1,)), 6)
    cc = camera_cov(base.flags, rot=1.5e-3, trans=3e-3)
    d = []
    for g in range(60):
        x = perturb(200 + g, base.cam_x, cc)
        sel = base.obs_key == g
        r = rigid_pose_gp3p(base.flags, base.const, x, base.model, *(a[sel] for a in base.obs()), threshold_px=6.0,
                              pixel_sigma=0.3, camera_cov=cc, gp3p_samples=32)  # fmt: skip
        if r.status[0] != STATUS_OK:
            continue
        e = r.pose[0] - base.truth[g]
        d.append(e @ np.linalg.solve(r.cov[0], e))
    d = np.array(d)
    assert len(d) >= 57
    assert abs(d.mean() - 6.0) < 4 * np.sqrt(12 / len(d)), d.mean()


def test_sparse_scene_share_posed_rises():
    b = sparse_bodies(31, n_frames=40)
    r0 = rigid_pose_robust(*b.rig(), b.model, *b.obs(), threshold_px=4.0)
    r = rigid_pose_gp3p(*b.rig(), b.model, *b.obs(), threshold_px=4.0, gp3p_samples=64)
    new = (r0.status != STATUS_OK) & (r.status == STATUS_OK)
    assert (r0.n_points < 3).mean() >= 0.2
    assert (r.status == STATUS_OK).mean() >= (r0.status == STATUS_OK).mean() + 0.15
    assert np.linalg.norm(r.pose[new, 3:] - b.truth[new, 3:], axis=1).max() < 0.05


def test_three_markers_with_two_exact_branches_are_ambiguous():
    """Two triangulated markers and a third seen by one camera whose ray meets the third marker's circle about the
    other two twice: gP3P gives two poses that fit every row, so the group is status 6 (pose and rmse reported, cov
    NaN).  A prior on either branch chooses it (status 0 there), and a fourth marker in one view leaves only the
    truth (status 0)."""
    b, model, obs, truth = ambiguous_three()
    fit = branches(b, model, obs)
    assert len(fit) == 2
    assert np.abs(fit[0] - fit[1]).max() > 0.1
    assert min(np.abs(q - truth).max() for q in fit) < 1e-4
    kw = dict(threshold_px=3.0, gp3p_samples=64, camera_cov=None)
    r = rigid_pose_gp3p(*b.rig(), model, *obs, **kw)
    assert r.n_points[0] == 2 and r.n_inliers[0] == 7 and r.slot[0] >= 1
    assert r.status[0] == STATUS_AMBIGUOUS
    assert np.isfinite(r.pose).all() and r.rmse_px[0] < 1e-6 and np.isnan(r.cov).all()
    other = r.pose[0].copy()
    # the rule is gP3P's alone: without it the group has no hypothesis
    assert rigid_pose_robust(*b.rig(), model, *obs, threshold_px=3.0).status[0] == STATUS_NO_CONSENSUS
    assert np.abs(truth - other).max() > 0.1
    for q in (truth, other):
        r = rigid_pose_gp3p(*b.rig(), model, *obs, prior=([0], q[None]), **kw)
        assert r.status[0] == STATUS_OK and r.slot[0] == 0 and np.isfinite(r.cov).all()
        np.testing.assert_allclose(r.pose[0], q, atol=1e-8)
    b4, model4, obs4, truth4 = ambiguous_three(fourth=True)
    r = rigid_pose_gp3p(*b4.rig(), model4, *obs4, **kw)
    assert r.status[0] == STATUS_OK and r.slot[0] >= 1 and r.n_inliers[0] == 8 and np.isfinite(r.cov).all()
    np.testing.assert_allclose(r.pose[0], truth4, atol=1e-9)


def test_sparse_scene_newly_posed_groups_are_calibrated():
    """DESIGN section 4.14's sparse scene (6 cameras, 8 markers, each row kept with probability 0.25, 3 % moved up to
    200 px), 1 000 frames.  Over the groups only gP3P poses (fewer than three triangulated markers, no prior), no
    status-0 group is beyond chi-square(6)'s 0.9999 quantile and the mean is within the chi-square band.  Frame 955 has
    nine rows on three markers, two of them triangulated; its winner is the wrong branch of two exact ones, 97 mm
    from the truth with a millimetre covariance unless it is status 6."""
    b = make_bodies(51, n_cams=6, n_frames=1000, n_model=8, noise=0.5, visible=0.25)
    b.obs_px, _ = plant_outliers(52, b.obs_px, 0.03, lo=10.0, hi=200.0)
    r = rigid_pose_gp3p(*b.rig(), b.model, *b.obs(), threshold_px=3.0, pixel_sigma=0.5, gp3p_samples=64)
    keys = np.unique(b.obs_key)
    only = (r.n_points < 3) & (r.count >= 4)
    d, ok = _chi2(r, b.truth[keys])
    d_new = d[only[ok]]
    print(f"gP3P groups {only.sum()}, status 0 {len(d_new)}, status 6 {(r.status[only] == STATUS_AMBIGUOUS).sum()}, "
          f"chi2 mean {d_new.mean():.2f} median {np.median(d_new):.2f} max {d_new.max():.1f}")  # fmt: skip
    assert len(d_new) >= 150
    assert r.status[keys == 955][0] == STATUS_AMBIGUOUS
    assert d_new.max() <= 27.86, d_new.max()  # chi-square(6) 0.9999 quantile
    assert abs(d_new.mean() - 6.0) < 4 * np.sqrt(12 / len(d_new)), d_new.mean()
