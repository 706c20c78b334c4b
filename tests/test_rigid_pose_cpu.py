"""The rigid-body pose oracle (oracle/rigid_pose_robust.py, DESIGN.md section 4.14) against independent references: the
true pose, scipy's least_squares, central differences, an SVD (Kabsch) fit, every status, both sample rules and the
chi-square calibration of its covariance."""
import numpy as np
import pytest
from scipy.optimize import least_squares

from oracle.ba_oracle import rodrigues
from oracle.resection_robust import candidate_samples, cameras, project, rot_log
from oracle.rigid_pose_robust import (STATUS_BEHIND, STATUS_FEW_ROWS, STATUS_MAX_ITER, STATUS_NO_CONSENSUS,
                                      STATUS_NOT_PD, STATUS_OK, body_jacobians, horn, refine_body, rigid_pose_robust)
from oracle.triangulation_robust import row_errors
from tests._rigid_cases import camera_cov, make_bodies, perturb


def _run(b, **kw):
    kw.setdefault("threshold_px", 3.0)
    return rigid_pose_robust(*b.rig(), b.model, *b.obs(), **kw)


@pytest.mark.parametrize("fisheye, free", [((), ()), ((1, 4), ()), ((), (0, 3, 5))])
def test_noise_free_recovers_the_truth(fisheye, free):
    b = make_bodies(1, n_frames=5, noise=0.0, fisheye=fisheye, free=free)
    r = _run(b)
    assert (r.status == STATUS_OK).all() and r.inlier.all()
    assert np.abs(r.pose - b.truth).max() <= 1e-9
    assert (r.n_points == len(b.model)).all()


def test_refinement_reaches_the_least_squares_optimum():
    b = make_bodies(2, n_frames=4, noise=0.5)
    r = _run(b)
    for g in range(4):
        rows = np.flatnonzero(r.inlier & (b.obs_key == g))

        def res(q):
            R = rodrigues(q[:3])[0]
            X = b.model[b.obs_pt[rows]] @ R.T + q[3:]
            from oracle.triangulation_refine import pixel_jacobians

            return pixel_jacobians(*b.rig(), b.obs_cam[rows], b.obs_px[rows], np.arange(len(rows)), X)[0].ravel()

        ls = least_squares(res, b.truth[g], method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15)
        assert r.status[g] == STATUS_OK
        np.testing.assert_allclose(r.pose[g], ls.x, atol=1e-9)
        np.testing.assert_allclose(r.rmse_px[g], np.sqrt(np.mean(ls.fun**2) * 2), rtol=1e-9)


def test_jacobian_matches_central_differences():
    b = make_bodies(3, n_frames=1, noise=0.2, free=(2,), fisheye=(5,))
    q = b.truth[0] + np.array([0.01, -0.02, 0.015, 0.003, -0.002, 0.004])
    M = b.model[b.obs_pt]
    _, J, _ = body_jacobians(*b.rig(), b.obs_cam, b.obs_px, M, q)
    num = np.zeros_like(J)
    for i in range(6):
        d = np.zeros(6)
        d[i] = 1e-6
        rp = body_jacobians(*b.rig(), b.obs_cam, b.obs_px, M, q + d)[0]
        rm = body_jacobians(*b.rig(), b.obs_cam, b.obs_px, M, q - d)[0]
        num[:, :, i] = (rp - rm) / 2e-6
    np.testing.assert_allclose(J, num, rtol=1e-6, atol=1e-5)
    H = np.einsum("nki,nkj->ij", J, J)
    Hn = np.einsum("nki,nkj->ij", num, num)
    np.testing.assert_allclose(H, Hn, rtol=1e-6)


def _kabsch(M, X):
    mb, xb = M.mean(axis=0), X.mean(axis=0)
    U, _, Vt = np.linalg.svd((M - mb).T @ (X - xb))
    D = np.diag([1.0, 1.0, np.sign(np.linalg.det(Vt.T @ U.T))])
    R = Vt.T @ D @ U.T
    return R, xb - R @ mb


def test_horn_equals_kabsch_on_exact_triples():
    rng = np.random.default_rng(4)
    for _ in range(200):
        M = rng.normal(size=(3, 3)) * rng.uniform(0.01, 2.0)
        R = rodrigues(rng.normal(size=3))[0]
        X = M @ R.T + rng.normal(size=3) * 3
        Rh, th = horn(M, X)
        Rk, tk = _kabsch(M, X)
        np.testing.assert_allclose(Rh, Rk, atol=1e-10)
        np.testing.assert_allclose(th, tk, atol=1e-10)
        np.testing.assert_allclose(Rh, R, atol=1e-9)
    M = np.array([[0.0, 0, 0], [1, 0, 0], [2, 1e-12, 0]])  # collinear: no hypothesis
    assert horn(M, M) is None


def _status_rig():
    return make_bodies(5, n_cams=6, n_frames=1, n_model=10, noise=0.0, visible=1.0)


def test_every_status_from_a_constructed_case():
    b = _status_rig()
    # 0
    assert _run(b).status[0] == STATUS_OK
    # 1: three rows
    r = rigid_pose_robust(*b.rig(), b.model, *(a[:3] for a in b.obs()), threshold_px=3.0)
    assert r.status[0] == STATUS_FEW_ROWS and np.isnan(r.pose).all()
    # 5: every marker seen by one camera only, no prior (no qualified point, no hypothesis)
    one = b.obs_cam == (b.obs_pt % 6)
    sub = [a[one] for a in b.obs()]
    r = rigid_pose_robust(*b.rig(), b.model, *sub, threshold_px=3.0)
    assert r.status[0] == STATUS_NO_CONSENSUS and r.n_points[0] == 0 and not r.inlier.any()
    # ... and 0 with the true pose as the prior
    r = rigid_pose_robust(*b.rig(), b.model, *sub, threshold_px=3.0, prior=([0], b.truth[:1]))
    assert r.status[0] == STATUS_OK and r.slot[0] == 0
    np.testing.assert_allclose(r.pose[0], b.truth[0], atol=1e-9)
    # 2: every consensus row on one marker (seen by all six cameras), the prior the winner
    m0 = b.obs_pt == 0
    sub = [a[m0] for a in b.obs()]
    r = rigid_pose_robust(*b.rig(), b.model, *sub, threshold_px=3.0, min_inliers=4, prior=([0], b.truth[:1]))
    assert r.status[0] == STATUS_NOT_PD and np.isnan(r.cov).all() and np.isfinite(r.pose).all()
    # 3: one iteration from a noisy start
    bn = make_bodies(5, n_cams=6, n_frames=1, n_model=10, noise=0.5, visible=1.0)
    r = _run(bn, max_iter=1)
    assert r.status[0] == STATUS_MAX_ITER and np.isfinite(r.cov).all()
    # 4: a marker that the refinement carries behind camera 0
    r = _behind_case()
    assert r.status[0] == STATUS_BEHIND and np.isfinite(r.cov).all()


def _behind_case():
    """A marker 0.05 m behind camera 0 on its optical axis at the true pose, seen by camera 0 alone at the principal
    point; two more markers are seen by two cameras, the rest by one, so no triple qualifies and the prior (the truth
    moved 0.1 m along camera 0's axis, where the marker is in front) is the only hypothesis.  Every pixel is exact at
    the truth, so the refinement reaches it, where the marker is behind."""
    b = _status_rig()
    cams = cameras(*b.rig())
    R0, t0 = rodrigues(cams[0].q[:3])[0], cams[0].q[3:6]
    z = R0[2]  # camera 0's optical axis in the world
    Rb, tb = rodrigues(b.truth[0, :3])[0], b.truth[0, 3:]
    Xw = R0.T @ (np.array([0.0, 0.0, -0.05]) - t0)
    model = np.r_[b.model, [Rb.T @ (Xw - tb)]]
    keep = (b.obs_pt < 2) & (b.obs_cam < 2) | (b.obs_pt >= 2) & (b.obs_cam == (b.obs_pt % 6))
    oc, ok, op, px = (a[keep] for a in b.obs())
    oc, ok, op = np.r_[oc, 0], np.r_[ok, 0], np.r_[op, len(model) - 1]
    px = np.r_[px, [[b.const[0, 2], b.const[0, 3]]]]
    prior = b.truth[:1].copy()
    prior[0, 3:] += 0.1 * z
    return rigid_pose_robust(*b.rig(), model, oc, ok, op, px, threshold_px=50.0, min_inliers=4, prior=([0], prior))


@pytest.mark.parametrize("n_q", [8, 9])
def test_sample_rule_around_max_samples(n_q):
    """C(8, 3) = 56 <= 64: every triple in lexicographic order; C(9, 3) = 84 > 64: the hashed draw.  The winner is the
    lowest score over exactly those candidates, found here by scoring them directly."""
    b = make_bodies(6, n_cams=6, n_frames=1, n_model=n_q, noise=0.8, visible=1.0)
    r = _run(b, max_samples=64)
    smp = candidate_samples(n_q, 64)
    assert len(smp) == (56 if n_q == 8 else 64)
    assert (smp == [(i, j, l) for i in range(n_q) for j in range(i + 1, n_q) for l in range(j + 1, n_q)]) == (n_q == 8)
    from oracle.rigid_pose_robust import point_hypotheses

    qg, qm, qx = point_hypotheses(*b.rig(), b.obs_cam, b.obs_px, np.zeros(len(b.obs_cam), np.int64), b.obs_pt, n_q,
                                  threshold_px=3.0, max_pairs=16)  # fmt: skip
    assert len(qm) == n_q
    rows = np.arange(len(b.obs_cam))
    scores = []
    for s in smp:
        if s is None:
            scores.append(np.inf)
            continue
        R, t = horn(b.model[qm[list(s)]], qx[list(s)])
        e2, zz = row_errors(*b.rig(), b.obs_cam, b.obs_px, rows, b.model[b.obs_pt] @ R.T + t)
        scores.append(np.where((zz > 0) & (e2 <= 9.0), e2, 9.0).sum())
    assert r.slot[0] == 1 + int(np.argmin(scores)) and r.best[0] == min(scores)


def _chi2(b, r, truth):
    ok = r.status == STATUS_OK
    e = r.pose[ok] - truth[ok]
    return np.array([ei @ np.linalg.solve(c, ei) for ei, c in zip(e, r.cov[ok])]), ok


def test_covariance_is_calibrated_without_camera_cov():
    b = make_bodies(7, n_frames=150, noise=0.5)
    r = _run(b, pixel_sigma=0.5)
    d, ok = _chi2(b, r, b.truth)
    assert ok.mean() > 0.99
    band = 4 * np.sqrt(12 / len(d))
    assert abs(d.mean() - 6.0) < band, d.mean()


def test_covariance_is_calibrated_with_camera_cov():
    """Each trial draws its own calibration error from camera_cov (the camera term is shared by every frame of one
    calibration, so only independent calibrations average out)."""
    base = make_bodies(8, n_frames=80, noise=0.3, free=(1,))
    cc = camera_cov(base.flags, rot=1.5e-3, trans=3e-3)
    d = []
    for g in range(80):
        x = perturb(100 + g, base.cam_x, cc)
        sel = base.obs_key == g
        r = rigid_pose_robust(base.flags, base.const, x, base.model, *(a[sel] for a in base.obs()), threshold_px=6.0,
                              pixel_sigma=0.3, camera_cov=cc)  # fmt: skip
        assert r.status[0] == STATUS_OK
        e = r.pose[0] - base.truth[g]
        d.append(e @ np.linalg.solve(r.cov[0], e))
        if g == 0:  # the camera term matters here: without it the same error is far outside the pixel-only band
            r0 = rigid_pose_robust(base.flags, base.const, x, base.model, *(a[sel] for a in base.obs()),
                                   threshold_px=6.0, pixel_sigma=0.3)  # fmt: skip
            assert np.trace(r.cov[0]) > 2 * np.trace(r0.cov[0])
    d = np.array(d)
    assert abs(d.mean() - 6.0) < 4 * np.sqrt(12 / len(d)), d.mean()


def test_refine_body_from_a_rotation_vector_start():
    """rot_log of the Horn R is the start: a winner near theta = pi still refines to the truth."""
    b = make_bodies(9, n_frames=1, noise=0.0)
    b.truth[0, :3] *= (np.pi - 1e-3) / np.linalg.norm(b.truth[0, :3])
    R = rodrigues(b.truth[0, :3])[0]
    cams = cameras(*b.rig())
    px = np.empty_like(b.obs_px)
    for i, (c, p) in enumerate(zip(b.obs_cam, b.obs_pt)):
        Rc = rodrigues(cams[c].q[:3])[0]
        px[i] = project(cams[c], Rc, cams[c].q[3:6], R @ b.model[p] + b.truth[0, 3:])[0]
    q0 = np.r_[rot_log(R), b.truth[0, 3:]]
    q, _, st = refine_body(*b.rig(), b.obs_cam, px, b.model[b.obs_pt], q0)
    assert st == STATUS_OK
    np.testing.assert_allclose(rodrigues(q[:3])[0], R, atol=1e-9)
