"""oracle/resection_robust.py, the statement of cb_resect_robust's rule (DESIGN.md section 4.9), checked on the CPU: its
P3P against OpenCV's, the candidate samples, planted outliers, the refinement against cv2.solvePnP, both covariance
terms against finite differences, and one hand-built group per status."""
from __future__ import annotations

import numpy as np
import pytest

from oracle.ba_oracle import rodrigues
from oracle.resection_robust import (bearings, cameras, candidate_samples, p3p, pose_covariance, pose_jacobians,
                                     refine_pose, resect_robust, rot_log, splitmix64)  # fmt: skip
from tests._resect_cases import camera_offsets, make_rig, perturb_cameras, plant_outliers

cv2 = pytest.importorskip("cv2")


def _triple(rng):
    X = rng.uniform(-1, 1, (3, 3))
    R = rodrigues(rng.normal(0, 0.6, 3))[0]
    t = np.array([0.0, 0.0, 5.0]) + rng.normal(0, 0.3, 3)
    Xc = X @ R.T + t
    return X, Xc[:, :2] / Xc[:, 2:]


def test_p3p_matches_opencv_both_ways():
    rng = np.random.default_rng(0)
    for _ in range(200):
        X, uv = _triple(rng)
        mine = [s for s in p3p(bearings(uv), X) if s is not None]
        _, rv, tv = cv2.solveP3P(X, uv, np.eye(3), None, flags=cv2.SOLVEPNP_P3P)
        theirs = [(cv2.Rodrigues(a)[0], b.ravel()) for a, b in zip(rv, tv)]

        def close(a, b):
            return (np.abs(a[0] - b[0]).max() <= 1e-9 and
                    np.abs(a[1] - b[1]).max() <= 1e-9 * np.abs(b[1]).max())  # fmt: skip

        assert len(mine) == len(theirs)
        assert all(any(close(a, b) for b in theirs) for a in mine)
        assert all(any(close(a, b) for a in mine) for b in theirs)


def test_splitmix64_reference_values():
    # splitmix64 generator outputs for the state sequence starting at 0 (Vigna's reference implementation)
    assert splitmix64(0) == 0xE220A8397B1DCDAF
    assert splitmix64(0x9E3779B97F4A7C15) == 0x6E789E6AA1B965F4


def test_candidate_samples():
    k = 7
    s = candidate_samples(k, 64)  # C(7, 3) = 35 <= 64: every triple, lexicographic
    assert s == sorted(s) and len(s) == 35 and len(set(s)) == 35
    k = 30
    s = candidate_samples(k, 64)
    assert len(s) == 64
    for m, smp in enumerate(s):
        got = []
        for t in range(16):
            v = splitmix64((m << 32) + t) % k
            if v not in got:
                got.append(v)
            if len(got) == 3:
                break
        assert smp == tuple(sorted(got))
        assert smp[0] < smp[1] < smp[2]
    # a group of 4 rows and 3 samples: the hashed rule, and 16 draws can run out of distinct positions
    assert all(x is None or len(set(x)) == 3 for x in candidate_samples(4, 3))


@pytest.mark.parametrize("fisheye,free", [((), ()), ((1, 3), ()), ((0,), (2, 4))])
def test_planted_outliers(fisheye, free):
    flags, const, cam_x, pts, oc, op, px = make_rig(3, 5, 40, fisheye=fisheye, free=free, noise=0.3)
    for frac, seed in ((0.05, 1), (0.3, 2)):
        pxo, moved = plant_outliers(seed, px, frac)
        prior = perturb_cameras(seed, flags, cam_x)
        r = resect_robust(flags, const, prior, pts, oc, oc.astype(np.int64), op, pxo, threshold_px=4.0)
        assert (r.status == 0).all()
        np.testing.assert_array_equal(r.inlier, ~moved)
        offs = camera_offsets(flags)
        for c in range(len(flags)):
            err = r.pose[c] - cam_x[offs[c] : offs[c] + 6]
            sd = np.sqrt(np.diag(r.cov[c])) * 0.3  # cov at pixel_sigma 1; the noise is 0.3 px
            assert np.all(np.abs(err) <= 5 * sd)


def test_refinement_matches_solvepnp():
    """On distortion-free pinhole cameras the refinement and cv2.solvePnP(SOLVEPNP_ITERATIVE, useExtrinsicGuess)
    minimise the same pixel cost from the same start.  Both stop at the optimum to within their own termination: this
    rule at |d| <= 1e-12 |q|, OpenCV's LM at a relative step of DBL_EPSILON or 20 iterations.  Near the optimum the
    cost is quadratic with curvature H, so two stopping points within the solver's tolerance of the optimum differ by
    at most about sqrt(eps) in the weakest direction: 1e-7 relative on the pose is the tolerance."""
    flags, const, cam_x, pts = make_rig(5, 4, 50)[:4]
    const[:, 4:] = 0.0
    cams = cameras(flags, const, cam_x)
    from oracle.resection_robust import project

    rng = np.random.default_rng(9)
    for c in range(4):
        R = rodrigues(cams[c].q[:3])[0]
        uv, _ = project(cams[c], R, cams[c].q[3:6], pts)
        obs = uv + rng.normal(0, 0.5, uv.shape)
        q0 = cams[c].q[:6] + np.r_[rng.normal(0, 0.01, 3), rng.normal(0, 0.02, 3)]
        q, _, st = refine_pose(cams[c], q0, pts, obs)
        assert st == 0
        K = np.array([[const[c, 0], 0, const[c, 2]], [0, const[c, 1], const[c, 3]], [0, 0, 1.0]])
        ok, rv, tv = cv2.solvePnP(pts, obs, K, None, q0[:3].copy(), q0[3:].copy(), useExtrinsicGuess=True,
                                  flags=cv2.SOLVEPNP_ITERATIVE)  # fmt: skip
        assert ok
        np.testing.assert_allclose(q, np.r_[rv.ravel(), tv.ravel()], rtol=1e-7, atol=1e-7)


def _group(seed=4, c=1):
    flags, const, cam_x, pts, oc, op, px = make_rig(seed, 4, 40, fisheye=(1,), free=(2,), noise=0.3)
    m = oc == c
    cam = cameras(flags, const, cam_x)[c]
    return cam, pts, op[m], px[m]


def test_covariance_pixel_term_is_inverse_central_difference_hessian():
    cam, pts, op, px = _group()
    X = pts[op]
    q, _, st = refine_pose(cam, cam.q[:6], X, px)
    assert st == 0
    h = 1e-6
    J = np.zeros((2 * len(X), 6))
    for i in range(6):
        dq = np.zeros(6)
        dq[i] = h
        rp, _, _ = pose_jacobians(cam, q + dq, X, px)
        rm, _, _ = pose_jacobians(cam, q - dq, X, px)
        J[:, i] = (rp - rm).ravel() / (2 * h)
    cov = pose_covariance(cam, q, X, px, op, 0.7)
    np.testing.assert_allclose(cov, 0.49 * np.linalg.inv(J.T @ J), rtol=1e-5, atol=0)


def test_covariance_point_term_first_order():
    """Moving the points by dX moves the re-solved pose by -H^-1 sum_p G_p dX_p to first order."""
    cam, pts, op, px = _group(seed=6)
    X = pts[op]
    q, _, _ = refine_pose(cam, cam.q[:6], X, px, max_iter=50, xtol=1e-15)
    _, J, JX = pose_jacobians(cam, q, X, px)
    H = np.einsum("nki,nkj->ij", J, J)
    G = np.einsum("nki,nkj->nij", J, JX)
    rng = np.random.default_rng(2)
    dP = rng.normal(0, 1e-6, pts.shape)
    pred = -np.linalg.solve(H, np.einsum("nij,nj->i", G, dP[op]))
    q2, _, _ = refine_pose(cam, q, (pts + dP)[op], px, max_iter=50, xtol=1e-15)
    np.testing.assert_allclose(q2 - q, pred, rtol=2e-3, atol=1e-12 + 2e-3 * np.abs(pred).max())
    # and the covariance term: sum_p G_p Sigma_p G_p^T with rows of a point summed first
    Sig = np.tile(np.eye(3) * 1e-6, (len(pts), 1, 1))
    op2 = np.r_[op, op[:3]]  # repeated rows of three points
    X2, px2 = pts[op2], np.r_[px, px[:3]]
    cov = pose_covariance(cam, q, X2, px2, op2, 0.0, Sig)
    _, J2, JX2 = pose_jacobians(cam, q, X2, px2)
    H2 = np.einsum("nki,nkj->ij", J2, J2)
    G2 = np.einsum("nki,nkj->nij", J2, JX2)
    M = sum(G2[op2 == p].sum(0) @ Sig[p] @ G2[op2 == p].sum(0).T for p in np.unique(op2))
    Hi = np.linalg.inv(H2)
    np.testing.assert_allclose(cov, Hi @ M @ Hi, rtol=1e-9, atol=0)


def test_status_codes():
    flags, const, cam_x, pts, oc, op, px = make_rig(8, 3, 30, noise=0.3)
    pts = pts.copy()
    m0 = oc == 0
    base = [(oc[m0], op[m0], px[m0])]  # status 0
    # status 1: three rows
    base.append((np.zeros(3, np.int32), np.arange(3), px[m0][:3]))
    # status 6: two cameras
    m1 = oc == 1
    base.append((np.r_[oc[m0][:5], oc[m1][:5]], np.r_[op[m0][:5], op[m1][:5]], np.r_[px[m0][:5], px[m1][:5]]))
    # status 5: pixels unrelated to the points
    base.append((np.zeros(10, np.int32), np.arange(10), np.random.default_rng(1).uniform(0, 1280, (10, 2))))
    rows_c, rows_p, rows_x, keys = [], [], [], []
    for g, (c, p, x) in enumerate(base):
        rows_c.append(c); rows_p.append(p); rows_x.append(x); keys.append(np.full(len(c), g))  # noqa: E702
    r = resect_robust(flags, const, cam_x, pts, np.concatenate(rows_c), np.concatenate(keys),
                      np.concatenate(rows_p), np.concatenate(rows_x), threshold_px=4.0)  # fmt: skip
    assert list(r.status) == [0, 1, 6, 5]
    assert np.isnan(r.pose[1:]).all() and (r.n_inliers[1:] == 0).all()

    # status 2: collinear points (rotation about their line is not observable)
    P = np.stack([np.linspace(-1, 1, 12), np.zeros(12), np.zeros(12)], axis=1)
    cam = cameras(flags, const, cam_x)[0]
    from oracle.resection_robust import project

    uv, _ = project(cam, rodrigues(cam.q[:3])[0], cam.q[3:6], P)
    r = resect_robust(flags, const, cam_x, P, np.zeros(12, np.int32), np.zeros(12, np.int64), np.arange(12), uv,
                      threshold_px=4.0, min_inliers=4)  # fmt: skip
    assert r.status[0] == 2 and np.isnan(r.cov[0]).all() and np.isfinite(r.pose[0]).all()

    # status 4: a consensus row in front of the winner but behind the camera at the refined pose.  The prior (the
    # winner) is the true pose moved 0.1 m back along the optical axis; every pixel is exact at the truth, and one point
    # sits on the optical axis 0.05 m behind the true camera: in front of the prior, projecting to the principal point
    # at both poses, so it is a consensus row, and the refinement reaches the truth, where it is behind.
    flags, const, cam_x, pts, oc, op, px = make_rig(10, 1, 20, noise=0.0)
    cam = cameras(flags, const, cam_x)[0]
    R, t = rodrigues(cam.q[:3])[0], cam.q[3:6]
    P = np.r_[pts, [R.T @ (np.array([0.0, 0.0, -0.05]) - t)]]
    uv, _ = project(cam, R, t, P)
    uv[-1] = [const[0, 2], const[0, 3]]
    prior = cam_x.copy()
    prior[5] += 0.1
    n = len(P)
    r = resect_robust(flags, const, prior, P, np.zeros(n, np.int32), np.zeros(n, np.int64), np.arange(n), uv,
                      threshold_px=50.0, max_samples=1)  # fmt: skip
    assert r.slot[0] == 0 and r.inlier.all()
    assert r.status[0] == 4
    np.testing.assert_allclose(r.pose[0], cam_x[:6], atol=1e-8)


def test_rot_log_matches_opencv():
    rng = np.random.default_rng(3)
    for r in list(rng.normal(0, 1.0, (50, 3))) + [np.array([np.pi - 1e-7, 0, 0]), np.array([1e-7, 0, 0]), np.zeros(3)]:
        R = rodrigues(r)[0]
        np.testing.assert_allclose(rot_log(R), cv2.Rodrigues(R)[0].ravel(), atol=1e-9)
