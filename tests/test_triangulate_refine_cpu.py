"""The NumPy oracle of triangulation refinement and point covariance (oracle/triangulation_refine.py refine_points,
point_covariance): derivatives, optimality, first-order covariance by Monte Carlo, and each status code."""
import numpy as np
import pytest

from caliscope_b200 import synthetic
from oracle import triangulation_refine as T


def _ncp(flags):
    return int(np.where(np.asarray(flags) & 1, 9, 6).sum())


def _rig(kind, seed=0, n_pts=30, noise_px=0.5):
    rig = synthetic.make_rig(6, n_pts, 6 * n_pts, refine_intrinsics=kind == "free9", seed=seed, noise_px=noise_px)
    flags, const = rig.cam_flags.copy(), rig.cam_const.copy()
    if kind == "fisheye":
        flags[::2] |= 2
        const[::2, 4:9] = (0.05, -0.01, 0.002, -0.0005, 0.0)
    return rig, flags, const


@pytest.mark.parametrize("kind", ["pinhole6", "free9", "fisheye"])
def test_pixel_jacobians_match_central_differences(kind):
    rig, flags, const = _rig(kind)
    ncp = _ncp(flags)
    cx = rig.x_true[:ncp].copy()
    X = rig.x_true[ncp:].reshape(-1, 3)
    grp = rig.obs_pt.astype(np.int64)
    args = (flags, const)
    _, JX, Jc = T.pixel_jacobians(*args, cx, rig.obs_cam, rig.obs_xy, grp, X)
    h = 1e-6
    for k in range(3):
        d = np.zeros(3)
        d[k] = h
        rp = T.pixel_jacobians(*args, cx, rig.obs_cam, rig.obs_xy, grp, X + d)[0]
        rm = T.pixel_jacobians(*args, cx, rig.obs_cam, rig.obs_xy, grp, X - d)[0]
        assert np.abs((rp - rm) / (2 * h) - JX[:, :, k]).max() < 1e-5 * np.abs(JX).max()
    offs = np.concatenate([[0], np.cumsum(np.where(flags & 1, 9, 6))])
    for q in range(9):
        cols = [o + q for c, o in enumerate(offs[:-1]) if q < offs[c + 1] - o]
        if not cols:
            continue
        cp, cm = cx.copy(), cx.copy()
        cp[cols] += h
        cm[cols] -= h
        rp = T.pixel_jacobians(*args, cp, rig.obs_cam, rig.obs_xy, grp, X)[0]
        rm = T.pixel_jacobians(*args, cm, rig.obs_cam, rig.obs_xy, grp, X)[0]
        assert np.abs((rp - rm) / (2 * h) - Jc[:, :, q]).max() < 1e-5 * max(np.abs(Jc[:, :, q]).max(), 1.0)


def test_noise_free_rig_refines_to_the_truth():
    rig, flags, const = _rig("pinhole6", seed=2, noise_px=0.0)
    ncp = _ncp(flags)
    truth = rig.x_true[ncp:].reshape(-1, 3)
    start = truth + np.random.default_rng(0).normal(0, 0.005, truth.shape)
    xyz, rmse, status, _ = T.refine_points(flags, const, rig.x_true[:ncp], rig.obs_cam, rig.obs_xy, rig.obs_pt, start)
    ok = np.bincount(rig.obs_pt, minlength=len(truth)) >= 2
    assert np.all(status[ok] == 0)
    assert np.abs(xyz[ok] - truth[ok]).max() < 1e-9
    assert rmse[ok].max() < 1e-6


@pytest.mark.parametrize("kind", ["pinhole6", "free9", "fisheye"])
def test_refined_rmse_is_never_above_the_dlt_rmse(kind):
    rig, flags, const = _rig(kind, seed=3, n_pts=200)
    ncp = _ncp(flags)
    cx = rig.x_true[:ncp]
    grp, G = T.group_rows(rig.obs_pt)
    x0 = T.dlt_start(flags, const, cx, rig.obs_cam, rig.obs_xy, grp, G)
    xyz, rmse, status, _ = T.refine_points(flags, const, cx, rig.obs_cam, rig.obs_xy, grp, x0)
    r0 = T.pixel_jacobians(flags, const, cx, rig.obs_cam, rig.obs_xy, grp, np.nan_to_num(x0))[0]
    n = np.bincount(grp, minlength=G)
    rmse0 = np.sqrt(np.bincount(grp, weights=(r0 * r0).sum(axis=1), minlength=G) / n)
    ok = status == 0
    assert ok.sum() > 0.9 * G
    assert np.all(rmse[ok] <= rmse0[ok])


def _mc_setup():
    rig = synthetic.make_rig(8, 400, 3200, seed=5, noise_px=0.0)
    ncp = _ncp(rig.cam_flags)
    cnt = np.bincount(rig.obs_pt, minlength=rig.n_pts)
    j = int(np.flatnonzero(cnt == 5)[0])  # one point seen by five cameras
    rows = np.flatnonzero(rig.obs_pt == j)
    return rig, ncp, rows, rig.x_true[ncp:].reshape(-1, 3)[j]


def _eig_ratio(emp, theory):
    w, V = np.linalg.eigh(theory)
    isq = V @ np.diag(w**-0.5) @ V.T
    return np.linalg.eigvalsh(isq @ emp @ isq)


def test_monte_carlo_pixel_term_matches_sigma2_hinv():
    rig, ncp, rows, X = _mc_setup()
    sigma, draws = 0.05, 2000
    rng = np.random.default_rng(11)
    k = len(rows)
    cam = np.tile(rig.obs_cam[rows], draws)
    px = np.tile(rig.obs_xy[rows], (draws, 1)) + rng.normal(0, sigma, (k * draws, 2))
    grp = np.repeat(np.arange(draws), k)
    xyz, _, status, _ = T.refine_points(rig.cam_flags, rig.cam_const, rig.x_true[:ncp], cam, px, grp, np.tile(X, (draws, 1)))
    assert np.all(status == 0)
    cov = T.point_covariance(rig.cam_flags, rig.cam_const, rig.x_true[:ncp], rig.obs_cam[rows], rig.obs_xy[rows],
                             np.zeros(k, np.int64), X[None], np.zeros(1, np.int32), sigma)[0]  # fmt: skip
    r = _eig_ratio(np.cov(xyz.T), cov)
    assert np.all(np.abs(r - 1) < 0.15), r


def test_monte_carlo_camera_term_matches_propagated_camera_covariance():
    rig, ncp, rows, X = _mc_setup()
    draws = 2000
    rng = np.random.default_rng(12)
    Lc = 2e-4 * (np.eye(ncp) + 0.3 * rng.normal(size=(ncp, ncp)) / np.sqrt(ncp))
    Sc = Lc @ Lc.T
    k = len(rows)
    # every draw gets its own copy of the cameras, so all draws refine in one call
    cams = rng.multivariate_normal(rig.x_true[:ncp], Sc, draws)
    flags = np.tile(rig.cam_flags, draws)
    const = np.tile(rig.cam_const, (draws, 1))
    cam = (rig.obs_cam[rows][None, :] + rig.n_cams * np.arange(draws)[:, None]).ravel()
    px = np.tile(rig.obs_xy[rows], (draws, 1))
    grp = np.repeat(np.arange(draws), k)
    xyz, _, status, _ = T.refine_points(flags, const, cams.ravel(), cam, px, grp, np.tile(X, (draws, 1)))
    assert np.all(status == 0)
    cov = T.point_covariance(rig.cam_flags, rig.cam_const, rig.x_true[:ncp], rig.obs_cam[rows], rig.obs_xy[rows],
                             np.zeros(k, np.int64), X[None], np.zeros(1, np.int32), 0.0, Sc)[0]  # fmt: skip
    r = _eig_ratio(np.cov(xyz.T), cov)
    assert np.all(np.abs(r - 1) < 0.15), r


def _pinhole(centres, f=1000.0):
    """Identity-rotation cameras at `centres`: (flags, const, cam_x)."""
    n = len(centres)
    const = np.tile([f, f, 640.0, 480.0, 0, 0, 0, 0, 0], (n, 1)).astype(float)
    x = np.concatenate([np.r_[0.0, 0.0, 0.0, -np.asarray(c, float)] for c in centres])
    return np.zeros(n, np.int32), const, x


def _px(X, c, f=1000.0):
    d = np.asarray(X, float) - np.asarray(c, float)
    return [f * d[0] / d[2] + 640.0, f * d[1] / d[2] + 480.0]


def test_status_codes():
    X = np.array([0.5, 0.1, 2.0])
    cen = [(0, 0, 0), (1, 0, 0), (0.5, 0, 4.0), (0.1, 0, 0)]
    flags, const, cx = _pinhole(cen)
    pts = {
        0: [(0, X), (1, X)],  # ok
        1: [(0, X)],  # one row
        2: [(0, X), (0, X)],  # two rows from one camera
        3: [(0, None), (3, None)],  # parallel rays: the same pixel in two cameras of equal orientation
        4: [(0, X), (1, X), (2, X)],  # behind camera 2
    }
    cam, px, grp = [], [], []
    for g, obs in pts.items():
        for c, P in obs:
            cam.append(c)
            px.append(_px(P, cen[c]) if P is not None else [740.0, 480.0])
            grp.append(g)
    cam, px, grp = np.array(cam, np.int32), np.array(px), np.array(grp, np.int64)
    x0 = T.dlt_start(flags, const, cx, cam, px, grp, 5)
    xyz, rmse, status, _ = T.refine_points(flags, const, cx, cam, px, grp, x0)
    assert status.tolist() == [0, 1, 2, 2, 4]
    assert np.abs(xyz[0] - X).max() < 1e-9 and np.abs(xyz[4] - X).max() < 1e-9
    assert np.isnan(xyz[1]).all() and np.isnan(rmse[1])
    assert np.array_equal(xyz[2], x0[2], equal_nan=True)
    cov = T.point_covariance(flags, const, cx, cam, px, grp, xyz, status, 1.0)
    assert np.isnan(cov[[1, 2, 3]]).all() and np.isfinite(cov[[0, 4]]).all()
    # the iteration limit
    _, _, st1, it1 = T.refine_points(flags, const, cx, cam, px, grp, x0 + 0.01, max_iter=1)
    assert st1[0] == 3 and it1[0] == 1
