"""cb_rigid_pose_robust (DESIGN.md section 4.14) against its oracle: pinhole, free-intrinsics and fisheye rigs, both lane
counts, camera tables on both sides of the shared-memory limit, priors and camera covariance on and off, groups without
enough triangulated markers, markers seen by one camera, caller order, device-resident inputs, repeatability, refused
arguments, the single-camera limit against resect_robust and a reduced tracking scene."""
import ctypes as C

import numpy as np
import pytest

from caliscope_b200 import _lib as L
from caliscope_b200.resection import resect_robust
from caliscope_b200.rigid import RigidStats, pose_rigid_robust
from oracle.ba_oracle import rodrigues
from oracle.resection_robust import rot_log
from oracle.rigid_pose_robust import rigid_pose_robust
from tests._rigid_cases import camera_cov, make_bodies, perturb, plant_outliers

pytestmark = pytest.mark.gpu


def _both(b, obs=None, **kw):
    obs = b.obs() if obs is None else obs
    kw.setdefault("threshold_px", 4.0)
    st = RigidStats()
    dev = pose_rigid_robust(*b.rig(), b.model, *obs, stats=st, **kw)
    orc = rigid_pose_robust(*b.rig(), b.model, *obs, **kw)
    return dev, orc, st


def _check(dev, orc, near_tie=1e-9, cov_rtol=1e-7):
    """Exact count / rep_row / n_points; status, inliers and n_inliers away from near-tie scores (the device's Horn pose
    is a Jacobi eigenvector, the oracle's LAPACK's: equal to rounding, so scores within rounding can swap); pose to
    1e-8, cov to cov_rtol."""
    np.testing.assert_array_equal(dev.count, orc.count)
    np.testing.assert_array_equal(dev.rep_row, orc.rep_row)
    np.testing.assert_array_equal(dev.n_points, orc.n_points)
    # an exact tie is a triple drawn twice by the hashed rule (the same hypothesis): both sides keep the lower slot
    with np.errstate(invalid="ignore"):
        gap = orc.second - orc.best
    tie = np.isfinite(orc.second) & (gap > 0) & (gap <= near_tie * np.maximum(1.0, orc.best))
    assert tie.mean() <= 0.1
    ok = ~tie
    np.testing.assert_array_equal(dev.status[ok], orc.status[ok])
    np.testing.assert_array_equal(dev.n_inliers[ok], orc.n_inliers[ok])
    both = ok & np.isin(orc.status, (0, 3, 4))
    sc = np.maximum(1.0, np.abs(orc.pose[both]))
    assert np.all(np.abs(dev.pose[both] - orc.pose[both]) <= 1e-8 * sc), np.abs(dev.pose[both] - orc.pose[both]).max()
    np.testing.assert_allclose(dev.rmse_px[both], orc.rmse_px[both], rtol=1e-8, atol=1e-12)
    c_o, c_d = orc.cov[both], dev.cov[both]
    cs = np.maximum(np.abs(c_o).max(axis=(1, 2), keepdims=True), 1e-300)
    assert np.all(np.abs(c_d - c_o) / cs <= cov_rtol), (np.abs(c_d - c_o) / cs).max()
    assert np.isnan(dev.pose[orc.status == 5]).all() and np.isnan(dev.cov[orc.status == 5]).all()
    return ok


def _inliers_agree(dev, orc, b, ok):
    keys = np.unique(b.obs_key)
    row_ok = ok[np.searchsorted(keys, b.obs_key)]
    np.testing.assert_array_equal(dev.inlier[row_ok], orc.inlier[row_ok])


@pytest.mark.parametrize("kind", ["pinhole", "free", "fisheye"])
@pytest.mark.parametrize("lanes", [8, 32])
def test_matches_oracle(kind, lanes):
    n_cams = 8 if lanes == 8 else 20  # 20 cameras x 12 markers x 0.7 ~ 168 rows per group: 32 lanes
    fisheye = tuple(range(0, n_cams, 3)) if kind == "fisheye" else ()
    free = tuple(range(1, n_cams, 2)) if kind == "free" else ()
    b = make_bodies(11, n_cams=n_cams, n_frames=24, fisheye=fisheye, free=free, noise=0.4)
    b.obs_px, _ = plant_outliers(12, b.obs_px, 0.05)
    cc = camera_cov(b.flags)
    prior = (np.arange(0, 24, 2), b.truth[::2] + 0.01)
    dev, orc, st = _both(b, prior=prior, camera_cov=cc, pixel_sigma=0.4)
    assert (n_cams * 12 * 0.7 > 96) == (lanes == 32)
    assert st.kernel_launches > 0 and st.n_groups == 24
    ok = _check(dev, orc)
    _inliers_agree(dev, orc, b, ok)
    assert (orc.status == 0).mean() > 0.9


@pytest.mark.parametrize("n_cams", [64, 160])
@pytest.mark.parametrize("with_prior, with_cov", [(False, False), (True, True)])
def test_camera_table_sides(n_cams, with_prior, with_cov):
    """64 cameras keep the camera table in shared memory, 160 read it from global memory."""
    b = make_bodies(13, n_cams=n_cams, n_frames=6, n_model=8, noise=0.3, visible=0.15, radius=4.0,
                    free=(3, 70) if n_cams > 70 else (3,))  # fmt: skip
    kw = {}
    if with_prior:
        kw["prior"] = (np.arange(6), b.truth + 0.005)
    if with_cov:
        kw["camera_cov"] = camera_cov(b.flags)
    dev, orc, _ = _both(b, **kw)
    ok = _check(dev, orc)
    _inliers_agree(dev, orc, b, ok)


def test_too_few_qualified_points_and_single_camera_markers():
    """A group whose markers are each seen by one camera has no qualified point: status 5 without a prior, 0 with one;
    markers seen by one camera take part in the consensus and refinement of every group."""
    b = make_bodies(14, n_cams=6, n_frames=10, n_model=10, noise=0.3, visible=1.0)
    single = b.obs_cam == (b.obs_pt % 6)
    keep = np.where(b.obs_key < 5, single, single | (b.obs_pt < 5))  # frames 5..9: markers 5..9 by one camera only
    obs = [a[keep] for a in b.obs()]
    dev, orc, _ = _both(b, obs=obs)
    assert (dev.status[:5] == 5).all() and (dev.n_points[:5] == 0).all()
    assert (dev.status[5:] == 0).all() and (dev.n_points[5:] == 5).all()
    _check(dev, orc)
    lone = keep & (b.obs_pt >= 5) & (b.obs_key >= 5)
    assert dev.inlier[np.flatnonzero(lone[keep])].all()
    dev, orc, _ = _both(b, obs=obs, prior=(np.arange(10), b.truth))
    assert (dev.status == 0).all()
    _check(dev, orc)


def test_caller_order_device_inputs_and_repeatability():
    torch = pytest.importorskip("torch")
    b = make_bodies(15, n_cams=8, n_frames=30, noise=0.3)
    b.obs_px, _ = plant_outliers(16, b.obs_px, 0.05)
    kw = dict(threshold_px=4.0, camera_cov=camera_cov(b.flags), prior=(np.arange(0, 30, 3), b.truth[::3]))
    a = pose_rigid_robust(*b.rig(), b.model, *b.obs(), **kw)
    a2 = pose_rigid_robust(*b.rig(), b.model, *b.obs(), **kw)
    for f in ("pose", "cov", "rmse_px", "status", "n_inliers", "inlier"):
        assert getattr(a, f).tobytes() == getattr(a2, f).tobytes(), f
    perm = np.random.default_rng(0).permutation(len(b.obs_cam))
    s = pose_rigid_robust(*b.rig(), b.model, *(x[perm] for x in b.obs()), **kw)
    # the order within a key changes the sample positions only through the sub-group order, which is by model point:
    # results are the same up to the order of sums
    np.testing.assert_array_equal(s.status, a.status)
    np.testing.assert_array_equal(s.inlier, a.inlier[perm])
    np.testing.assert_allclose(s.pose, a.pose, rtol=0, atol=1e-9)
    dev = [torch.as_tensor(np.ascontiguousarray(x), device="cuda:0") for x in
           (b.obs_cam.astype(np.int32), b.obs_key.astype(np.int64), b.obs_pt.astype(np.int32), b.obs_px)]  # fmt: skip
    d = pose_rigid_robust(*b.rig(), b.model, *dev, **kw)
    for f in ("pose", "cov", "rmse_px", "status", "n_inliers", "inlier", "key"):
        assert getattr(d, f).tobytes() == getattr(a, f).tobytes(), f


def _raw(b, **over):
    lib = L.load()
    n = len(b.obs_cam)
    flags = np.ascontiguousarray(b.flags, np.int32)
    const = np.ascontiguousarray(b.const)
    cx = np.ascontiguousarray(b.cam_x)
    model = np.ascontiguousarray(b.model)
    cam, key = np.ascontiguousarray(b.obs_cam, np.int32), np.ascontiguousarray(b.obs_key, np.int64)
    pt, px = np.ascontiguousarray(b.obs_pt, np.int32), np.ascontiguousarray(b.obs_px)
    a = dict(threshold_px=4.0, min_inliers=6, max_pairs=16, max_samples=64, pkey=np.zeros(0, np.int64),
             ppose=np.zeros((0, 6)), pixel_sigma=1.0, max_iter=20, xtol=1e-12, n_model=len(model))  # fmt: skip
    a.update(over)
    outs = [np.zeros((n, 6)), np.zeros((n, 36)), np.zeros(n)] + [np.zeros(n, np.int32) for _ in range(5)]
    inl = np.zeros(n, np.uint8)
    ng = C.c_int32(0)
    st = L.RigidStats()
    p = lambda x: x.ctypes.data_as(C.c_void_p)  # noqa: E731
    code = lib.cb_rigid_pose_robust(len(flags), p(flags), p(const), p(cx), None, a["n_model"], p(model), n, p(cam),
                                    p(key), p(pt), p(px), 0, a["threshold_px"], a["min_inliers"], a["max_pairs"],
                                    a["max_samples"], len(a["pkey"]), p(np.ascontiguousarray(a["pkey"])),
                                    p(np.ascontiguousarray(a["ppose"])), a["pixel_sigma"], a["max_iter"], a["xtol"], n,
                                    C.byref(ng), *(p(o) for o in outs), p(inl), C.byref(st), 0, None)  # fmt: skip
    return code, st, (lib.cb_ba_last_error() or b"").decode()


def test_refused_arguments():
    b = make_bodies(17, n_cams=6, n_frames=3)
    code, st, _ = _raw(b)
    assert code == 0 and st.kernel_launches > 0
    bad = [dict(threshold_px=0.0), dict(threshold_px=np.inf), dict(min_inliers=3), dict(max_pairs=0),
           dict(max_samples=0), dict(max_samples=4097), dict(pixel_sigma=-1.0), dict(max_iter=0), dict(xtol=np.nan),
           dict(pkey=np.array([2, 1]), ppose=np.zeros((2, 6))), dict(pkey=np.array([1, 1]), ppose=np.zeros((2, 6))),
           dict(pkey=np.array([0]), ppose=np.full((1, 6), np.nan))]  # fmt: skip
    for kw in bad:
        code, st, err = _raw(b, **kw)
        assert code == -1 and "cb_rigid_pose_robust" in err, kw
        assert st.kernel_launches == 0 and st.total_ms == 0.0, kw
    code, _, err = _raw(b, n_model=len(b.model) - 1)  # obs_pt out of range: found on the device
    assert code == -1 and "model point index out of range" in err
    code, st, _ = _raw(b)
    assert code == 0


def test_single_camera_with_prior_reaches_resection_optimum():
    """A body seen by one camera, its prior near the truth: the pose is resect_robust's camera pose (model frame as the
    world) composed with the camera's pose in the rig."""
    b = make_bodies(18, n_cams=4, n_frames=5, n_model=16, noise=0.0, visible=1.0)
    sel = b.obs_cam == 2
    obs = [a[sel] for a in b.obs()]
    prior = (np.arange(5), b.truth + 0.002)
    dev = pose_rigid_robust(*b.rig(), b.model, *obs, threshold_px=4.0, prior=prior)
    assert (dev.status == 0).all() and (dev.n_points == 0).all()
    # resection of camera 2 against the model: one camera per frame, x = the camera's intrinsics
    off = np.concatenate([[0], np.cumsum(np.where(b.flags & 1, 9, 6))])
    qc = b.cam_x[off[2] : off[3]]
    Rc, tc = rodrigues(qc[:3])[0], qc[3:6]
    flags1, const1 = b.flags[2:3], b.const[2:3]
    for g in range(5):
        rows = obs[1] == g
        x0 = qc.copy()
        Rb = rodrigues(prior[1][g, :3])[0]
        Rp = Rc @ Rb
        x0[:3], x0[3:6] = rot_log(Rp), Rc @ prior[1][g, 3:] + tc
        r = resect_robust(flags1, const1, x0, b.model, np.zeros(rows.sum(), np.int32), np.zeros(rows.sum(), np.int64),
                          obs[2][rows], obs[3][rows], threshold_px=4.0)  # fmt: skip
        assert r.status[0] == 0
        Rr, tr = rodrigues(r.pose[0, :3])[0], r.pose[0, 3:]
        Rw, tw = Rc.T @ Rr, Rc.T @ (tr - tc)
        np.testing.assert_allclose(rodrigues(dev.pose[g, :3])[0], Rw, atol=1e-8)
        np.testing.assert_allclose(dev.pose[g, 3:], tw, atol=1e-8)


def test_reduced_track_scene():
    """DESIGN section 4.9's track scene, reduced: a 0.2 m cluster of 12 markers 3 m from 8 cameras, 5 % of the rows
    moved up to 200 px."""
    b = make_bodies(19, n_cams=8, n_frames=2000, n_model=12, noise=0.5, visible=1.0, size=0.2, radius=3.0)
    b.obs_px, moved = plant_outliers(20, b.obs_px, 0.05, lo=10.0, hi=200.0)
    r = pose_rigid_robust(*b.rig(), b.model, *b.obs(), threshold_px=3.0, pixel_sigma=0.5)
    ok = r.status == 0
    assert ok.mean() >= 0.99
    assert (~r.inlier[moved]).mean() >= 0.99
    e = r.pose[ok] - b.truth[ok]
    d = np.einsum("gi,gi->g", e, np.linalg.solve(r.cov[ok], e[:, :, None])[:, :, 0])
    assert abs(d.mean() - 6.0) < 4 * np.sqrt(12 / len(d)) + 0.3, d.mean()
    cc = camera_cov(b.flags, rot=5e-4, trans=1e-3)
    rc = pose_rigid_robust(b.flags, b.const, perturb(21, b.cam_x, cc), b.model, *b.obs(), threshold_px=3.0,
                           pixel_sigma=0.5, camera_cov=cc)  # fmt: skip
    assert (rc.status == 0).mean() >= 0.99 and np.isfinite(rc.cov[rc.status == 0]).all()
