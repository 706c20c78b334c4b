"""cb_rigid_pose_robust_gp3p (DESIGN.md section 4.14, gP3P hypotheses) against its oracle: pinhole, free-intrinsics and
fisheye sparse rigs, both lane counts, camera tables on both sides of the shared-memory limit, priors and camera
covariance on and off; groups with three or more triangulated markers bit-identical to a call without gP3P, and that
call bit-identical to cb_rigid_pose_robust; the single-camera limit against resect_robust without a prior; the sample
rule's edges; repeatability, device-resident inputs, caller order, refused arguments and a reduced sparse tracking
scene."""
import ctypes as C

import numpy as np
import pytest

from caliscope_b200 import _lib as L
from caliscope_b200.resection import resect_robust
from caliscope_b200.rigid import RigidStats, pose_rigid_robust
from oracle.ba_oracle import rodrigues
from oracle.resection_robust import rot_log
from oracle.rigid_pose_gp3p import rigid_pose_gp3p
from tests._gp3p_cases import mixed, one_view, sparse_bodies
from tests._rigid_cases import camera_cov, make_bodies, plant_outliers
from tests.test_gpu_rigid_pose import _check, _inliers_agree

pytestmark = pytest.mark.gpu

FIELDS = ("pose", "cov", "rmse_px", "count", "n_inliers", "n_points", "rep_row", "status")


def _both(b, obs=None, **kw):
    obs = b.obs() if obs is None else obs
    kw.setdefault("threshold_px", 4.0)
    kw.setdefault("gp3p_samples", 64)
    st = RigidStats()
    dev = pose_rigid_robust(*b.rig(), b.model, *obs, stats=st, **kw)
    orc = rigid_pose_gp3p(*b.rig(), b.model, *obs, **kw)
    return dev, orc, st


def _mixed(seed, n_cams, n_frames, n_model=12, keep=0.85, **kw):
    """Even frames with every marker in one random camera's row (no triangulated marker), the rows of odd frames kept
    with probability `keep`."""
    b = make_bodies(seed, n_cams=n_cams, n_frames=n_frames, n_model=n_model, visible=1.0, **kw)
    return mixed(b, seed, np.arange(0, n_frames, 2), keep)


@pytest.mark.parametrize("kind", ["pinhole", "free", "fisheye"])
@pytest.mark.parametrize("lanes", [8, 32])
@pytest.mark.parametrize("with_prior_cov", [False, True])
def test_matches_oracle(kind, lanes, with_prior_cov):
    n_cams = 8 if lanes == 8 else 20  # 20 cameras: about 110 rows per group on average, so 32 lanes
    fisheye = tuple(range(0, n_cams, 3)) if kind == "fisheye" else ()
    free = tuple(range(1, n_cams, 2)) if kind == "free" else ()
    b = _mixed(31, n_cams, 24, fisheye=fisheye, free=free, noise=0.4)
    b.obs_px, _ = plant_outliers(32, b.obs_px, 0.03)
    kw = {}
    if with_prior_cov:
        kw = dict(prior=(np.arange(0, 24, 4), b.truth[::4] + 0.01), camera_cov=camera_cov(b.flags), pixel_sigma=0.4)
    dev, orc, st = _both(b, **kw)
    assert (len(b.obs_cam) / 24 > 96) == (lanes == 32)
    assert st.kernel_launches > 0 and st.n_groups == 24
    ok = _check(dev, orc)
    _inliers_agree(dev, orc, b, ok)
    assert (dev.n_points[::2] == 0).all() and (dev.status[::2] == 0).mean() >= 0.9


@pytest.mark.parametrize("n_cams", [64, 160])
@pytest.mark.parametrize("with_prior, with_cov", [(False, False), (True, True)])
def test_camera_table_sides(n_cams, with_prior, with_cov):
    """64 cameras keep the camera table in shared memory, 160 read it from global memory."""
    b = make_bodies(33, n_cams=n_cams, n_frames=6, n_model=8, noise=0.3, visible=1.0, radius=4.0,
                    free=(3, 70) if n_cams > 70 else (3,))  # fmt: skip
    b = mixed(b, 34, [0, 2, 4], 0.15)
    kw = {}
    if with_prior:
        kw["prior"] = (np.array([1, 3]), b.truth[[1, 3]] + 0.005)
    if with_cov:
        kw["camera_cov"] = camera_cov(b.flags)
    dev, orc, _ = _both(b, **kw)
    ok = _check(dev, orc)
    _inliers_agree(dev, orc, b, ok)


def test_groups_with_triangulated_markers_are_bit_identical():
    b = _mixed(35, 8, 40, noise=0.4)
    b.obs_px, _ = plant_outliers(36, b.obs_px, 0.05)
    kw = dict(threshold_px=4.0, camera_cov=camera_cov(b.flags), prior=(np.arange(0, 40, 5), b.truth[::5] + 0.01))
    off = pose_rigid_robust(*b.rig(), b.model, *b.obs(), **kw)
    keys = np.unique(b.obs_key)
    for g in (1, 64, 4096):
        on = pose_rigid_robust(*b.rig(), b.model, *b.obs(), gp3p_samples=g, **kw)
        keep = off.n_points >= 3
        assert keep.sum() == 20
        for f in FIELDS:
            assert getattr(on, f)[keep].tobytes() == getattr(off, f)[keep].tobytes(), (g, f)
        rows = keep[np.searchsorted(keys, b.obs_key)]
        assert on.inlier[rows].tobytes() == off.inlier[rows].tobytes()
        assert (on.status[~keep] == 0).sum() > (off.status[~keep] == 0).sum()


def _raw(b, symbol="cb_rigid_pose_robust_gp3p", cov=None, **over):
    lib = L.load()
    n = len(b.obs_cam)
    flags = np.ascontiguousarray(b.flags, np.int32)
    const = np.ascontiguousarray(b.const)
    cx = np.ascontiguousarray(b.cam_x)
    model = np.ascontiguousarray(b.model)
    cam, key = np.ascontiguousarray(b.obs_cam, np.int32), np.ascontiguousarray(b.obs_key, np.int64)
    pt, px = np.ascontiguousarray(b.obs_pt, np.int32), np.ascontiguousarray(b.obs_px)
    a = dict(threshold_px=4.0, min_inliers=6, max_pairs=16, max_samples=64, gp3p_samples=0,
             pkey=np.zeros(0, np.int64), ppose=np.zeros((0, 6)), pixel_sigma=1.0, max_iter=20, xtol=1e-12)  # fmt: skip
    a.update(over)
    outs = [np.zeros((n, 6)), np.zeros((n, 36)), np.zeros(n)] + [np.zeros(n, np.int32) for _ in range(5)]
    inl = np.zeros(n, np.uint8)
    ng = C.c_int32(0)
    st = L.RigidStats()
    p = lambda x: x.ctypes.data_as(C.c_void_p)  # noqa: E731
    gp = [a["gp3p_samples"]] if symbol.endswith("gp3p") else []
    cc = None if cov is None else p(np.ascontiguousarray(cov))
    code = getattr(lib, symbol)(len(flags), p(flags), p(const), p(cx), cc, len(model), p(model), n, p(cam), p(key),
                                p(pt), p(px), 0, a["threshold_px"], a["min_inliers"], a["max_pairs"], a["max_samples"],
                                *gp, len(a["pkey"]), p(np.ascontiguousarray(a["pkey"])),
                                p(np.ascontiguousarray(a["ppose"])), a["pixel_sigma"], a["max_iter"], a["xtol"], n,
                                C.byref(ng), *(p(o) for o in outs), p(inl), C.byref(st), 0, None)  # fmt: skip
    return code, st, (lib.cb_ba_last_error() or b"").decode(), [o[: ng.value] for o in outs] + [inl]


def test_off_through_the_new_symbol_equals_the_old_symbol():
    b = _mixed(37, 8, 20, noise=0.4)
    cc = camera_cov(b.flags)
    kw = dict(pkey=np.arange(0, 20, 3), ppose=b.truth[::3] + 0.01)
    c_old, _, _, old = _raw(b, "cb_rigid_pose_robust", cov=cc, **kw)
    c_new, _, _, new = _raw(b, cov=cc, gp3p_samples=0, **kw)
    assert c_old == 0 and c_new == 0
    for o, n in zip(old, new):
        assert o.tobytes() == n.tobytes()


def test_single_camera_without_prior_reaches_resection_optimum():
    """A body seen by one camera and no prior: gP3P reduces to P3P, and the pose is resect_robust's camera pose (model
    frame as the world) composed with the camera's pose in the rig."""
    b = make_bodies(38, n_cams=4, n_frames=5, n_model=16, noise=0.0, visible=1.0)
    sel = b.obs_cam == 2
    obs = [a[sel] for a in b.obs()]
    dev = pose_rigid_robust(*b.rig(), b.model, *obs, threshold_px=4.0, gp3p_samples=64)
    assert (dev.status == 0).all() and (dev.n_points == 0).all()
    off = np.concatenate([[0], np.cumsum(np.where(b.flags & 1, 9, 6))])
    qc = b.cam_x[off[2] : off[3]]
    Rc, tc = rodrigues(qc[:3])[0], qc[3:6]
    flags1, const1 = b.flags[2:3], b.const[2:3]
    for g in range(5):
        rows = obs[1] == g
        x0 = qc.copy()
        Rb = rodrigues(b.truth[g, :3] + 0.002)[0]
        x0[:3], x0[3:6] = rot_log(Rc @ Rb), Rc @ (b.truth[g, 3:] + 0.002) + tc
        r = resect_robust(flags1, const1, x0, b.model, np.zeros(rows.sum(), np.int32), np.zeros(rows.sum(), np.int64),
                          obs[2][rows], obs[3][rows], threshold_px=4.0)  # fmt: skip
        assert r.status[0] == 0
        Rr, tr = rodrigues(r.pose[0, :3])[0], r.pose[0, 3:]
        np.testing.assert_allclose(rodrigues(dev.pose[g, :3])[0], Rc.T @ Rr, atol=1e-8)
        np.testing.assert_allclose(dev.pose[g, 3:], Rc.T @ (tr - tc), atol=1e-8)


@pytest.mark.parametrize("g", [20, 19, 1, 4096])
def test_sample_rule_edges(g):
    """k = 6 rows per group: C(6, 3) = 20 at gp3p_samples and one past it, and the ends of the range.  Six rows from six
    cameras hold the depth weakly, so the refinement gets 100 iterations: at 20 a few groups stop at the limit on one
    side and converge on the other."""
    b = one_view(make_bodies(39, n_cams=6, n_frames=40, n_model=6, noise=0.4, visible=1.0), 40)
    assert (np.bincount(b.obs_key) == 6).all()
    dev, orc, _ = _both(b, gp3p_samples=g, threshold_px=3.0, max_iter=100)
    ok = _check(dev, orc)
    _inliers_agree(dev, orc, b, ok)
    if g >= 19:
        assert (dev.status == 0).mean() >= 0.9


def test_caller_order_device_inputs_repeatability_and_refusals():
    torch = pytest.importorskip("torch")
    b = _mixed(41, 8, 30, noise=0.3)
    b.obs_px, _ = plant_outliers(42, b.obs_px, 0.05)
    kw = dict(threshold_px=4.0, camera_cov=camera_cov(b.flags), gp3p_samples=64)
    a = pose_rigid_robust(*b.rig(), b.model, *b.obs(), **kw)
    a2 = pose_rigid_robust(*b.rig(), b.model, *b.obs(), **kw)
    for f in ("pose", "cov", "rmse_px", "status", "n_inliers", "inlier"):
        assert getattr(a, f).tobytes() == getattr(a2, f).tobytes(), f
    # caller order within a key changes the gP3P samples (row positions): the same poses up to the consensus rows
    perm = np.random.default_rng(0).permutation(len(b.obs_cam))
    s = pose_rigid_robust(*b.rig(), b.model, *(x[perm] for x in b.obs()), **kw)
    both = (s.status == 0) & (a.status == 0)
    assert both.mean() >= 0.9
    assert np.abs(s.pose[both, 3:] - a.pose[both, 3:]).max() < 0.02
    orc = rigid_pose_gp3p(*b.rig(), b.model, *(x[perm] for x in b.obs()), **kw)
    _check(s, orc)
    dev = [torch.as_tensor(np.ascontiguousarray(x), device="cuda:0") for x in
           (b.obs_cam.astype(np.int32), b.obs_key.astype(np.int64), b.obs_pt.astype(np.int32), b.obs_px)]  # fmt: skip
    d = pose_rigid_robust(*b.rig(), b.model, *dev, **kw)
    for f in ("pose", "cov", "rmse_px", "status", "n_inliers", "inlier", "key"):
        assert getattr(d, f).tobytes() == getattr(a, f).tobytes(), f
    for bad in (-1, 4097):
        with pytest.raises(ValueError, match="gp3p_samples"):
            pose_rigid_robust(*b.rig(), b.model, *b.obs(), threshold_px=4.0, gp3p_samples=bad)
        code, st, err, _ = _raw(b, gp3p_samples=bad)
        assert code == -1 and "cb_rigid_pose_robust_gp3p" in err
        assert st.kernel_launches == 0 and st.total_ms == 0.0
    code, st, _, _ = _raw(b, gp3p_samples=4096)
    assert code == 0 and st.kernel_launches > 0


def test_reduced_sparse_track_scene():
    """6 cameras, 8 markers, each (marker, camera) row kept with probability 0.25, 3 % of the rows moved up to 200 px:
    about a fifth of the frames have fewer than three triangulated markers.  gP3P poses most of them, and the groups it
    newly poses are within 20 mm of the truth."""
    b = sparse_bodies(43, n_cams=6, n_frames=2000, n_model=8, noise=0.5, visible=0.25)
    b.obs_px, _ = plant_outliers(44, b.obs_px, 0.03, lo=10.0, hi=200.0)
    off = pose_rigid_robust(*b.rig(), b.model, *b.obs(), threshold_px=3.0, pixel_sigma=0.5)
    on = pose_rigid_robust(*b.rig(), b.model, *b.obs(), threshold_px=3.0, pixel_sigma=0.5, gp3p_samples=64)
    assert (off.n_points < 3).mean() >= 0.15
    assert (on.status == 0).mean() >= (off.status == 0).mean() + 0.1
    new = (off.status != 0) & (on.status == 0)
    e = np.linalg.norm(on.pose[new, 3:] - b.truth[new, 3:], axis=1)
    assert np.median(e) < 5e-3 and np.percentile(e, 95) < 2e-2, (np.median(e), np.percentile(e, 95))
