"""cb_rigid_model_refine on the GPU against its oracle (oracle/rigid_model.py): rigs, body sizes, several bodies,
cluster sizes, device-resident inputs, caller order, repeatability, refused arguments and the round trip through
rigid-body pose."""
from __future__ import annotations

import numpy as np
import pytest

from oracle.rigid_model import rigid_model_refine
from tests._rigid_cases import camera_cov
from tests._rigid_model_cases import behind_scene, check, kabsch_error, make_scene, multi_body, one_camera_marker_scene

pytestmark = pytest.mark.gpu


def _dev(sc, **kw):
    from caliscope_b200 import rigid

    b = sc.bodies
    return rigid.refine_rigid_model(b.flags, b.const, b.cam_x, sc.nominal, b.obs_cam, b.obs_key, b.obs_pt, b.obs_px,
                                    (sc.start_key, sc.start_pose), bodies=sc.body_start, **kw)  # fmt: skip


@pytest.mark.parametrize("with_cam", [False, True])
@pytest.mark.parametrize("kw", [dict(), dict(free=(0, 2, 5)), dict(fisheye=(1, 4))])
@pytest.mark.parametrize("K", [3, 4, 32])
def test_against_oracle(kw, K, with_cam):
    sc = make_scene(40 + K, n_model=K, n_frames=10, **kw)
    ccov = camera_cov(sc.bodies.flags) if with_cam else None
    o = rigid_model_refine(*sc.args(), body_start=sc.body_start, pixel_sigma=0.5, camera_cov=ccov)
    check(_dev(sc, pixel_sigma=0.5, camera_cov=ccov), o)


@pytest.mark.parametrize("with_cam", [False, True])
def test_multi_body(with_cam):
    sc = multi_body(41, free=(1,))
    ccov = camera_cov(sc.bodies.flags) if with_cam else None
    check(_dev(sc, camera_cov=ccov), rigid_model_refine(*sc.args(), body_start=sc.body_start, camera_cov=ccov))


def test_statuses():
    sc = make_scene(43, n_model=5, n_frames=8)
    o = rigid_model_refine(*sc.args(), body_start=sc.body_start, max_iter=1)
    assert o.status[0] == 3
    check(_dev(sc, max_iter=1), o)
    sc.nominal = np.outer([-1.5, -0.5, 0.5, 1.5, 2.5], [0.03, -0.02, 0.05])  # collinear
    o = rigid_model_refine(*sc.args(), body_start=sc.body_start)
    assert o.status[0] == 2
    check(_dev(sc), o)
    for sc, st in ((one_camera_marker_scene(45), 2), (behind_scene(45), 4)):
        o = rigid_model_refine(*sc.args(), body_start=sc.body_start, camera_cov=camera_cov(sc.bodies.flags))
        assert o.status[0] == st
        check(_dev(sc, camera_cov=camera_cov(sc.bodies.flags)), o)
    sc = make_scene(47, n_model=5, n_frames=8)  # a marker never seen, and a frame with two markers
    b = sc.bodies
    keep = (b.obs_pt != 4) & ((b.obs_key != 0) | (b.obs_pt < 2))
    for name in ("obs_cam", "obs_key", "obs_pt", "obs_px"):
        setattr(b, name, getattr(b, name)[keep])
    o = rigid_model_refine(*sc.args(), body_start=sc.body_start)
    assert o.status[0] == 1 and (o.frame_status == 1).all()
    check(_dev(sc), o)


@pytest.mark.parametrize("n_frames", [5, 64, 65, 300])
def test_cluster_edges(n_frames):
    sc = make_scene(47, n_model=4, n_frames=n_frames, visible=0.8)
    check(_dev(sc), rigid_model_refine(*sc.args(), body_start=sc.body_start))


def test_inputs_order_and_repeatability():
    import torch

    sc = make_scene(53, n_model=6, n_frames=40)
    a, b = _dev(sc), _dev(sc)
    assert np.array_equal(a.model, b.model) and np.array_equal(a.pose, b.pose)
    assert np.array_equal(a.cov[0], b.cov[0], equal_nan=True)
    bo = sc.bodies
    dev = [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in bo.obs()]
    from caliscope_b200 import rigid

    c = rigid.refine_rigid_model(bo.flags, bo.const, bo.cam_x, sc.nominal, *dev, (sc.start_key, sc.start_pose),
                                 bodies=sc.body_start)  # fmt: skip
    assert np.array_equal(a.model, c.model) and np.array_equal(a.pose, c.pose) and np.array_equal(a.key, c.key)
    perm = np.random.default_rng(0).permutation(len(bo.obs_cam))
    for name in ("obs_cam", "obs_key", "obs_pt", "obs_px"):
        setattr(bo, name, getattr(bo, name)[perm])
    d = _dev(sc)
    assert np.abs(d.model - a.model).max() <= 1e-10 and np.abs(d.pose - a.pose).max() <= 1e-9


def test_refused_arguments():
    from caliscope_b200._lib import EngineError

    sc = make_scene(59, n_model=4, n_frames=6)
    for kw in (dict(max_iter=0), dict(pixel_sigma=np.inf), dict(pixel_sigma=np.nan), dict(xtol=np.nan)):
        with pytest.raises(EngineError, match="cb_rigid_model_refine"):
            _dev(sc, **kw)
    for bs in ([0, 2, 4], [0, 3], [1, 4], [0, 4, 3]):  # K = 2, not ending at n_model, not from 0, descending
        sc.body_start = np.array(bs)
        with pytest.raises(EngineError, match="cb_rigid_model_refine"):
            _dev(sc)
    sc.body_start = np.array([0, 4])
    big = make_scene(61, n_model=33, n_frames=4)
    with pytest.raises(EngineError, match="cb_rigid_model_refine"):
        _dev(big)
    sc.start_key = sc.start_key[::-1].copy()
    sc.start_pose = sc.start_pose[::-1].copy()
    with pytest.raises(EngineError, match="cb_rigid_model_refine"):
        _dev(sc)
    sc = make_scene(59, n_model=6, n_frames=6)  # every key spans both bodies
    sc.body_start = np.array([0, 3, 6])
    with pytest.raises(EngineError, match="cb_rigid_model_refine"):
        _dev(sc)


def test_round_trip_through_rigid_pose():
    from caliscope_b200 import rigid

    sc = make_scene(67, n_model=6, n_frames=20, noise=0.3)
    d = _dev(sc)
    b = sc.bodies
    p = rigid.pose_rigid_robust(b.flags, b.const, b.cam_x, d.model, b.obs_cam, b.obs_key, b.obs_pt, b.obs_px,
                                threshold_px=50.0, prior=(d.key, d.pose), max_iter=50)  # fmt: skip
    assert (p.status == 0).all() and (p.key == d.key).all()
    assert np.abs(p.pose - d.pose).max() <= 1e-8


def _world_error(sc, layout, keys, poses):
    """RMS over frames and markers of the world position of the truth's markers predicted by (layout, pose)."""
    from oracle.ba_oracle import rodrigues

    b = sc.bodies
    idx = np.searchsorted(np.unique(b.obs_key), keys)
    e = []
    for q, i in zip(poses, idx):
        t = b.truth[i]
        e.append(layout @ rodrigues(q[:3])[0].T + q[3:] - (sc.truth_model @ rodrigues(t[:3])[0].T + t[3:]))
    return float(np.sqrt(np.mean(np.square(e))))


def test_reduced_track_scene():
    """From poses that pose_rigid_robust gives on a 2 mm-off nominal layout: the layout error against the truth and
    the re-posed frames' errors fall by the factors the oracle gives."""
    from caliscope_b200 import rigid

    sc = make_scene(71, n_model=10, n_frames=200, noise=0.5, model_off=2e-3)
    b = sc.bodies
    p1 = rigid.pose_rigid_robust(b.flags, b.const, b.cam_x, sc.nominal, b.obs_cam, b.obs_key, b.obs_pt, b.obs_px,
                                 threshold_px=4.0)  # fmt: skip
    use = p1.inlier
    for name in ("obs_cam", "obs_key", "obs_pt", "obs_px"):
        setattr(b, name, getattr(b, name)[use])
    sc.start_key, sc.start_pose = p1.key, p1.pose
    o = rigid_model_refine(*sc.args(), body_start=sc.body_start)
    d = _dev(sc)
    check(d, o)
    e0 = np.linalg.norm(kabsch_error(sc.nominal, sc.truth_model))
    eo, ed = np.linalg.norm(kabsch_error(o.model, sc.truth_model)), np.linalg.norm(kabsch_error(d.model, sc.truth_model))
    assert ed < 0.5 * e0 and abs(e0 / ed - e0 / eo) <= 1e-6 * (e0 / eo)
    p2 = rigid.pose_rigid_robust(b.flags, b.const, b.cam_x, d.model, b.obs_cam, b.obs_key, b.obs_pt, b.obs_px,
                                 threshold_px=4.0, prior=(d.key, d.pose))  # fmt: skip
    w1 = _world_error(sc, sc.nominal, p1.key, p1.pose)
    w2, wo = _world_error(sc, d.model, p2.key, p2.pose), _world_error(sc, o.model, o.key, o.pose)
    assert w2 < w1 and abs(w1 / w2 - w1 / wo) <= 1e-3 * (w1 / wo)
