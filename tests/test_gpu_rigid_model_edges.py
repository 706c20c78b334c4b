"""cb_rigid_model_refine on the GPU against its oracle (oracle/rigid_model.py) at the edges of its device path: used-frame
counts at every cluster-size and round edge, bodies of 3 to 32 markers with gaps in their frames' masks, frames at the
frame-use boundary, every status in one call, camera-term runs of one row and of more than 32, 64-camera rigs, extreme
and shuffled keys, the iteration limit, and long and many-body calls.  The scenes are in tests/_rigid_model_edges.py;
tests/test_rigid_model_edges_cpu.py checks without a GPU that each one hits the edge it claims."""
from __future__ import annotations

import numpy as np
import pytest

from oracle.rigid_model import rigid_model_refine
from tests._rigid_cases import camera_cov
from tests._rigid_model_cases import behind_scene, check, make_scene, multi_body
from tests._rigid_model_edges import (BOUNDARY_KEYS, EXTREME_KEYS, MIX_MAX_ITER, MIX_STATUS, MIXED_FRAMES, body_alone,
                                      camterm_scene, cluster_scene, cluster_size, far_scene, key_scene,
                                      marker_scene, mixed_cluster_scene, rounds, status_mix, boundary_scene)  # fmt: skip

pytestmark = pytest.mark.gpu


def _dev(sc, **kw):
    from caliscope_b200 import rigid

    b = sc.bodies
    return rigid.refine_rigid_model(b.flags, b.const, b.cam_x, sc.nominal, b.obs_cam, b.obs_key, b.obs_pt, b.obs_px,
                                    (sc.start_key, sc.start_pose), bodies=sc.body_start, **kw)  # fmt: skip


def _both(sc, cam=False, **kw):
    """The device and the oracle on sc (with the camera term when cam), checked against each other."""
    if cam:
        kw["camera_cov"] = camera_cov(sc.bodies.flags)
    d = _dev(sc, **kw)
    o = rigid_model_refine(*sc.args(), body_start=sc.body_start, **kw)
    check(d, o)
    return d, o


@pytest.mark.parametrize("nf", [1, 32, 33, 224, 225, 256, 257])
def test_cluster_and_round_edges(nf):
    """cs = 1, 1, 2, 7, 8, 8, 8 CTAs and 1, 4, 3, 4, 4, 4, 5 rounds: one active warp, a non-power-of-two cluster, a
    partial last round, full rounds and one warp in the last round; with the camera term."""
    d, _ = _both(cluster_scene(nf), cam=True)
    assert d.n_frames.tolist() == [nf]


def test_small_bodies_on_large_clusters():
    """Bodies of 1 and 5 frames beside one of 300 run on 8-CTA clusters, mostly idle: the same results as alone, up
    to summation order."""
    sc = mixed_cluster_scene()
    d, _ = _both(sc, cam=True)
    assert d.n_frames.tolist() == list(MIXED_FRAMES) and cluster_size(max(MIXED_FRAMES)) == 8
    for i in (0, 1):
        lo, hi = sc.body_start[i], sc.body_start[i + 1]
        a = _dev(body_alone(sc, i), camera_cov=camera_cov(sc.bodies.flags))
        assert a.status[0] == d.status[i] == 0 and a.n_frames[0] == MIXED_FRAMES[i]
        assert np.abs(a.model - d.model[lo:hi]).max() <= 1e-10
        idx = np.searchsorted(d.key, a.key)
        assert (d.key[idx] == a.key).all()
        assert np.abs(a.pose - d.pose[idx]).max() <= 1e-10
        np.testing.assert_allclose(a.rmse_px, d.rmse_px[i : i + 1], rtol=1e-10)
        np.testing.assert_allclose(a.frame_rmse_px, d.frame_rmse_px[idx], rtol=1e-10)
        assert np.abs(a.cov[0] - d.cov[i]).max() <= 1e-9 * np.abs(d.cov[i]).max()


@pytest.mark.parametrize("K", [3, 5, 6, 7, 8, 12, 13, 23, 24, 31, 32])
def test_marker_counts(K):
    """nr = 3K - 6 across 32 and 64 (rmod_solve's lane-strided dots), (3K)^2 across 256 (rmod_accumulate), nr^2 across
    256 (rmod_factor) and the full 32-bit mask, with frames missing marker 0, marker K-1 or every odd marker."""
    d, _ = _both(marker_scene(K))
    assert d.n_frames.tolist() == [12] and d.status[0] == 0


def test_frame_use_boundary():
    """Frames of 3 rows, of 2 markers and without a start pose take no part; a frame of exactly 4 rows and 3 markers
    does; a start key without rows is no frame."""
    sc = boundary_scene()
    d, o = _both(sc)
    k = BOUNDARY_KEYS
    assert k["no_rows"] not in d.key and len(d.key) == 13
    at = {name: int(np.searchsorted(d.key, key)) for name, key in k.items() if name != "no_rows"}
    assert [d.frame_status[at[n]] for n in ("three_rows", "two_markers", "minimal", "no_start")] == [1, 1, 0, 1]
    assert [d.count[at[n]] for n in ("three_rows", "two_markers", "minimal")] == [3, 4, 4]
    unused = d.frame_status == 1
    assert np.isnan(d.frame_rmse_px[unused]).all() and np.isfinite(d.frame_rmse_px[~unused]).all()
    assert np.isnan(d.pose[at["no_start"]]).all()
    for n in ("three_rows", "two_markers"):  # the start pose, as given
        assert np.array_equal(d.pose[at[n]], sc.start_pose[np.searchsorted(sc.start_key, k[n])])
    assert d.n_frames.tolist() == [10] and d.n_rows[0] == d.count[~unused].sum()


def test_status_mix_repeatable():
    """Statuses 0, 1 (with used frames), 1 (without), 2, 4 and 3 in one call with the camera term; a second call is
    bit-identical, NaN patterns included."""
    sc = status_mix()
    kw = dict(cam=True, max_iter=MIX_MAX_ITER)
    d, _ = _both(sc, **kw)
    assert tuple(d.status) == MIX_STATUS and d.n_frames.tolist() == [8, 7, 0, 8, 6, 8]
    e = _dev(sc, camera_cov=camera_cov(sc.bodies.flags), max_iter=MIX_MAX_ITER)
    for name in ("model", "pose", "rmse_px", "frame_rmse_px", "status", "iterations", "frame_status", "key"):
        assert np.array_equal(getattr(d, name), getattr(e, name), equal_nan=name in ("pose", "rmse_px", "frame_rmse_px"))
    for a, b in zip(d.cov, e.cov):
        assert np.array_equal(a, b, equal_nan=True)


@pytest.mark.parametrize("pixel_sigma", [0.0, 0.5])
@pytest.mark.parametrize("free", [(), (0, 3, 6)], ids=["P6", "P9"])
def test_camera_term_runs(free, pixel_sigma):
    """Runs of 33 and 64 rows (rmod_run_kernel's second staging batch), a one-row run, a frame seen by one camera and a
    camera that sees no frame of a body; pixel_sigma = 0 leaves the camera term alone."""
    d, o = _both(camterm_scene(free=free), cam=True, pixel_sigma=pixel_sigma)
    assert d.n_frames.tolist() == [8, 6] and (d.status == 0).all()
    assert all(np.abs(c).max() > 0 for c in o.cov)


@pytest.mark.parametrize("free", [(), (0, 17, 40, 63)], ids=["P6", "P9"])
def test_camera_term_64_cameras(free):
    sc = make_scene(137, n_model=5, n_frames=8, n_cams=64, visible=0.25, free=free)
    d, _ = _both(sc, cam=True)
    assert len(sc.bodies.flags) == 64 and d.n_frames.tolist() == [8]


def test_keys():
    """Keys 0, 2^62 and 2^63 - 1 with gaps, start poses for some keys only, rows in shuffled order."""
    sc = key_scene()
    d, _ = _both(sc)
    assert np.array_equal(d.key, EXTREME_KEYS) and d.n_frames.tolist() == [6]


def test_negative_key_refused():
    from caliscope_b200._lib import EngineError

    sc = key_scene()
    sc.bodies.obs_key[sc.bodies.obs_key == 7] = -1
    with pytest.raises(EngineError, match="cb_rigid_model_refine.*negative group key"):
        _dev(sc)


@pytest.mark.parametrize("max_iter", [1, 2, 3])
def test_iteration_limit(max_iter):
    """From a far start the iteration count, status 3 and the result after 1, 2 and 3 steps match the oracle."""
    d, o = _both(far_scene(), max_iter=max_iter)
    assert (d.status == 3).all() and (d.iterations == o.iterations).all() and d.iterations[0] == max_iter


def test_behind_at_iteration_limit():
    """A row behind its camera with the iteration limit reached: status 3, not 4."""
    d, _ = _both(behind_scene(45), cam=True, max_iter=1)
    assert d.status[0] == 3


def test_long_track():
    """One body of 10 markers over 2000 frames: 8-CTA clusters, 32 rounds; with the camera term."""
    d, _ = _both(make_scene(139, n_model=10, n_frames=2000), cam=True)
    assert d.n_frames.tolist() == [2000] and cluster_size(2000) == 8 and rounds(2000, 8) == 32


def test_many_bodies():
    """32 bodies of 3 to 8 markers, 60 frames each, in one launch."""
    d, _ = _both(multi_body(141, sizes=tuple(3 + i % 6 for i in range(32)), n_frames=60))
    assert (d.n_frames == 60).all() and len(d.status) == 32
