"""Each scene of tests/_rigid_model_edges.py hits the edge that tests/test_gpu_rigid_model_edges.py claims for it: used-
frame counts and the cluster size and rounds they give, frame masks, frames at the frame-use boundary, statuses by the
oracle, camera-term run sizes and keys.  No GPU."""
from __future__ import annotations

import numpy as np
import pytest

from oracle.rigid_model import frame_table, rigid_model_refine
from tests._rigid_cases import camera_cov
from tests._rigid_model_cases import behind_scene
from tests._rigid_model_edges import (BOUNDARY_KEYS, CAMTERM_RUNS, CAMTERM_SINGLE, CAMTERM_UNSEEN, EXTREME_KEYS,
                                      MIX_MAX_ITER, MIX_STATUS, MIXED_FRAMES, boundary_scene, camterm_scene,
                                      cluster_scene, cluster_size, far_scene, key_scene, marker_scene,
                                      mixed_cluster_scene, rounds, run_sizes, status_mix, used_frames)  # fmt: skip


@pytest.mark.parametrize("nf,cs,rd", [(1, 1, 1), (32, 1, 4), (33, 2, 3), (224, 7, 4), (225, 8, 4), (256, 8, 4),
                                      (257, 8, 5)])  # fmt: skip
def test_cluster_edges(nf, cs, rd):
    u = used_frames(cluster_scene(nf))
    assert u.tolist() == [nf] and cluster_size(nf) == cs and rounds(nf, cs) == rd
    # the last round's active warps: one at nf = 1 and 257, a partial round at 225, none idle at 256
    assert nf - (rd - 1) * 8 * cs == {1: 1, 32: 8, 33: 1, 224: 56, 225: 33, 256: 64, 257: 1}[nf]


def test_mixed_cluster():
    u = used_frames(mixed_cluster_scene())
    assert tuple(u) == MIXED_FRAMES and cluster_size(u.max()) == 8 and rounds(1, 8) == rounds(5, 8) == 1


@pytest.mark.parametrize("K", [3, 5, 6, 7, 8, 12, 13, 23, 24, 31, 32])
def test_marker_masks(K):
    """Every frame used; at K >= 4 rounds of warps with four different masks, one without marker 0 and one without
    marker K-1 (bit 31 at K = 32)."""
    sc = marker_scene(K)
    b = sc.bodies
    keys, rows, _, used = frame_table(b.obs_key, b.obs_pt, sc.start_key, sc.start_pose)
    assert used.all() and len(keys) == 12
    masks = [sum(1 << int(k) for k in np.unique(b.obs_pt[r])) for r in rows]
    full = (1 << K) - 1
    if K == 3:
        assert set(masks) == {full}
        return
    odd = sum(1 << k for k in range(1, K, 2))
    want = [full, full & ~1, full & ~(1 << (K - 1)), full & ~odd]
    assert masks == want * 3 and len(set(masks[:8])) == 4  # the 8 warps of the first round hold 4 masks


def test_frame_use_boundary():
    sc = boundary_scene()
    b = sc.bodies
    keys, rows, pose, used = frame_table(b.obs_key, b.obs_pt, sc.start_key, sc.start_pose)
    k = BOUNDARY_KEYS
    assert k["no_rows"] not in keys and k["no_rows"] in sc.start_key and k["no_start"] not in sc.start_key
    at = {name: int(np.searchsorted(keys, key)) for name, key in k.items() if name != "no_rows"}
    shape = {n: (len(rows[at[n]]), len(np.unique(b.obs_pt[rows[at[n]]]))) for n in at}
    assert shape["three_rows"] == (3, 3) and shape["two_markers"] == (4, 2) and shape["minimal"] == (4, 3)
    assert shape["no_start"][0] >= 4 and shape["no_start"][1] >= 3
    assert [bool(used[at[n]]) for n in ("three_rows", "two_markers", "minimal", "no_start")] == [False, False, True, False]
    assert used.sum() == 10 and np.isnan(pose[at["no_start"]]).all()
    # the boundary frames sit between used frames in key order
    assert all(used[at[n] - 1] and used[at[n] + 1] for n in at)


def test_status_mix():
    sc = status_mix()
    assert used_frames(sc).tolist() == [8, 7, 0, 8, 6, 8]
    o = rigid_model_refine(*sc.args(), body_start=sc.body_start, camera_cov=camera_cov(sc.bodies.flags),
                           max_iter=MIX_MAX_ITER)  # fmt: skip
    assert tuple(o.status) == MIX_STATUS
    # body 1's marker 4 has rows, all in an unused frame; its other frames are used and its frames' status is 1
    b = sc.bodies
    keys, rows, _, used = frame_table(b.obs_key, b.obs_pt, sc.start_key, sc.start_pose)
    m4 = [f for f, r in enumerate(rows) if (b.obs_pt[r] == sc.body_start[1] + 4).any()]
    assert len(m4) == 1 and not used[m4[0]]
    assert (o.iterations[[0, 4]] < MIX_MAX_ITER).all() and o.iterations[5] == MIX_MAX_ITER


@pytest.mark.parametrize("free", [(), (0, 3, 6)])
def test_camterm_runs(free):
    sc = camterm_scene(free=free)
    b = sc.bodies
    assert used_frames(sc).tolist() == [8, 6]
    sizes = run_sizes(sc)
    assert sizes.max() == 64 and 33 in sizes and 1 in sizes
    for key, (cam, n) in CAMTERM_RUNS.items():
        assert ((b.obs_key == key) & (b.obs_cam == cam)).sum() == n
    key, cam = CAMTERM_SINGLE
    assert set(b.obs_cam[b.obs_key == key]) == {cam} and len(np.unique(b.obs_pt[b.obs_key == key])) == 32
    assert not ((b.obs_pt >= sc.body_start[1]) & (b.obs_cam == CAMTERM_UNSEEN)).any()
    assert ((b.obs_pt < sc.body_start[1]) & (b.obs_cam == CAMTERM_UNSEEN)).any()
    assert (np.asarray(b.flags) & 1).any() == bool(free)


def test_keys():
    sc = key_scene()
    b = sc.bodies
    keys, _, _, used = frame_table(b.obs_key, b.obs_pt, sc.start_key, sc.start_pose)
    assert np.array_equal(keys, EXTREME_KEYS) and used.sum() == 6
    assert (np.diff(b.obs_key) < 0).any()  # not in key order


def test_iteration_edges():
    for max_iter in (1, 2, 3):
        sc = far_scene()
        o = rigid_model_refine(*sc.args(), body_start=sc.body_start, max_iter=max_iter)
        assert o.status[0] == 3 and o.iterations[0] == max_iter
    sc = behind_scene(45)
    kw = dict(body_start=sc.body_start, camera_cov=camera_cov(sc.bodies.flags))
    assert rigid_model_refine(*sc.args(), max_iter=1, **kw).status[0] == 3
    assert rigid_model_refine(*sc.args(), **kw).status[0] == 4


def test_size_edges():
    assert cluster_size(2000) == 8 and rounds(2000, 8) == 32 and cluster_size(60) == 2 and rounds(60, 2) == 4
