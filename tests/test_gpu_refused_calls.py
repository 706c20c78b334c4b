"""A call that the engine refuses after it has queued device work leaves the library usable: the same call with correct
arguments afterwards returns what it returned before the refusal, bit for bit.  The refusals are a group count one above
max_groups (found by the device grouping), a camera row out of range (found by the device validation of the rows) and a
repeated camera in a problem's cam_order (found in the index build, after its first sorts were queued)."""
import ctypes as C

import numpy as np
import pytest

import caliscope_b200 as cb
from caliscope_b200 import _lib as L
from caliscope_b200 import synthetic
from tests.test_gpu_triangulate_refine import _rig_case

pytestmark = pytest.mark.gpu


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _last_error():
    return (L.load().cb_ba_last_error() or b"").decode()


def _check_refusals(call, cam, n_cams):
    """call(max_groups, cam) -> (return code, reported group count, outputs)."""
    code, n_groups, before = call(len(cam), cam)
    assert code == 0 and n_groups > 1
    code, ng, _ = call(n_groups - 1, cam)
    assert code == -1 and ng == n_groups
    assert f"{n_groups} groups but room for {n_groups - 1}" in _last_error()
    bad = cam.copy()
    bad[len(bad) // 2] = n_cams
    code, _, _ = call(n_groups, bad)
    assert code == -1 and "camera index out of range" in _last_error()
    code, ng, after = call(n_groups, cam)
    assert code == 0 and ng == n_groups
    for a, b in zip(before, after):
        assert a.tobytes() == b.tobytes()


def _grouped_rows():
    rig = synthetic.make_rig(8, 600, 4000, seed=1)
    proj, xy = synthetic.exact_normalized_observations(rig)
    proj = np.ascontiguousarray(proj)
    cam = np.ascontiguousarray(rig.obs_cam, np.int32)
    key = np.ascontiguousarray(rig.obs_pt, np.int64)
    return rig, proj, cam, key, np.ascontiguousarray(xy, np.float64)


def _dlt_outputs(n):
    return [np.zeros((n, 3)), np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros((n, 2), np.uint64)]


@pytest.mark.parametrize("undistort", [False, True])
def test_triangulate_dlt(undistort):
    lib = L.load()
    rig, proj, cam0, key, xy = _grouped_rows()
    nc = len(proj)
    fish = np.zeros(nc, np.int32)
    k = np.ascontiguousarray(np.concatenate([rig.cam_const[:, :4], np.zeros((nc, 1))], axis=1))
    dist = np.zeros((nc, 12))
    dist[:, :5] = rig.cam_const[:, 4:9]
    px = np.ascontiguousarray(rig.obs_xy, np.float64)

    def call(max_groups, cam):
        n = len(cam)
        out = _dlt_outputs(n)
        ng = C.c_int32(0)
        tail = (n, _p(cam), _p(key), _p(px if undistort else xy), 0, max_groups, C.byref(ng), *map(_p, out), None, 0, None)
        if undistort:
            code = lib.cb_undistort_triangulate(nc, _p(fish), _p(k), _p(dist), _p(proj), *tail)
        else:
            code = lib.cb_triangulate_dlt(nc, _p(proj), *tail)
        return code, ng.value, [o[: ng.value] for o in out]

    _check_refusals(call, cam0, nc)


@pytest.mark.parametrize("robust", [False, True])
def test_triangulate_calibrated(robust):
    lib = L.load()
    flags, const, cx, cam0, key, px = _rig_case("p6")
    flags = np.ascontiguousarray(flags, np.int32)
    const = np.ascontiguousarray(const, np.float64)
    cx = np.ascontiguousarray(cx, np.float64)
    cam0 = np.ascontiguousarray(cam0, np.int32)
    key = np.ascontiguousarray(key, np.int64)
    px = np.ascontiguousarray(px, np.float64)
    nc = len(flags)

    def call(max_groups, cam):
        n = len(cam)
        xyz, cov, rmse = np.zeros((n, 3)), np.zeros((n, 3, 3)), np.zeros(n)
        count, n_in, rep, status = (np.zeros(n, np.int32) for _ in range(4))
        inlier = np.zeros(n, np.uint8)
        ng = C.c_int32(0)
        head = (nc, _p(flags), _p(const), _p(cx), None, n, _p(cam), _p(key), _p(px), 0)
        if robust:
            code = lib.cb_triangulate_robust(*head, 4.0, 2, 64, 1.0, 20, 1e-12, max_groups, C.byref(ng), _p(xyz), _p(cov),
                                             _p(rmse), _p(count), _p(n_in), _p(rep), _p(status), _p(inlier), None, 0,
                                             None)  # fmt: skip
        else:
            code = lib.cb_triangulate_refine(*head, 1.0, 20, 1e-12, max_groups, C.byref(ng), _p(xyz), _p(cov), _p(rmse),
                                             _p(count), _p(rep), _p(status), None, 0, None)  # fmt: skip
        g = ng.value
        out = [xyz[:g], cov[:g], rmse[:g], count[:g], rep[:g], status[:g]]
        return code, g, out + [n_in[:g], inlier] if robust else out

    _check_refusals(call, cam0, nc)


def test_pnp_ippe():
    lib = L.load()
    ses = synthetic.make_board_session(6, 12, seed=1)
    slot = {int(c): i for i, c in enumerate(ses.cam_ids)}
    cam0 = np.array([slot[int(c)] for c in ses.cam_id], np.int32)
    sync = ses.sync_index.astype(np.int64)
    obj_id = ses.object_id.astype(np.int64)
    key = np.ascontiguousarray((cam0 * (sync.max() + 1) + sync) * (obj_id.max() + 1) + obj_id, np.int64)
    nc = len(ses.cam_ids)
    fish = np.ascontiguousarray(ses.cam_fisheye, np.int32)
    k = np.ascontiguousarray(ses.cam_k, np.float64)
    dist = np.ascontiguousarray(ses.cam_dist, np.float64)
    px = np.ascontiguousarray(ses.img_xy, np.float64)
    obj = np.ascontiguousarray(ses.obj_xyz, np.float64)

    def call(max_groups, cam):
        n = len(cam)
        R, t, rmse = np.zeros((n, 3, 3)), np.zeros((n, 3)), np.zeros(n)
        status, count, rep = (np.zeros(n, np.int32) for _ in range(3))
        ng = C.c_int32(0)
        code = lib.cb_pnp_ippe(nc, _p(fish), _p(k), _p(dist), n, _p(cam), _p(key), _p(px), _p(obj), 4, max_groups,
                               C.byref(ng), _p(R), _p(t), _p(rmse), _p(status), _p(count), _p(rep), None, 0, None)  # fmt: skip
        g = ng.value
        return code, g, [R[:g], t[:g], rmse[:g], status[:g], count[:g], rep[:g]]

    _check_refusals(call, cam0, nc)


def test_problem_after_a_refused_camera_order():
    rig = synthetic.make_rig(8, 500, 6000, seed=3)
    args = (rig.cam_flags, rig.cam_const, rig.n_pts, rig.obs_cam, rig.obs_pt, rig.obs_xy)

    def evaluate():
        with cb.BAProblem(*args) as prob:
            return prob.residuals(rig.x0), prob.normal_equations(rig.x0, 1e-3)

    r0, ne0 = evaluate()
    order = np.arange(rig.n_cams)
    order[3] = order[5]
    with pytest.raises(L.EngineError, match="cam_order is not a permutation"):
        cb.BAProblem(*args, cam_order=order)
    r1, ne1 = evaluate()
    assert r0.tobytes() == r1.tobytes()
    assert ne0.keys() == ne1.keys()
    for name in ne0:
        assert np.asarray(ne0[name]).tobytes() == np.asarray(ne1[name]).tobytes(), name
