"""Lens undistortion on the device (undistort_kernel through cb_undistort_points and the fused undistort + DLT call)
against live OpenCV, the definition it implements, on every distortion model and branch of the inverse maps
(tests/_undistort_cases.py).

Tolerance: pinhole bit-exact (the kernel evaluates OpenCV's expressions unfused, in OpenCV's order).  Fisheye at most
one float32 ulp on finite values, for the device tan() against libm's; NaN and infinite values, and the (-1e6, -1e6)
failure sentinel, exact."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from caliscope_b200 import _lib as L
from caliscope_b200.triangulation import triangulate_groups, undistort_points
from tests import _undistort_cases as U

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")

CAMS = U.cameras()
OUTPUTS = ["normalized", "pixels"]


def _tables():
    return np.stack([c.K for c in CAMS]), [c.d for c in CAMS], np.array([c.fisheye for c in CAMS], np.int32)


def _rig(seed=3):
    """Every camera's point sets as one shuffled list: (camera row, pixels); n is not a multiple of 256."""
    rows, pts = [], []
    for r, c in enumerate(CAMS):
        p = U.all_points(c, seed=seed + r)
        assert U.branches(c, p) >= c.reaches, c.name
        rows.append(np.full(len(p), r, np.int32))
        pts.append(p)
    rows, pts = np.concatenate(rows), np.concatenate(pts)
    perm = np.random.default_rng(seed).permutation(len(rows))
    if len(perm) % 256 == 0:
        perm = perm[:-1]
    return rows[perm], pts[perm]


def _check_against_cv2(cam, got, pts, output):
    """`got` (float32) against cv2 for camera `cam`, with the exact fraction in every message."""
    ref = U.cv2_undistort(cam, pts, output)
    got = np.asarray(got, np.float32)
    exact = np.mean((got == ref) | (np.isnan(got) & np.isnan(ref)))
    what = f"{cam.name} {output}: exact fraction {exact:.6f}"
    assert np.array_equal(np.isnan(got), np.isnan(ref)), f"{what}; NaN positions differ"
    if not cam.fisheye:
        U.assert_same_f32(got, ref, what)
        return
    special = ~np.isfinite(ref) | (ref == np.float32(U.SENTINEL)).all(axis=1, keepdims=True)
    special &= ~np.isnan(ref)
    assert np.array_equal(got[special], ref[special]), f"{what}; sentinel or infinite values differ"
    fin = np.isfinite(ref) & ~special
    e = U.ulp32(got[fin], ref[fin])
    assert e.max(initial=0) <= 1, f"{what}; max {e.max()} ulp at {pts[np.argwhere(fin)[np.argmax(e)][0]]}"


@pytest.mark.parametrize("output", OUTPUTS)
def test_all_cameras_in_one_launch_equal_cv2(output):
    mats, dists, fish = _tables()
    rows, pts = _rig()
    assert len(rows) % 256 != 0
    got = undistort_points(pts, rows, mats, dists, fish, output=output)
    for r, c in enumerate(CAMS):
        _check_against_cv2(c, got[rows == r], pts[rows == r], output)


@pytest.mark.parametrize("output", OUTPUTS)
def test_device_resident_input_and_output_equal_the_host_call(output):
    """on_device = 1: rows, points and results stay in device memory (torch tensors)."""
    import torch

    from caliscope_b200.triangulation import _camera_tables

    mats, dists, fish = _tables()
    rows, pts = _rig(seed=11)
    host = undistort_points(pts, rows, mats, dists, fish, output=output)
    f, k, d = _camera_tables(mats, dists, fish)
    d_rows = torch.from_numpy(rows).cuda()
    d_pts = torch.from_numpy(np.ascontiguousarray(pts)).cuda()
    d_out = torch.full_like(d_pts, 7.0)
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    L.check(L.load().cb_undistort_points(len(f), p(f), p(k), p(d), len(pts), C.c_void_p(d_rows.data_ptr()),
                                         C.c_void_p(d_pts.data_ptr()), 1, int(output == "pixels"),
                                         C.c_void_p(d_out.data_ptr()), 0, None), "undistort_points")  # fmt: skip
    torch.cuda.synchronize()
    dev = d_out.cpu().numpy()
    assert np.array_equal(dev, dev.astype(np.float32).astype(np.float64), equal_nan=True)  # float32 values
    assert np.array_equal(dev.astype(np.float32).view(np.int32), host.view(np.int32))  # bit for bit, NaNs included
    for r, c in enumerate(CAMS):
        _check_against_cv2(c, dev[rows == r], pts[rows == r], output)


@pytest.mark.parametrize("cam", CAMS, ids=[c.name for c in CAMS])
def test_single_camera_without_rows_equals_cv2(cam):
    """obs_cam = NULL: one camera, every point."""
    pts = U.all_points(cam, seed=5)
    for output in OUTPUTS:
        got = undistort_points(pts, None, cam.K[None], [cam.d], [cam.fisheye], output=output)
        _check_against_cv2(cam, got, pts, output)


def test_fused_undistort_triangulate_is_one_computation():
    """cb_undistort_triangulate with host pixels (float32-staged, undistort_kernel<float>), with device-resident pixels
    (undistort_kernel<double>) and cb_undistort_points + cb_triangulate_dlt give bit-identical groups, on a rig of every
    camera model including fisheye sentinel rows and non-finite pixels."""
    import torch

    from caliscope_b200.triangulation import _camera_tables

    mats, dists, fish = _tables()
    cam, px = _rig(seed=17)
    rng = np.random.default_rng(17)
    proj = np.empty((len(CAMS), 3, 4))
    for r in range(len(CAMS)):
        a = rng.uniform(-0.3, 0.3, 3)
        R = cv2.Rodrigues(a)[0]
        proj[r] = np.hstack([R, rng.normal(0, 0.2, (3, 1)) + [[0.0], [0.0], [3.0]]])
    # groups of 1..6 rows drawn across cameras (single-row groups come out NaN)
    sizes = rng.integers(1, 7, len(cam))
    key = np.repeat(np.arange(len(sizes), dtype=np.int64), sizes)[: len(cam)]
    wild = [r for r, c in enumerate(CAMS) if c.name == "fish_wild"][0]
    und = undistort_points(px, cam, mats, dists, fish)
    assert (und[cam == wild] == np.float32(U.SENTINEL)).all(axis=1).any() and np.isnan(und).any()

    two = triangulate_groups(proj, cam, key, und.astype(np.float64))
    host = triangulate_groups(proj, cam, key, px, undistort=(mats, dists, fish))

    f, k, d = _camera_tables(mats, dists, fish)
    n = len(cam)
    xyz, count, rep = np.empty((n, 3)), np.empty(n, np.int32), np.empty(n, np.int32)
    sig, ng, st = np.empty((n, 2), np.uint64), C.c_int32(0), L.TriStats()
    dev_in = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (cam, key, px)]
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    L.check(L.load().cb_undistort_triangulate(len(f), p(f), p(k), p(d), p(np.ascontiguousarray(proj)), n,
                                              *(C.c_void_p(t.data_ptr()) for t in dev_in), 1, n, C.byref(ng), p(xyz),
                                              p(count), p(rep), p(sig), C.byref(st), 0, None),
            "undistort_triangulate")  # fmt: skip
    g = ng.value
    dev = (xyz[:g], count[:g], rep[:g], sig[:g])
    assert g == len(two[0]) == len(np.unique(key))
    assert np.isnan(two[0]).any() and np.isfinite(two[0]).any()
    for name, a, b, c in zip(("xyz", "count", "rep_row", "camset_sig"), two, host, dev):
        assert np.array_equal(a, b, equal_nan=True), f"{name}: host-input fused call differs from the two calls"
        assert np.array_equal(a, c, equal_nan=True), f"{name}: device-input fused call differs from the two calls"
