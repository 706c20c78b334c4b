"""cb_resect_robust on the device against oracle/resection_robust.py: both consensus shapes (lanes per group with 8 or
32 lanes, and the (chunk, hypothesis) tiles of long groups), P = 6 and 9, fisheye, repeated point rows, NaN points,
with and without a point covariance, prior on and off, exhaustive and hashed samples; device-resident inputs, repeat
calls, refused calls, and the calibration of the covariance end to end."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from oracle.resection_robust import resect_robust as oracle_resect
from tests._resect_bank import check as _check
from tests._resect_bank import inlier_check as _inlier_check
from tests._resect_cases import camera_offsets, make_rig, perturb_cameras, plant_outliers

pytestmark = pytest.mark.gpu


def _resect():
    from caliscope_b200.resection import resect_robust

    return resect_robust


def _case(seed, *, n_cams=6, n_pts=40, fisheye=(), free=(), frac=0.15, frames=1, nan_pts=0, repeat=0):
    flags, const, cam_x, pts, oc, op, px = make_rig(seed, n_cams, n_pts, fisheye=fisheye, free=free)
    rng = np.random.default_rng(seed + 100)
    if frames > 1:  # key = (camera, frame): each frame sees 8-20 of the camera's points
        sel, keys = [], []
        for c in range(n_cams):
            rows_c = np.flatnonzero(oc == c)
            for f in range(frames):
                idx = rng.choice(rows_c, int(rng.integers(8, 21)), replace=False)
                sel.append(idx)
                keys.append(np.full(len(idx), c * frames + f, np.int64))
        sel = np.concatenate(sel)
        oc, op, px, key = oc[sel], op[sel], px[sel], np.concatenate(keys)
    else:
        key = oc.astype(np.int64)
    if repeat:
        r = rng.choice(len(oc), repeat, replace=False)
        oc, op, key = np.r_[oc, oc[r]], np.r_[op, op[r]], np.r_[key, key[r]]
        px = np.r_[px, px[r] + rng.normal(0, 0.2, (repeat, 2))]
    px, _ = plant_outliers(seed + 1, px, frac)
    if nan_pts:
        pts = pts.copy()
        pts[rng.choice(len(pts), nan_pts, replace=False)] = np.nan
    perm = rng.permutation(len(oc))
    return flags, const, perturb_cameras(seed + 2, flags, cam_x), pts, oc[perm], key[perm], op[perm], px[perm]


def _pts_cov(seed, n, nan_at=None):
    rng = np.random.default_rng(seed)
    A = rng.normal(0, 1e-3, (n, 3, 3))
    cov = A @ np.transpose(A, (0, 2, 1)) + 1e-7 * np.eye(3)
    if nan_at is not None:
        cov[nan_at] = np.nan
    return cov


VARIANTS = {
    # name: (case kwargs, call kwargs)
    "short8_p6": (dict(frames=12), dict()),
    "short8_fisheye_p9_noprior": (dict(frames=12, fisheye=(1, 4), free=(2,)), dict(use_prior=False)),
    "short8_exhaustive": (dict(frames=10, n_pts=40), dict(max_samples=4096)),
    "short32_repeat_nan": (dict(n_pts=150, repeat=30, nan_pts=3), dict()),
    "short32_noprior_hashed": (dict(n_pts=150, fisheye=(0,), free=(3,)), dict(use_prior=False, max_samples=16)),
    "long_p6": (dict(n_cams=3, n_pts=700), dict()),
    "long_fisheye_p9_noprior_nan": (dict(n_cams=3, n_pts=700, fisheye=(1,), free=(2,), nan_pts=5), dict(use_prior=False)),
}


@pytest.mark.parametrize("name", sorted(VARIANTS))
@pytest.mark.parametrize("with_cov", [False, True])
def test_device_matches_oracle(name, with_cov):
    case_kw, call_kw = VARIANTS[name]
    flags, const, cam_x, pts, oc, key, op, px = _case(11, **case_kw)
    pcov = _pts_cov(5, len(pts)) if with_cov else None
    kw = dict(threshold_px=4.0, min_inliers=6, points_cov=pcov, pixel_sigma=0.5, **call_kw)
    dev = _resect()(flags, const, cam_x, pts, oc, key, op, px, **kw)
    orc = oracle_resect(flags, const, cam_x, pts, oc, key, op, px, **kw)
    assert (orc.status == 0).mean() > 0.5
    tie = _check(dev, orc)
    _inlier_check(dev, orc, key, tie)


def test_nan_point_cov_and_statuses():
    """A NaN point covariance in the consensus set makes that group's cov NaN; hand-built groups give 1, 5 and 6."""
    flags, const, cam_x, pts, oc, key, op, px = _case(3, n_cams=4, n_pts=30, frac=0.0)
    pcov = _pts_cov(1, len(pts), nan_at=0)
    extra_key = key.max() + 1
    # status 1 (3 rows), 6 (two cameras), 5 (every row far off)
    oc2 = np.r_[oc, [0, 0, 0], [0, 1, 0, 1, 0], [2] * 8]
    key2 = np.r_[key, [extra_key] * 3, [extra_key + 1] * 5, [extra_key + 2] * 8]
    op2 = np.r_[op, [0, 1, 2], [0, 1, 2, 3, 4], np.arange(8)]
    px2 = np.r_[px, np.zeros((3, 2)), np.zeros((5, 2)), np.random.default_rng(0).uniform(-5e4, 5e4, (8, 2))]
    kw = dict(threshold_px=4.0, points_cov=pcov)
    dev = _resect()(flags, const, cam_x, pts, oc2, key2, op2, px2, **kw)
    orc = oracle_resect(flags, const, cam_x, pts, oc2, key2, op2, px2, **kw)
    _check(dev, orc)
    assert list(dev.status[-3:]) == [1, 6, 5]
    assert np.isnan(dev.cov[:4]).all()  # point 0 is in every camera's consensus set
    assert (dev.status[:4] == 0).all()


def test_device_inputs_and_repeat_bit_identical():
    torch = pytest.importorskip("torch")
    for kw_case in (dict(frames=12), dict(n_cams=3, n_pts=700)):
        flags, const, cam_x, pts, oc, key, op, px = _case(21, **kw_case)
        kw = dict(threshold_px=4.0, points_cov=_pts_cov(2, len(pts)))
        a = _resect()(flags, const, cam_x, pts, oc, key, op, px, **kw)
        b = _resect()(flags, const, cam_x, pts, oc, key, op, px, **kw)
        t = [torch.as_tensor(v).cuda() for v in (oc, key, op, px)]
        d = _resect()(flags, const, cam_x, pts, t[0], t[1], t[2], t[3], **kw)
        for other in (b, d):
            for f in ("cam", "pose", "cov", "rmse_px", "count", "n_inliers", "rep_row", "status", "inlier"):
                np.testing.assert_array_equal(getattr(a, f), getattr(other, f), err_msg=f)


def test_refusals_and_next_call():
    from caliscope_b200 import _lib as L
    from caliscope_b200.resection import resect_robust

    flags, const, cam_x, pts, oc, key, op, px = _case(31, frames=12)
    kw = dict(threshold_px=4.0)
    ref = resect_robust(flags, const, cam_x, pts, oc, key, op, px, **kw)
    for bad in (dict(threshold_px=0.0), dict(threshold_px=np.inf), dict(threshold_px=4.0, min_inliers=3),
                dict(threshold_px=4.0, max_samples=0), dict(threshold_px=4.0, max_samples=4097),
                dict(threshold_px=4.0, max_iter=0), dict(threshold_px=4.0, points_cov=np.zeros((2, 3, 3)))):  # fmt: skip
        with pytest.raises(ValueError):
            resect_robust(flags, const, cam_x, pts, oc, key, op, px, **bad)
    # refused inside the engine after device work was queued: a point index out of range, too few group slots
    op_bad = op.copy()
    op_bad[5] = len(pts)
    with pytest.raises(Exception, match="point index out of range"):
        resect_robust(flags, const, cam_x, pts, oc, key, op_bad, px, **kw)
    lib = L.load()
    n = len(oc)
    cam_p = np.ascontiguousarray(oc, np.int32)
    key_p = np.ascontiguousarray(key, np.int64)
    pt_p = np.ascontiguousarray(op, np.int32)
    px_p = np.ascontiguousarray(px, np.float64)
    outs = [np.empty(n, np.int32), np.empty((n, 6)), np.empty((n, 36)), np.empty(n), np.empty(n, np.int32),
            np.empty(n, np.int32), np.empty(n, np.int32), np.empty(n, np.int32), np.empty(n, np.uint8)]  # fmt: skip
    ng = C.c_int32(0)

    def call(max_groups, min_inliers=6, max_samples=64):
        p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        return lib.cb_resect_robust(len(flags), p(np.ascontiguousarray(flags, np.int32)), p(np.ascontiguousarray(const)),
                                    p(np.ascontiguousarray(cam_x)), len(pts), p(np.ascontiguousarray(pts)), None, n,
                                    p(cam_p), p(key_p), p(pt_p), p(px_p), 0, 4.0, min_inliers, max_samples, 1, 1.0, 20,
                                    1e-12, max_groups, C.byref(ng), *(p(o) for o in outs), None, 0, None)  # fmt: skip

    assert call(n, min_inliers=3) != 0
    assert call(n, max_samples=5000) != 0
    assert call(2) != 0 and b"groups but room for" in lib.cb_ba_last_error()
    again = resect_robust(flags, const, cam_x, pts, oc, key, op, px, **kw)
    for f in ("pose", "rmse_px", "status", "inlier", "n_inliers"):
        np.testing.assert_array_equal(getattr(ref, f), getattr(again, f), err_msg=f)


def test_covariance_calibration_end_to_end():
    """Resect each camera against points triangulated (robustly) from the true other cameras without its rows, with
    points_cov = those points' covariance.  Over all cameras of a few seeds, the mean squared Mahalanobis distance of
    (pose - truth) under cov is chi^2 with 6 degrees of freedom per camera: mean 6.  With 24 cameras the standard error
    of the mean is sqrt(12 / 24) = 0.71, so the band [6 - 2.5, 6 + 2.5] holds by ~3.5 standard errors while a covariance
    off by a factor 1.6 in either direction (mean 3.75 or 9.6) would fail."""
    from caliscope_b200.resection import resect_robust
    from caliscope_b200.triangulation import triangulate_robust

    d2 = []
    for seed in range(4):
        flags, const, cam_x, pts_true, oc, op, px = make_rig(40 + seed, n_cams=6, n_pts=80, noise=0.5)
        offs = camera_offsets(flags)
        for c in range(len(flags)):
            other = oc != c
            tri = triangulate_robust(flags, const, cam_x, oc[other], op[other].astype(np.int64), px[other],
                                     threshold_px=4.0, pixel_sigma=0.5)  # fmt: skip
            assert len(tri.xyz) == len(pts_true)
            mine = oc == c
            res = resect_robust(flags, const, perturb_cameras(seed, flags, cam_x), tri.xyz, oc[mine], oc[mine].astype(np.int64),
                                op[mine], px[mine], threshold_px=4.0, pixel_sigma=0.5, points_cov=tri.cov)  # fmt: skip
            assert res.status[0] == 0
            e = res.pose[0] - cam_x[offs[c] : offs[c] + 6]
            d2.append(float(e @ np.linalg.solve(res.cov[0], e)))
    assert 3.5 <= np.mean(d2) <= 8.5, (np.mean(d2), d2)
