"""cb_calibrate_intrinsics on the H100 against oracle/intrinsics.py (and cv2 where it imports): every CPU case, the
cluster shapes of 1 camera x 3000 views and 64 cameras x 300 views, device-resident inputs, repeatability, refused calls
and the calibration of the standard deviations over 240 seeded cameras."""
from __future__ import annotations

import numpy as np
import pytest

from caliscope_b200 import _lib as L
from caliscope_b200 import intrinsics as I
from oracle import intrinsics as OI
from tests._intrinsics_cases import STRONG, WEBCAM, board, camera_status_case, make_case

pytestmark = pytest.mark.gpu


def _gpu(case, flags=None, guess=None, **kw):
    fixed = None if flags is None else np.asarray(flags) & 0x1FF
    return I.calibrate_cameras(case.obs_cam, case.obs_key, case.obs_obj, case.obs_px, case.image_size, fixed=fixed,
                               guess=guess, **kw)  # fmt: skip


def _oracle(case, flags=None, guess=None, **kw):
    nc = len(case.image_size)
    return OI.calibrate(case.obs_cam, case.obs_key, case.obs_obj, case.obs_px, case.image_size,
                        np.zeros(nc, int) if flags is None else flags, guess, **kw)  # fmt: skip


def _rel(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return float(np.nanmax(np.abs(a - b) / np.maximum(np.abs(b), 1e-300))) if a.size else 0.0


def _same(g, o, rtol=1e-9, std_rtol=1e-8):
    assert np.array_equal(g.status, o.status)
    assert np.array_equal(g.view_status, o.view_status)
    assert np.array_equal(g.view_cam, o.view_cam) and np.array_equal(g.view_count, o.view_count)
    assert np.array_equal(g.view_rep, o.view_rep)
    assert np.array_equal(g.n_views, o.n_views) and np.array_equal(g.n_rows, o.n_rows)
    assert np.array_equal(np.isnan(g.params), np.isnan(o.params))
    ok = np.isin(o.status, (0, 4))
    for c in np.flatnonzero(ok):
        # relative to the parameter vector (LM stops on |d| <= xtol |x|, so small coefficients are only determined to
        # that absolute level), and far inside the parameters' standard deviations
        d = np.abs(g.params[c] - o.params[c])
        assert d.max() <= rtol * np.linalg.norm(o.params[c]), (c, g.params[c], o.params[c])
        assert np.all(d <= 1e-6 * o.std[c]), (c, d / o.std[c])
        assert _rel(g.rms[c], o.rms[c]) <= std_rtol
        assert _rel(g.std[c], o.std[c]) <= std_rtol
        assert _rel(g.cov[c], o.cov[c]) <= std_rtol or np.abs(g.cov[c] - o.cov[c]).max() <= std_rtol * np.abs(o.cov[c]).max()
    used = o.view_status == 0
    used &= np.isin(o.status[o.view_cam], (0, 4))
    assert np.abs(g.view_pose[used] - o.view_pose[used]).max(initial=0) <= 1e-8
    assert _rel(g.view_std[used], o.view_std[used]) <= std_rtol
    assert _rel(g.view_rmse[used], o.view_rmse[used]) <= std_rtol


@pytest.mark.parametrize("lens,n_views,seed", [(WEBCAM, 20, 1), (WEBCAM, 60, 2), (STRONG, 30, 3), (STRONG, 45, 4)])
def test_device_matches_oracle(lens, n_views, seed):
    case = make_case(seed, [lens], n_views)
    _same(_gpu(case), _oracle(case))


def test_device_matches_oracle_cameras_of_different_sizes():
    case = make_case(5, [WEBCAM, STRONG, WEBCAM], [25, 30, 20])
    _same(_gpu(case), _oracle(case))


@pytest.mark.parametrize("fixed_bits,use_guess", [(0b1100, False), (0b11000000, False), (0b100110000, False),
                                                  (0, True), (0b11, True), (0b11001100, True)])  # fmt: skip
def test_device_matches_oracle_fixed_and_guess(fixed_bits, use_guess):
    case = make_case(7, [STRONG, WEBCAM], 30)
    guess = None
    if use_guess:
        guess = np.array([STRONG[2], WEBCAM[2]]) * np.array([1.02, 0.98, 1.0, 1.0, 0.8, 1.1, 0.5, 0.5, 0.9])
    flags = np.array([fixed_bits | (OI.USE_GUESS if use_guess else 0)] * 2)
    _same(_gpu(case, flags, guess), _oracle(case, flags, guess))


def test_device_against_cv2():
    cv2 = pytest.importorskip("cv2")
    case = make_case(3, [STRONG], 30)
    g = _gpu(case)
    objs = [case.obs_obj[case.obs_key == k].astype(np.float32) for k in np.unique(case.obs_key)]
    imgs = [case.obs_px[case.obs_key == k].reshape(-1, 1, 2).astype(np.float32) for k in np.unique(case.obs_key)]
    crit = (cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, 200, np.finfo(float).eps)
    rms, K, d, _, _, si, _, pve = cv2.calibrateCameraExtended(objs, imgs, tuple(int(v) for v in case.image_size[0]),
                                                             None, None, criteria=crit)  # fmt: skip
    th = np.array([K[0, 0], K[1, 1], K[0, 2], K[1, 2], *d.ravel()[:5]])
    assert np.all(np.abs(g.params[0] - th) <= 1e-6 * si.ravel()[:9])
    assert abs(g.rms[0] / rms - 1) <= 1e-10
    assert np.allclose(g.std[0], si.ravel()[:9], rtol=2e-5, atol=0)
    assert np.allclose(g.view_rmse, pve.ravel(), rtol=1e-6, atol=0)
    out = I.calibrate_camera(objs, imgs, tuple(int(v) for v in case.image_size[0]))
    assert out[0] == g.rms[0] and np.array_equal(out[5][:9, 0], g.std[0]) and np.all(out[5][9:] == 0)


def test_excluded_views_and_camera_statuses():
    case = make_case(11, [WEBCAM, STRONG], 24)
    X = board()
    rng = np.random.default_rng(0)
    nxt = int(case.obs_key.max()) + 1
    extra = [(np.r_[np.zeros(27, np.int32), np.ones(27, np.int32)], X),
             (np.zeros(3, np.int32), X[:3]),
             (np.zeros(54, np.int32), X + np.c_[np.zeros((54, 2)), X[:, 0] * 0.1]),
             (np.zeros(9, np.int32), X[:9]),
             (np.full(54, 2, np.int32), X)]  # camera 2: one view only  # fmt: skip
    cam = np.concatenate([case.obs_cam] + [e[0] for e in extra])
    key = np.concatenate([case.obs_key] + [np.full(len(e[0]), nxt + j, np.int64) for j, e in enumerate(extra)])
    obj = np.concatenate([case.obs_obj] + [e[1] for e in extra])
    px = np.concatenate([case.obs_px] + [rng.uniform(100, 900, (len(e[0]), 2)) for e in extra])
    full = type(case)(cam, key, obj, px, np.r_[case.image_size, [[640, 480]]], case.truth)
    g, o = _gpu(full), _oracle(full)
    _same(g, o)
    assert list(g.status) == [0, 0, 1]
    assert sorted(set(g.view_status.tolist())) == [0, 1, 2, 5, 6]


def test_shapes_one_camera_3000_views_and_64_cameras_300_views():
    for lenses, nv, seed in (([WEBCAM], 3000, 21), ([WEBCAM, STRONG] * 32, 300, 22)):
        case = make_case(seed, lenses, nv)
        st = I.IntrinsicsStats()
        g = _gpu(case, stats=st)
        assert (g.status == 0).all() and (g.n_views == nv).all()
        err = np.abs(g.params - case.truth) / g.std
        assert np.nanmax(err) < 6.0, np.nanmax(err)
        sub = make_case(seed, lenses[:1], min(nv, 300))
        _same(_gpu(sub), _oracle(sub))
        assert st.kernel_launches > 0 and st.lm_ms > 0


def test_device_resident_inputs_and_repeatability():
    torch = pytest.importorskip("torch")
    case = make_case(9, [WEBCAM, STRONG, WEBCAM], 40)
    a, b = _gpu(case), _gpu(case)
    dev = I.calibrate_cameras(torch.tensor(case.obs_cam, dtype=torch.int32, device="cuda:0"),
                              torch.tensor(case.obs_key, dtype=torch.int64, device="cuda:0"),
                              torch.tensor(case.obs_obj, dtype=torch.float64, device="cuda:0"),
                              torch.tensor(case.obs_px, dtype=torch.float64, device="cuda:0"), case.image_size)  # fmt: skip
    for f in ("params", "std", "cov", "rms", "sigma2", "iterations", "status", "view_pose", "view_std", "view_rmse",
              "view_status", "view_count", "view_rep", "view_cam"):  # fmt: skip
        assert np.array_equal(getattr(a, f), getattr(b, f), equal_nan=getattr(a, f).dtype.kind == "f"), f
        assert np.array_equal(getattr(a, f), getattr(dev, f), equal_nan=getattr(a, f).dtype.kind == "f"), f


def test_camera_statuses_on_the_device():
    """Statuses 1 (one view), 2 (no Zhang start) and 3 (S not positive definite at the solution: std / cov NaN, the
    last iterate and its view poses returned) as the oracle gives them; status 4 from a small max_iter."""
    case, flags, guess = camera_status_case()
    g, o = _gpu(case, flags, guess), _oracle(case, flags, guess)
    assert list(g.status) == [OI.CAM_TOO_FEW_VIEWS, OI.CAM_NO_START, OI.CAM_NOT_PD]
    _same(g, o)
    assert np.isnan(g.std[2]).all() and np.isnan(g.cov[2]).all() and np.isfinite(g.params[2]).all()
    v2 = g.view_cam == 2
    assert np.isnan(g.view_std[v2]).all() and np.isfinite(g.view_pose[v2]).all()
    assert np.isnan(g.params[1]).all() and np.isnan(g.view_pose[g.view_cam == 1]).all()
    case = make_case(3, [STRONG, WEBCAM], 30)
    g, o = _gpu(case, max_iter=3), _oracle(case, max_iter=3)
    assert list(g.status) == [OI.CAM_MAX_ITER] * 2 and list(g.iterations) == [3, 3]
    _same(g, o)


def test_refused_calls():
    import ctypes as C

    case = make_case(1, [WEBCAM], 8)
    with pytest.raises(ValueError):
        I.calibrate_cameras(case.obs_cam, case.obs_key, case.obs_obj, case.obs_px, case.image_size, fixed=[1 << 10])
    with pytest.raises(ValueError):
        I.calibrate_cameras(case.obs_cam, case.obs_key, case.obs_obj, case.obs_px, case.image_size, min_points=3)
    lib = L.load()
    nv = C.c_int32(0)
    isz = np.array([[640, 480]], np.int32)
    cam = case.obs_cam.astype(np.int32)
    key = case.obs_key.astype(np.int64)
    obj, px = np.ascontiguousarray(case.obs_obj), np.ascontiguousarray(case.obs_px)
    # (cam_flags, cam_fixed, expected): the fisheye flag every other call takes, a fixed aspect ratio and an unknown bit
    # are CB_E_UNSUPPORTED; a guess flag without a guess and fixed bits beyond the 9 parameters are CB_E_INVALID
    for flags, fixed, code in ((L.CB_CAM_FISHEYE, 0, -4), (0x200, 0, -4), (1 << 12, 0, -4), (I.CB_INTR_USE_GUESS, 0, -1),
                               (0, 1 << 9, -1), (L.CB_CAM_FREE_INTRINSICS, 0, 0)):  # fmt: skip
        fl, fx = np.array([flags], np.int32), np.array([fixed], np.int32)
        out = [np.empty(max(81, 6 * len(cam))) for _ in range(16)]
        before = L.load().cb_ba_launch_count()
        r = lib.cb_calibrate_intrinsics(1, isz.ctypes.data, fl.ctypes.data, fx.ctypes.data, None, len(cam),
                                        cam.ctypes.data, key.ctypes.data, obj.ctypes.data, px.ctypes.data, 0, 4, 2, 10,
                                        0.0, len(cam), C.byref(nv), *[o.ctypes.data for o in out], None, 0, None)  # fmt: skip
        assert r == code, (flags, fixed, r)
        if code:
            assert lib.cb_ba_launch_count() == before  # refused before any device work
    with pytest.raises(NotImplementedError):
        I.calibrate_camera([np.c_[np.random.rand(10, 2), np.random.rand(10)]] * 3, [np.random.rand(10, 2)] * 3, (640, 480))
    with pytest.raises(ValueError):
        I.calibrate_camera([board()] * 3, [np.random.rand(54, 2)] * 3, (640, 480), flags=I.CALIB_USE_INTRINSIC_GUESS)


def test_standard_deviations_are_calibrated():
    """(theta_hat - theta_true) / std over 240 seeded cameras (one call): mean within 4 standard errors of 0, variance
    within [0.75, 1.3] for every parameter (the chi-square spread of 240 samples is about +-0.18 at 2 sigma)."""
    n = 240
    lenses = [WEBCAM if k % 2 == 0 else STRONG for k in range(n)]
    case = make_case(123, lenses, 25)
    g = _gpu(case, with_cov=False)
    assert (g.status == 0).all()
    z = (g.params - case.truth) / g.std
    m, v = z.mean(0), z.var(0)
    assert np.all(np.abs(m) < 4.0 / np.sqrt(n)), m
    assert np.all((v > 0.75) & (v < 1.3)), v
