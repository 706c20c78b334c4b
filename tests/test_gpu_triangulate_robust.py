"""cb_triangulate_robust against the NumPy oracle (oracle/triangulation_robust.py robust_points) at every shape-selected
variant, with planted outliers: P = 6 and 9, fisheye, sampled pairs (dense groups), 8 and 32 lanes per group, same-camera
pairs, and the camera table in and out of shared memory."""
import numpy as np
import pytest

from caliscope_b200.triangulation import RobustStats, triangulate_refined, triangulate_robust
from oracle import triangulation_refine as T
from oracle import triangulation_robust as R
from tests.test_gpu_triangulate_refine import CASES, _camera_cov, _rig_case
from tests.test_triangulate_robust_cpu import status_cases

pytestmark = pytest.mark.gpu

TAU = 4.0
FIELDS = ("xyz", "cov", "rmse_px", "count", "n_inliers", "rep_row", "status", "inlier")


def _with_outliers(name, seed=21):
    flags, const, cx, cam, key, px = _rig_case(name)
    rng = np.random.default_rng(seed)
    px = px.copy()
    bad = rng.uniform(0, 1, len(px)) < rng.uniform(0.05, 0.10)
    px[bad] += rng.choice([-1.0, 1.0], (bad.sum(), 2)) * rng.uniform(20.0, 200.0, (bad.sum(), 2))
    return flags, const, cx, cam, key, px


def _device(cam, key, px):
    import torch

    return (torch.from_numpy(np.ascontiguousarray(cam, np.int32)).cuda(),
            torch.from_numpy(np.ascontiguousarray(key, np.int64)).cuda(),
            torch.from_numpy(np.ascontiguousarray(px, np.float64)).cuda())  # fmt: skip


def _check(flags, const, cx, cam, key, px, *, camera_cov=None, sigma=0.5, tau=TAU, min_ok=0.85, **kw):
    st = RobustStats()
    out = triangulate_robust(flags, const, cx, cam, key, px, threshold_px=tau, pixel_sigma=sigma, camera_cov=camera_cov,
                             stats=st, **kw)  # fmt: skip
    ref = R.robust_points(flags, const, cx, cam, px, key, threshold_px=tau, pixel_sigma=sigma, cam_cov=camera_cov, **kw)
    cs = ref.consensus
    grp, G = T.group_rows(key)
    assert G == len(out.xyz) == st.n_groups
    assert np.array_equal(out.count, cs.count)
    assert np.array_equal(out.rep_row, np.array([np.flatnonzero(grp == g)[0] for g in range(G)]))
    assert np.array_equal(out.status, ref.status)
    assert np.array_equal(out.n_inliers, np.bincount(grp, weights=out.inlier, minlength=G).astype(np.int32))
    # the inlier masks agree wherever the oracle's two best scores are not a near-tie.  A best score of k tau^2 means no
    # row is within tau of any hypothesis: the consensus set is empty whichever wins, so such a tie is not counted.
    tie = (np.isfinite(cs.best) & (np.abs(cs.second - cs.best) <= 1e-9 * np.abs(cs.best))
           & (cs.best < cs.count * tau * tau))  # fmt: skip
    assert tie.mean() < 1e-3
    same = np.array([np.array_equal(out.inlier[grp == g], cs.inlier[grp == g]) for g in range(G)])
    assert same[~tie].all()
    assert np.array_equal(out.n_inliers[~tie], cs.n_inliers[~tie])
    m = same & ~tie
    # The hypotheses differ in the last bits (Jacobi on the device, LAPACK in the oracle), so the refinement starts from
    # slightly different points and stops at its convergence floor: a 1e-12 relative change of the oracle's own start
    # moves its refined points by up to 1.4e-9 relative on these rigs (rmse and cov by < 2e-10).  Status 2 keeps the
    # hypothesis.
    refined = m & np.isin(ref.status, (0, 3, 4))
    scale = np.linalg.norm(ref.xyz[refined], axis=1, keepdims=True)
    assert np.max(np.abs(out.xyz[refined] - ref.xyz[refined]) / scale, initial=0.0) < 1e-8
    at_hyp = m & (ref.status == 2)
    scale = np.linalg.norm(ref.xyz[at_hyp], axis=1, keepdims=True)
    assert np.max(np.abs(out.xyz[at_hyp] - ref.xyz[at_hyp]) / scale, initial=0.0) < 1e-6
    nan = np.isin(ref.status, (1, 5))
    assert np.isnan(out.xyz[nan]).all() and np.isnan(out.rmse_px[nan]).all() and np.isnan(out.cov[nan]).all()
    assert np.max(np.abs(out.rmse_px[refined] - ref.rmse_px[refined]) / np.maximum(ref.rmse_px[refined], 1e-3),
                  initial=0.0) < 1e-8  # fmt: skip
    ok = refined & np.isfinite(ref.cov).all(axis=(1, 2))
    assert np.array_equal(ok, refined & np.isfinite(out.cov).all(axis=(1, 2)))
    nrm = np.linalg.norm(ref.cov[ok], axis=(1, 2))[:, None, None]
    assert np.max(np.abs(out.cov[ok] - ref.cov[ok]) / nrm, initial=0.0) < 1e-8
    assert (ref.status == 0).mean() > min_ok
    return out, st


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("with_cov", [False, True])
def test_robust_matches_oracle(name, with_cov):
    flags, const, cx, cam, key, px = _with_outliers(name)
    out, _ = _check(flags, const, cx, cam, key, px, camera_cov=_camera_cov(len(cx), 9) if with_cov else None)
    assert (~out.inlier).sum() > 0


@pytest.mark.parametrize("name", ["p9", "repeated"])
def test_device_resident_observations(name):
    flags, const, cx, cam, key, px = _with_outliers(name)
    c = _camera_cov(len(cx), 3)
    host = triangulate_robust(flags, const, cx, cam, key, px, threshold_px=TAU, camera_cov=c)
    dev = triangulate_robust(flags, const, cx, *_device(cam, key, px), threshold_px=TAU, camera_cov=c)
    for f in FIELDS:
        assert np.array_equal(getattr(host, f), getattr(dev, f), equal_nan=True), f


def test_two_calls_are_bit_identical():
    flags, const, cx, cam, key, px = _with_outliers("dense")
    c = _camera_cov(len(cx), 4)
    a = triangulate_robust(flags, const, cx, cam, key, px, threshold_px=TAU, camera_cov=c)
    b = triangulate_robust(flags, const, cx, cam, key, px, threshold_px=TAU, camera_cov=c)
    for f in FIELDS:
        assert np.array_equal(getattr(a, f), getattr(b, f), equal_nan=True), f


def test_max_pairs_and_min_inliers():
    flags, const, cx, cam, key, px = _with_outliers("mocap")
    # two-view groups have fewer than 3 consensus rows: status 5
    _check(flags, const, cx, cam, key, px, max_pairs=3, min_inliers=3, min_ok=0.7)


def test_status_codes_on_the_device():
    flags, const, cx, cam, key, px, expect = status_cases()
    out = triangulate_robust(flags, const, cx, cam, key, px, threshold_px=4.0)
    assert out.status.tolist() == expect
    assert out.inlier[key == 4].tolist() == [True, True, True, False]
    assert out.inlier[key == 5].all() and out.n_inliers.tolist() == [0, 0, 0, 0, 3, 4]
    assert triangulate_robust(flags, const, cx, cam, key, px, threshold_px=4.0, min_inliers=4).status[4] == 5


def test_huge_threshold_on_clean_data_is_the_plain_refinement():
    flags, const, cx, cam, key, px = _rig_case("mocap")
    rob = triangulate_robust(flags, const, cx, cam, key, px, threshold_px=1e6)
    ref = triangulate_refined(flags, const, cx, cam, key, px)
    assert np.array_equal(rob.count, ref.count) and np.array_equal(rob.rep_row, ref.rep_row)
    m = (rob.status == 0) & (ref.status == 0)
    assert m.mean() > 0.9
    assert np.all(rob.n_inliers[m] == rob.count[m])
    rel = np.linalg.norm(rob.xyz[m] - ref.xyz[m], axis=1) / np.linalg.norm(ref.xyz[m], axis=1)
    assert rel.max() < 1e-8


def test_bad_arguments_are_refused():
    from caliscope_b200 import _lib as L

    flags, const, cx, cam, key, px = _rig_case("p6")
    with pytest.raises(L.EngineError):
        triangulate_robust(flags, const, cx, cam, key, px, threshold_px=TAU, max_iter=0)
    with pytest.raises(L.EngineError):
        triangulate_robust(flags, const, cx, np.where(cam == 0, 99, cam), key, px, threshold_px=TAU)
    for kw in ({"threshold_px": 0.0}, {"threshold_px": np.inf}, {"threshold_px": np.nan},
               {"threshold_px": TAU, "min_inliers": 1}, {"threshold_px": TAU, "max_pairs": 0}):  # fmt: skip
        with pytest.raises(ValueError):
            triangulate_robust(flags, const, cx, cam, key, px, **kw)
    with pytest.raises(ValueError):
        triangulate_robust(flags, const, cx, cam, key, px, threshold_px=TAU, camera_cov=np.eye(3))
    # the engine's own argument check, below the Python one
    import ctypes as C

    lib = L.load()
    ng = C.c_int32(0)
    f32 = np.ascontiguousarray(flags, np.int32)
    c9 = np.ascontiguousarray(const, np.float64)
    xx = np.ascontiguousarray(cx, np.float64)
    cm = np.ascontiguousarray(cam, np.int32)
    ky = np.ascontiguousarray(key, np.int64)
    pp = np.ascontiguousarray(px, np.float64)
    n = len(cm)
    bufs = [np.empty((n, 9)) for _ in range(3)] + [np.empty(n, np.int32) for _ in range(4)] + [np.empty(n, np.uint8)]
    ptr = [b.ctypes.data_as(C.c_void_p) for b in bufs]
    for tau, mi, mp in ((0.0, 2, 64), (-1.0, 2, 64), (np.nan, 2, 64), (TAU, 1, 64), (TAU, 2, 0)):
        code = lib.cb_triangulate_robust(len(f32), f32.ctypes.data_as(C.c_void_p), c9.ctypes.data_as(C.c_void_p),
                                         xx.ctypes.data_as(C.c_void_p), None, n, cm.ctypes.data_as(C.c_void_p),
                                         ky.ctypes.data_as(C.c_void_p), pp.ctypes.data_as(C.c_void_p), 0, tau, mi, mp,
                                         1.0, 20, 1e-12, n, C.byref(ng), ptr[0], ptr[1], ptr[2], ptr[3], ptr[4],
                                         ptr[5], ptr[6], ptr[7], None, 0, None)  # fmt: skip
        with pytest.raises(L.EngineError):
            L.check(code, "triangulate_robust")
