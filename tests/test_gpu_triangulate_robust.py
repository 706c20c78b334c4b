"""cb_triangulate_robust against the NumPy oracle (oracle/triangulation_robust.py robust_points) at every shape-selected
variant, with planted outliers: P = 6 and 9, fisheye, sampled pairs (dense groups), 8 and 32 lanes per group, same-camera
pairs, and the camera table in and out of shared memory; the pair table at T = max_pairs, groups with T above 2^31 and
2^32, a long group under 8 lanes, and decisive rows at a group's first and last position."""
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


# ---- pair-table edges, huge groups, skewed lanes, decisive rows -------------------------------------------------------------
def _ring(n_cams=64, seed=0):
    """n_cams pinhole / fisheye cameras on a ring around the origin (tests/_resect_cases.make_rig's cameras)."""
    from tests._resect_cases import make_rig

    flags, const, cx, _, _, _, _ = make_rig(seed, n_cams, 1, fisheye=tuple(range(0, n_cams, 5)), free=(3, 7))
    return flags, const, cx


def _views(flags, const, cx, X, cams, noise, rng):
    from oracle.ba_oracle import rodrigues
    from oracle.resection_robust import cameras, project

    cs = cameras(flags, const, cx)
    px = np.empty((len(cams), 2))
    for c in np.unique(cams):
        m = cams == c
        uv, _ = project(cs[c], rodrigues(cs[c].q[:3])[0], cs[c].q[3:6], X)
        px[m] = uv + rng.normal(0, noise, (m.sum(), 2))
    return px


def _point_group(flags, const, cx, k, rng, *, noise=0.3, X=None):
    X = rng.uniform(-0.5, 0.5, 3) if X is None else X
    cams = np.sort(rng.choice(len(flags), k, replace=k > len(flags))).astype(np.int32)
    rng.shuffle(cams)
    return cams, _views(flags, const, cx, X, cams, noise, rng)


def _lanes_of(cam):
    return 32 if len(cam) // len(np.unique(cam)) > 96 else 8


@pytest.mark.parametrize("k,max_pairs", [(12, 66), (12, 65), (2, 1)])
def test_pair_table_edges(k, max_pairs):
    """T = k (k - 1) / 2 against max_pairs: 66 at k = 12 (every pair, the table full), 65 (sampled ranks), and k = 2 at
    max_pairs = 1; 40 groups each with 20 % outliers."""
    flags, const, cx = _ring(16, 1)
    rng = np.random.default_rng(k + max_pairs)
    cam, key, px = [], [], []
    for g in range(40):
        c, p = _point_group(flags, const, cx, k, rng)
        bad = rng.random(k) < 0.2
        p[bad] += rng.uniform(20, 200, (bad.sum(), 2))
        cam.append(c), key.append(np.full(k, g, np.int64)), px.append(p)
    cam, key, px = np.concatenate(cam), np.concatenate(key), np.concatenate(px)
    T = k * (k - 1) // 2
    print(f"k {k}, max_pairs {max_pairs}: T {T}, {'every pair' if T <= max_pairs else 'sampled ranks'}, "
          f"lanes {_lanes_of(key)}")  # fmt: skip
    _check(flags, const, cx, cam, key, px, max_pairs=max_pairs, min_ok=0.0)


@pytest.mark.parametrize("k", [65537, 100000])
def test_huge_groups_rank_exactly(k):
    """One point in k rows from 64 cameras: T = 2,147,516,416 (> 2^31 - 1) and 4,999,950,000 (> 2^32) pairs, ranks
    floor(m T / 64).  With max_iter = 1 and 0.5 px of noise the output is one step from the selected pair's point, so
    status, inliers and xyz show which rank won."""
    flags, const, cx = _ring(64, 2)
    rng = np.random.default_rng(k)
    cam, px = _point_group(flags, const, cx, k, rng, noise=0.5)
    bad = rng.random(k) < 0.1
    px[bad] += rng.uniform(20, 200, (bad.sum(), 2))
    key = np.zeros(k, np.int64)
    T = k * (k - 1) // 2
    assert T > (1 << 31) - 1 and (k < 100000 or T > 1 << 32)
    out, st = _check(flags, const, cx, cam, key, px, max_pairs=64, max_iter=1, min_ok=-1.0)
    print(f"k {k}: T {T}, sampled ranks, lanes {_lanes_of(key)}, launches {st.kernel_launches}, status {out.status}")
    assert out.status[0] == 3


def test_skewed_lanes():
    """A 5000-row group among 300 two-view groups (mean ~ 18 rows: 8 lanes), and the same group alone (32 lanes)."""
    flags, const, cx = _ring(64, 3)
    rng = np.random.default_rng(7)
    c0, p0 = _point_group(flags, const, cx, 5000, rng)
    bad = rng.random(5000) < 0.15
    p0[bad] += rng.uniform(20, 200, (bad.sum(), 2))
    cam, key, px = [c0], [np.zeros(5000, np.int64)], [p0]
    for g in range(300):
        c, p = _point_group(flags, const, cx, 2, rng)
        cam.append(c), key.append(np.full(2, g + 1, np.int64)), px.append(p)
    cam, key, px = np.concatenate(cam), np.concatenate(key), np.concatenate(px)
    mixed, _ = _check(flags, const, cx, cam, key, px, min_ok=0.5)
    alone, _ = _check(flags, const, cx, c0, np.zeros(5000, np.int64), p0)
    assert _lanes_of(key) == 8 and _lanes_of(np.zeros(5000)) == 32
    print(f"skewed: lanes 8 with {len(np.unique(key))} groups, 32 alone; status {mixed.status[0]}, {mixed.n_inliers[0]} inliers")
    np.testing.assert_array_equal(mixed.inlier[:5000], alone.inlier)
    assert mixed.n_inliers[0] == alone.n_inliers[0] and mixed.status[0] == alone.status[0]


def _decisive_group(flags, const, cx, k, at, rng):
    """Rows of two points A and B 0.3 m apart, exact under their point (A's with 0.01 px of noise so that A's pairs do not
    tie), A with one more row than B and A's rows at `at`: A's best pair wins by about tau^2; a score without one of A's
    rows ties B at best, and B's exact pairs then win."""
    XA = np.array([0.1, -0.05, 0.2])
    XB = XA + np.array([0.0, 0.0, 0.3])
    cam = (np.arange(k) % len(flags)).astype(np.int32)
    rng.shuffle(cam)
    n_a = k // 2 + 1
    role = np.zeros(k, bool)
    role[list(at)] = True
    rest = np.flatnonzero(~role)
    role[rng.choice(rest, n_a - role.sum(), replace=False)] = True
    pa = _views(flags, const, cx, XA, cam, 0.01, rng)
    pb = _views(flags, const, cx, XB, cam, 0.0, rng)
    assert (np.linalg.norm(pa - pb, axis=1) > 4 * TAU).all()
    return cam, np.where(role[:, None], pa, pb), role


@pytest.mark.parametrize("lanes", [8, 32])
def test_decisive_rows(lanes):
    """The deciding row (one of A's) at the group's first and last position, in an 8-lane call (among two-view groups)
    and a 32-lane call (alone)."""
    flags, const, cx = _ring(64, 4)
    rng = np.random.default_rng(lanes)
    k = 21 if lanes == 8 else 201  # odd: A has (k + 1) / 2 rows, B one fewer
    cam0, px0, role = _decisive_group(flags, const, cx, k, (0, k - 1), rng)
    cam, key, px = [cam0], [np.zeros(k, np.int64)], [px0]
    if lanes == 8:
        for g in range(40):
            c, p = _point_group(flags, const, cx, 2, rng)
            cam.append(c), key.append(np.full(2, g + 1, np.int64)), px.append(p)
    cam, key, px = np.concatenate(cam), np.concatenate(key), np.concatenate(px)
    assert _lanes_of(key) == lanes
    max_pairs = k * (k - 1) // 2 if lanes == 8 else 64
    out, st = _check(flags, const, cx, cam, key, px, max_pairs=max_pairs, min_ok=0.0)
    print(f"decisive rows: lanes {lanes}, k {k}, {'every pair' if lanes == 8 else 'sampled ranks'}, "
          f"{out.n_inliers[0]} inliers")  # fmt: skip
    np.testing.assert_array_equal(out.inlier[:k], role)
