"""GPU parity of the step in front of bundle adjustment (SURVEY.md §8(f) rank 3): lens undistortion
and DLT triangulation through the C ABI, against the reference's golden vectors and the oracle.

Tolerances: undistortion is float32-valued like the reference — bit-exact for pinhole cameras, one
float32 ulp allowed for fisheye (device tan() vs libm); triangulation 1e-9 m on well-posed groups (the kernel takes the
smallest eigenvector of the 4x4 normal matrix in fp64, the reference an SVD of the 2k x 4 system)."""
from __future__ import annotations

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def g(golden_dir):
    return np.load(golden_dir / "triangulation.npz")


def _ulp32(a, b):
    a32, b32 = a.astype(np.float32), b.astype(np.float32)
    return np.abs(a32.view(np.int32).astype(np.int64) - b32.view(np.int32).astype(np.int64)).max()


@pytest.mark.parametrize("case", ["s4", "syn"])
def test_triangulate_image_points_matches_reference_golden(g, case):
    from caliscope_b200.triangulation import triangulate_image_points

    pm = {int(c): g[f"{case}_proj"][i] for i, c in enumerate(g[f"{case}_cam_ids"])}
    s, o, k, xyz = triangulate_image_points(pm, g[f"{case}_sync"], g[f"{case}_cam"], g[f"{case}_obj"], g[f"{case}_kp"],
                                            g[f"{case}_xy"])  # fmt: skip
    assert s.dtype == np.int64 and o.dtype == np.int64 and k.dtype == np.int64
    assert np.array_equal(s, g[f"{case}_out_sync"])  # same keys in the reference's by-camera-set order
    assert np.array_equal(o, g[f"{case}_out_obj"])
    assert np.array_equal(k, g[f"{case}_out_kp"])
    assert np.abs(xyz - g[f"{case}_out_xyz"]).max() < 1e-9


def test_triangulate_matches_oracle_on_a_larger_seeded_case():
    from caliscope_b200.triangulation import triangulate_image_points
    from oracle import triangulation as T

    rng = np.random.default_rng(5)
    cam_ids = np.arange(0, 24, 2)
    pm = {}
    for c in cam_ids:
        a = rng.uniform(0, 2 * np.pi)
        R = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
        pm[int(c)] = np.hstack([R, np.array([[0.0], [0.0], [3.0]]) + rng.normal(0, 0.1, (3, 1))])
    rows = []
    for j in range(3000):
        X = rng.uniform(-0.5, 0.5, 3)
        cams = rng.choice(cam_ids, size=int(rng.integers(1, 10)), replace=False)
        for c in cams:
            h = pm[int(c)] @ np.append(X, 1.0)
            rows.append((j // 50, int(c), j % 3, j % 50, *(h[:2] / h[2] + rng.normal(0, 1e-3, 2))))
    rows = np.array(rows)
    rng.shuffle(rows)
    a = (rows[:, 0].astype(np.int64), rows[:, 1].astype(np.int64), rows[:, 2].astype(np.int64), rows[:, 3].astype(np.int64),
         np.ascontiguousarray(rows[:, 4:6]))  # fmt: skip
    ref = T.triangulate_image_points(pm, *a)
    got = triangulate_image_points(pm, *a)
    for i in range(3):
        assert np.array_equal(ref[i], got[i])
    assert np.abs(ref[3] - got[3]).max() < 1e-9


def test_triangulate_edge_cases():
    from caliscope_b200.triangulation import triangulate_image_points

    pm = {0: np.hstack([np.eye(3), [[0.0], [0.0], [2.0]]]), 1: np.hstack([np.eye(3), [[0.5], [0.0], [2.0]]])}
    i64 = lambda *v: np.array(v, dtype=np.int64)  # noqa: E731
    # fewer than two observations -> four empty arrays (point_data.py:136-142)
    out = triangulate_image_points(pm, i64(0), i64(0), i64(0), i64(0), np.zeros((1, 2)))
    assert [len(x) for x in out] == [0, 0, 0, 0] and out[3].shape == (0, 3)
    # only single-view groups -> empty (point_data.py:174-180)
    out = triangulate_image_points(pm, i64(0, 1), i64(0, 1), i64(0, 0), i64(0, 0), np.zeros((2, 2)))
    assert [len(x) for x in out] == [0, 0, 0, 0]
    # unknown camera id -> KeyError like the reference's dict lookup
    with pytest.raises(KeyError):
        triangulate_image_points(pm, i64(0, 0), i64(0, 7), i64(0, 0), i64(0, 0), np.zeros((2, 2)))
    # exact two-view point
    X = np.array([0.1, -0.2, 0.4])
    xy = np.stack([(pm[c] @ np.append(X, 1))[:2] / (pm[c] @ np.append(X, 1))[2] for c in (0, 1)])
    s, o, k, xyz = triangulate_image_points(pm, i64(5, 5), i64(0, 1), i64(2, 2), i64(9, 9), xy)
    assert (s[0], o[0], k[0]) == (5, 2, 9)
    assert np.abs(xyz[0] - X).max() < 1e-12


def test_triangulate_roundtrip_at_full_size():
    """cfg4 scale (64 cameras, 50 000 points, 2 M observations): exact projections triangulate back to
    the points they came from — the size-independent property of the DLT step."""
    from caliscope_b200 import synthetic
    from caliscope_b200.triangulation import TriangulationStats, triangulate_groups

    rig = synthetic.cfg4()
    proj, xy = synthetic.exact_normalized_observations(rig)
    st = TriangulationStats()
    xyz, count, rep, sig = triangulate_groups(proj, rig.obs_cam, rig.obs_pt.astype(np.int64), xy, stats=st)
    assert len(xyz) == rig.n_pts and count.sum() == rig.n_obs
    truth = rig.x_true[-3 * rig.n_pts :].reshape(-1, 3)
    assert np.abs(xyz - truth).max() < 1e-9
    assert st.kernel_launches > 0 and st.dlt_ms > 0


def test_undistort_points_matches_reference_golden(g):
    from caliscope_b200.triangulation import undistort_points

    pts = g["und_pts"]
    for fish, K, d, tag in ((False, g["und_Kp"], g["und_d5"], "pinhole"), (True, g["und_Kf"], g["und_d4"], "fisheye")):
        for mode, key in (("normalized", "norm"), ("pixels", "px")):
            got = undistort_points(pts, None, K[None], [d], [fish], output=mode)
            ref = g[f"und_{tag}_{key}"]
            assert got.dtype == np.float32 and got.shape == ref.shape
            if fish:
                assert _ulp32(got, ref) <= 1, (tag, mode)
                assert np.mean(got.astype(np.float64) == ref) > 0.999
            else:  # no tan(): OpenCV's arithmetic, unfused, gives OpenCV's bits
                assert np.array_equal(got.astype(np.float64), ref), (tag, mode)


def test_undistort_all_cameras_in_one_launch_matches_per_camera_reference(g):
    """_undistort_batch (point_data.py:236-252) loops cameras; the engine takes the camera row per point."""
    from caliscope_b200.triangulation import undistort_points

    rows = np.searchsorted(g["s4_cam_ids"], g["s4_px_cam"])
    got = undistort_points(g["s4_px"], rows, g["s4_K"], list(g["s4_dist"]), np.zeros(len(g["s4_K"]), np.int32))
    assert np.array_equal(got.astype(np.float64), g["s4_px_undist"])  # pinhole cameras: bit-exact
    with pytest.raises(ValueError):
        undistort_points(g["s4_px"], rows, g["s4_K"], list(g["s4_dist"]), np.zeros(len(g["s4_K"]), np.int32), output="mm")
    with pytest.raises(ValueError):  # fisheye needs 4 coefficients (camera_array / reprojection.py:26-27 behaviour)
        undistort_points(g["und_pts"], None, g["und_Kf"][None], [g["und_d5"]], [True])


def test_undistort_then_triangulate_reproduces_reference_world_points(g):
    """ImagePoints.triangulate (point_data.py:416-559) at array level: pixels -> undistort -> DLT."""
    from caliscope_b200.triangulation import triangulate_image_points, undistort_points

    rows = np.searchsorted(g["s4_cam_ids"], g["s4_px_cam"])
    und = undistort_points(g["s4_px"], rows, g["s4_K"], list(g["s4_dist"]), np.zeros(len(g["s4_K"]), np.int32))
    pm = {int(c): g["s4_proj"][i] for i, c in enumerate(g["s4_cam_ids"])}
    # the recorded call received exactly these undistorted rows (same order as the image-point table)
    assert np.abs(und.astype(np.float64) - g["s4_xy"]).max() < 1e-6
    out = triangulate_image_points(pm, g["s4_sync"], g["s4_cam"], g["s4_obj"], g["s4_kp"], und.astype(np.float64))
    assert np.abs(out[3] - g["s4_world_xyz"]).max() < 1e-5  # float32-ulp input differences amplified by the DLT


def test_fused_undistort_triangulate_equals_the_two_calls(g):
    """cb_undistort_triangulate == cb_undistort_points followed by cb_triangulate_dlt, bit for bit."""
    from caliscope_b200.triangulation import pack_keys, triangulate_groups, undistort_points

    rows = np.searchsorted(g["s4_cam_ids"], g["s4_px_cam"])
    fish = np.zeros(len(g["s4_K"]), np.int32)
    und = undistort_points(g["s4_px"], rows, g["s4_K"], list(g["s4_dist"]), fish)
    key = pack_keys(g["s4_sync"], g["s4_obj"], g["s4_kp"])
    assert len(key) == len(rows)
    two = triangulate_groups(g["s4_proj"], rows, key, und.astype(np.float64))
    one = triangulate_groups(g["s4_proj"], rows, key, g["s4_px"], undistort=(g["s4_K"], list(g["s4_dist"]), fish))
    for a, b in zip(one, two):
        assert np.array_equal(a, b, equal_nan=True)
