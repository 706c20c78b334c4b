"""The covariance statement (oracle/covariance.py), the gauge choice and the pose conversion (caliscope_b200.uncertainty),
without a GPU."""
from __future__ import annotations

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from caliscope_b200 import uncertainty as U
from oracle import covariance as OC
from tests import _covariance_cases as CC

PIVOT_RTOL = 1e-10  # CB_COV_PIVOT_RTOL, include/caliscope_b200.h


@pytest.mark.parametrize("name", [c[0] for c in CC.FIXTURES] + ["degenerate"])
def test_dense_and_schur_forms_agree(name):
    if name == "degenerate":
        rig, x = CC.degenerate_rig()
        loss, fs = "linear", 1.0
    else:
        rig, x, loss, fs = CC.fixture_case(name)
    fixed = CC.gauge(rig, x)
    d = OC.dense_covariance(x, rig, fixed, loss, fs)
    s = OC.schur_covariance(x, rig, fixed, loss, fs)
    assert CC.rel_fro(s["cameras"], d["cameras"]) < 1e-10
    assert np.array_equal(s["point_rank"], d["point_rank"]) and s["dof"] == d["dof"]
    if rig.n_constraints == 0:  # component points are NaN in both
        assert CC.rel_fro(s["points"], d["points"]) < 1e-10
    if name == "degenerate":
        assert (d["point_rank"][::7] == 0).all() and (d["point_rank"] == 2).any()


def test_default_gauge_fixes_seven_or_six_and_skips_unobserved_cameras():
    rig, x, _, _ = CC.fixture_case("small_pinhole_refine0.npz")
    f = CC.gauge(rig, x)
    assert len(f) == 7 and list(f[:6]) == list(range(6)) and f[6] in range(rig.cam_offsets[1] + 3, rig.cam_offsets[-1])
    rig, x, _, _ = CC.fixture_case("small_pinhole_constraints.npz")
    assert list(CC.gauge(rig, x)) == list(range(6))
    rig, x = CC.degenerate_rig()
    observed = OC.observed_cameras(rig)
    observed[0] = False  # camera 0 unobserved: camera 1 becomes the reference
    f = U.default_gauge(x, rig.cam_offsets, observed, False)
    assert list(f[:6]) == list(range(rig.cam_offsets[1], rig.cam_offsets[1] + 6))
    o4 = rig.cam_offsets[4]
    assert not np.isin(f, np.arange(o4, o4 + 6)).any()  # camera 4 has no observations


def test_pivot_threshold_separates_gauge_fixed_from_singular_systems():
    for name in ("small_pinhole_refine0.npz", "small_pinhole_refine1.npz", "session4_softl1.npz", "mixed_fisheye.npz"):
        rig, x, loss, fs = CC.fixture_case(name)
        good = OC.reduced_pivots(x, rig, CC.gauge(rig, x), loss, fs).min()
        bad = OC.reduced_pivots(x, rig, np.arange(6), loss, fs).min()
        assert good > 1e4 * PIVOT_RTOL and bad < 1e-2 * PIVOT_RTOL, (name, good, bad)


def test_gauge_invariance_of_a_relative_rotation_angle():
    rig, x, loss, fs = CC.fixture_case("session4_softl1.npz")
    g = CC.fd_gradient(lambda xx: CC.rel_angle(xx, rig.cam_offsets, 1, 2), x, rig.n_camera_params)
    a = OC.schur_covariance(x, rig, CC.gauge(rig, x), loss, fs)["cameras"]
    b = OC.schur_covariance(x, rig, CC.alt_gauge(rig, x), loss, fs)["cameras"]
    va, vb = g @ a @ g, g @ b @ g
    assert abs(va - vb) < 1e-6 * va
    # a gauge-dependent quantity (camera 1's centre) does change
    gc = CC.fd_gradient(lambda xx: U.camera_centers(xx, rig.cam_offsets)[1, 0], x, rig.n_camera_params)
    assert abs(gc @ a @ gc - gc @ b @ gc) > 1e-3 * (gc @ a @ gc)


def test_pose_conversion_matches_finite_difference_propagation():
    rig, x, loss, fs = CC.fixture_case("small_pinhole_refine0.npz")
    cam = OC.dense_covariance(x, rig, CC.gauge(rig, x), loss, fs)["cameras"]
    poses = U.camera_poses(x, rig.cam_offsets, cam)
    assert np.all(poses[0].position_cov == 0) and poses[0].orientation_std_deg == 0
    for c in (1, 2):
        o = rig.cam_offsets[c]
        r0, t0 = x[o : o + 3], x[o + 3 : o + 6]
        R0 = U.rodrigues(r0)

        def f(p):
            R = U.rodrigues(p[:3])
            e = Rotation.from_matrix(R0.T @ R).as_rotvec()
            return np.concatenate([-R.T @ p[3:], e])

        p0 = np.concatenate([r0, t0])
        G = np.stack([(f(p0 + h) - f(p0 - h)) / 2e-7 for h in 1e-7 * np.eye(6)], axis=1)
        ref = G @ cam[o : o + 6, o : o + 6] @ G.T
        assert np.allclose(poses[c].position_cov, ref[:3, :3], rtol=1e-5, atol=1e-6 * np.abs(ref[:3, :3]).max())
        assert np.allclose(poses[c].orientation_cov, ref[3:, 3:], rtol=1e-5, atol=1e-6 * np.abs(ref[3:, 3:]).max())
        assert poses[c].position_std > 0 and poses[c].orientation_std_deg > 0
