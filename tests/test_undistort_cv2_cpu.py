"""oracle.triangulation.undistort_points against live OpenCV, the definition it restates, on every distortion model
and branch of the inverse maps (tests/_undistort_cases.py): bit-exact float32, NaN positions equal."""
from __future__ import annotations

import numpy as np
import pytest

from oracle.triangulation import undistort_points
from tests import _undistort_cases as U

cv2 = pytest.importorskip("cv2")

CAMS = U.cameras()


@pytest.mark.parametrize("cam", CAMS, ids=[c.name for c in CAMS])
@pytest.mark.parametrize("output", ["normalized", "pixels"])
def test_oracle_undistort_equals_cv2(cam, output):
    sets = U.point_sets(cam)
    pts = np.concatenate(list(sets.values()))
    assert U.branches(cam, pts) >= cam.reaches, cam.name
    with np.errstate(invalid="ignore", over="ignore"):
        got = undistort_points(pts, cam.K, cam.d, cam.fisheye, output=output)
    ref = U.cv2_undistort(cam, pts, output)
    start = 0
    for name, p in sets.items():
        U.assert_same_f32(got[start : start + len(p)], ref[start : start + len(p)], f"{cam.name} {output} {name}")
        start += len(p)


def test_cases_reach_every_branch():
    """The case set as a whole keeps covering the branches the kernel and oracle have."""
    reached = set().union(*(U.branches(c, U.all_points(c)) for c in CAMS))
    assert reached == {"icdist_neg", "sentinel", "theta_tiny", "nonfinite"}
    assert any(c.K[0, 1] != 0 for c in CAMS if c.fisheye) and any(c.K[0, 1] != 0 for c in CAMS if not c.fisheye)
    assert {len(c.d) for c in CAMS if not c.fisheye} == {4, 5, 8, 12}
    assert {c.name for c in CAMS if not c.fisheye and not np.any(c.d)} == {"pin0", "pin0_skew"}
    for c in CAMS:
        r = U.point_sets(c)["rounding"]
        assert (r.astype(np.float32).astype(np.float64) != r).all()


def test_fisheye_sentinel_and_nan_edges():
    """The two fisheye edges where OpenCV differs from mapping every result through K, pinned by value."""
    wild = next(c for c in CAMS if c.name == "fish_wild")
    p = np.array([[1200.0, 480.0], [np.nan, 100.0]])
    norm = undistort_points(p, wild.K, wild.d, True)
    px = undistort_points(p, wild.K, wild.d, True, output="pixels")
    assert (norm[0] == U.SENTINEL).all() and (px[0] == U.SENTINEL).all()
    # NaN theta_d clamps to -pi/2 and iterates, so y keeps a value in normalised output; pixels are (NaN, NaN)
    assert np.isnan(norm[1, 0]) and np.isfinite(norm[1, 1]) and np.isnan(px[1]).all()
    U.assert_same_f32(norm, U.cv2_undistort(wild, p, "normalized"), "normalized")
    U.assert_same_f32(px, U.cv2_undistort(wild, p, "pixels"), "pixels")
