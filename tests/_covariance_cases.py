"""Problems and helpers shared by the covariance tests (test infrastructure)."""
from __future__ import annotations

import numpy as np

from oracle import ba_oracle as O
from oracle import covariance as OC
from tests._util import load_golden

# (fixture, solution key, loss)
FIXTURES = [
    ("small_pinhole_refine0.npz", "x_default", "linear"),
    ("small_pinhole_refine1.npz", "x_default", "linear"),
    ("mixed_fisheye.npz", "x1", "linear"),
    ("session4_softl1.npz", "x_default", "soft_l1"),
    ("small_pinhole_constraints.npz", "x_default", "linear"),
    ("aruco_constraints_refine0.npz", "x_default", "linear"),
]


def fixture_case(name):
    fx, key, loss = next(c for c in FIXTURES if c[0] == name)
    g, rig = load_golden(fx)
    fs = float(g["f_scale"]) if "f_scale" in g else 1.0
    return rig, g[key], loss, fs


def degenerate_rig():
    """Single-view points (every 5th point keeps one observation), unobserved points (every 7th) and an unobserved
    camera (4), like the solve's test_unobserved_points_and_cameras_are_left_untouched."""
    from caliscope_b200 import synthetic

    r = synthetic.make_rig(6, 300, 3000, seed=5)
    keep = (r.obs_pt % 7 != 0) & (r.obs_cam != 4)
    first = np.zeros(len(keep), bool)
    _, idx = np.unique(r.obs_pt, return_index=True)
    first[idx] = True
    keep &= (r.obs_pt % 5 != 0) | first | (r.obs_pt % 7 == 0)
    rig = O.Rig(r.cam_flags, r.cam_const, r.n_pts, r.obs_cam[keep], r.obs_pt[keep], r.obs_xy[keep])
    return rig, r.x0


def gauge(rig, x):
    from caliscope_b200 import uncertainty

    return uncertainty.default_gauge(x, rig.cam_offsets, OC.observed_cameras(rig), rig.n_constraints > 0)


def alt_gauge(rig, x):
    """A second valid gauge: the extrinsics of the LAST observed camera and, without constraints, the translation
    component of the camera farthest from it that default_gauge's rule picks."""
    from caliscope_b200 import uncertainty

    order = np.nonzero(OC.observed_cameras(rig))[0][::-1]
    f = list(range(rig.cam_offsets[order[0]], rig.cam_offsets[order[0]] + 6))
    if rig.n_constraints == 0:
        C = uncertainty.camera_centers(x, rig.cam_offsets)
        c1 = int(order[1:][np.argmax(np.linalg.norm(C[order[1:]] - C[order[0]], axis=1))])
        d = uncertainty.rodrigues(x[rig.cam_offsets[c1] : rig.cam_offsets[c1] + 3]) @ (C[order[0]] - C[c1])
        f.append(int(rig.cam_offsets[c1]) + 3 + int(np.argmax(np.abs(d))))
    return np.asarray(f, np.int32)


def rel_angle(x, offs, a, b):
    from caliscope_b200 import uncertainty as U

    Ra = U.rodrigues(x[offs[a] : offs[a] + 3])
    Rb = U.rodrigues(x[offs[b] : offs[b] + 3])
    return float(np.arccos(np.clip((np.trace(Ra @ Rb.T) - 1) / 2, -1, 1)))


def baseline_ratio(x, offs, a, b, c, d):
    from caliscope_b200 import uncertainty as U

    C = U.camera_centers(x, offs)
    return float(np.linalg.norm(C[a] - C[b]) / np.linalg.norm(C[c] - C[d]))


def fd_gradient(fun, x, ncp, h=1e-6):
    """Central-difference gradient of fun(x) over the camera section."""
    g = np.zeros(ncp)
    for i in range(ncp):
        xp = x.copy()
        xm = x.copy()
        xp[i] += h
        xm[i] -= h
        g[i] = (fun(xp) - fun(xm)) / (2 * h)
    return g


def rel_fro(a, b) -> float:
    m = np.isfinite(b)
    assert np.array_equal(m, np.isfinite(a)), "NaN pattern differs"
    return float(np.linalg.norm(a[m] - b[m]) / np.linalg.norm(b[m]))
