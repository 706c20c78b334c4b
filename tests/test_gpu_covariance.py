"""cb_ba_covariance / BAProblem.covariance against the NumPy statement in oracle/covariance.py, and the statistical meaning
of the prediction (Monte Carlo)."""
from __future__ import annotations

import numpy as np
import pytest

from oracle import ba_oracle as O
from oracle import covariance as OC
from tests import _covariance_cases as CC
from tests import _engine_cases as EC

pytestmark = pytest.mark.gpu


def make_problem(rig: O.Rig):
    import caliscope_b200 as cb

    cons = (rig.groups_a, rig.groups_b, rig.distances, rig.weights) if rig.n_constraints else None
    return cb.BAProblem(rig.cam_flags, rig.cam_const, rig.n_pts, rig.obs_cam, rig.obs_pt, rig.obs_xy, constraints=cons)


def _check(cov, ref, tol, tag):
    e_cam = CC.rel_fro(cov.cameras, ref["cameras"])
    ok = np.isfinite(ref["points"][:, 0, 0])
    e_pt = CC.rel_fro(cov.points[ok], ref["points"][ok]) if ok.any() else 0.0
    print(f"{tag}: camera block rel. Frobenius error {e_cam:.2e}, point blocks {e_pt:.2e}, s2 {cov.variance_factor:.6e}, "
          f"dof {cov.dof}")
    assert np.array_equal(cov.point_rank, ref["point_rank"])
    assert np.isnan(cov.points[~ok]).all()
    assert cov.dof == ref["dof"]
    assert abs(cov.variance_factor - ref["variance_factor"]) <= 1e-9 * ref["variance_factor"]
    assert e_cam < tol and e_pt < tol


@pytest.mark.parametrize("name", [c[0] for c in CC.FIXTURES])
def test_covariance_matches_dense_oracle_on_fixtures(name):
    rig, x, loss, fs = CC.fixture_case(name)
    with make_problem(rig) as p:
        cov = p.covariance(x, loss=loss, f_scale=fs)
    ref = OC.dense_covariance(x, rig, cov.fixed, loss, fs)
    assert np.array_equal(cov.fixed, CC.gauge(rig, x))
    _check(cov, ref, 1e-8, name)
    if rig.n_constraints:
        assert (cov.point_rank[OC.constrained_points(rig)] == -1).all()


def test_covariance_with_single_view_and_unobserved_points_and_cameras():
    rig, x = CC.degenerate_rig()
    with make_problem(rig) as p:
        cov = p.covariance(x)
    ref = OC.dense_covariance(x, rig, cov.fixed)
    _check(cov, ref, 1e-8, "degenerate rig")
    assert (cov.point_rank[::7] == 0).all() and (cov.point_rank == 2).any()
    o = rig.cam_offsets[4]
    assert np.isnan(cov.cameras[o : o + 6]).all() and np.isnan(cov.cameras[:, o : o + 6]).all()
    assert (cov.cameras[np.ix_(cov.fixed, cov.fixed)] == 0).all()


@pytest.mark.parametrize("case", EC.COVARIANCE_CASES)
def test_covariance_all_tile_shapes(case):
    """The rigs of test_schur_system_all_tile_shapes (30 .. 600 reduced parameters: every Schur tile shape, direct and
    PCG-sized systems, 1 .. 19 pivot blocks of the sweep), plus the rigs whose points carry more than 96 rows (the
    32-lane variant of the covariance point pass, with and without repeated rows) and the 240-camera dome (camera table
    in global memory, 1440 reduced parameters).  Cameras with fewer than 20 observations lose them all: on the
    100-camera ring, cameras 80..99 see at most a handful of points, which leaves their poses undetermined (the call would
    rightly refuse the singular system); unobserved, they are masked and the reduced system keeps its 600 parameters."""
    c = EC.CASES[case]
    r = c.make()
    keep = np.bincount(r.obs_cam, minlength=c.n_cams)[r.obs_cam] >= 20
    rig = EC.oracle_rig(r, keep)
    with make_problem(rig) as p:
        if c.stats:
            EC.check_stats(p, c)
        cov = p.covariance(r.x0)
    ref = OC.schur_covariance(r.x0, rig, cov.fixed)
    _check(cov, ref, 1e-8, case)


def test_covariance_without_scale_gauge_names_the_singular_parameter():
    from caliscope_b200 import EngineError

    rig, x, loss, fs = CC.fixture_case("small_pinhole_refine0.npz")
    with make_problem(rig) as p:
        with pytest.raises(EngineError) as ei:
            p.covariance(x, fixed=np.arange(6))
        msg = str(ei.value)
        print(msg)
        assert "singular" in msg and "camera" in msg and "parameter" in msg
        p.covariance(x)  # the problem stays usable


def test_covariance_is_gauge_invariant_for_invariant_quantities():
    rig, x, loss, fs = CC.fixture_case("session4_softl1.npz")
    offs = rig.cam_offsets
    g = CC.fd_gradient(lambda xx: CC.rel_angle(xx, offs, 1, 2), x, rig.n_camera_params)
    with make_problem(rig) as p:
        a = p.covariance(x, loss=loss, f_scale=fs, points=False)
        b = p.covariance(x, loss=loss, f_scale=fs, fixed=CC.alt_gauge(rig, x), points=False)
    assert not np.array_equal(a.fixed, b.fixed)
    va, vb = g @ a.cameras @ g, g @ b.cameras @ g
    print(f"var of the relative angle of cameras 1, 2 under two gauges: {va:.6e} {vb:.6e}")
    assert abs(va - vb) < 1e-6 * va


def test_monte_carlo_variance_matches_prediction():
    """cfg2-sized rig (8 cameras, equal fx), exact pixels + seeded N(0, sigma) noise, 500 solves.  The empirical variance
    of similarity-invariant quantities against the prediction at the truth with s2 = (sigma / fx)^2.  For N = 500 normal
    samples the variance ratio has a relative standard deviation sqrt(2 / 499) = 0.063, so [0.8, 1.25] is a band of more
    than 3 standard deviations on either side."""
    import caliscope_b200 as cb
    from caliscope_b200 import synthetic

    sigma, n_runs = 0.5, 500
    r = synthetic.make_rig(8, 2000, 40000, seed=21, noise_px=0.0)
    rig = O.Rig(r.cam_flags, r.cam_const, r.n_pts, r.obs_cam, r.obs_pt, r.obs_xy)
    xt = r.x_true
    fx = float(rig.cam_const[0, 0])
    assert np.all(rig.cam_const[:, 0] == fx)
    exact = O.reproj_errors_px(xt, rig) + rig.obs_xy  # projections of the truth
    offs = rig.cam_offsets
    quantities = {  # relative rotation angles away from 0 and 180 degrees (arccos is not differentiable there)
        "angle(2,5)": lambda x: CC.rel_angle(x, offs, 2, 5),
        "angle(1,3)": lambda x: CC.rel_angle(x, offs, 1, 3),
        "baseline |C1-C4| / |C2-C6|": lambda x: CC.baseline_ratio(x, offs, 1, 4, 2, 6),
        "baseline |C3-C5| / |C0-C7|": lambda x: CC.baseline_ratio(x, offs, 3, 5, 0, 7),
    }
    with cb.BAProblem(rig.cam_flags, rig.cam_const, rig.n_pts, rig.obs_cam, rig.obs_pt, exact) as p:
        cov = p.covariance(xt, variance_factor=(sigma / fx) ** 2, points=False)
    pred = {k: (lambda g: float(g @ cov.cameras @ g))(CC.fd_gradient(f, xt, rig.n_camera_params)) for k, f in quantities.items()}
    rng = np.random.default_rng(2024)
    samples = {k: [] for k in quantities}
    for _ in range(n_runs):
        obs = exact + rng.normal(0.0, sigma, exact.shape)
        with cb.BAProblem(rig.cam_flags, rig.cam_const, rig.n_pts, rig.obs_cam, rig.obs_pt, obs) as q:
            res = q.solve(xt, ftol=1e-12, xtol=1e-12, gtol=1e-12)
        assert res.status > 0
        for k, f in quantities.items():
            samples[k].append(f(res.x))
    ratios = {k: np.var(samples[k], ddof=1) / pred[k] for k in quantities}
    for k, v in ratios.items():
        print(f"Monte Carlo {k}: empirical / predicted variance = {v:.3f} (N = {n_runs})")
    assert all(0.8 <= v <= 1.25 for v in ratios.values()), ratios
