"""Gaussian priors on cameras and points in the engine (DESIGN.md section 4.13): every shape-selected variant forms the
oracle's system with fixed sets (section 4.12) alone and with priors beside them, a solve is scipy's least_squares on the augmented residuals, zero information changes
nothing, stiff information approaches the fixed solve, the covariance is the posterior, and the refused inputs are
refused before any device work."""
from __future__ import annotations

import numpy as np
import pytest

from oracle import ba_oracle as O
from oracle import lm_schur as LS
from tests import _engine_cases as EC
from tests import _held_oracle as HO

pytestmark = pytest.mark.gpu


def _width(rig, c):
    return int(rig.cam_offsets[c + 1] - rig.cam_offsets[c])


def _spd(rng, n, scale):
    A = rng.standard_normal((n, n))
    M = A @ A.T / n + np.eye(n)
    return scale * M / np.abs(M).max()


def _add_cam(pr, rig, c, mean_w, info_w, slots=None):
    """A camera prior: mean over the camera's width, info over ``slots`` of it (all by default), padded to 9."""
    w = _width(rig, c)
    slots = np.arange(w) if slots is None else np.asarray(slots)
    m = np.zeros(9)
    m[:w] = mean_w
    L = np.zeros((9, 9))
    L[np.ix_(slots, slots)] = info_w
    pr.cams = np.append(pr.cams, c).astype(np.int64)
    pr.cam_mean = np.concatenate([pr.cam_mean, m[None]])
    pr.cam_info = np.concatenate([pr.cam_info, L[None]])


def _add_pt(pr, j, mean, info):
    pr.pts = np.append(pr.pts, j).astype(np.int64)
    pr.pt_mean = np.concatenate([pr.pt_mean, np.asarray(mean, np.float64)[None]])
    pr.pt_info = np.concatenate([pr.pt_info, np.asarray(info, np.float64)[None]])


def _case_priors(rig, x, seed=0):
    """Priors in every form, scaled to the data's own information, and fixed sets beside them:
    - camera 0: a full prior (6 x 6 or 9 x 9);
    - camera 2: a full prior with two of its rotation parameters fixed (the prior still pulls the rest);
    - the first other 9-parameter camera: s, k1, k2 only; under P = 9 the first other 6-parameter camera: a full prior;
    - every 11th point: a full-rank prior; every 13th (not 11th) point: a rank-1 prior;
    - fixed: the two parameters above and every 7th point that has no prior.
    Means are x plus noise of the start's own size."""
    rng = np.random.default_rng(seed)
    lin = LS.linearize(x, rig)
    u = float(np.median(np.einsum("cii->ci", lin.U)[lin.U[:, 0, 0] > 0]))
    v = float(np.median(np.einsum("jii->ji", lin.V)))
    pr = HO.Priors()
    ncp = rig.n_camera_params

    def cam_mean(c):
        o, w = rig.cam_offsets[c], _width(rig, c)
        return x[o : o + w] + 1e-3 * rng.standard_normal(w)

    for c in (0, 2):
        _add_cam(pr, rig, c, cam_mean(c), _spd(rng, _width(rig, c), u))
    wide = [c for c in range(1, rig.n_cams) if _width(rig, c) == 9 and c != 2]
    if wide:
        _add_cam(pr, rig, wide[0], cam_mean(wide[0]), _spd(rng, 3, u), slots=[6, 7, 8])
        narrow = [c for c in range(1, rig.n_cams) if _width(rig, c) == 6 and c != 2]
        if narrow:
            _add_cam(pr, rig, narrow[0], cam_mean(narrow[0]), _spd(rng, 6, u))
    X = x[ncp:].reshape(-1, 3)
    for j in range(0, rig.n_pts, 11):
        _add_pt(pr, j, X[j] + 1e-3 * rng.standard_normal(3), _spd(rng, 3, v))
    for j in range(0, rig.n_pts, 13):
        if j % 11:
            a = rng.standard_normal(3)
            _add_pt(pr, j, X[j] + 1e-3 * rng.standard_normal(3), v * np.outer(a, a) / (a @ a))
    fc = [int(rig.cam_offsets[2]), int(rig.cam_offsets[2]) + 1]
    fp = [j for j in range(3, rig.n_pts, 7) if j % 11 and j % 13]
    return pr, fc, fp


def _case_fixed_sets(rig):
    """Camera 0 whole, s, k1, k2 of the first other camera with free intrinsics (if any), every seventh point."""
    fc = list(range(rig.cam_offsets[0], rig.cam_offsets[1]))
    wide = [c for c in range(1, rig.n_cams) if _width(rig, c) == 9]
    fc += [int(rig.cam_offsets[c]) + a for c in wide[:1] for a in (6, 7, 8)]
    return fc, list(range(3, rig.n_pts, 7))


# ---------------------------------------------------------------------------------------------
# 1. every shape-selected variant forms the oracle's system, with fixed sets alone and with priors beside them
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("held", ["fixed", "priors+fixed"])
@pytest.mark.parametrize("case", list(EC.CASES) + ["relabelled-sparse-lists"])
def test_every_variant_forms_the_held_system(case, held):
    """The engine's U, g_c, V, g_p and cost, its masked reduced system and step, and a solve: the fixed entries come back
    bit for bit and the cost is at or below scipy's on the free subvector."""
    if case == "relabelled-sparse-lists":
        rig, x0, xt = EC.relabelled_sparse_case()
        c = None
    else:
        c = EC.CASES[case]
        r = c.make()
        rig, x0, xt = EC.oracle_rig(r), r.x0, r.x_true
    if held == "fixed":
        pr, (fc, fp) = None, _case_fixed_sets(rig)
    else:
        pr, fc, fp = _case_priors(rig, x0)
    free = EC.free_mask(rig, fc, fp)
    # known values at the fixed entries, as a caller's are: held at a noisy start, a fixed camera or point contradicts
    # the observations, and the solve crawls along a flat valley where the termination tests stop at scattered points
    x0 = np.where(free, x0, xt)
    lam = 1e-3
    with EC.problem(rig, pr, fixed_cam_params=fc, fixed_points=fp) as p:
        if c is not None and c.stats:
            EC.check_stats(p, c)
        if c is None:
            print(f"{case}: compacted Schur lists {int(p.stat(0))}")
            assert p.stat(EC.REORDERED) == 1 and p.stat(0) == 1  # relabelled, compacted lists
        mode = int(p.stat(EC.SOLVE))
        P = p.cam_stride
        ne = p.normal_equations(x0, lam)
        res = p.solve(x0)
    whole = HO.linearize(x0, rig, None, pr)  # what the engine's U, g_c slot, V, g_p hold: every observation, the priors
    lin = HO.linearize(x0, rig, free, pr)
    Dc2, Dp2 = HO.scaling(x0, rig, pr)
    fcs, fps = HO.free_slots(free, rig, P)
    active = np.zeros(rig.n_cams * P, bool)
    for k in range(rig.n_cams):
        active[k * P : k * P + _width(rig, k)] = True
    S, b, Einv, Wd = HO.schur_system(lin, rig, lam, Dc2, Dp2, active & ~fcs, ~fps)
    n_cp, n_pp = (0, 0) if pr is None else (len(pr.cams), len(pr.pts))
    print(f"{case} {held}: P {P} solve mode {mode}, {n_cp} camera and {n_pp} point priors")
    assert abs(ne["cost"] - whole.cost) <= 1e-12 * whole.cost
    for k, ref in (("U", whole.U), ("gc", whole.gc), ("V", whole.V), ("gp", whole.gp)):
        err = np.abs(ne[k] - ref).max() / np.abs(ref).max()
        assert err < 1e-10, (k, err)
    assert np.abs(ne["S"] - S).max() < 1e-9 * np.abs(S).max()
    assert np.abs(ne["b"] - b).max() < 1e-9 * np.abs(b).max()
    EC.check_step(ne["S"], ne["b"], ne["dc"], mode, case)
    assert np.all(ne["dc"].ravel()[active & ~fcs] == 0.0) and np.all(ne["dp"][~fps] == 0.0)
    dp = -np.einsum("jab,jb->ja", Einv, lin.gp + np.einsum("jcpa,cp->ja", Wd, ne["dc"]))
    assert np.abs(ne["dp"] - dp).max() < 1e-9 * np.abs(dp).max()
    ref = HO.solve_scipy(rig, x0, free, pr)
    print(f"{case} {held}: gpu status {res.status} nfev {res.nfev} cost {res.cost:.15e} | scipy nfev {ref.nfev} "
          f"cost {ref.cost:.15e}")  # fmt: skip
    assert res.status in (1, 2, 3, 4)
    assert np.array_equal(res.x[~free], x0[~free])
    assert res.cost <= ref.cost * (1 + 1e-8)


def test_prior_point_without_observations():
    """A point no camera sees, with a definite prior: its block is the prior's information alone, the solve puts it at
    the prior mean, and its covariance is s2 info^-1 (rank 3) from the ordinary pseudo-inverse path."""
    from caliscope_b200 import synthetic

    r = synthetic.make_rig(8, 300, 3000, seed=31)
    rig = O.Rig(r.cam_flags, r.cam_const, r.n_pts + 1, r.obs_cam, r.obs_pt, r.obs_xy)
    j = r.n_pts
    x0 = np.concatenate([r.x0, [0.3, -0.2, 2.0]])
    mean = np.array([0.31, -0.18, 2.05])
    info = np.array([[4e3, 1e3, 0.0], [1e3, 3e3, 5e2], [0.0, 5e2, 2e3]])
    pr = HO.Priors()
    _add_pt(pr, j, mean, info)
    pr_s = HO.Priors()
    for jj, m in ((j, mean), (0, x0[rig.n_camera_params : rig.n_camera_params + 3]), (1, x0[rig.n_camera_params + 3 :][:3]),
                  (2, x0[rig.n_camera_params + 6 :][:3])):  # fmt: skip
        _add_pt(pr_s, jj, m, info)  # three more priors on seen points fix the gauge for the covariance
    with EC.problem(rig, pr) as p:
        ne = p.normal_equations(x0, 1e-3)
        assert np.array_equal(ne["V"][j], info)
        assert np.allclose(ne["gp"][j], info @ (x0[-3:] - mean), rtol=1e-14)
        res = p.solve(x0)
    assert res.status in (1, 2, 3, 4)
    assert np.abs(res.x[-3:] - mean).max() < 1e-6  # where ftol stops the approach
    with EC.problem(rig, pr_s) as p:
        res = p.solve(x0)
        cov = p.covariance(res.x)
    ref = HO.dense_covariance(res.x, rig, priors=pr_s)
    assert cov.point_rank[j] == 3 and ref["point_rank"][j] == 3
    want = cov.variance_factor * np.linalg.inv(info)
    assert np.allclose(cov.points[j], want, rtol=1e-9)
    assert cov.dof == ref["dof"]


# ---------------------------------------------------------------------------------------------
# 2. solves against scipy on the augmented residuals
# ---------------------------------------------------------------------------------------------
def _pulled_case(n_cams, n_pts, n_obs, seed):
    """Free intrinsics; camera 0 and point `anchor` fixed at their true values (gauge and scale), priors on cameras 3, 5
    and every 9th point with means away from the truth, information of the data's own size.  Returns the rig, x0, free
    mask, the priors and the fixed sets."""
    from caliscope_b200 import synthetic

    r = synthetic.make_rig(n_cams, n_pts, n_obs, seed=seed, refine_intrinsics=True)
    rig = EC.oracle_rig(r)
    rng = np.random.default_rng(seed)
    lin = LS.linearize(r.x_true, rig)
    ncp = rig.n_camera_params
    seen = np.bincount(rig.obs_pt, minlength=rig.n_pts)
    anchor = int(np.argmax(seen))
    fc, fp = list(range(rig.cam_offsets[0], rig.cam_offsets[1])), [anchor]
    pr = HO.Priors()
    for c in (3, 5):
        o, w = rig.cam_offsets[c], _width(rig, c)
        L = np.diag(np.einsum("ii->i", lin.U[c])[:w])
        _add_cam(pr, rig, c, r.x_true[o : o + w] + 3e-3 * rng.standard_normal(w), L)
    X = r.x_true[ncp:].reshape(-1, 3)
    for j in range(1, rig.n_pts, 9):
        if j != anchor:
            _add_pt(pr, j, X[j] + 5e-3 * rng.standard_normal(3), lin.V[j] + 1e-3 * np.eye(3))
    free = EC.free_mask(rig, fc, fp)
    x0 = np.where(free, r.x0, r.x_true)
    return rig, x0, free, pr, fc, fp


@pytest.mark.parametrize("n_cams,n_pts,n_obs", [(8, 300, 3000), (16, 500, 6000)])
@pytest.mark.parametrize("loss", ["linear", "soft_l1"])
@pytest.mark.parametrize("with_fixed", [True, False])
def test_solve_matches_scipy_with_priors(n_cams, n_pts, n_obs, loss, with_fixed):
    """The bar of test_gpu_fixed_params.test_solve_matches_scipy_on_the_free_subvector: cost at or below scipy's; the
    RMSE (linear) or the cost (soft_l1) within scipy's own default-vs-tight termination noise.  The engine's cost and
    initial cost are the augmented objective's."""
    from caliscope_b200 import synthetic

    rig, x0, free, pr, fc, fp = _pulled_case(n_cams, n_pts, n_obs, n_cams + 40)
    if not with_fixed:
        free, fc, fp = np.ones(rig.n_params, bool), [], []
    fs = 2.0 / synthetic.WEBCAM_F
    ref = HO.solve_scipy(rig, x0, free, pr, loss=loss, f_scale=fs)
    tight = HO.solve_scipy(rig, x0, free, pr, loss=loss, f_scale=fs, ftol=1e-15, xtol=1e-15, gtol=1e-15, max_nfev=200)
    with EC.problem(rig, pr, fixed_cam_params=fc, fixed_points=fp) as p:
        res = p.solve(x0, loss=loss, f_scale=fs)
        rm = p.overall_rmse_px(res.x)
    rm_ref, rm_tight = O.overall_rmse_px(ref.x, rig), O.overall_rmse_px(tight.x, rig)
    print(f"{n_cams} cams {loss} fixed={with_fixed}: gpu status {res.status} nfev {res.nfev} cost {res.cost:.15e} "
          f"rmse {rm:.10f} | scipy nfev {ref.nfev} cost {ref.cost:.15e} rmse {rm_ref:.10f} | tight cost "
          f"{tight.cost:.15e} rmse {rm_tight:.10f}")  # fmt: skip
    assert res.status in (1, 2, 3, 4)
    assert np.array_equal(res.x[~free], x0[~free])
    assert res.cost <= ref.cost * (1 + 1e-8)
    if loss == "linear":
        assert abs(rm - rm_ref) < 3 * abs(rm_ref - rm_tight) + 1e-6
    else:
        assert abs(res.cost - tight.cost) < 1e-6 * tight.cost
    for x, c in ((res.x, res.cost), (x0, res.initial_cost)):
        want = O.robust_cost(O.residuals(x, rig), loss, fs) + HO.prior_cost(x, rig, pr)
        assert abs(c - want) <= 1e-10 * want


def test_huber_and_cauchy_match_scipy_with_priors():
    """Robust refinement after a linear solve, the way the robust losses are used: from the linear solution of the same
    augmented problem.  (From the rig's synthetic start, where nearly every row lies outside the loss's quadratic zone,
    the engine's huber and cauchy solves reject every trial from the first linearisation on, with or without priors and
    fixed sets, while scipy's converge; that start is left out here.)"""
    from caliscope_b200 import synthetic

    rig, x0, free, pr, fc, fp = _pulled_case(8, 300, 3000, 77)
    fs = 2.0 / synthetic.WEBCAM_F
    with EC.problem(rig, pr, fixed_cam_params=fc, fixed_points=fp) as p:
        xs = p.solve(x0).x
        for loss in ("huber", "cauchy"):
            res = p.solve(xs, loss=loss, f_scale=fs)
            ref = HO.solve_scipy(rig, xs, free, pr, loss=loss, f_scale=fs)
            print(f"{loss}: gpu status {res.status} nfev {res.nfev} cost {res.cost:.15e} | scipy nfev {ref.nfev} "
                  f"{ref.cost:.15e}")  # fmt: skip
            # scipy crawls here (huber: some 1800 evaluations to stop at a cost 2e-8 above the engine's); the engine's
            # cost is checked to be the augmented objective at its x, so lower is better, not different
            assert res.status in (1, 2, 3, 4)
            assert res.cost <= ref.cost * (1 + 1e-8)
            want = O.robust_cost(O.residuals(res.x, rig), loss, fs) + HO.prior_cost(res.x, rig, pr)
            assert abs(res.cost - want) <= 1e-10 * want


def test_cost_and_optimality_include_the_priors():
    """gtol above the start's gradient: the solve stops at x0 with status 1, so cost, initial_cost and optimality are
    the augmented objective's at x0 exactly -- and differ from the prior-free ones."""
    rig, x0, free, pr, fc, fp = _pulled_case(8, 300, 3000, 48)
    c = 7  # a prior whose mean is far off: its gradient is the largest
    o = rig.cam_offsets[c]
    u = LS.linearize(x0, rig).U[c]
    _add_cam(pr, rig, c, x0[o : o + 9] + np.r_[0.0, 0.0, 0.0, 1.0, 1.0, 1.0, 0.0, 0.0, 0.0], np.diag(np.diag(u)))
    lin = HO.linearize(x0, rig, free, pr)
    g = LS.join_x(lin.gc, lin.gp, rig)
    gmax = np.abs(g[free]).max()
    lin0 = HO.linearize(x0, rig, free)
    g0 = np.abs(LS.join_x(lin0.gc, lin0.gp, rig)[free]).max()
    with EC.problem(rig, pr, fixed_cam_params=fc, fixed_points=fp) as p:
        res = p.solve(x0, gtol=2 * max(gmax, g0))
    print(f"optimality {res.optimality:.12e} (augmented {gmax:.12e}, prior-free {g0:.12e}); cost {res.cost:.12e} "
          f"(augmented {lin.cost:.12e}, prior-free {lin0.cost:.12e})")  # fmt: skip
    assert res.status == 1 and np.array_equal(res.x, x0)
    assert abs(res.optimality - gmax) <= 1e-9 * gmax and gmax > 2 * g0
    assert abs(res.cost - lin.cost) <= 1e-12 * lin.cost and res.initial_cost == res.cost
    assert lin.cost - lin0.cost > 1e-3 * lin.cost


def test_prior_pulls_between_the_free_solve_and_the_mean():
    """A camera and points whose prior means sit off the free solution, with information of the data's size: the
    solution lies between the free solve and the mean (on the segment's interior, in both distances)."""
    rig, x0, free, _, fc, fp = _pulled_case(8, 300, 3000, 51)
    with EC.problem(rig, fixed_cam_params=fc, fixed_points=fp) as p:
        xf = p.solve(x0, ftol=1e-12, xtol=1e-12, gtol=1e-12).x
    rng = np.random.default_rng(5)
    lin = LS.linearize(xf, rig)
    pr = HO.Priors()
    c = 4
    o, w = rig.cam_offsets[c], _width(rig, c)
    # isotropic information a I: to second order the solution is a + (H + a I)^-1 a (m - a), whose matrix is symmetric
    # with eigenvalues in (0, 1), so it lands strictly inside the segment in both distances
    _add_cam(pr, rig, c, xf[o : o + w] + 2e-3 * rng.standard_normal(w), np.trace(lin.U[c]) / w * np.eye(w))
    ncp = rig.n_camera_params
    pts = [j for j in range(2, rig.n_pts, 23) if j not in fp][:8]
    for j in pts:
        _add_pt(pr, j, xf[ncp + 3 * j : ncp + 3 * j + 3] + 0.01 * rng.standard_normal(3), np.trace(lin.V[j]) / 3 * np.eye(3))
    with EC.problem(rig, pr, fixed_cam_params=fc, fixed_points=fp) as p:
        xp = p.solve(x0, ftol=1e-12, xtol=1e-12, gtol=1e-12).x
    for cols, mean, _ in HO.blocks(rig, pr):
        a, m, b = xf[cols], mean, xp[cols]
        t = (b - a) @ (m - a) / ((m - a) @ (m - a))
        print(f"x{cols[0]}..: pulled {t:.3f} of the way to the mean")
        assert 0.0 < t < 1.0
        assert np.linalg.norm(b - m) < np.linalg.norm(a - m) and np.linalg.norm(b - a) < np.linalg.norm(m - a)


# ---------------------------------------------------------------------------------------------
# 3. zero information changes nothing; stiff information approaches fixed
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["ring16-direct-nP96", "ring11-refine-pcg-cl6-nP99", "dome70-refine-pcg-l2-nP630",
                                  "static-ring12-lanes32-dups"])  # fmt: skip
def test_zero_information_is_bit_identical(case):
    """Priors with info = 0 on every camera and point run the prior variants of the kernels; every term they add is an
    exact zero (x + 0.0, fma(0, d, v)), so the solve is the prior-free one bit for bit."""
    r = EC.CASES[case].make()
    rig = EC.oracle_rig(r)
    pr = HO.Priors()
    for c in range(rig.n_cams):
        _add_cam(pr, rig, c, r.x0[rig.cam_offsets[c] : rig.cam_offsets[c + 1]] + 0.01, np.zeros((6, 6)), slots=range(6))
    for j in range(rig.n_pts):
        _add_pt(pr, j, r.x0[rig.n_camera_params + 3 * j :][:3] - 0.02, np.zeros((3, 3)))
    with EC.problem(rig) as p:
        a = p.solve(r.x0)
    with EC.problem(rig, pr) as p:
        b = p.solve(r.x0)
    print(f"{case}: nfev {a.nfev} / {b.nfev}, cost {a.cost!r} / {b.cost!r}")
    assert np.array_equal(a.x, b.x) and a.cost == b.cost and a.nfev == b.nfev and a.njev == b.njev
    assert a.initial_cost == b.initial_cost and a.optimality == b.optimality


def test_stiff_priors_approach_fixed():
    """info = 1e12 I at known values on a whole camera, and on four surveyed points: within 1e-7 (x units) of the solve
    that holds the same parameters fixed.  Both run to tight tolerances, so where they stop is the optimum, not the
    termination test."""
    from caliscope_b200 import synthetic

    r = synthetic.make_rig(12, 400, 5000, seed=12)
    rig = EC.oracle_rig(r)
    ncp = rig.n_camera_params
    x0 = r.x0.copy()
    picks = [5, 50, 120, 300]
    for j in picks:
        x0[ncp + 3 * j : ncp + 3 * j + 3] = r.x_true[ncp + 3 * j : ncp + 3 * j + 3]
    c = 3
    fc = list(range(rig.cam_offsets[c], rig.cam_offsets[c + 1]))
    x0[fc] = r.x_true[fc]
    pr = HO.Priors()
    _add_cam(pr, rig, c, x0[fc], 1e12 * np.eye(6))
    for j in picks:
        _add_pt(pr, j, x0[ncp + 3 * j : ncp + 3 * j + 3], 1e12 * np.eye(3))
    tight = dict(ftol=1e-12, xtol=1e-12, gtol=1e-12)
    with EC.problem(rig, fixed_cam_params=fc, fixed_points=picks) as p:
        a = p.solve(x0, **tight)
    with EC.problem(rig, pr) as p:
        b = p.solve(x0, **tight)
    err = np.abs(a.x - b.x).max()
    print(f"stiff priors vs fixed: max |dx| {err:.2e}, cost {a.cost:.12e} / {b.cost:.12e}, nfev {a.nfev} / {b.nfev}")
    assert b.status in (1, 2, 3, 4)
    assert err < 1e-7
    assert abs(a.cost - b.cost) <= 1e-6 * a.cost


# ---------------------------------------------------------------------------------------------
# 4. covariance: the posterior
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("refine", [False, True])
def test_covariance_is_the_posterior(refine):
    """Priors on three surveyed points (fixing the gauge with fixed=None), on one camera and on further points, with
    info = vf Sigma^-1 for a physical Sigma: the covariance matches the dense (J^T J + info)^-1 at the solution, with its
    dof and s2, and each prior block's posterior is below its prior Sigma in the Loewner order."""
    from caliscope_b200 import synthetic, uncertainty

    r = synthetic.make_rig(10, 400, 5000, seed=60 + refine, refine_intrinsics=refine)
    rig = EC.oracle_rig(r)
    ncp = rig.n_camera_params
    X = r.x_true[ncp:].reshape(-1, 3)
    seen = np.bincount(rig.obs_pt, minlength=rig.n_pts) >= 3
    cand = np.nonzero(seen)[0]
    surveyed = [cand[np.argmin(X[cand, 2])], cand[np.argmax(X[cand, 0])], cand[np.argmax(X[cand, 1])]]
    pixel_sigma, fx = 0.5, float(rig.cam_const[0, 0])
    vf = (pixel_sigma / fx) ** 2
    rng = np.random.default_rng(61)
    pr = HO.Priors()
    sig = {}
    for j in surveyed + [7, 19, 44]:
        S = np.diag([1e-6, 2e-6, 4e-6]) if j in surveyed else np.diag([1e-4, 1e-4, 1e-4])
        _add_pt(pr, j, X[j] + rng.multivariate_normal(np.zeros(3), S), uncertainty.prior_information(S, pixel_sigma, fx))
        sig[("p", j)] = S
    c = 6
    w = _width(rig, c)
    o = rig.cam_offsets[c]
    Sc = np.diag(np.full(w, 1e-6))
    _add_cam(pr, rig, c, r.x_true[o : o + w] + rng.multivariate_normal(np.zeros(w), Sc),
             uncertainty.prior_information(Sc, pixel_sigma, fx))  # fmt: skip
    x0 = r.x0.copy()
    with EC.problem(rig, pr) as p:
        res = p.solve(x0)
        cov = p.covariance(res.x)
        cov_vf = p.covariance(res.x, variance_factor=vf)
    ref = HO.dense_covariance(res.x, rig, priors=pr)
    e_cam = np.linalg.norm(cov.cameras - ref["cameras"]) / np.linalg.norm(ref["cameras"])
    ok = ref["point_rank"] == 3
    e_pt = np.linalg.norm(cov.points[ok] - ref["points"][ok]) / np.linalg.norm(ref["points"][ok])
    print(f"posterior covariance: cameras {e_cam:.2e}, points {e_pt:.2e}, dof {cov.dof} / {ref['dof']}, s2 "
          f"{cov.variance_factor:.6e} / {ref['variance_factor']:.6e}")  # fmt: skip
    assert res.status in (1, 2, 3, 4) and len(cov.fixed) == 0
    assert cov.dof == ref["dof"]
    assert abs(cov.variance_factor - ref["variance_factor"]) <= 1e-9 * ref["variance_factor"]
    assert np.array_equal(cov.point_rank, ref["point_rank"])
    assert e_cam < 1e-8 and e_pt < 1e-8
    for (kind, j), S in sig.items():
        post = cov_vf.points[j]
        d = np.linalg.eigvalsh(S - post)
        assert d.min() >= -1e-9 * np.abs(S).max(), (j, d)
    post = cov_vf.cameras[o : o + w, o : o + w]
    d = np.linalg.eigvalsh(Sc - 0.5 * (post + post.T))
    assert d.min() >= -1e-9 * np.abs(Sc).max()


# ---------------------------------------------------------------------------------------------
# 5. carry-over
# ---------------------------------------------------------------------------------------------
def test_cull_keeps_the_priors():
    from caliscope_b200 import filtering, synthetic

    r = synthetic.make_rig(10, 600, 7000, seed=10, outlier_frac=0.02)
    rig = EC.oracle_rig(r)
    pr, fc, fp = _case_priors(rig, r.x0, seed=3)
    free = EC.free_mask(rig, fc, fp)
    with EC.problem(rig, pr, fixed_cam_params=fc, fixed_points=fp) as p:
        a = p.solve(r.x0)
        _, thr = filtering.percentile_thresholds(p, a.x, 95.0, want_err=False)
        p2, keep = p.cull(a.x, thr, 10)
        with p2:
            assert p2.has_priors and np.array_equal(p2.point_priors[0], pr.pts)
            ne = p2.normal_equations(a.x, 1e-3)
            c = p2.solve(a.x)
    assert not keep.all()
    rig2 = EC.oracle_rig(r, keep)
    whole = HO.linearize(a.x, rig2, None, pr)
    assert abs(ne["cost"] - whole.cost) <= 1e-12 * whole.cost
    assert np.abs(ne["gc"] - whole.gc).max() <= 1e-10 * np.abs(whole.gc).max()
    ref = HO.solve_scipy(rig2, a.x, free, pr)
    print(f"after cull: gpu cost {c.cost:.15e} nfev {c.nfev} | scipy cost {ref.cost:.15e}")
    assert c.status in (1, 2, 3, 4) and c.cost <= ref.cost * (1 + 1e-8)
    assert np.array_equal(c.x[~free], r.x0[~free])


# ---------------------------------------------------------------------------------------------
# 6. refusals
# ---------------------------------------------------------------------------------------------
def test_refused_inputs_launch_nothing():
    import caliscope_b200 as cb
    from caliscope_b200 import _lib as L
    from caliscope_b200 import synthetic

    lib = L.load()
    r = synthetic.make_rig(6, 200, 2000, seed=6)
    rig = EC.oracle_rig(r)
    ga = np.array([[0, 0, 0, 0], [5, 5, 5, 5]], np.int32)
    gb = np.array([[1, 1, 1, 1], [6, 6, 6, 6]], np.int32)
    cons = (ga, gb, np.array([0.1, 0.1]), np.array([1.0, 1.0]))
    I6, I3 = np.pad(np.eye(6), ((0, 3), (0, 3))), np.eye(3)
    z9, z3 = np.zeros(9), np.zeros(3)

    def cams(idx, mean=None, info=None):
        k = len(idx)
        return dict(camera_priors=(idx, np.stack([z9] * k) if mean is None else mean,
                                   np.stack([I6] * k) if info is None else info))  # fmt: skip

    def pts(idx, mean=None, info=None):
        k = len(idx)
        return dict(point_priors=(idx, np.stack([z3] * k) if mean is None else mean,
                                  np.stack([I3] * k) if info is None else info))  # fmt: skip

    asym = I6.copy()
    asym[0, 1] = 1e-6
    neg = I6.copy()
    neg[2, 2] = -1e-3
    outside = I6.copy()
    outside[7, 7] = 1.0
    nanm = z9.copy()
    nanm[4] = np.nan
    infi = I3.copy()
    infi[1, 1] = np.inf
    cases = [
        (cams([6]), None, -1, "out of range"),
        (cams([-1]), None, -1, "out of range"),
        (cams([2, 2]), None, -1, "repeated"),
        (pts([rig.n_pts]), None, -1, "out of range"),
        (pts([7, 8, 7]), None, -1, "repeated"),
        (cams([1], mean=nanm[None]), None, -1, "non-finite mean"),
        (pts([3], info=infi[None]), None, -1, "non-finite information"),
        (cams([1], info=asym[None]), None, -1, "not symmetric"),
        (cams([1], info=neg[None]), None, -1, "semi-definite"),
        (pts([4], info=-I3[None]), None, -1, "semi-definite"),
        (cams([1], info=outside[None]), None, -1, "outside its 6 x 6"),
        (dict(fixed_points=[9], **pts([9])), None, -1, "both fixed"),
        (pts([6]), cons, -4, "rigid-distance"),
    ]
    codes = {v: k for k, v in vars(L).items() if k.startswith("CB_E_")}
    for kw, cn, code, msg in cases:
        n0 = lib.cb_ba_launch_count()
        with pytest.raises(cb.EngineError, match=msg) as ei:
            cb.BAProblem(rig.cam_flags, rig.cam_const, rig.n_pts, rig.obs_cam, rig.obs_pt, rig.obs_xy, constraints=cn, **kw)
        assert ei.value.code == code, (msg, codes.get(ei.value.code))
        assert lib.cb_ba_launch_count() == n0, msg
    # a symmetric information within 1e-12 relative and a rank-deficient one are accepted; so is a point prior outside
    # every constraint row beside constraints
    ok = I6.copy()
    ok[0, 1] = 1e-13
    tiny_neg = np.diag([1.0, 1.0, -1e-14])
    with cb.BAProblem(rig.cam_flags, rig.cam_const, rig.n_pts, rig.obs_cam, rig.obs_pt, rig.obs_xy, constraints=cons,
                      **cams([1], info=ok[None]), **pts([7], info=tiny_neg[None])) as p:  # fmt: skip
        assert p.solve(r.x0).status in (1, 2, 3, 4)
    # a sharded solve (here the all-reduce callback, on one GPU) is refused
    with EC.problem(rig, **pts([7])) as p:
        called = []
        n0 = lib.cb_ba_launch_count()
        with pytest.raises(cb.EngineError, match="sharded") as ei:
            p.solve(r.x0, allreduce=lambda user, buf, n, stream: called.append(n) or 0)
        assert ei.value.code == -4 and not called
        assert lib.cb_ba_launch_count() == n0
