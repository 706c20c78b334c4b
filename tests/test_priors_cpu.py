"""The oracle's statement of Gaussian priors (DESIGN.md section 4.13), pinned on the CPU: with zero information it is the
prior-free reference, its mixed loss is scipy's named loss where there are no prior rows, its reduced system gives the
step of the dense augmented normal equations, and ``uncertainty.prior_information`` turns covariances into information
the way the docs say."""
from __future__ import annotations

import numpy as np
import pytest

from caliscope_b200 import _lib as L
from caliscope_b200 import uncertainty
from oracle import ba_oracle as O
from oracle import lm_schur as LS
from tests import _engine_cases as EC
from tests import _held_oracle as HO


def _rig(refine: bool, seed: int = 4):
    from caliscope_b200 import synthetic

    r = synthetic.make_rig(4, 40, 300, seed=seed, refine_intrinsics=refine)
    return r, EC.oracle_rig(r)


def _spd(rng, n, scale=1.0):
    A = rng.standard_normal((n, n))
    return scale * (A @ A.T + n * np.eye(n))


def _priors(rig, x, rng, zero=False, scale=1e6):
    """Full priors on cameras 0 and 2 and every fifth point, means the start values plus noise."""
    pr = HO.Priors()
    cams = [0, 2]
    pr.cams = np.array(cams)
    pr.cam_mean = np.zeros((2, 9))
    pr.cam_info = np.zeros((2, 9, 9))
    for k, c in enumerate(cams):
        o, w = rig.cam_offsets[c], rig.cam_offsets[c + 1] - rig.cam_offsets[c]
        pr.cam_mean[k, :w] = x[o : o + w] + 1e-3 * rng.standard_normal(w)
        pr.cam_info[k, :w, :w] = 0.0 if zero else _spd(rng, w, scale)
    pr.pts = np.arange(0, rig.n_pts, 5)
    ncp = rig.n_camera_params
    pr.pt_mean = x[ncp:].reshape(-1, 3)[pr.pts] + 1e-3 * rng.standard_normal((len(pr.pts), 3))
    pr.pt_info = np.stack([np.zeros((3, 3)) if zero else _spd(rng, 3, scale) for _ in pr.pts])
    return pr


@pytest.mark.parametrize("refine,loss", [(False, "linear"), (True, "soft_l1"), (False, "cauchy")])
def test_zero_information_is_the_prior_free_reference(refine, loss):
    r, rig = _rig(refine)
    pr = _priors(rig, r.x0, np.random.default_rng(1), zero=True)
    fs = 2e-3  # a scale at which the robust solves converge in a few steps instead of crawling
    ref = O.solve_scipy(rig, r.x0, loss=loss, f_scale=fs)
    got = HO.solve_scipy(rig, r.x0, priors=pr, loss=loss, f_scale=fs)
    print(f"P{'9' if refine else '6'} {loss}: prior-oracle nfev {got.nfev} cost {got.cost:.15e} | scipy nfev {ref.nfev} "
          f"cost {ref.cost:.15e}")  # fmt: skip
    # a robust loss goes through scipy's callable-loss path in the one and its named path in the other: the same rho in
    # different rounding, which moves the last steps of a slow solve (nfev) and, along the gauge's null space, x -- not
    # the cost it ends at beyond a hundred times ftol = 1e-8
    tol = 1e-12 if loss == "linear" else 1e-6
    if loss == "linear":
        assert got.nfev == ref.nfev and got.status == ref.status
        assert np.abs(got.x - ref.x).max() <= 1e-9 * np.abs(ref.x).max()
    assert abs(got.cost - ref.cost) <= tol * ref.cost
    # and with a fixed set: the free-subvector reference
    free = np.ones(rig.n_params, bool)
    free[rig.cam_offsets[1] : rig.cam_offsets[2]] = False
    free[rig.n_camera_params : rig.n_camera_params + 6] = False
    ref = HO.solve_scipy(rig, r.x0, free, loss=loss, f_scale=fs)
    got = HO.solve_scipy(rig, r.x0, free, pr, loss=loss, f_scale=fs)
    if loss == "linear":
        assert got.nfev == ref.nfev
        # scipy's iterative (lsmr) trust-region solve rounds x further than the cost
        assert np.abs(got.x - ref.x).max() <= 1e-6 * np.abs(ref.x).max()
    assert abs(got.cost - ref.cost) <= tol * ref.cost
    assert np.array_equal(got.x[~free], r.x0[~free])


@pytest.mark.parametrize("loss", list(L.LOSS_IDS))
def test_mixed_loss_is_the_named_loss_without_prior_rows(loss):
    from scipy.optimize._lsq.least_squares import construct_loss_function

    rng = np.random.default_rng(2)
    f = rng.standard_normal(50) * 3.0
    fs = 0.7
    named = construct_loss_function(len(f), loss, fs)
    mixed = construct_loss_function(len(f), HO.mixed_loss(len(f), loss, fs), fs)
    want = named(f) if named is not None else np.stack([f * f, np.ones_like(f), np.zeros_like(f)])
    assert np.allclose(mixed(f), want, rtol=1e-14, atol=0.0)
    # prior rows after them are linear whatever the loss: rho = f^2, rho' = 1, rho'' = 0 after scipy's scaling
    g = np.concatenate([f, rng.standard_normal(7)])
    got = construct_loss_function(len(g), HO.mixed_loss(len(f), loss, fs), fs)(g)
    assert np.allclose(got[:, : len(f)], want, rtol=1e-14, atol=0.0)
    assert np.allclose(got[0, len(f) :], g[len(f) :] ** 2, rtol=1e-14) and np.all(got[1, len(f) :] == 1.0)
    assert np.all(got[2, len(f) :] == 0.0)
    # and the whole solve without priors is oracle.ba_oracle.solve_scipy's
    r, rig = _rig(False, seed=6)
    ref = O.solve_scipy(rig, r.x0, loss=loss, f_scale=2e-4)
    got = HO.solve_scipy(rig, r.x0, priors=HO.Priors(), loss=loss, f_scale=2e-4)
    assert abs(got.cost - ref.cost) <= 1e-9 * ref.cost


@pytest.mark.parametrize("refine,fixed", [(False, False), (True, False), (True, True)])
def test_prior_reduced_system_gives_the_dense_augmented_step(refine, fixed):
    """The Schur reduction of the prior linearisation solves the dense damped normal equations of the augmented J."""
    r, rig = _rig(refine)
    rng = np.random.default_rng(3)
    pr = _priors(rig, r.x0, rng, scale=1e4)
    P = LS.cam_stride(rig)
    free = np.ones(rig.n_params, bool)
    if fixed:
        free[rig.cam_offsets[2] + 6 : rig.cam_offsets[2] + 9] = False  # s, k1, k2 of a camera with a prior
        free[rig.n_camera_params + 3 : rig.n_camera_params + 6] = False  # point 1 (no prior)
    lam = 1e-3
    lin = HO.linearize(r.x0, rig, free, pr)
    Dc2, Dp2 = HO.scaling(r.x0, rig, pr)
    fcs, fps = HO.free_slots(free, rig, P)
    active = np.zeros(rig.n_cams * P, bool)
    for k in range(rig.n_cams):
        active[k * P : k * P + rig.cam_offsets[k + 1] - rig.cam_offsets[k]] = True
    S, b, Einv, Wd = HO.schur_system(lin, rig, lam, Dc2, Dp2, active & ~fcs, ~fps)
    sl = np.nonzero(active)[0]
    dc = np.zeros(rig.n_cams * P)
    dc[sl] = np.linalg.solve(S[np.ix_(sl, sl)], -b[sl])
    dp = -np.einsum("jab,jb->ja", Einv, lin.gp + np.einsum("jcpa,cp->ja", Wd, dc.reshape(rig.n_cams, P)))
    # dense: H = J^T J + info over the free parameters, damped by lam * D (D from the unmasked blocks)
    J = O.jacobian(r.x0, rig).toarray()
    H = J.T @ J + HO.info_matrix(rig, pr)
    g = J.T @ O.residuals(r.x0, rig) + HO.info_matrix(rig, pr) @ (r.x0 - _mean_vector(rig, pr, r.x0))
    D = np.concatenate([LS.join_x(Dc2, np.zeros((rig.n_pts, 3)), rig)[: rig.n_camera_params], Dp2.ravel()])
    fi = np.nonzero(free)[0]
    d = np.zeros(rig.n_params)
    d[fi] = np.linalg.solve((H + lam * np.diag(D))[np.ix_(fi, fi)], -g[fi])
    got = LS.join_x(dc.reshape(rig.n_cams, P), dp, rig)
    assert np.abs(got - d).max() <= 1e-8 * np.abs(d).max()
    assert np.all(got[~free] == 0.0)
    assert abs(lin.cost - (0.5 * O.residuals(r.x0, rig) @ O.residuals(r.x0, rig) + HO.prior_cost(r.x0, rig, pr))) < 1e-12


def _mean_vector(rig, pr, x):
    m = np.array(x, dtype=np.float64)
    for c, mu, _ in HO.blocks(rig, pr):
        m[c] = mu
    return m


def test_dense_covariance_is_the_inverse_of_the_augmented_normal_matrix():
    """Priors on every camera pose and point fix the gauge: (J^T J + info)^-1 over everything, s2 from the augmented
    cost and m = 2 n_obs + sum rank(info)."""
    r, rig = _rig(False)
    rng = np.random.default_rng(5)
    pr = _priors(rig, r.x0, rng, scale=1e2)
    pr.cams = np.arange(rig.n_cams)
    pr.cam_mean = np.concatenate([r.x0[: rig.n_camera_params].reshape(-1, 6), np.zeros((rig.n_cams, 3))], axis=1)
    pr.cam_info = np.zeros((rig.n_cams, 9, 9))
    pr.cam_info[:, :6, :6] = _spd(rng, 6, 1e2)
    cov = HO.dense_covariance(r.x0, rig, priors=pr)
    J = O.jacobian(r.x0, rig).toarray()
    H = J.T @ J + HO.info_matrix(rig, pr)
    f = O.residuals(r.x0, rig)
    cost = 0.5 * f @ f + HO.prior_cost(r.x0, rig, pr)
    m = 2 * rig.n_obs + 6 * rig.n_cams + 3 * len(pr.pts)
    assert cov["dof"] == m - rig.n_params
    s2 = 2 * cost / cov["dof"]
    Sig = s2 * np.linalg.inv(H)
    ncp = rig.n_camera_params
    assert np.allclose(cov["cameras"], Sig[:ncp, :ncp], rtol=1e-8, atol=1e-12 * np.abs(Sig).max())
    j = 7
    assert np.allclose(cov["points"][j], Sig[ncp + 3 * j : ncp + 3 * j + 3, ncp + 3 * j : ncp + 3 * j + 3], rtol=1e-8)


# ---------------------------------------------------------------------------------------------
# uncertainty.prior_information
# ---------------------------------------------------------------------------------------------
def test_prior_information_inverts_and_scales():
    rng = np.random.default_rng(7)
    A = rng.standard_normal((6, 6))
    cov = A @ A.T + 6 * np.eye(6)
    info = uncertainty.prior_information(cov, 0.5, 800.0)
    assert np.allclose(info, (0.5 / 800.0) ** 2 * np.linalg.inv(cov), rtol=1e-12)
    assert np.array_equal(info, info.T)


def test_prior_information_infinite_variance_is_unconstrained():
    rng = np.random.default_rng(8)
    A = rng.standard_normal((3, 3))
    sub = A @ A.T + 3 * np.eye(3)
    cov = np.full((9, 9), 0.0)
    cov[:6, :6] = np.diag(np.full(6, np.inf))
    cov[6:, 6:] = sub
    cov[0, 7] = cov[7, 0] = 5.0  # an entry in an unconstrained row is ignored
    info = uncertainty.prior_information(cov, 1.0, 2.0)
    assert np.all(info[:6, :] == 0.0) and np.all(info[:, :6] == 0.0)
    assert np.allclose(info[6:, 6:], 0.25 * np.linalg.inv(sub), rtol=1e-12)
    assert np.all(uncertainty.prior_information(np.diag([np.inf, np.inf]), 1.0, 1.0) == 0.0)


@pytest.mark.parametrize("bad,msg", [
    (np.diag([1.0, 0.0, 2.0]), "zero variance"),
    (np.array([[1.0, 1.0], [1.0, 1.0]]), "singular"),
    (np.array([[2.0, 0.5], [0.4, 2.0]]), "not symmetric"),
    (np.array([[1.0, 2.0], [2.0, 1.0]]), "singular"),  # indefinite
    (np.diag([1.0, -1.0]), "negative"),
    (np.ones((2, 3)), "square"),
])  # fmt: skip
def test_prior_information_refuses(bad, msg):
    with pytest.raises(ValueError, match=msg):
        uncertainty.prior_information(bad, 1.0, 1.0)
