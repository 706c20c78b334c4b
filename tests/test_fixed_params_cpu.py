"""The oracle's statement of fixed parameters (DESIGN.md section 4.12), pinned on the CPU: the masked dense LM iteration
reaches the cost of scipy's least_squares on the free subvector, the masked reduced system gives the step of the dense
normal equations over the free parameters, and the masked dense covariance is that of J with the fixed columns deleted."""
from __future__ import annotations

import numpy as np
import pytest

from oracle import ba_oracle as O
from oracle import lm_schur as LS
from tests import _engine_cases as EC
from tests import _held_oracle as HO


def _rig(refine: bool, seed: int = 4):
    from caliscope_b200 import synthetic

    r = synthetic.make_rig(4, 40, 300, seed=seed, refine_intrinsics=refine)
    return r, EC.oracle_rig(r)


def _free(rig, cams=(), cam_slots=(), points=()):
    """Boolean over x: False for every parameter of the cameras in ``cams``, for the x indices ``cam_slots`` and for the
    coordinates of ``points``."""
    free = np.ones(rig.n_params, bool)
    for c in cams:
        free[rig.cam_offsets[c] : rig.cam_offsets[c + 1]] = False
    free[list(cam_slots)] = False
    for j in points:
        free[rig.n_camera_params + 3 * j : rig.n_camera_params + 3 * j + 3] = False
    return free


def _fixed_sets(rig, kind):
    if kind == "camera+points":
        return dict(cams=(1,), points=range(0, rig.n_pts, 10))
    if kind == "intrinsic-slots":  # s, k1, k2 of cameras 0 and 2 (9-parameter blocks)
        return dict(cam_slots=[rig.cam_offsets[c] + a for c in (0, 2) for a in (6, 7, 8)])
    return dict(cam_slots=[rig.cam_offsets[3] + 7], points=(3, 17))  # one k1 and two points


@pytest.mark.parametrize("refine,loss,kind", [
    (False, "linear", "camera+points"),
    (False, "soft_l1", "camera+points"),
    (True, "linear", "intrinsic-slots"),
    (True, "soft_l1", "intrinsic-slots"),
    (True, "linear", "camera+points"),
    (True, "soft_l1", "single-slot+points"),
])  # fmt: skip
def test_masked_dense_lm_reaches_free_subvector_scipy(refine, loss, kind):
    r, rig = _rig(refine)
    free = _free(rig, **_fixed_sets(rig, kind))
    fs = 2e-4
    ref = HO.solve_scipy(rig, r.x0, free, loss=loss, f_scale=fs)
    got = HO.lm_solve_dense(rig, r.x0, free, loss=loss, f_scale=fs)
    print(f"{kind} P{'9' if refine else '6'} {loss}: dense status {got['status']} nfev {got['nfev']} cost "
          f"{got['cost']:.12e} | scipy status {ref.status} nfev {ref.nfev} cost {ref.cost:.12e}")  # fmt: skip
    assert np.array_equal(got["x"][~free], r.x0[~free]) and np.array_equal(ref.x[~free], r.x0[~free])
    assert got["status"] in (1, 2, 3, 4)
    assert got["cost"] <= ref.cost * (1 + 1e-8)
    if loss == "linear":  # under a robust loss the RMSE is not what either minimises
        # with free intrinsics scipy's own default-vs-tight runs differ by a few 1e-6 px (SURVEY 7.1)
        tol = 1e-5 if refine else 1e-6
        assert abs(O.overall_rmse_px(got["x"], rig) - O.overall_rmse_px(ref.x, rig)) < tol
    if refine:  # bounds hold on the free intrinsics
        lo, hi = rig.bounds()
        assert np.all(got["x"] >= lo) and np.all(got["x"] <= hi)


def test_dense_lm_with_every_parameter_free_is_the_oracles():
    r, rig = _rig(False)
    a = LS.lm_solve_dense(rig, r.x0)
    b = HO.lm_solve_dense(rig, r.x0, np.ones(rig.n_params, bool))
    assert np.array_equal(a["x"], b["x"]) and a["cost"] == b["cost"] and a["nfev"] == b["nfev"]


@pytest.mark.parametrize("refine", [False, True])
def test_masked_reduced_system_gives_the_free_subvector_step(refine):
    """Unit rows and columns of S for fixed camera slots, Einv = 0 for fixed points: the camera and point steps of the
    dense damped normal equations restricted to the free parameters, and zero for the fixed ones."""
    r, rig = _rig(refine)
    sets = _fixed_sets(rig, "intrinsic-slots" if refine else "camera+points")
    if refine:
        sets["points"] = (5, 6, 30)
    free = _free(rig, **sets)
    lam, P = 1e-3, LS.cam_stride(rig)
    lin = LS.linearize(r.x0, rig)
    Dc2 = np.where(np.einsum("cii->ci", lin.U) > 0, np.einsum("cii->ci", lin.U), 1.0)
    Dp2 = np.where(np.einsum("jii->ji", lin.V) > 0, np.einsum("jii->ji", lin.V), 1.0)
    fc, fp = HO.free_slots(free, rig, P)
    active = np.zeros(rig.n_cams * P, bool)
    for c in range(rig.n_cams):
        active[c * P : c * P + rig.cam_offsets[c + 1] - rig.cam_offsets[c]] = True
    S, b, Einv, Wd = HO.schur_system(lin, rig, lam, Dc2, Dp2, fixed_slots=active & ~fc, fixed_pts=~fp)
    dc = np.linalg.solve(S, -b).reshape(rig.n_cams, P)
    dp = -np.einsum("jab,jb->ja", Einv, lin.gp + np.einsum("jcpa,cp->ja", Wd, dc))
    # the same step from the full dense system over the free parameters
    f = O.residuals(r.x0, rig)
    J = O.jacobian(r.x0, rig).toarray()
    H, g = J.T @ J, J.T @ f
    D = np.diag(H).copy()
    D[D <= 0] = 1.0
    fi = np.nonzero(free)[0]
    d = np.zeros(rig.n_params)
    d[fi] = np.linalg.solve((H + lam * np.diag(D))[np.ix_(fi, fi)], -g[fi])
    ncp = rig.n_camera_params
    dc_x = LS.join_x(dc, np.zeros((rig.n_pts, 3)), rig)[:ncp]
    assert np.abs(dc_x - d[:ncp]).max() <= 1e-9 * np.abs(d[:ncp]).max()
    assert np.abs(dp.ravel() - d[ncp:]).max() <= 1e-9 * np.abs(d[ncp:]).max()
    assert np.all(dc.ravel()[active & ~fc] == 0.0) and np.all(dp[~fp] == 0.0)
    # linearize's own mask: the Jacobian of the free parameters, fixed columns zero
    lin_f = HO.linearize(r.x0, rig, free)
    assert np.all(lin_f.gc.ravel()[active & ~fc] == 0.0) and np.all(lin_f.V[~fp] == 0.0)


def test_masked_dense_covariance_is_that_of_the_free_columns():
    """Four surveyed points and one whole camera fixed: no gauge is left, and the covariance is s2 (J_F^T J_F)^-1 over the
    remaining columns; fixed points get zero blocks, rank -2, and 3 fewer parameters each in dof."""
    from caliscope_b200 import synthetic

    r = synthetic.make_rig(5, 60, 280, seed=9)
    rig = EC.oracle_rig(r)
    x = O.solve_scipy(rig, r.x0).x
    fixed_pts = np.array([2, 11, 23, 40])
    fixed = np.arange(6, 12)  # camera 1
    ref = HO.dense_covariance(x, rig, fixed, fixed_pts)
    free = _free(rig, cams=(1,), points=fixed_pts)
    J = O.jacobian(x, rig).toarray()[:, free]
    assert np.linalg.matrix_rank(J) == J.shape[1]  # every point is seen twice or more: nothing to deflate
    dof = J.shape[0] - J.shape[1]
    s2 = 2.0 * O.robust_cost(O.residuals(x, rig), "linear", 1.0) / dof
    Sig = np.zeros((rig.n_params, rig.n_params))
    Sig[np.ix_(free, free)] = s2 * np.linalg.inv(J.T @ J)
    ncp = rig.n_camera_params
    assert ref["dof"] == dof
    assert np.abs(ref["cameras"] - Sig[:ncp, :ncp]).max() <= 1e-9 * np.abs(Sig[:ncp, :ncp]).max()
    pts = np.stack([Sig[ncp + 3 * j : ncp + 3 * j + 3, ncp + 3 * j : ncp + 3 * j + 3] for j in range(rig.n_pts)])
    assert np.abs(ref["points"] - pts).max() <= 1e-9 * np.abs(pts).max()
    assert np.all(ref["point_rank"][fixed_pts] == -2) and np.all(ref["points"][fixed_pts] == 0.0)
