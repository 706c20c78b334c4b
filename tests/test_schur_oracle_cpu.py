"""oracle.lm_schur.component_schur, the reduced system with rigid-distance rows that the GPU constraint tests compare the
engine with, pinned on the CPU: without constraints it is schur_system, and with them its step is the dense solve of the
full damped normal equations."""
from __future__ import annotations

import numpy as np
import pytest

from oracle import ba_oracle as O
from oracle import lm_schur as LS
from tests import _constraint_cases as CCS
from tests import _engine_cases as EC
from tests._util import load_golden


@pytest.mark.parametrize("refine,loss", [(False, "linear"), (True, "soft_l1")])
def test_component_schur_without_constraints_is_schur_system(refine, loss):
    from caliscope_b200 import synthetic

    r = synthetic.make_rig(7, 300, 2000, seed=3, refine_intrinsics=refine)
    rig = EC.oracle_rig(r)
    lam, fs = 1e-3, 5e-4
    cs = LS.component_schur(r.x0, rig, lam, loss, fs)
    lin = LS.linearize(r.x0, rig, loss, fs)
    Dc2 = np.einsum("cii->ci", lin.U)
    Dp2 = np.einsum("jii->ji", lin.V)
    S, b, Einv, Wd = LS.schur_system(lin, rig, lam, np.where(Dc2 > 0, Dc2, 1.0), np.where(Dp2 > 0, Dp2, 1.0))
    assert abs(cs.cost - lin.cost) <= 1e-14 * lin.cost
    assert np.abs(cs.S - S).max() <= 1e-12 * np.abs(S).max()
    assert np.abs(cs.b - b).max() <= 1e-12 * np.abs(b).max()
    dp = -np.einsum("jab,jb->ja", Einv, lin.gp + np.einsum("jcpa,cp->ja", Wd, cs.dc))
    assert np.abs(cs.backsub(cs.dc) - dp).max() <= 1e-12 * np.abs(dp).max()


@pytest.mark.parametrize("name,loss,lam", [
    ("small_pinhole_constraints.npz", "linear", 1e-3),
    ("aruco_constraints_refine0.npz", "linear", 1e-4),
    ("aruco_constraints_refine1.npz", "soft_l1", 1e-2),
    ("board_truss_constraints_refine0.npz", "linear", 1e-3),
])  # fmt: skip
def test_component_schur_step_equals_dense_normal_equations(name, loss, lam):
    """The same dense solve as test_damped_step_with_constraints_equals_dense_normal_equations."""
    g, rig = load_golden(name)
    fs, x0 = 5e-4, g["x0"]
    cs = LS.component_schur(x0, rig, lam, loss, fs)
    f = O.residuals(x0, rig)
    J = O.jacobian(x0, rig).toarray()
    js, fsc = O.robust_row_scales(f, loss, fs)
    Js = J * js[:, None]
    H, grad = Js.T @ Js, Js.T @ fsc
    D = np.diag(H).copy()
    D[D <= 0] = 1.0
    d = np.linalg.solve(H + lam * np.diag(D), -grad)
    ncp = rig.n_camera_params
    assert abs(cs.cost - O.robust_cost(f, loss, fs)) <= 1e-14 * cs.cost
    dc = cs.dc.reshape(-1)[cs.slot]
    assert np.abs(dc - d[:ncp]).max() <= 1e-10 * np.abs(d[:ncp]).max()
    dp = cs.backsub(cs.dc).ravel()
    assert np.abs(dp - d[ncp:]).max() <= 1e-10 * np.abs(d[ncp:]).max()


def test_constrained_rig_helper_builds_the_requested_components():
    """tie / pick_components: reference-format rows, one component per requested point set, exact distances at the truth,
    and the degenerate points (unobserved, single-view) inside components."""
    c = CCS.CASES["ring40-sparse-spread"]
    r, rig, comps = c.make()
    assert rig.groups_a.shape == rig.groups_b.shape == (rig.n_constraints, 4)
    got = LS.constraint_components(rig)
    assert sorted(map(tuple, (np.sort(k) for k in comps))) == sorted(map(tuple, got))
    assert np.abs(O.constraint_residuals(r.x_true, rig)).max() < 1e-12
    assert np.all(rig.weights == CCS.WEIGHT)
    p2p = (rig.groups_a == rig.groups_a[:, :1]).all(axis=1)
    assert p2p.any() and (~p2p).any()
    assert all(len(np.unique(a)) == 4 for a in rig.groups_a[~p2p])
    n_obs = np.bincount(rig.obs_pt, minlength=rig.n_pts)
    assert n_obs[comps[0][0]] == 0 and n_obs[comps[-1][-1]] == 1
    # the components reach more than one 96-column tile in the caller's camera order
    tiles = [np.unique(rig.obs_cam[np.isin(rig.obs_pt, k)] * 6 // 96) for k in comps]
    assert all(len(t) > 1 for t in tiles)
