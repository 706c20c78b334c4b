"""The point pass writes the Schur factor Zt as whole 64-byte granules from pieces staged in shared memory.  These rigs put
the edges of that path in play: a last granule of a row that is only partly inside n_cams * P columns, 72-byte pieces
(P = 9) that straddle granules, several 96-column tiles, 32 lanes per point, a rigid-distance constraint rig
(untransformed W rows) and the covariance pass.  Rigs with repeated (camera, point) rows take the run-summed variants,
which store their pieces as they are; two of them stay here so that both store paths write the same factor under the
same checks (tests/test_gpu_engine_paths.py covers points whose rows are not in camera-slot order, which also store their
pieces as they are).  Every granule carries zeros
for the cameras a point does not see; a wrong value there, or a structural zero of Zt left non-zero, enters
S = U - Z Z^T directly, so the reduced system is checked against the NumPy oracle, and checked again at the same point
after a solve has run its passes over the same factor (at the solution itself b is close to zero and its relative
error says nothing)."""
from __future__ import annotations

import numpy as np
import pytest

from oracle import covariance as OC
from oracle import lm_schur as LS
from tests import _constraint_cases as CCS
from tests import _engine_cases as EC

pytestmark = pytest.mark.gpu

CASES = {
    c.id: c
    for c in [
        # 42 columns: the last granule of a row holds 2 of 8
        EC.Case("ring7-nP42", 7, 400, 2400, stats={EC.LANES: 8, EC.DUPS: 0}),
        # 117 columns, two column tiles, 72-byte pieces at 8-byte alignment
        EC.Case("ring13-refine-nP117", 13, 700, 6000, True, stats={EC.LANES: 8, EC.DUPS: 0}),
        # 138 columns over two tiles, with local visibility (few cameras per point, granules at both ends of a run)
        EC.Case("ring23-local-nP138", 23, 900, 5400, cams_per_point=6, stats={EC.LANES: 8, EC.DUPS: 0}),
        # 32 lanes per point over eight tiles (staged path)
        EC.CASES["dome128-lanes32"],
        # repeated rows (run-summed variants, pieces stored as they are): 8 lanes at 90 columns, 32 lanes at 117
        EC.CASES["ring10-refine-direct-nP90"],
        EC.Case("static-ring13-refine-lanes32-dups", 13, 100, 13000, True, stats={EC.LANES: 32, EC.DUPS: 1}),
    ]
}


def _problem(rig):
    import caliscope_b200 as cb

    cons = CCS.constraints_of(rig) if rig.n_constraints else None
    return cb.BAProblem(rig.cam_flags, rig.cam_const, rig.n_pts, rig.obs_cam, rig.obs_pt, rig.obs_xy, constraints=cons)


def _check_schur(ne, rig, x, lam, tag):
    lin = LS.linearize(x, rig)
    Dc2 = np.einsum("cii->ci", lin.U)
    Dp2 = np.einsum("jii->ji", lin.V)
    S, b, _, _ = LS.schur_system(lin, rig, lam, np.where(Dc2 > 0, Dc2, 1.0), np.where(Dp2 > 0, Dp2, 1.0))
    eS = np.abs(ne["S"] - S).max() / np.abs(S).max()
    eb = np.abs(ne["b"] - b).max() / np.abs(b).max()
    print(f"{tag}: S {eS:.1e}, b {eb:.1e}")
    assert eS < 1e-12 and eb < 1e-12


@pytest.mark.parametrize("case", list(CASES))
def test_zt_granules_give_the_oracle_schur_system_before_and_after_a_solve(case):
    c = CASES[case]
    r = c.make()
    rig = EC.oracle_rig(r)
    lam = 1e-3
    with _problem(rig) as p:
        EC.check_stats(p, c)
        _check_schur(p.normal_equations(r.x0, lam), rig, r.x0, lam, f"{case} at x0")
        res = p.solve(r.x0)
        assert res.status in (1, 2, 3, 4)
        _check_schur(p.normal_equations(r.x0, lam), rig, r.x0, lam, f"{case} at x0 after the solve")


def test_zt_granules_with_rigid_distance_constraints():
    """Points in a constraint component write W = Jc^T Jp, not Z, through the same staged stores."""
    from tests.test_gpu_constraints import _check_normal_equations

    name = next(iter(CCS.CASES))
    r, rig, _ = CCS.CASES[name].make()
    lam = 1e-3
    with _problem(rig) as p:
        mode = int(p.stat(EC.SOLVE))
        _check_normal_equations(p.normal_equations(r.x0, lam), rig, r.x0, lam, mode, name)
        res = p.solve(r.x0)
        assert res.status in (1, 2, 3, 4)
        _check_normal_equations(p.normal_equations(r.x0, lam), rig, r.x0, lam, mode, f"{name} at x0 after the solve")


@pytest.mark.parametrize("case", ["ring13-refine-nP117", "static-ring13-refine-lanes32-dups"])
def test_zt_granules_in_the_covariance_pass(case):
    """The covariance pass writes Z = W R^T through the same stores."""
    r = CASES[case].make()
    rig = EC.oracle_rig(r)
    with _problem(rig) as p:
        cov = p.covariance(r.x0)
    ref = OC.schur_covariance(r.x0, rig, cov.fixed)
    from tests.test_gpu_covariance import _check

    _check(cov, ref, 1e-8, case)
