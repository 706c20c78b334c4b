"""The host side of one solve: the start state, the bounds, the upload of x0 and the download of the result, at the
PCG shapes the camera step runs at on large rigs (the slab streamed from L2 above 96 cameras; 64 cameras with free
intrinsics in registers).  Each solve must start from the same device state whatever ran before it on the problem, and
the device loop must return what direct launches return."""
from __future__ import annotations

import numpy as np
import pytest

from tests import _engine_cases as EC

pytestmark = pytest.mark.gpu

CASES = [
    EC.Case("dome128-pcg-l2", 128, 300, 33000, layout="dome", stats={EC.SOLVE: EC.PCG_L2}),
    EC.Case("ring64-refine-pcg-reg-nP576", 64, 700, 9000, True, stats={EC.SOLVE: EC.PCG_REG, EC.PCG_CL: 18}),
]


def _problem(rig, **kw):
    import caliscope_b200 as cb

    return cb.BAProblem(rig.cam_flags, rig.cam_const, rig.n_pts, rig.obs_cam, rig.obs_pt, rig.obs_xy, **kw)


def _same(a, b) -> bool:
    return a.nfev == b.nfev and a.nit == b.nit and a.status == b.status and np.array_equal(a.x, b.x)


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_device_loop_and_direct_launches_agree_and_leave_x0_alone(case):
    rig = case.make()
    x0 = rig.x0.copy()
    with _problem(rig) as p:
        for key, want in case.stats.items():
            assert p.stat(key) == want, (case.id, key)
        loop = p.solve(x0, max_nfev=4)
        direct = p.solve(x0, max_nfev=4, time_kernels=True)
        again = p.solve(x0, max_nfev=4)
    assert loop.used_graph_mode == 2 and direct.used_graph_mode == 0
    assert loop.nfev > 1 and not np.array_equal(loop.x, x0)
    assert _same(loop, direct), "device loop and direct launches differ"
    assert _same(loop, again), "a second solve on the same problem starts from a different state"
    assert np.array_equal(x0, rig.x0), "solve wrote into x0"
    assert not np.shares_memory(loop.x, x0) and not np.shares_memory(loop.x, again.x)


def test_bounds_follow_use_bounds_from_solve_to_solve():
    """Free intrinsics carry bounds (focal scale in [0.5, 2]).  With the fixed focal lengths three times the true ones
    the optimal scale is 1/3, so the bound binds; switching use_bounds on one problem gives what a fresh problem gives."""
    import caliscope_b200 as cb

    rig = CASES[1].make()
    const = rig.cam_const.copy()
    const[:, :2] *= 3.0

    def problem():
        return cb.BAProblem(rig.cam_flags, const, rig.n_pts, rig.obs_cam, rig.obs_pt, rig.obs_xy)

    with problem() as p:
        free = p.solve(rig.x0, use_bounds=False, max_nfev=6)
        bounded = p.solve(rig.x0, use_bounds=True, max_nfev=6)
        free2 = p.solve(rig.x0, use_bounds=False, max_nfev=6)
    with problem() as q:
        bounded_fresh = q.solve(rig.x0, use_bounds=True, max_nfev=6)
    assert not _same(free, bounded), "the bounds did not bind: the test checks nothing"
    assert _same(bounded, bounded_fresh)
    assert _same(free, free2)
