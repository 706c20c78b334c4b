"""Problems that live side by side.  Problems of the same camera stride, lanes per point and repeated-row flag launch the
same kernel instantiations (DESIGN.md §4, "Where the variants are chosen"), and a kernel's dynamic shared-memory limit
belongs to the kernel, not to a problem: creating a smaller problem must leave a larger one able to launch."""
from __future__ import annotations

import numpy as np
import pytest

from tests import _engine_cases as EC

pytestmark = pytest.mark.gpu

# (larger, smaller).  Fixed intrinsics: the point pass asks for 63.7 KB with 64 cameras and 54.3 KB with 32 (camera table +
# Zt staging).  Free intrinsics: both take the register PCG with 18 columns per lane, 83 KB against 73 KB of shared memory.
PAIRS = {
    "P6-64-then-32": (EC.CASES["64-False"], EC.Case("32-False", 32, 700, 9000)),
    "P9-64-then-48-same-pcg": (EC.CASES["ring64-refine-pcg-cl18-nP576"], EC.Case("48-True", 48, 700, 9000, True)),
}


def _problem(rig):
    import caliscope_b200 as cb

    return cb.BAProblem(rig.cam_flags, rig.cam_const, rig.n_pts, rig.obs_cam, rig.obs_pt, rig.obs_xy)


@pytest.mark.parametrize("pair", list(PAIRS))
def test_creating_a_smaller_problem_leaves_a_larger_one_solvable(pair):
    big, small = (c.make() for c in PAIRS[pair])
    with _problem(EC.oracle_rig(big)) as p:
        alone = p.solve(big.x0, max_nfev=50)
    with _problem(EC.oracle_rig(big)) as p, _problem(EC.oracle_rig(small)) as q:
        sp, sq = EC.stats(p), EC.stats(q)
        print(f"{pair}: P {p.cam_stride} / {q.cam_stride}, stat keys {sp} / {sq}")
        # the two share the point pass, the back-substitution and (free intrinsics) the PCG kernel
        assert p.cam_stride == q.cam_stride
        assert all(sp[k] == sq[k] for k in (EC.LANES, EC.DUPS, EC.CAM_SMEM, EC.SOLVE))
        if p.cam_stride == 9:
            assert sp[EC.SOLVE] == EC.PCG_REG and sp[EC.PCG_CL] == sq[EC.PCG_CL]
        both = p.solve(big.x0, max_nfev=50)
        other = q.solve(small.x0, max_nfev=50)
    assert alone.status > 0 and other.status > 0
    assert np.array_equal(both.x, alone.x) and both.cost == alone.cost and both.nfev == alone.nfev
    assert both.kernel_launches == alone.kernel_launches
