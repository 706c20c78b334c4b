"""The dense Schur product loads each pipeline stage with one 2-D tensor box per column tile: SY_KC rows of 100 columns,
the 96 of the tile and 4 that land on the padding of the shared-memory row and are never read.  They are the next tile's
columns, or, past the last tile, out of bounds of Zt and filled with zeros.  Rigs with compacted row lists (sparse
visibility) keep one row copy per lane.  These rigs cover 1, 2, 3, 4, 6 and 7 column tiles (an odd count leaves one
diagonal tile on its own), P = 6 and P = 9, and a row-list rig beside dense ones; the reduced system is checked against
the NumPy oracle, and two evaluations must agree bit for bit."""
from __future__ import annotations

import numpy as np
import pytest

from oracle import lm_schur as LS
from tests import _engine_cases as EC

pytestmark = pytest.mark.gpu

SCHUR_SPARSE = 0  # BAProblem.stat key: 1 when the product runs on compacted row lists

CASES = {
    c.id: c
    for c in [
        # 96 columns: one tile, the box's extra columns all past the end of Zt
        EC.Case("ring16-tiles1", 16, 1500, 12000),
        EC.Case("ring30-tiles2", 30, 1500, 12000),
        # three tiles: one diagonal pair and one diagonal tile on its own
        EC.Case("ring40-tiles3", 40, 1500, 15000),
        EC.Case("ring64-tiles4", 64, 3000, 40000),
        # P = 9: 576 columns over six tiles
        EC.Case("ring64-refine-tiles6", 64, 3000, 40000, True),
        # seven tiles, 600 columns: the last tile's box reaches 72 columns past the end of Zt
        EC.Case("dome100-tiles7", 100, 2000, 60000, layout="dome"),
        # local visibility, fed once from compacted row lists and once from tensor boxes
        EC.Case("ring40-local", 40, 3000, 18000, seed=5, cams_per_point=6),
    ]
}
# CB_SY_SPARSE forces the row lists (1) or the dense tiles (0); unset, the engine picks by visibility
MODES = [(case, None) for case in CASES if case != "ring40-local"] + [("ring40-local", "1"), ("ring40-local", "0")]


def _schur_error(ne, rig, x, lam):
    lin = LS.linearize(x, rig)
    Dc2 = np.einsum("cii->ci", lin.U)
    Dp2 = np.einsum("jii->ji", lin.V)
    S, b, _, _ = LS.schur_system(lin, rig, lam, np.where(Dc2 > 0, Dc2, 1.0), np.where(Dp2 > 0, Dp2, 1.0))
    return np.abs(ne["S"] - S).max() / np.abs(S).max(), np.abs(ne["b"] - b).max() / np.abs(b).max()


@pytest.mark.parametrize("case,rows", MODES)
def test_schur_feed_gives_the_oracle_reduced_system(case, rows, monkeypatch):
    import caliscope_b200 as cb

    if rows is None:
        monkeypatch.delenv("CB_SY_SPARSE", raising=False)
    else:
        monkeypatch.setenv("CB_SY_SPARSE", rows)
    c = CASES[case]
    r = c.make()
    rig = EC.oracle_rig(r)
    lam = 1e-3
    with cb.BAProblem(rig.cam_flags, rig.cam_const, rig.n_pts, rig.obs_cam, rig.obs_pt, rig.obs_xy) as p:
        sparse = int(p.stat(SCHUR_SPARSE))
        assert sparse == (rows == "1"), f"{case}: schur_sparse {sparse}"
        ne = p.normal_equations(r.x0, lam)
        eS, eb = _schur_error(ne, rig, r.x0, lam)
        print(f"{case}: nP {p.n_cams * p.cam_stride}, schur_sparse {sparse}: S {eS:.1e}, b {eb:.1e}")
        assert eS < 1e-12 and eb < 1e-12
        again = p.normal_equations(r.x0, lam)
        assert np.array_equal(again["S"], ne["S"]) and np.array_equal(again["b"], ne["b"])
