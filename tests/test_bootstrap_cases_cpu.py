"""CPU anchor of the rig-scale bootstrap tests (tests/test_gpu_bootstrap_shapes.py): the OpenCV reference helpers
``oracle.bootstrap.pnp_cv2`` / ``stereo_rmse_cv2`` against the unmodified reference's outputs, and every case's shape
assertions, without a GPU."""
from __future__ import annotations

from pathlib import Path

import numpy as np
import pytest

from oracle import bootstrap as OB
from tests import _bootstrap_cases as BC
from tests.test_bootstrap_host import tables

cv2 = pytest.importorskip("cv2")
GOLD = Path(__file__).parent / "golden"


@pytest.mark.parametrize("name", ["session4", "session11"])
def test_cv2_helpers_match_reference_goldens(name):
    """pnp_cv2 == the reference's PnP poses (1e-6 outside its fallback groups, same groups and order); stereo_rmse_cv2 on
    the reference's aggregated pairs == its stereo RMSE (2e-5 relative, float32), with the same None positions."""
    g = dict(np.load(GOLD / f"bootstrap_{name}.npz"))
    norm = OB.undistort_all(g["cam_ids"], g["cam_k"], g["cam_dist"], g["cam_fisheye"], g["cam_id"], g["img_xy"])
    keys, R, t, rmse, status = OB.pnp_cv2(norm, g["cam_id"], g["sync_index"], g["object_id"], g["obj_xyz"])
    live = status != OB.PNP_TOO_FEW
    assert keys[live].tolist() == g["pnp_keys"].tolist()
    R, t, rmse, status = R[live], t[live], rmse[live], status[live]
    fin = np.isfinite(g["pnp_R"]).all(axis=(1, 2))
    assert np.array_equal(fin, status != OB.PNP_DEGENERATE)
    ok = fin & (status == OB.PNP_OK)
    assert ok.sum() > 0.95 * len(ok)
    assert np.abs(R[ok] - g["pnp_R"][ok]).max() < 1e-6 and np.abs(t[ok] - g["pnp_t"][ok]).max() < 1e-6
    assert np.all(np.abs(rmse[ok] - g["pnp_rmse"][ok]) <= 1e-4 * g["pnp_rmse"][ok] + 1e-8)
    tab = tables(g)
    r2, cnt = OB.stereo_rmse_cv2(g["agg_pairs"], g["agg_R"], g["agg_t"], tab.cam_ids, tab.ignore, norm, g["cam_id"],
                                 g["sync_index"], g["object_id"], g["keypoint_id"])  # fmt: skip
    gold = g["rmse_pair"]
    assert np.array_equal(np.isnan(r2), np.isnan(gold))
    has = ~np.isnan(gold)
    assert np.array_equal(cnt[has], g["rmse_common"][has])
    assert np.all(np.abs(r2[has] - gold[has]) <= 2e-5 * gold[has])


@pytest.mark.parametrize("name", sorted(BC.BUILDERS))
def test_case_reaches_its_shapes(name):
    c = BC.BUILDERS[name]()
    got = BC.reached(c)
    structural = c.reaches - {"iqr_t", "iqr_r"}
    assert structural <= got, f"{name} no longer reaches {sorted(structural - got)}"
    assert len(np.unique(np.stack([c.cam_id, c.sync_index, c.object_id, c.keypoint_id], axis=1), axis=0)) == c.n_obs


def test_outlier_case_reaches_both_iqr_rules():
    """ring64_outliers: with OpenCV's poses, both the translation rule and the rotation rule reject rows of pairs with at
    least 5 samples (the GPU test checks the same with the device's poses)."""
    c = BC.ring64_outliers()
    norm = OB.undistort_all(c.tab.cam_ids, c.tab.k, c.tab.dist, c.tab.fisheye, c.cam_id, c.img_xy)
    keys, R, t, _, status = OB.pnp_cv2(norm, c.cam_id, c.sync_index, c.object_id, c.obj_xyz)
    live = status != OB.PNP_TOO_FEW
    n_t, n_r = BC.iqr_rejections(c, keys[live], R[live], t[live])
    assert n_t > 0 and n_r > 0


def test_planted_degenerate_groups_under_opencv():
    """The planted 40-row groups behave under cv2 as the case claims: IPPE gives up on 39 collinear points plus one (the
    ITERATIVE fallback runs), all-collinear points give a NaN pose, NaN z is solved as z = 0, 3 rows are too few."""
    c = BC.planted()
    norm = OB.undistort_all(c.tab.cam_ids, c.tab.k, c.tab.dist, c.tab.fisheye, c.cam_id, c.img_xy)
    keys, _, _, _, status = OB.pnp_cv2(norm, c.cam_id, c.sync_index, c.object_id, c.obj_xyz)
    st = {int(k[1]): int(s) for k, s in zip(keys, status) if k[0] == 0 and k[1] >= BC.PLANTED_SYNC}
    s0 = BC.PLANTED_SYNC
    assert st == {s0: OB.PNP_OK_FALLBACK, s0 + 1: OB.PNP_DEGENERATE, s0 + 2: OB.PNP_OK, s0 + 3: OB.PNP_TOO_FEW, s0 + 4: OB.PNP_OK}
