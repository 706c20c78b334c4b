"""Fixed camera parameters and fixed points in the engine (DESIGN.md section 4.12): a solve is scipy's least_squares on
the free subvector, the fixed entries of x come back bit for bit, and the refused inputs are refused before any device
work.  Every shape-selected variant is tested with the priors, in test_gpu_priors.py."""
from __future__ import annotations

import numpy as np
import pytest

from oracle import ba_oracle as O
from tests import _engine_cases as EC
from tests import _held_oracle as HO

pytestmark = pytest.mark.gpu


def _whole_camera(rig, c):
    return list(range(rig.cam_offsets[c], rig.cam_offsets[c + 1]))


def _intrinsics_of(rig, cams):
    return [int(rig.cam_offsets[c]) + a for c in cams for a in (6, 7, 8)]


def _known(x0, x_true, free):
    """The start vector with the fixed entries at their true values, as a caller's known values are.  Held at a noisy
    start instead, a fixed camera or point contradicts the observations, and the solve crawls along a flat valley where
    the termination tests (scipy's as much as the engine's) stop at points that differ by 1e-5 in cost."""
    x = np.array(x0, dtype=np.float64)
    x[~free] = x_true[~free]
    return x


# ---------------------------------------------------------------------------------------------
# 1. against live SciPy on the free subvector
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_cams,n_pts,n_obs", [(8, 300, 3000), (16, 500, 6000)])
@pytest.mark.parametrize("fixed", ["camera+points", "intrinsics"])
@pytest.mark.parametrize("loss", ["linear", "soft_l1"])
def test_solve_matches_scipy_on_the_free_subvector(n_cams, n_pts, n_obs, fixed, loss):
    """Free intrinsics.  One whole camera and every tenth point fixed, or s, k1, k2 of every other camera.  The bar is
    test_gpu_parity.py's for free intrinsics unfixed: cost at or below scipy's; the RMSE (linear) or the cost (soft_l1)
    within scipy's own default-vs-tight termination noise."""
    from caliscope_b200 import synthetic

    r = synthetic.make_rig(n_cams, n_pts, n_obs, seed=n_cams + 100, refine_intrinsics=True)
    rig = EC.oracle_rig(r)
    if fixed == "camera+points":
        fc, fp = _whole_camera(rig, 1), list(range(0, n_pts, 10))
    else:
        fc, fp = _intrinsics_of(rig, range(0, n_cams, 2)), []
    free = EC.free_mask(rig, fc, fp)
    x0 = _known(r.x0, r.x_true, free)
    fs = 2.0 / synthetic.WEBCAM_F
    ref = HO.solve_scipy(rig, x0, free, loss=loss, f_scale=fs)
    # tolerances 1e-15 never trigger here: 200 evaluations stand for "run to convergence"
    tight = HO.solve_scipy(rig, x0, free, loss=loss, f_scale=fs, ftol=1e-15, xtol=1e-15, gtol=1e-15, max_nfev=200)
    with EC.problem(rig, fixed_cam_params=fc, fixed_points=fp) as p:
        res = p.solve(x0, loss=loss, f_scale=fs)
        rm = p.overall_rmse_px(res.x)
    rm_ref, rm_tight = O.overall_rmse_px(ref.x, rig), O.overall_rmse_px(tight.x, rig)
    print(f"{n_cams} cams {fixed} {loss}: gpu status {res.status} nfev {res.nfev} cost {res.cost:.15e} rmse {rm:.10f} | "
          f"scipy nfev {ref.nfev} cost {ref.cost:.15e} rmse {rm_ref:.10f} | tight cost {tight.cost:.15e} "
          f"rmse {rm_tight:.10f}")  # fmt: skip
    assert res.status in (1, 2, 3, 4)
    assert np.array_equal(res.x[~free], x0[~free])
    assert res.cost <= ref.cost * (1 + 1e-8)
    if loss == "linear":
        assert abs(rm - rm_ref) < 3 * abs(rm_ref - rm_tight) + 1e-6
    else:
        assert abs(res.cost - tight.cost) < 1e-6 * tight.cost


# ---------------------------------------------------------------------------------------------
# 2. fixed s, k1, k2 at their locked values == the same camera without free intrinsics
# ---------------------------------------------------------------------------------------------
def test_fixed_intrinsics_equal_a_camera_without_free_intrinsics():
    from caliscope_b200 import synthetic

    r = synthetic.make_rig(12, 600, 7000, seed=12, refine_intrinsics=True)
    free_cams = np.arange(r.n_cams) % 3 != 0
    flags = free_cams.astype(np.int32)
    blocks = r.x0[: 9 * r.n_cams].reshape(r.n_cams, 9)
    pts = r.x0[9 * r.n_cams :]
    k = 4  # a free-intrinsics camera
    a_flags = flags.copy()
    b_flags = flags.copy()
    b_flags[k] = 0
    a_blocks = [blocks[c] if free_cams[c] else blocks[c, :6] for c in range(r.n_cams)]
    a_blocks[k] = np.concatenate([blocks[k, :6], [1.0, r.cam_const[k, 4], r.cam_const[k, 5]]])
    b_blocks = [blocks[c] if b_flags[c] else blocks[c, :6] for c in range(r.n_cams)]
    xa = np.concatenate(a_blocks + [pts])
    xb = np.concatenate(b_blocks + [pts])
    rig_a = O.Rig(a_flags, r.cam_const, r.n_pts, r.obs_cam, r.obs_pt, r.obs_xy)
    rig_b = O.Rig(b_flags, r.cam_const, r.n_pts, r.obs_cam, r.obs_pt, r.obs_xy)
    fc = _intrinsics_of(rig_a, [k])
    with EC.problem(rig_a, fixed_cam_params=fc) as p:
        assert p.cam_stride == 9
        ra = p.solve(xa)
    with EC.problem(rig_b) as p:
        rb = p.solve(xb)
    keep = np.ones(len(xa), bool)
    keep[fc] = False
    err = np.abs(ra.x[keep] - rb.x).max()
    print(f"fixed s, k1, k2 vs locked camera: status {ra.status} / {rb.status}, nfev {ra.nfev} / {rb.nfev}, max |dx| {err:.2e}")
    assert ra.status == rb.status and ra.nfev == rb.nfev
    assert err <= 1e-12
    assert np.array_equal(ra.x[fc], xa[fc])


# ---------------------------------------------------------------------------------------------
# 3. surveyed points: scale and frame from the solve, and a covariance without a gauge argument
# ---------------------------------------------------------------------------------------------
def _centres(x, rig):
    out = []
    for c in range(rig.n_cams):
        o = rig.cam_offsets[c]
        out.append(-O.rodrigues(x[o : o + 3])[0].T @ x[o + 3 : o + 6])
    return np.array(out)


def test_surveyed_points_set_scale_and_frame():
    from caliscope_b200 import synthetic

    r = synthetic.make_rig(16, 400, 5000, seed=21)
    rig = EC.oracle_rig(r)
    ncp = rig.n_camera_params
    X = r.x_true[ncp:].reshape(-1, 3)
    seen = np.bincount(rig.obs_pt, minlength=rig.n_pts) >= 3
    cand = np.nonzero(seen)[0]
    picks = [cand[np.argmin(X[cand, 2])], cand[np.argmax(X[cand, 2])], cand[np.argmax(X[cand, 0])],
             cand[np.argmax(X[cand, 1])]]  # fmt: skip
    A = X[picks[1:]] - X[picks[0]]
    assert abs(np.linalg.det(A)) > 1e-3  # not coplanar
    x0 = r.x0.copy()
    for j in picks:
        x0[ncp + 3 * j : ncp + 3 * j + 3] = X[j]
    with EC.problem(rig, fixed_points=picks) as p:
        res = p.solve(x0)
        cov = p.covariance(res.x)
    ct, c0, c1 = _centres(r.x_true, rig), _centres(r.x0, rig), _centres(res.x, rig)
    e0, e1 = np.linalg.norm(c0 - ct, axis=1).max(), np.linalg.norm(c1 - ct, axis=1).max()
    print(f"surveyed points: camera centres within {e1 * 1e3:.2f} mm of the truth (start {e0 * 1e3:.2f} mm); "
          f"status {res.status} nfev {res.nfev}")  # fmt: skip
    assert res.status in (1, 2, 3, 4)
    assert e1 < 0.01 and e1 < 0.5 * e0  # the start's translation noise is 0.01 m per axis
    ref = HO.dense_covariance(res.x, rig, [], picks)
    e_cam = np.linalg.norm(cov.cameras - ref["cameras"]) / np.linalg.norm(ref["cameras"])
    ok = np.isfinite(ref["points"][:, 0, 0]) & (ref["point_rank"] == 3)
    e_pt = np.linalg.norm(cov.points[ok] - ref["points"][ok]) / np.linalg.norm(ref["points"][ok])
    print(f"covariance with no gauge argument: cameras {e_cam:.2e}, points {e_pt:.2e}, dof {cov.dof}")
    assert len(cov.fixed) == 0
    assert np.array_equal(cov.point_rank, ref["point_rank"]) and np.all(cov.point_rank[picks] == -2)
    assert np.all(cov.points[picks] == 0.0)
    assert cov.dof == ref["dof"]
    assert abs(cov.variance_factor - ref["variance_factor"]) <= 1e-9 * ref["variance_factor"]
    assert e_cam < 1e-8 and e_pt < 1e-8


# ---------------------------------------------------------------------------------------------
# 4. adding a camera to a calibrated rig
# ---------------------------------------------------------------------------------------------
def test_adding_a_camera_keeps_the_calibrated_rig():
    from caliscope_b200 import resection, synthetic

    r = synthetic.make_rig(9, 500, 5000, seed=9)
    rig = EC.oracle_rig(r)
    new = 8
    old_rows = rig.obs_cam != new
    rig_old = EC.oracle_rig(r, old_rows)
    with EC.problem(rig_old) as p:
        x_old = p.solve(r.x0).x
    ncp = rig.n_camera_params
    X = x_old[ncp:].reshape(-1, 3)
    rows = ~old_rows
    poses = resection.resect_robust(rig.cam_flags, rig.cam_const, x_old[:ncp], X, rig.obs_cam[rows],
                                    rig.obs_cam[rows].astype(np.int64), rig.obs_pt[rows], rig.obs_xy[rows],
                                    threshold_px=5.0)  # fmt: skip
    assert poses.status[0] == 0 and poses.cam[0] == new
    x1 = x_old.copy()
    o = rig.cam_offsets[new]
    x1[o : o + 6] = poses.pose[0]
    fc = list(range(rig.cam_offsets[new]))  # every old camera
    with EC.problem(rig, fixed_cam_params=fc) as p:
        rm0 = p.overall_rmse_px(x1)
        res = p.solve(x1)
        rm1 = p.overall_rmse_px(res.x)
    print(f"added camera: resection rmse {poses.rmse_px[0]:.4f} px; rig rmse {rm0:.6f} -> {rm1:.6f} px, status "
          f"{res.status} nfev {res.nfev}")  # fmt: skip
    assert res.status in (1, 2, 3, 4)
    assert np.array_equal(res.x[fc], x_old[fc])
    cam_rm = np.sqrt(np.mean(np.sum(O.reproj_errors_px(res.x, rig)[rows] ** 2, axis=1)))
    assert cam_rm <= poses.rmse_px[0] + 1e-9 and rm1 <= rm0


# ---------------------------------------------------------------------------------------------
# 5. carry-over and repeatability
# ---------------------------------------------------------------------------------------------
def test_cull_keeps_the_fixed_sets_and_solves_repeat():
    from caliscope_b200 import filtering, synthetic

    r = synthetic.make_rig(10, 600, 7000, seed=10, outlier_frac=0.02)
    rig = EC.oracle_rig(r)
    fc, fp = _whole_camera(rig, 2) + [3, 4], list(range(0, rig.n_pts, 9))
    free = EC.free_mask(rig, fc, fp)
    with EC.problem(rig, fixed_cam_params=fc, fixed_points=fp) as p:
        a = p.solve(r.x0)
        b = p.solve(r.x0)
        assert np.array_equal(a.x, b.x) and a.cost == b.cost and a.nfev == b.nfev and a.nit == b.nit
        _, thr = filtering.percentile_thresholds(p, a.x, 95.0, want_err=False)
        p2, keep = p.cull(a.x, thr, 10)
        with p2:
            assert np.array_equal(p2.fixed_cam_params, np.unique(fc)) and np.array_equal(p2.fixed_points, fp)
            c = p2.solve(a.x)
    assert not keep.all()
    assert np.array_equal(a.x[~free], r.x0[~free]) and np.array_equal(c.x[~free], r.x0[~free])
    ref = HO.solve_scipy(EC.oracle_rig(r, keep), a.x, free)
    print(f"after cull: gpu cost {c.cost:.15e} nfev {c.nfev} | scipy cost {ref.cost:.15e}")
    assert c.status in (1, 2, 3, 4) and c.cost <= ref.cost * (1 + 1e-8)


def test_empty_fixed_lists_equal_the_plain_problem():
    from caliscope_b200 import synthetic

    for refine in (False, True):
        r = synthetic.make_rig(12, 700, 9000, seed=3, refine_intrinsics=refine)
        rig = EC.oracle_rig(r)
        with EC.problem(rig) as p:
            a = p.solve(r.x0)
        with EC.problem(rig, fixed_cam_params=[], fixed_points=[]) as p:
            b = p.solve(r.x0)
        assert np.array_equal(a.x, b.x) and a.cost == b.cost and a.nfev == b.nfev and a.nit == b.nit, refine


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
    ncp = rig.n_camera_params
    ga = np.array([[0, 0, 0, 0], [5, 5, 5, 5]], np.int32)
    gb = np.array([[1, 1, 1, 1], [6, 6, 6, 6]], np.int32)
    cons = (ga, gb, np.array([0.1, 0.1]), np.array([1.0, 1.0]))
    cases = [
        (dict(fixed_cam_params=[ncp]), None, -1, "out of range"),
        (dict(fixed_cam_params=[-1]), None, -1, "out of range"),
        (dict(fixed_cam_params=[3, 3]), None, -1, "repeated"),
        (dict(fixed_points=[rig.n_pts]), None, -1, "out of range"),
        (dict(fixed_points=[7, 8, 7]), None, -1, "repeated"),
        (dict(fixed_cam_params=list(range(ncp)), fixed_points=list(range(rig.n_pts))), None, -1, "every parameter"),
        (dict(fixed_points=[6]), cons, -4, "rigid-distance"),
    ]
    codes = {v: k for k, v in vars(L).items() if k.startswith("CB_E_")}
    for kw, cn, code, msg in cases:
        n0 = lib.cb_ba_launch_count()
        with pytest.raises(cb.EngineError, match=msg) as ei:
            cb.BAProblem(rig.cam_flags, rig.cam_const, rig.n_pts, rig.obs_cam, rig.obs_pt, rig.obs_xy, constraints=cn, **kw)
        assert ei.value.code == code, (kw, codes.get(ei.value.code))
        assert lib.cb_ba_launch_count() == n0, kw
    # a fixed point outside every constraint row is accepted beside constraints
    with cb.BAProblem(rig.cam_flags, rig.cam_const, rig.n_pts, rig.obs_cam, rig.obs_pt, rig.obs_xy, constraints=cons,
                      fixed_points=[7]) as p:  # fmt: skip
        assert p.solve(r.x0).status in (1, 2, 3, 4)
    # a sharded solve (here the all-reduce callback, on one GPU) is refused
    with EC.problem(rig, fixed_points=[7]) as p:
        called = []
        n0 = lib.cb_ba_launch_count()
        with pytest.raises(cb.EngineError, match="sharded") as ei:
            p.solve(r.x0, allreduce=lambda user, buf, n, stream: called.append(n) or 0)
        assert ei.value.code == -4 and not called
        assert lib.cb_ba_launch_count() == n0
