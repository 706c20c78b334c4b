"""What the engine decides at problem creation, seen from outside: the internal camera order (every output is mapped back
to the caller's numbering), device-resident observation lists (read in place, so their layout is checked first) and the
largest reduced system the PCG can hold."""
from __future__ import annotations

import numpy as np
import pytest

from oracle import ba_oracle as O
from tests import _engine_cases as EC

pytestmark = pytest.mark.gpu


def _problem(rig, **kw):
    import caliscope_b200 as cb

    return cb.BAProblem(rig.cam_flags, rig.cam_const, rig.n_pts, rig.obs_cam, rig.obs_pt, rig.obs_xy, **kw)


def _rel(a, b) -> float:
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


def _mixed_intrinsics_rig():
    """48 cameras, local visibility (6 cameras per point); two cameras in three refine their intrinsics (P = 9), the third
    keeps 6 parameters, so the reduced system has padding slots that move with the camera order."""
    from caliscope_b200 import synthetic

    r = synthetic.make_rig(48, 4000, 24000, seed=7, cams_per_point=6, refine_intrinsics=True)
    free = np.arange(r.n_cams) % 3 != 0
    flags = free.astype(np.int32)
    const = r.cam_const.copy()
    const[~free, :2] = synthetic.WEBCAM_F
    blocks = r.x0[: 9 * r.n_cams].reshape(r.n_cams, 9)
    x = np.concatenate([blocks[c] if free[c] else blocks[c, :6] for c in range(r.n_cams)] + [r.x0[9 * r.n_cams :]])
    return O.Rig(flags, const, r.n_pts, r.obs_cam, r.obs_pt, r.obs_xy), x


def _relabel(rig, x, perm):
    """The same problem with camera k of the new numbering = camera perm[k] of the old.  Returns the rig, its x and
    xmap: old camera-parameter index -> new index."""
    inv = np.argsort(perm)
    rig2 = O.Rig(rig.cam_flags[perm], rig.cam_const[perm], rig.n_pts, inv[rig.obs_cam].astype(np.int32), rig.obs_pt,
                 rig.obs_xy)  # fmt: skip
    off, off2 = rig.cam_offsets, rig2.cam_offsets
    xmap = np.empty(rig.n_camera_params, np.int64)
    for k, c in enumerate(perm):
        xmap[off[c] : off[c + 1]] = np.arange(off2[k], off2[k + 1])
    x2 = x.copy()
    x2[xmap] = x[: rig.n_camera_params]
    return rig2, x2, xmap


def test_camera_relabelling_permutes_every_output():
    """The engine lays the reduced camera system out in its own camera order (chosen from co-visibility, or given as
    cam_order) and maps every output back to the caller's numbering.  Relabelling the cameras must permute the outputs
    and change nothing else: per-observation and per-camera reductions bitwise, the reduced system to rounding, the step,
    the solve and the covariance to 1e-9 (the PCG step to 1e-8)."""
    from caliscope_b200 import filtering

    rig, x = _mixed_intrinsics_rig()
    perm = np.random.default_rng(2024).permutation(rig.n_cams)
    rig2, x2, xmap = _relabel(rig, x, perm)
    lam, q = 1e-3, 90.0
    out = []
    for rg, xx in ((rig, x), (rig2, x2)):
        with _problem(rg) as p:
            st = EC.stats(p)
            o = dict(stats=st, P=p.cam_stride, r=p.residuals(xx), J=p.jacobian_blocks(xx), e=p.reproj_errors_px(xx),
                     rmse=p.rmse_px(xx), ost=p.error_order_stats(xx, q), ne=p.normal_equations(xx, lam))  # fmt: skip
            _, thr = filtering.percentile_thresholds(p, xx, 100.0 - q, want_err=False)
            p2, keep = p.cull(xx, thr, 10)
            with p2:
                o.update(thr=thr, keep=keep, r_cull=p2.residuals(xx))
            o["sol"] = p.solve(xx)
            out.append(o)
    a, b = out
    print(f"caller's numbering: stat keys {a['stats']}; relabelled: stat keys {b['stats']}")
    assert a["P"] == b["P"] == 9
    assert b["stats"][EC.REORDERED] == 1
    # per observation: bitwise
    assert np.array_equal(a["r"], b["r"])
    assert np.array_equal(a["J"][0], b["J"][0]) and np.array_equal(a["J"][1], b["J"][1])
    assert np.array_equal(a["e"], b["e"])
    # per camera: bitwise, permuted; the overall RMSE sums the cameras in slot order
    assert np.array_equal(a["rmse"][1][perm], b["rmse"][1])
    assert abs(a["rmse"][0] - b["rmse"][0]) <= 1e-14 * a["rmse"][0]
    assert np.array_equal(a["ost"][0], b["ost"][0])
    for k in (1, 2, 3):
        assert np.array_equal(a["ost"][k][perm], b["ost"][k])
    assert np.array_equal(a["thr"][perm], b["thr"])
    assert np.array_equal(a["keep"], b["keep"]) and not a["keep"].all()
    assert np.array_equal(a["r_cull"], b["r_cull"])
    # the linearisation and the reduced system, permuted blockwise
    na, nb, nc, P = a["ne"], b["ne"], rig.n_cams, 9
    Sa = na["S"].reshape(nc, P, nc, P)[perm][:, :, perm].reshape(nc * P, nc * P)
    errs = {"U": _rel(na["U"][perm], nb["U"]), "gc": _rel(na["gc"][perm], nb["gc"]), "V": _rel(na["V"], nb["V"]),
            "gp": _rel(na["gp"], nb["gp"]), "S": _rel(Sa, nb["S"]), "b": _rel(na["b"].reshape(nc, P)[perm], nb["b"].reshape(nc, P)),
            "dc": _rel(na["dc"][perm], nb["dc"]), "dp": _rel(na["dp"], nb["dp"]),
            "cost": abs(na["cost"] - nb["cost"]) / na["cost"]}  # fmt: skip
    sa, sb = a["sol"], b["sol"]
    xa = sa.x.copy()
    xa[xmap] = sa.x[: rig.n_camera_params]
    errs.update(solve_x=_rel(xa, sb.x), solve_cost=abs(sa.cost - sb.cost) / sa.cost)
    # covariance at the solution, in the same gauge expressed in each numbering
    with _problem(rig) as p:
        ca = p.covariance(sa.x)
    with _problem(rig2) as p:
        cb_ = p.covariance(sb.x, fixed=xmap[ca.fixed])
    errs.update(cov_cameras=_rel(cb_.cameras[np.ix_(xmap, xmap)], ca.cameras),
                cov_points=_rel(ca.points[ca.point_rank == 3], cb_.points[cb_.point_rank == 3]))  # fmt: skip
    print(f"relabelled vs caller's numbering (nfev {sa.nfev} / {sb.nfev}): " + ", ".join(f"{k} {v:.1e}" for k, v in errs.items()))
    for k in ("U", "gc", "V", "gp", "S", "b"):
        assert errs[k] <= 1e-12, k
    # the step comes from a PCG, which amplifies the rounding-level differences of the two S (2e-16) to ~1e-9
    for k in ("dc", "dp"):
        assert errs[k] <= 1e-8, k
    for k in ("cost", "solve_x", "solve_cost", "cov_cameras", "cov_points"):
        assert errs[k] <= 1e-9, k
    assert np.array_equal(ca.point_rank, cb_.point_rank)
    # the caller's own numbering, passed explicitly, is kept
    with _problem(rig2, cam_order=np.arange(rig.n_cams)) as p:
        assert EC.stats(p)[EC.REORDERED] == 0
        r_id = p.residuals(x2)
        ne_id = p.normal_equations(x2, lam)
    assert np.array_equal(r_id, b["r"])
    assert _rel(ne_id["S"], nb["S"]) <= 1e-12 and _rel(ne_id["b"], nb["b"]) <= 1e-12
    assert _rel(ne_id["dc"], nb["dc"]) <= 1e-8 and _rel(ne_id["dp"], nb["dp"]) <= 1e-8


def test_device_resident_observations_are_validated_and_read_in_place():
    """CUDA tensors are read in place: int32 and int16 camera indices give exactly what NumPy input gives; any other
    dtype, a CPU tensor, a strided view or unequal lengths are refused before the engine reads a byte (an int64 camera
    tensor would otherwise be read as int32 words: half the list, every other index 0, all in range)."""
    torch = pytest.importorskip("torch")
    import caliscope_b200 as cb
    from caliscope_b200 import synthetic

    r = synthetic.make_rig(12, 800, 9000, seed=2)
    rig = EC.oracle_rig(r)
    with _problem(rig) as p:
        ref = (p.residuals(r.x0), p.normal_equations(r.x0, 1e-3), p.solve(r.x0))
    dev = torch.device("cuda", 0)
    pt = torch.from_numpy(r.obs_pt).to(dev)
    xy = torch.from_numpy(np.ascontiguousarray(r.obs_xy)).to(dev)
    for dt in (np.int32, np.int16):
        cam = torch.from_numpy(r.obs_cam.astype(dt)).to(dev)
        with cb.BAProblem(rig.cam_flags, rig.cam_const, rig.n_pts, cam, pt, xy) as p:
            got = (p.residuals(r.x0), p.normal_equations(r.x0, 1e-3), p.solve(r.x0))
        assert np.array_equal(got[0], ref[0]), dt
        for k, v in ref[1].items():
            assert np.array_equal(got[1][k], v), (dt, k)
        assert np.array_equal(got[2].x, ref[2].x) and got[2].cost == ref[2].cost and got[2].nfev == ref[2].nfev, dt
    cam = torch.from_numpy(r.obs_cam).to(dev)
    bad = {
        "obs_cam": [(cam.long(), pt, xy), (cam.cpu(), pt, xy), (cam.float(), pt, xy)],
        "obs_pt": [(cam, pt.long(), xy), (cam, torch.stack([pt, pt], 1)[:, 0], xy)],
        "obs_xy": [(cam, pt, xy.float()), (cam, pt, torch.cat([xy, xy], 1)[:, :2]), (cam, pt, xy.reshape(-1))],
    }
    for name, cases in bad.items():
        for c, q, w in cases:
            with pytest.raises(ValueError, match=name):
                cb.BAProblem(rig.cam_flags, rig.cam_const, rig.n_pts, c, q, w)
    with pytest.raises(ValueError, match="same length"):
        cb.BAProblem(rig.cam_flags, rig.cam_const, rig.n_pts, cam, pt[:-1], xy)


def test_reduced_system_above_the_pcg_shared_memory_limit_is_refused():
    """The L2-streamed PCG keeps 9 vectors of n_camera_params and the P x P preconditioner blocks in one CTA's shared
    memory, (15 nP + 544) doubles at P = 6: above about 316 cameras (P = 6) the 227 KB of an H100 CTA do not hold it and
    problem creation fails with an error that names the PCG configuration."""
    import caliscope_b200 as cb
    from caliscope_b200 import synthetic

    r = synthetic.make_rig(400, 300, 20000, seed=400, layout="dome")
    with pytest.raises(cb.EngineError, match="PCG cluster configuration"):
        _problem(EC.oracle_rig(r))
