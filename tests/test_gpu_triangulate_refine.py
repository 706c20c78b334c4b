"""cb_triangulate_refine against the NumPy oracle (oracle/triangulation_refine.py refine_points / point_covariance) at every
shape-selected variant: P = 6 and 9, 8 and 32 lanes per group, the camera table in and out of shared memory."""
import numpy as np
import pytest

from caliscope_b200 import synthetic
from caliscope_b200.triangulation import RefineStats, triangulate_groups, triangulate_refined
from oracle import triangulation_refine as T

pytestmark = pytest.mark.gpu


def _ncp(flags):
    return int(np.where(np.asarray(flags) & 1, 9, 6).sum())


def _camera_cov(ncp, seed):
    rng = np.random.default_rng(seed)
    L = 1e-4 * (np.eye(ncp) + 0.3 * rng.normal(size=(ncp, ncp)) / np.sqrt(ncp))
    return L @ L.T


def _check(flags, const, cx, obs_cam, obs_key, obs_px, *, camera_cov=None, sigma=0.5, on_device=False):
    args = (obs_cam, obs_key, obs_px)
    if on_device:
        import torch

        args = (torch.from_numpy(np.ascontiguousarray(obs_cam, np.int32)).cuda(),
                torch.from_numpy(np.ascontiguousarray(obs_key, np.int64)).cuda(),
                torch.from_numpy(np.ascontiguousarray(obs_px, np.float64)).cuda())  # fmt: skip
    st = RefineStats()
    out = triangulate_refined(flags, const, cx, *args, pixel_sigma=sigma, camera_cov=camera_cov, stats=st)
    # the DLT start of the same call: cb_undistort_triangulate on cameras derived from the BA layout
    proj, mats, dists, fish = T.dlt_camera_models(flags, const, cx)
    x0, count, rep, _ = triangulate_groups(proj, obs_cam, obs_key, obs_px, undistort=(mats, dists, fish))
    assert np.array_equal(out.count, count) and np.array_equal(out.rep_row, rep)
    grp, G = T.group_rows(obs_key)
    assert G == len(out.xyz) == st.n_groups
    xyz, rmse, status, _ = T.refine_points(flags, const, cx, obs_cam, obs_px, grp, x0)
    assert np.array_equal(out.status, status)
    ref = status != T.STATUS_NOT_PD
    assert np.array_equal(out.xyz[~ref], x0[~ref], equal_nan=True)
    scale = np.linalg.norm(xyz[ref], axis=1, keepdims=True)
    assert np.nanmax(np.abs(out.xyz[ref] - xyz[ref]) / scale, initial=0.0) < 1e-9
    assert np.array_equal(np.isnan(out.rmse_px), np.isnan(rmse))
    assert np.nanmax(np.abs(out.rmse_px - rmse) / np.maximum(rmse, 1e-3), initial=0.0) < 1e-8
    cov = T.point_covariance(flags, const, cx, obs_cam, obs_px, grp, xyz, status, sigma, camera_cov)
    ok = np.isfinite(cov).all(axis=(1, 2))
    assert np.array_equal(ok, np.isfinite(out.cov).all(axis=(1, 2)))
    nrm = np.linalg.norm(cov[ok], axis=(1, 2))[:, None, None]
    assert np.max(np.abs(out.cov[ok] - cov[ok]) / nrm, initial=0.0) < 1e-8
    assert (status == 0).mean() > 0.9
    return out, st


def _rig_case(name):
    if name == "p6":
        rig = synthetic.make_rig(8, 600, 4000, seed=1)
    elif name == "p9":
        rig = synthetic.make_rig(16, 600, 6000, refine_intrinsics=True, seed=2)
    elif name == "fisheye_mixed":  # fisheye cameras with locked intrinsics next to free Brown-Conrady ones
        from oracle import ba_oracle as O

        rig = synthetic.make_rig(8, 600, 4000, refine_intrinsics=True, seed=3)
        flags, const = rig.cam_flags.copy(), rig.cam_const.copy()
        flags[::2] = 2
        const[::2, 4:9] = (0.05, -0.01, 0.002, -0.0005, 0.0)
        cx = np.concatenate([rig.x_true[9 * c : 9 * c + (6 if flags[c] & 2 else 9)] for c in range(8)])
        orc = O.Rig(flags, const, rig.n_pts, rig.obs_cam, rig.obs_pt, rig.obs_xy)
        uv = O._project(np.concatenate([cx, rig.x_true[72:]]), orc, False)[0]
        px = uv + np.random.default_rng(3).normal(0, 0.5, uv.shape)
        key = rig.obs_pt.astype(np.int64)
        key[0] = rig.n_pts + 5
        return flags, const, cx, rig.obs_cam, key, px
    elif name == "dense":  # 40 of 64 cameras per point
        rig = synthetic.make_rig(64, 300, 12_000, layout="dome", seed=4)
    elif name == "mocap":  # 2-8 cameras per point
        rig = synthetic.make_rig(8, 3000, 12_000, cams_per_point=8, seed=5)
    elif name == "repeated":  # repeated (camera, point) rows; > 96 rows per group: 32 lanes
        rig = synthetic.make_rig(8, 20, 2400, seed=6)
    elif name == "cams_global":  # 150 cameras: the camera table does not fit in shared memory
        rig = synthetic.make_rig(150, 400, 8000, layout="dome", seed=7)
    else:
        raise KeyError(name)
    ncp = _ncp(rig.cam_flags)
    # the truth's cameras observe noisy pixels; one single-row group (status 1)
    key = rig.obs_pt.astype(np.int64)
    key[0] = rig.n_pts + 5
    return rig.cam_flags, rig.cam_const, rig.x_true[:ncp], rig.obs_cam, key, rig.obs_xy


CASES = ["p6", "p9", "fisheye_mixed", "dense", "mocap", "repeated", "cams_global"]


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("with_cov", [False, True])
def test_refine_matches_oracle(name, with_cov):
    flags, const, cx, cam, key, px = _rig_case(name)
    _check(flags, const, cx, cam, key, px, camera_cov=_camera_cov(len(cx), 9) if with_cov else None)


@pytest.mark.parametrize("name", ["p9", "repeated"])
def test_device_resident_observations(name):
    flags, const, cx, cam, key, px = _rig_case(name)
    host, _ = _check(flags, const, cx, cam, key, px, camera_cov=_camera_cov(len(cx), 3))
    dev, _ = _check(flags, const, cx, cam, key, px, camera_cov=_camera_cov(len(cx), 3), on_device=True)
    for f in ("xyz", "cov", "rmse_px", "count", "rep_row", "status"):
        assert np.array_equal(getattr(host, f), getattr(dev, f), equal_nan=True), f


def test_two_calls_are_bit_identical():
    flags, const, cx, cam, key, px = _rig_case("dense")
    c = _camera_cov(len(cx), 4)
    a = triangulate_refined(flags, const, cx, cam, key, px, camera_cov=c)
    b = triangulate_refined(flags, const, cx, cam, key, px, camera_cov=c)
    for f in ("xyz", "cov", "rmse_px", "count", "rep_row", "status"):
        assert np.array_equal(getattr(a, f), getattr(b, f), equal_nan=True), f


def test_status_codes_on_the_device():
    X = np.array([0.5, 0.1, 2.0])
    cen = np.array([(0, 0, 0), (1, 0, 0), (0.5, 0, 4.0), (0.1, 0, 0)], float)
    const = np.tile([1000.0, 1000.0, 640.0, 480.0, 0, 0, 0, 0, 0], (4, 1))
    cx = np.concatenate([np.r_[0.0, 0.0, 0.0, -c] for c in cen])

    def px(c):
        d = X - cen[c]
        return [1000.0 * d[0] / d[2] + 640.0, 1000.0 * d[1] / d[2] + 480.0]

    rows = [(0, 0, px(0)), (0, 1, px(1)), (1, 0, px(0)), (2, 0, px(0)), (2, 0, px(0)), (3, 0, [740.0, 480.0]),
            (3, 3, [740.0, 480.0]), (4, 0, px(0)), (4, 1, px(1)), (4, 2, px(2))]  # fmt: skip
    key = np.array([r[0] for r in rows], np.int64)
    cam = np.array([r[1] for r in rows], np.int32)
    obs = np.array([r[2] for r in rows], float)
    out = triangulate_refined(np.zeros(4, np.int32), const, cx, cam, key, obs)
    assert out.status.tolist() == [0, 1, 2, 2, 4]
    assert np.abs(out.xyz[[0, 4]] - X).max() < 1e-9
    assert np.isnan(out.cov[[1, 2, 3]]).all() and np.isfinite(out.cov[[0, 4]]).all()
    assert triangulate_refined(np.zeros(4, np.int32), const, cx, cam, key, obs + 3.0, max_iter=1).status[0] == 3


def test_solve_covariance_then_refined_triangulation():
    import caliscope_b200 as cb

    sigma = 0.5
    rig = synthetic.make_rig(8, 800, 6000, seed=8, noise_px=sigma)
    ncp = _ncp(rig.cam_flags)
    with cb.BAProblem(rig.cam_flags, rig.cam_const, rig.n_pts, rig.obs_cam, rig.obs_pt, rig.obs_xy) as prob:
        res = prob.solve(rig.x0)
        cov = prob.covariance(res.x, variance_factor=(sigma / rig.cam_const[0, 0]) ** 2, points=False)
    # new observations of new points with the calibrated rig
    new = synthetic.make_rig(8, 500, 4000, seed=9, noise_px=sigma)
    out, _ = _check(rig.cam_flags, rig.cam_const, res.x[:ncp], new.obs_cam, new.obs_pt.astype(np.int64), new.obs_xy,
                    camera_cov=cov.cameras, sigma=sigma)  # fmt: skip
    # the camera term adds to the pixel term
    pix = triangulate_refined(rig.cam_flags, rig.cam_const, res.x[:ncp], new.obs_cam, new.obs_pt, new.obs_xy,
                              pixel_sigma=sigma)  # fmt: skip
    ok = out.status == 0
    assert np.all(np.trace(out.cov[ok], axis1=1, axis2=2) >= np.trace(pix.cov[ok], axis1=1, axis2=2))


def test_bad_arguments_are_refused():
    from caliscope_b200 import _lib as L

    flags, const, cx, cam, key, px = _rig_case("p6")
    with pytest.raises(L.EngineError):
        triangulate_refined(flags, const, cx, cam, key, px, max_iter=0)
    with pytest.raises(L.EngineError):
        triangulate_refined(flags, const, cx, np.where(cam == 0, 99, cam), key, px)
    with pytest.raises(ValueError):
        triangulate_refined(flags, const, cx, cam, key, px, camera_cov=np.eye(3))
