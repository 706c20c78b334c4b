"""cb_relative_pose_robust on the GPU against oracle/relative_pose.py."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from oracle.relative_pose import relative_poses_robust as oracle_relpose
from tests._relpose_cases import assert_report, compare, scene

pytestmark = pytest.mark.gpu


def _run(*a, **k):
    from caliscope_b200.epipolar import relative_poses_robust

    return relative_poses_robust(*a, **k)


CASES = {
    "exhaustive-8lanes": dict(n_cams=4, n_pts=9, seed=11, noise_px=0.3, kw=dict(min_inliers=5, max_samples=200)),
    "hashed-32lanes": dict(n_cams=3, n_pts=400, seed=12, noise_px=0.5, outlier_frac=0.05, kw=dict(max_samples=48)),
    "fisheye-nan-repeat-free": dict(n_cams=4, n_pts=50, seed=13, noise_px=0.5, outlier_frac=0.03, nan_rows=7,
                                    fisheye=(2,), free=(1,), repeat=1, kw=dict(max_samples=32)),
    "below-min-inliers": dict(n_cams=3, n_pts=12, seed=14, noise_px=0.5, kw=dict(min_inliers=15)),
}


@pytest.mark.parametrize("name", list(CASES))
def test_device_matches_oracle(name):
    c = dict(CASES[name])
    kw = c.pop("kw")
    flags, const, x, cam, key, px, *_ = scene(**c)
    dev = _run(flags, const, cam, key, px, cam_x=x, threshold_px=3.0, **kw)
    orc = oracle_relpose(flags, const, x, cam, key, px, threshold_px=3.0, **kw)
    assert_report(compare(dev, orc), name)
    if name == "below-min-inliers":
        assert (dev.status == 1).all()
    else:
        assert (dev.status == 0).sum() >= 1


def test_device_inputs_repeatability_and_refusals():
    import torch

    from caliscope_b200 import _lib as L

    flags, const, x, cam, key, px, *_ = scene(3, 60, seed=15, noise_px=0.5, outlier_frac=0.05)
    a = _run(flags, const, cam, key, px, cam_x=x, threshold_px=3.0)
    b = _run(flags, const, cam, key, px, cam_x=x, threshold_px=3.0)
    d = _run(flags, const, torch.from_numpy(cam).cuda(), torch.from_numpy(key).cuda(), torch.from_numpy(px).cuda(),
             cam_x=x, threshold_px=3.0)
    for f in ("pose", "cov", "rmse_px", "parallax_deg", "count", "n_inliers", "status"):
        assert np.array_equal(getattr(a, f), getattr(b, f), equal_nan=True), f
        assert np.array_equal(getattr(a, f), getattr(d, f), equal_nan=True), f
    lib = L.load()
    fl, co, xx = (np.ascontiguousarray(v) for v in (flags, const, x))
    out = [np.empty(64, np.int32) for _ in range(2)] + [np.empty(6 * 64), np.empty(36 * 64), np.empty(64), np.empty(64)]
    out += [np.empty(64, np.int32) for _ in range(3)]
    ptr = lambda v: v.ctypes.data_as(C.c_void_p)  # noqa: E731
    npairs = C.c_int32(0)

    def call(tau=3.0, mi=15, ms=64, sig=1.0, it=20, xt=1e-12, c=cam):
        c = np.ascontiguousarray(c, np.int32)
        return lib.cb_relative_pose_robust(len(fl), ptr(fl), ptr(co), ptr(xx), len(c), ptr(c), ptr(key), ptr(px), 0, tau,
                                           mi, ms, sig, it, xt, 64, C.byref(npairs), *[ptr(o) for o in out], None, 0,
                                           None)  # fmt: skip

    assert call() == 0
    for kw in (dict(tau=0.0), dict(tau=float("nan")), dict(mi=4), dict(ms=0), dict(ms=4097), dict(it=0),
               dict(xt=-1.0), dict(sig=float("inf")), dict(c=np.where(cam == 0, 7, cam))):
        assert call(**kw) == -1, kw  # CB_E_INVALID


def _umeyama(src, dst):
    """s, R, t minimising |s R src + t - dst|^2."""
    ms, md = src.mean(0), dst.mean(0)
    S, D = src - ms, dst - md
    U, sv, Vt = np.linalg.svd(D.T @ S / len(src))
    d = np.sign(np.linalg.det(U @ Vt))
    R = U @ np.diag([1.0, 1.0, d]) @ Vt
    s = (sv * [1.0, 1.0, d]).sum() / (S * S).sum() * len(src)
    return s, R, md - s * R @ ms


def _rot(r):
    import cv2

    return cv2.Rodrigues(np.asarray(r, np.float64))[0]


@pytest.mark.parametrize("shape", ["ring16", "stacked64"])
def test_epipolar_start_end_to_end(shape):
    from caliscope_b200 import synthetic
    from caliscope_b200.epipolar import epipolar_start
    from caliscope_b200.problem import BAProblem

    if shape == "ring16":
        rig = synthetic.make_rig(16, 2000, 16000, seed=1, noise_px=0.5, outlier_frac=0.02)
    else:
        rig = synthetic.make_rig(64, 20000, 120000, seed=2, noise_px=0.5, outlier_frac=0.02, cams_per_point=6)
    mi = 15
    key = rig.obs_pt.astype(np.int64)
    st = epipolar_start(rig.cam_flags, rig.cam_const, rig.obs_cam, key, rig.obs_xy, threshold_px=3.0, min_inliers=mi)
    nc = rig.n_cams
    # every camera that shares at least min_inliers points with another camera is posed
    shared = np.zeros(nc, int)
    for c in range(nc):
        pts_c = np.unique(rig.obs_pt[rig.obs_cam == c])
        others = np.unique(rig.obs_pt[rig.obs_cam != c])
        shared[c] = len(np.intersect1d(pts_c, others))
    assert st.posed[shared >= mi].all(), np.flatnonzero((shared >= mi) & ~st.posed)
    # similarity alignment of the posed centres to the truth
    xt = rig.x_true[: 6 * nc].reshape(nc, 6)
    xe = st.x[: 6 * nc].reshape(nc, 6)
    cams = np.flatnonzero(st.posed)
    Rt = np.array([_rot(xt[c, :3]) for c in cams])
    Re = np.array([_rot(xe[c, :3]) for c in cams])
    Ct = np.einsum("nji,nj->ni", Rt, xt[cams, 3:])
    Ce = np.einsum("nji,nj->ni", Re, xe[cams, 3:])
    Ct, Ce = -Ct, -Ce
    s, R, t = _umeyama(Ce, Ct)
    diam = np.max(np.linalg.norm(Ct[:, None] - Ct[None], axis=2))
    cerr = np.linalg.norm(s * Ce @ R.T + t - Ct, axis=1).max() / diam
    rerrs = [np.degrees(np.linalg.norm(_log_rot(Rt[i] @ (Re[i] @ R.T).T))) for i in range(len(cams))]
    rerr = max(rerrs)
    worst = cams[int(np.argmax(rerrs))]
    print(f"{shape}: {len(cams)} of {nc} posed, rounds {st.rounds}, centre error {cerr:.2e} of the diameter, "
          f"rotation error {rerr:.4f} deg (camera {worst}, {(st.obs_cam == worst).sum()} rows), rmse {st.rmse_px:.6f} px")
    assert cerr <= 1e-3 and rerr <= 0.05
    # the final bundle adjustment reaches the minimum a bundle adjustment from the true poses reaches on the same rows
    slot = np.full(nc, -1)
    slot[cams] = np.arange(len(cams))
    x_truth = np.concatenate([xt[cams].ravel(), rig.x_true[6 * nc :].reshape(-1, 3)[st.pt_key].ravel()])
    with BAProblem(rig.cam_flags[cams], rig.cam_const[cams], len(st.pt_key), slot[st.obs_cam].astype(np.int32),
                   st.obs_pt, st.obs_xy) as prob:  # fmt: skip
        ref = prob.overall_rmse_px(prob.solve(x_truth).x)
    assert abs(st.rmse_px - ref) <= 1e-6, (st.rmse_px, ref)


def _log_rot(R):
    import cv2

    return cv2.Rodrigues(R)[0].ravel()
