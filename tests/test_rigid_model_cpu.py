"""The rigid-body layout refinement oracle (oracle/rigid_model.py) against the truth, scipy's least_squares, the dense
covariance, its gauge rule, every status and the chi-square calibration of its covariance."""
from __future__ import annotations

import numpy as np
import pytest
from scipy.optimize import least_squares

from oracle.ba_oracle import rodrigues
from oracle.resection_robust import rot_log
from oracle.rigid_model import (STATUS_BEHIND, STATUS_MAX_ITER, STATUS_NOT_PD, STATUS_OK, STATUS_UNUSED,
                                gauge_basis, gauge_constraints, rigid_model_refine)  # fmt: skip
from oracle.rigid_pose_robust import body_jacobians
from tests._rigid_cases import camera_cov, perturb
from tests._rigid_model_cases import behind_scene, kabsch_error, make_scene, multi_body, one_camera_marker_scene


def _solve(sc, **kw):
    return rigid_model_refine(*sc.args(), body_start=sc.body_start, **kw)


def _residuals(sc, M, poses):
    b = sc.bodies
    keys = np.unique(b.obs_key)
    out = []
    for f, k in enumerate(keys):
        rows = np.flatnonzero(b.obs_key == k)
        r, _, _ = body_jacobians(b.flags, b.const, b.cam_x, b.obs_cam[rows], b.obs_px[rows], M[b.obs_pt[rows]], poses[f])
        out.append(r.ravel())
    return np.concatenate(out)


def test_noise_free_reaches_truth():
    sc = make_scene(3, n_model=6, n_frames=12, noise=0.0, model_off=5e-3, rot_deg=2.0, trans=5e-3)
    r = _solve(sc)
    assert r.status[0] == STATUS_OK
    assert np.abs(kabsch_error(r.model, sc.truth_model)).max() < 1e-9
    # the poses are the truth's seen through the gauge's rigid motion: X_w of every marker is the truth's
    for f in range(len(r.key)):
        q, t = r.pose[f], sc.bodies.truth[f]
        Xr = r.model @ rodrigues(q[:3])[0].T + q[3:]
        Xt = sc.truth_model @ rodrigues(t[:3])[0].T + t[3:]
        assert np.abs(Xr - Xt).max() < 1e-9


def test_optimum_matches_least_squares():
    sc = make_scene(5, n_model=5, n_frames=8, noise=0.5)
    r = _solve(sc)
    N = gauge_basis(sc.nominal)
    nz, F = N.shape[1], len(sc.start_key)

    def fun(p):
        M = sc.nominal + (N @ p[:nz]).reshape(-1, 3)
        return _residuals(sc, M, p[nz:].reshape(F, 6))

    ls = least_squares(fun, np.concatenate([np.zeros(nz), sc.start_pose.ravel()]), method="lm", xtol=1e-15,
                       ftol=1e-15, gtol=1e-15)  # fmt: skip
    M = sc.nominal + (N @ ls.x[:nz]).reshape(-1, 3)
    assert np.abs(r.model - M).max() <= 1e-8 * np.abs(M).max()
    assert np.abs(r.pose - ls.x[nz:].reshape(F, 6)).max() <= 1e-8 * np.abs(r.pose).max()


@pytest.mark.parametrize("with_cam", [False, True])
def test_covariance_equals_dense_inverse(with_cam):
    sc = make_scene(7, n_model=4, n_frames=6, noise=0.3, free=(1, 3))
    b = sc.bodies
    ccov = camera_cov(b.flags) if with_cam else None
    r = _solve(sc, pixel_sigma=0.7, camera_cov=ccov)
    N = gauge_basis(sc.nominal)
    nz, F = N.shape[1], len(r.key)
    # dense J over (z, q) at the solution, and the camera Jacobian
    rows_all, J, Jc_all = [], [], []
    nc = 6 * F + nz
    widths = np.where(b.flags & 1, 9, 6)
    offs = np.concatenate([[0], np.cumsum(widths)])
    for f, k in enumerate(r.key):
        rows = np.flatnonzero(b.obs_key == k)
        res, Jq, Jc = body_jacobians(b.flags, b.const, b.cam_x, b.obs_cam[rows], b.obs_px[rows],
                                     r.model[b.obs_pt[rows]], r.pose[f])  # fmt: skip
        R = rodrigues(r.pose[f][:3])[0]
        for i, row in enumerate(rows):
            Ji = np.zeros((2, nc))
            JM = Jq[i][:, 3:6] @ R
            Ji[:, :nz] = JM @ N[3 * b.obs_pt[row] : 3 * b.obs_pt[row] + 3]
            Ji[:, nz + 6 * f : nz + 6 * f + 6] = Jq[i]
            J.append(Ji)
            Jci = np.zeros((2, offs[-1]))
            c = b.obs_cam[row]
            Jci[:, offs[c] : offs[c] + widths[c]] = Jc[i][:, : widths[c]]
            Jc_all.append(Jci)
    J, Jc = np.concatenate(J), np.concatenate(Jc_all)
    Hi = np.linalg.inv(J.T @ J)
    cov_z = 0.49 * Hi
    if with_cam:
        G = J.T @ Jc
        cov_z = cov_z + Hi @ G @ ccov @ G.T @ Hi
    dense = N @ cov_z[:nz, :nz] @ N.T
    assert np.abs(r.cov[0] - dense).max() <= 1e-8 * np.abs(dense).max()


def test_gauge_constraints_and_rigid_motion():
    sc = make_scene(11, n_model=7, n_frames=10, noise=0.4)
    r = _solve(sc)
    C = gauge_constraints(sc.nominal)
    d = (r.model - sc.nominal).ravel()
    assert np.abs(C.T @ d).max() <= 1e-10 * np.abs(r.model).max()
    # one rigid motion g of the start layout: poses compose with g^-1, the result moves by g
    Rg, tg = rodrigues(np.array([0.3, -0.2, 0.5]))[0], np.array([0.05, -0.02, 0.1])
    sc2 = make_scene(11, n_model=7, n_frames=10, noise=0.4)
    sc2.nominal = sc.nominal @ Rg.T + tg
    for f in range(len(sc2.start_pose)):
        R = rodrigues(sc.start_pose[f][:3])[0]
        sc2.start_pose[f] = np.concatenate([rot_log(R @ Rg.T), sc.start_pose[f][3:] - R @ Rg.T @ tg])
    r2 = _solve(sc2)
    assert np.abs(r2.model - (r.model @ Rg.T + tg)).max() <= 1e-9


def test_statuses():
    sc = make_scene(13, n_model=5, n_frames=8, noise=0.3)
    b = sc.bodies
    assert _solve(sc, max_iter=1).status[0] == STATUS_MAX_ITER
    # a marker never seen: status 1, start layout, NaN cov
    keep = b.obs_pt != 4
    sc.bodies.obs_cam, sc.bodies.obs_key = b.obs_cam[keep], b.obs_key[keep]
    sc.bodies.obs_pt, sc.bodies.obs_px = b.obs_pt[keep], b.obs_px[keep]
    r = _solve(sc)
    assert r.status[0] == STATUS_UNUSED and np.isnan(r.cov[0]).all() and (r.model == sc.nominal).all()
    # a frame with two markers takes no part
    sc = make_scene(13, n_model=5, n_frames=8, noise=0.3)
    b = sc.bodies
    keep = (b.obs_key != 0) | (b.obs_pt < 2)
    for name in ("obs_cam", "obs_key", "obs_pt", "obs_px"):
        setattr(b, name, getattr(b, name)[keep])
    r = _solve(sc)
    assert r.frame_status[0] == STATUS_UNUSED and r.status[0] == STATUS_OK and (r.frame_status[1:] == 0).all()
    # collinear markers: the rotation about their line is free
    sc = make_scene(17, n_model=4, n_frames=8, noise=0.3)
    line = np.array([0.03, -0.02, 0.05])
    sc.nominal = np.outer([-1.5, -0.5, 0.5, 1.5], line)
    r = _solve(sc)
    assert r.status[0] == STATUS_NOT_PD and np.isnan(r.cov[0]).all()
    # a marker seen by camera 0 only, in frames that all share one pose: its depth along the ray is free
    r = _solve(one_camera_marker_scene(19))
    assert r.status[0] == STATUS_NOT_PD and np.isnan(r.cov[0]).all() and np.isnan(r.rmse_px[0])
    # a camera at camera 0's centre looking the other way: its rows are behind it at the solution
    r = _solve(behind_scene(19))
    assert r.status[0] == STATUS_BEHIND and np.isfinite(r.cov[0]).all()


def _chi2(seeds, with_cam, term):
    vals = []
    for s in seeds:
        sc = make_scene(100 + s, n_model=4, n_frames=10, noise=0.2, model_off=2e-3)
        b = sc.bodies
        ccov = camera_cov(b.flags, rot=2e-3, trans=5e-3)
        if with_cam:
            b.cam_x = perturb(1000 + s, b.cam_x, ccov)
        r = _solve(sc, pixel_sigma=0.2, camera_cov=ccov if term else None)
        e = kabsch_error(r.model, sc.truth_model)
        vals.append(e @ np.linalg.pinv(r.cov[0], rcond=1e-10) @ e)
    return np.mean(vals)


@pytest.mark.parametrize("with_cam,term,inside", [(False, False, True), (True, True, True), (True, False, False)])
def test_chi2_calibration(with_cam, term, inside):
    n, dof = 200, 3 * 4 - 6
    m = _chi2(range(n), with_cam, term)
    half = 4.0 * np.sqrt(2 * dof / n)
    assert (abs(m - dof) <= half) == inside, m


def test_multi_body():
    sc = multi_body(23)
    r = _solve(sc)
    assert (r.status == 0).all() and [c.shape for c in r.cov] == [(12, 12), (18, 18), (9, 9)]
    for b in range(3):
        lo, hi = sc.body_start[b], sc.body_start[b + 1]
        assert r.n_frames[b] == 12
        assert np.isfinite(r.model[lo:hi]).all()
