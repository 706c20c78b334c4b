"""Scenes for the rigid-body layout refinement tests: tracked frames of one or several bodies from
``_rigid_cases.make_bodies``, and a nominal layout and start poses perturbed from the truth."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from oracle.ba_oracle import rodrigues
from oracle.resection_robust import rot_log
from tests._rigid_cases import Bodies, make_bodies

__all__ = ["Scene", "make_scene", "multi_body", "kabsch_error", "one_camera_marker_scene", "behind_scene", "check"]


@dataclass
class Scene:
    bodies: Bodies
    truth_model: np.ndarray  # (n_model, 3)
    nominal: np.ndarray  # the start layout
    start_key: np.ndarray
    start_pose: np.ndarray
    body_start: np.ndarray
    frame_keys: np.ndarray | None = None  # the key of each row of bodies.truth

    def args(self):
        b = self.bodies
        return (b.flags, b.const, b.cam_x, self.nominal, b.obs_cam, b.obs_key, b.obs_pt, b.obs_px,
                (self.start_key, self.start_pose))  # fmt: skip


def perturb_pose(rng, q, rot_deg, trans):
    ax = rng.normal(size=3)
    dR = rodrigues(ax / np.linalg.norm(ax) * np.deg2rad(rot_deg))[0]
    return np.concatenate([rot_log(dR @ rodrigues(q[:3])[0]), q[3:] + rng.normal(0, trans, 3)])


def make_scene(seed, *, n_model=8, n_frames=20, n_cams=8, noise=0.3, model_off=2e-3, rot_deg=1.0, trans=2e-3,
               **kw) -> Scene:  # fmt: skip
    """make_bodies, with a nominal layout `model_off` (per coordinate, normal) off the truth and start poses
    `rot_deg` and `trans` off."""
    b = make_bodies(seed, n_cams=n_cams, n_frames=n_frames, n_model=n_model, noise=noise, **kw)
    rng = np.random.default_rng(seed + 7919)
    nominal = b.model + rng.normal(0, model_off, b.model.shape)
    keys = np.unique(b.obs_key)
    idx = np.searchsorted(np.asarray(kw.get("frame_keys", np.arange(n_frames))), keys)
    start = np.array([perturb_pose(rng, b.truth[i], rot_deg, trans) for i in idx])
    return Scene(b, b.model.copy(), nominal, keys, start, np.array([0, n_model]),
                 np.asarray(kw.get("frame_keys", np.arange(n_frames)), np.int64))  # fmt: skip


def multi_body(seed, sizes=(4, 6, 3), n_frames=12, **kw) -> Scene:
    """Bodies on disjoint model ranges and disjoint keys, seen by the same rig."""
    parts = [make_scene(seed + 31 * i, n_model=k, n_frames=n_frames,
                        frame_keys=np.arange(n_frames) + 1000 * i, **kw) for i, k in enumerate(sizes)]  # fmt: skip
    base = parts[0].bodies
    off = np.concatenate([[0], np.cumsum(sizes)])
    # every part uses the same rig (make_rig is seeded by the seed): re-project the other parts with the first rig
    from oracle.resection_robust import cameras, project

    cams = cameras(base.flags, base.const, base.cam_x)
    oc, ok, op, px, truth_pose = [], [], [], [], []
    for i, p in enumerate(parts):
        b = p.bodies
        for r in range(len(b.obs_cam)):
            f = int(b.obs_key[r] - 1000 * i)
            q = b.truth[f]
            Xw = b.model[b.obs_pt[r]] @ rodrigues(q[:3])[0].T + q[3:]
            c = cams[b.obs_cam[r]]
            uv, _ = project(c, rodrigues(c.q[:3])[0], c.q[3:6], Xw[None])
            oc.append(b.obs_cam[r]); ok.append(b.obs_key[r]); op.append(b.obs_pt[r] + off[i])
            px.append(uv[0])
    rng = np.random.default_rng(seed + 17)
    noise = kw.get("noise", 0.3)
    px = np.array(px) + rng.normal(0, noise, (len(px), 2))
    model = np.concatenate([p.truth_model for p in parts])
    bodies = Bodies(base.flags, base.const, base.cam_x, model, np.concatenate([p.bodies.truth for p in parts]),
                    np.array(oc, np.int32), np.array(ok, np.int64), np.array(op, np.int32), px)  # fmt: skip
    return Scene(bodies, model.copy(), np.concatenate([p.nominal for p in parts]),
                 np.concatenate([p.start_key for p in parts]), np.concatenate([p.start_pose for p in parts]),
                 off.astype(np.int64))  # fmt: skip


def kabsch_error(M, truth):
    """M minus the truth rigidly aligned onto M (Kabsch), flattened."""
    M, T = np.asarray(M, np.float64), np.asarray(truth, np.float64)
    mc, tc = M.mean(axis=0), T.mean(axis=0)
    U, _, Vt = np.linalg.svd((T - tc).T @ (M - mc))
    D = np.diag([1.0, 1.0, np.sign(np.linalg.det(U @ Vt))])
    R = (U @ D @ Vt).T
    return (M - ((T - tc) @ R.T + mc)).ravel()


def _reproject(b, poses, noise, seed):
    """b's pixels recomputed from the truth layout at `poses` (one per row's frame index), plus noise."""
    from oracle.resection_robust import cameras, project

    cams = cameras(b.flags, b.const, b.cam_x)
    keys = np.unique(b.obs_key)
    fidx = np.searchsorted(keys, b.obs_key)
    rng = np.random.default_rng(seed)
    px = np.empty_like(b.obs_px)
    for r in range(len(b.obs_cam)):
        q = poses[fidx[r]]
        Xw = b.model[b.obs_pt[r]] @ rodrigues(q[:3])[0].T + q[3:]
        c = cams[b.obs_cam[r]]
        px[r] = project(c, rodrigues(c.q[:3])[0], c.q[3:6], Xw[None])[0][0]
    return px + rng.normal(0, noise, px.shape)


def one_camera_marker_scene(seed) -> Scene:
    """Status 2: every frame at one pose and the last marker seen by camera 0 only, so its depth along that ray is free."""
    sc = make_scene(seed, n_model=5, n_frames=6, visible=1.0)
    b = sc.bodies
    b.truth[:] = b.truth[0]
    b.obs_px = _reproject(b, b.truth, 0.2, seed)
    keep = (b.obs_pt != 4) | (b.obs_cam == 0)
    for name in ("obs_cam", "obs_key", "obs_pt", "obs_px"):
        setattr(b, name, getattr(b, name)[keep])
    sc.start_pose[:] = sc.start_pose[0]
    return sc


def behind_scene(seed) -> Scene:
    """Status 4: a camera at camera 0's centre looking the other way sees every marker behind it, with the pixels the
    engine's projection gives there, so the noise-free solution keeps those rows behind it."""
    sc = make_scene(seed, n_model=5, n_frames=6, noise=0.0, visible=1.0)
    b = sc.bodies
    Q = np.diag([-1.0, 1.0, -1.0])  # a half turn about the camera's y axis
    R0 = rodrigues(b.cam_x[:3])[0]
    x_new = np.concatenate([rot_log(Q @ R0), Q @ b.cam_x[3:6]])
    n_cams = len(b.flags)
    b.flags = np.append(b.flags, b.flags[0]).astype(np.int32)
    b.const = np.vstack([b.const, b.const[0]])
    b.cam_x = np.concatenate([b.cam_x, x_new])
    extra = np.flatnonzero(b.obs_cam == 0)
    b.obs_cam = np.concatenate([b.obs_cam, np.full(len(extra), n_cams, np.int32)])
    b.obs_key = np.concatenate([b.obs_key, b.obs_key[extra]])
    b.obs_pt = np.concatenate([b.obs_pt, b.obs_pt[extra]])
    b.obs_px = np.vstack([b.obs_px, np.zeros((len(extra), 2))])
    b.obs_px = _reproject(b, b.truth, 0.0, seed)
    return sc


def check(d, o):
    """A device result d against the oracle's o: statuses, the frame table and counts exactly, iterations at the limit,
    layout, poses, rmse and cov to rounding-level tolerances (NaN where the oracle has NaN)."""
    assert (d.status == o.status).all()
    assert (d.frame_status == o.frame_status).all() and (d.key == o.key).all() and (d.count == o.count).all()
    assert (d.n_frames == o.n_frames).all() and (d.n_rows == o.n_rows).all()
    # iteration counts agree at the limit; below it the last steps compare costs at rounding level
    assert (d.iterations[d.status == 3] == o.iterations[o.status == 3]).all()
    ok = np.isin(d.status, (0, 3, 4))
    scale = max(1.0, np.abs(o.model).max())
    assert np.abs(d.model - o.model).max() <= 1e-7 * scale
    fin = np.isfinite(o.pose).all(axis=1)
    assert (np.isfinite(d.pose).all(axis=1) == fin).all()
    if fin.any():
        assert np.abs(d.pose[fin] - o.pose[fin]).max() <= 1e-7 * max(1.0, np.abs(o.pose[fin]).max())
    np.testing.assert_allclose(d.rmse_px, o.rmse_px, rtol=1e-7, atol=1e-9)  # NaN where the oracle has NaN
    np.testing.assert_allclose(d.frame_rmse_px, o.frame_rmse_px, rtol=1e-7, atol=1e-9)
    for b in range(len(d.status)):
        if ok[b]:
            assert np.abs(d.cov[b] - o.cov[b]).max() <= 1e-6 * np.abs(o.cov[b]).max()
        else:
            assert np.isnan(d.cov[b]).all()
