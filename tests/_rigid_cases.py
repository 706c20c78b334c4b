"""Synthetic rigs for the rigid-body pose tests: cameras on a ring around a marker cluster, the cluster at a known pose in
every frame, each (marker, camera) row kept with some probability, pixel noise and planted outliers."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from oracle.ba_oracle import rodrigues
from oracle.resection_robust import cameras, project
from tests._resect_cases import camera_offsets, make_rig, plant_outliers

__all__ = ["Bodies", "make_bodies", "plant_outliers", "camera_offsets", "camera_cov", "perturb", "pose_error"]


@dataclass
class Bodies:
    flags: np.ndarray
    const: np.ndarray
    cam_x: np.ndarray
    model: np.ndarray  # (n_model, 3)
    truth: np.ndarray  # (n_frames, 6) the body pose (r, t) of every frame
    obs_cam: np.ndarray
    obs_key: np.ndarray  # the frame
    obs_pt: np.ndarray
    obs_px: np.ndarray

    def rig(self):
        return self.flags, self.const, self.cam_x

    def obs(self):
        return self.obs_cam, self.obs_key, self.obs_pt, self.obs_px


def make_bodies(seed, n_cams=8, n_frames=20, n_model=12, *, fisheye=(), free=(), noise=0.3, visible=0.7, size=0.2,
                radius=3.0, spread=0.3, frame_keys=None) -> Bodies:  # fmt: skip
    """A rig of n_cams cameras on a ring of `radius` looking at the origin, a cluster of n_model markers in a cube of
    `size`, one random pose per frame within `spread` of the origin.  Each (frame, marker, camera) row is kept with
    probability `visible`; rows are ordered by frame, then marker, then camera."""
    rng = np.random.default_rng(seed)
    flags, const, cam_x, _, _, _, _ = make_rig(seed, n_cams, 1, fisheye=fisheye, free=free, radius=radius)
    cams = cameras(flags, const, cam_x)
    model = rng.uniform(-size / 2, size / 2, (n_model, 3))
    keys = np.arange(n_frames) if frame_keys is None else np.asarray(frame_keys)
    truth = np.zeros((n_frames, 6))
    oc, ok, op, px = [], [], [], []
    for f in range(n_frames):
        ax = rng.normal(size=3)
        truth[f, :3] = ax / np.linalg.norm(ax) * rng.uniform(0, np.pi * 0.8)
        truth[f, 3:] = rng.uniform(-spread, spread, 3)
        R = rodrigues(truth[f, :3])[0]
        Xw = model @ R.T + truth[f, 3:]
        for c in range(n_cams):
            Rc = rodrigues(cams[c].q[:3])[0]
            uv, _ = project(cams[c], Rc, cams[c].q[3:6], Xw)
            keep = rng.random(n_model) < visible
            m = np.flatnonzero(keep)
            oc.append(np.full(len(m), c))
            ok.append(np.full(len(m), keys[f]))
            op.append(m)
            px.append(uv[m] + rng.normal(0, noise, (len(m), 2)))
    order = np.lexsort((np.concatenate(oc), np.concatenate(op), np.concatenate(ok)))
    return Bodies(flags, const, cam_x, model, truth, np.concatenate(oc).astype(np.int32)[order],
                  np.concatenate(ok).astype(np.int64)[order], np.concatenate(op).astype(np.int32)[order],
                  np.concatenate(px)[order])  # fmt: skip


def camera_cov(flags, rot=1e-3, trans=2e-3, intr=(1e-3, 1e-3, 1e-3)):
    """A block-diagonal camera covariance in x's layout: rotation, translation and (s, k1, k2) variances."""
    offs = camera_offsets(flags)
    var = []
    for f in flags:
        var += [rot**2] * 3 + [trans**2] * 3 + ([v**2 for v in intr] if f & 1 else [])
    assert len(var) == offs[-1]
    return np.diag(var)


def perturb(seed, cam_x, cov):
    """cam_x moved by one draw of N(0, cov)."""
    rng = np.random.default_rng(seed)
    return cam_x + np.linalg.cholesky(cov) @ rng.normal(size=len(cam_x))


def pose_error(pose, truth):
    """(r, t) difference; the rotation part is the difference of rotation vectors (first order)."""
    return np.asarray(pose) - np.asarray(truth)
