"""Synthetic rigs for the robust-resection tests: cameras on a ring around a cloud of known points, every camera seeing
every point, pixel noise and planted outliers."""
from __future__ import annotations

import numpy as np

from oracle.ba_oracle import rodrigues
from oracle.resection_robust import cameras, project, rot_log


def look_at(center, target=(0.0, 0.0, 0.0)):
    """(r, t) of a camera at `center` looking at `target` (z forward, y down)."""
    c = np.asarray(center, np.float64)
    z = np.asarray(target, np.float64) - c
    z /= np.linalg.norm(z)
    x = np.cross([0.0, 0.0, -1.0], z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z])
    return rot_log(R), -R @ c


def make_rig(seed, n_cams=6, n_pts=40, *, fisheye=(), free=(), noise=0.3, radius=4.0, spread=1.0):
    """cam_flags, cam_const, cam_x, pts, and the rows (obs_cam, obs_pt, obs_px) of every camera seeing every point."""
    rng = np.random.default_rng(seed)
    flags = np.zeros(n_cams, np.int32)
    const = np.zeros((n_cams, 9))
    xs = []
    for c in range(n_cams):
        a = 2 * np.pi * c / n_cams
        r, t = look_at([radius * np.cos(a), radius * np.sin(a), 0.8 + 0.3 * np.sin(3 * a)])
        fish = c in fisheye
        flags[c] = (2 if fish else 0) | (1 if c in free else 0)
        if fish:
            const[c] = [600.0, 600.0, 640.0, 480.0, 0.02, -0.01, 0.003, -0.001, 0.0]
        else:
            const[c] = [900.0 + 10 * c, 905.0 + 10 * c, 640.0, 480.0, -0.08, 0.02, 0.001, -0.0005, 0.001]
        q = list(r) + list(t)
        if c in free:
            q += [1.01, const[c, 4] * 1.1, const[c, 5] * 0.9]
        xs.append(np.array(q))
    cam_x = np.concatenate(xs)
    pts = rng.uniform(-spread, spread, (n_pts, 3))
    cams = cameras(flags, const, cam_x)
    oc, op, px = [], [], []
    for c in range(n_cams):
        R = rodrigues(cams[c].q[:3])[0]
        uv, _ = project(cams[c], R, cams[c].q[3:6], pts)
        oc.append(np.full(n_pts, c))
        op.append(np.arange(n_pts))
        px.append(uv + rng.normal(0, noise, uv.shape))
    return flags, const, cam_x, pts, np.concatenate(oc).astype(np.int32), np.concatenate(op).astype(np.int32), np.concatenate(px)


def plant_outliers(seed, px, frac, lo=20.0, hi=200.0):
    """px with `frac` of the rows moved by lo..hi pixels in a random direction; returns (px, moved mask)."""
    rng = np.random.default_rng(seed)
    px = px.copy()
    moved = rng.random(len(px)) < frac
    ang = rng.uniform(0, 2 * np.pi, moved.sum())
    mag = rng.uniform(lo, hi, moved.sum())
    px[moved] += np.stack([np.cos(ang), np.sin(ang)], axis=1) * mag[:, None]
    return px, moved


def perturb_cameras(seed, flags, cam_x, rot=0.02, trans=0.05):
    """cam_x with every camera's pose moved a little (a prior that is near, not at, the truth)."""
    rng = np.random.default_rng(seed)
    x = cam_x.copy()
    o = 0
    for f in flags:
        x[o : o + 3] += rng.normal(0, rot, 3)
        x[o + 3 : o + 6] += rng.normal(0, trans, 3)
        o += 9 if f & 1 else 6
    return x


def camera_offsets(flags):
    return np.concatenate([[0], np.cumsum(np.where(np.asarray(flags) & 1, 9, 6))])
