"""Seeded 2-D-only scenes for the relative-pose tests: cameras on a ring looking at the origin, points near it, every
point seen by every camera (key = point), with pixel noise, planted outliers and NaN rows."""
from __future__ import annotations

import cv2
import numpy as np


def look_at(c):
    """World-to-camera R, t of a camera at c looking at the origin (y down)."""
    z = -np.asarray(c, np.float64) / np.linalg.norm(c)
    x = np.cross([0.0, -1.0, 0.0], z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z])
    return R, -R @ c


def scene(n_cams=4, n_pts=60, seed=0, noise_px=0.0, outlier_frac=0.0, nan_rows=0, fisheye=(), free=(), repeat=0):
    """(cam_flags, cam_const, cam_x, obs_cam, obs_key, obs_px, truth R (n, 3, 3), truth t (n, 3), outlier mask)."""
    rng = np.random.default_rng(seed)
    flags = np.zeros(n_cams, np.int32)
    const = np.zeros((n_cams, 9))
    Rs, ts, xs = [], [], []
    for c in range(n_cams):
        ang = 2 * np.pi * c / n_cams + rng.uniform(-0.1, 0.1)
        R, t = look_at(np.array([3.0 * np.cos(ang), rng.uniform(-0.3, 0.3), 3.0 * np.sin(ang)]))
        Rs.append(R)
        ts.append(t)
        f = rng.uniform(700, 900)
        const[c] = [f, f * rng.uniform(0.98, 1.02), 640 + rng.uniform(-5, 5), 360 + rng.uniform(-5, 5),
                    rng.uniform(-0.05, 0.05), rng.uniform(-0.01, 0.01), 0.0, 0.0, 0.0]  # fmt: skip
        if c in fisheye:
            flags[c] |= 2
            const[c, 4:8] = [0.01, -0.005, 0.001, 0.0]
        if c in free:
            flags[c] |= 1
        q = np.r_[cv2.Rodrigues(R)[0].ravel(), t]
        xs.append(np.r_[q, 1.0, const[c, 4], const[c, 5]] if c in free else q)
    X = rng.uniform(-0.8, 0.8, (n_pts, 3))
    cam, key, px = [], [], []
    for p in range(n_pts):
        for c in range(n_cams):
            K = np.array([[const[c, 0], 0, const[c, 2]], [0, const[c, 1], const[c, 3]], [0, 0, 1.0]])
            rv = cv2.Rodrigues(Rs[c])[0]
            if flags[c] & 2:
                uv = cv2.fisheye.projectPoints(X[p][None, None], rv, ts[c], K, const[c, 4:8])[0].reshape(2)
            else:
                uv = cv2.projectPoints(X[p][None], rv, ts[c], K, const[c, [4, 5, 6, 7, 8]])[0].reshape(2)
            for _ in range(1 + (repeat if p % 7 == 0 and c == 0 else 0)):
                cam.append(c)
                key.append(p)
                px.append(uv + rng.normal(0, noise_px, 2))
    cam, key, px = np.array(cam, np.int32), np.array(key, np.int64), np.array(px)
    out = rng.random(len(px)) < outlier_frac
    px[out] = rng.uniform([0, 0], [1280, 720], (out.sum(), 2))
    if nan_rows:
        px[rng.choice(len(px), nan_rows, replace=False)] = np.nan
    perm = rng.permutation(len(px))
    return flags, const, np.concatenate(xs), cam[perm], key[perm], px[perm], np.array(Rs), np.array(ts), out[perm]


def relative_truth(Rs, ts, a, b):
    """R, unit t of camera b relative to camera a (X_b = R X_a + t)."""
    R = Rs[b] @ Rs[a].T
    t = ts[b] - R @ ts[a]
    return R, t / np.linalg.norm(t)
