"""Seeded planar-board views of synthetic cameras for the intrinsic-calibration tests (CPU oracle and GPU)."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from oracle.ba_oracle import rodrigues

WEBCAM = (1920, 1080, np.array([1400.0, 1405.0, 962.0, 538.0, 0.08, -0.15, 0.0008, -0.0006, 0.02]))
STRONG = (1280, 800, np.array([620.0, 618.0, 645.0, 395.0, -0.30, 0.09, 0.0015, 0.0010, -0.012]))


def board(cols=9, rows=6, square=0.03):
    """54-corner chessboard (9 x 6 inner corners) in the board frame, z = 0."""
    g = np.stack(np.meshgrid(np.arange(cols), np.arange(rows)), -1).reshape(-1, 2) * square
    return np.concatenate([g, np.zeros((len(g), 1))], 1)


@dataclass
class Case:
    obs_cam: np.ndarray
    obs_key: np.ndarray
    obs_obj: np.ndarray
    obs_px: np.ndarray
    image_size: np.ndarray  # (C, 2)
    truth: np.ndarray  # (C, 9)


def project(theta, R, t, X):
    fx, fy, cx, cy, k1, k2, p1, p2, k3 = theta
    Xc = X @ R.T + t
    a, b = Xc[:, 0] / Xc[:, 2], Xc[:, 1] / Xc[:, 2]
    r2 = a * a + b * b
    cd = 1 + r2 * (k1 + r2 * (k2 + r2 * k3))
    xd = a * cd + 2 * p1 * a * b + p2 * (r2 + 2 * a * a)
    yd = b * cd + p1 * (r2 + 2 * b * b) + 2 * p2 * a * b
    return np.stack([fx * xd + cx, fy * yd + cy], 1)


def make_views(rng, w, h, theta, n_views, X):
    """Board poses that keep every corner in the image, seen from 0.35-0.9 m with tilts up to ~40 degrees."""
    out = []
    ctr = X.mean(0)
    while len(out) < n_views:
        r = rng.normal(0, 0.35, 3)
        r[2] = rng.uniform(-0.4, 0.4)
        R = rodrigues(r)[0]
        z = rng.uniform(0.35, 0.9)
        xy = rng.uniform(-0.25, 0.25, 2) * z
        t = np.array([xy[0], xy[1], z]) - R @ ctr
        uv = project(theta, R, t, X)
        Xc = X @ R.T + t
        if (Xc[:, 2] > 0.1).all() and (uv[:, 0] > 5).all() and (uv[:, 0] < w - 6).all() and (uv[:, 1] > 5).all() \
                and (uv[:, 1] < h - 6).all():
            out.append(uv)
    return out


def make_case(seed, lenses, n_views, noise=0.5, X=None) -> Case:
    """One call's rows: lenses = [(w, h, theta)] per camera, n_views per camera (int or list), keys camera-major with
    the views of different cameras interleaved in key order."""
    rng = np.random.default_rng(seed)
    X = board() if X is None else X
    nv = [n_views] * len(lenses) if np.isscalar(n_views) else list(n_views)
    cam, key, obj, px = [], [], [], []
    for c, (w, h, th) in enumerate(lenses):
        for v, uv in enumerate(make_views(rng, w, h, th, nv[c], X)):
            cam.append(np.full(len(X), c, np.int32))
            key.append(np.full(len(X), v * len(lenses) + c, np.int64))
            obj.append(X.astype(np.float32).astype(np.float64))  # what cv2 sees (float32 inputs)
            px.append((uv + rng.normal(0, noise, uv.shape)).astype(np.float32).astype(np.float64))
    perm = rng.permutation(sum(len(k) for k in key))
    cat = lambda a: np.concatenate(a)[perm]  # noqa: E731
    return Case(cat(cam), cat(key), cat(obj), cat(px), np.array([[w, h] for w, h, _ in lenses], np.int32),
                np.array([th for _, _, th in lenses]))


def cv2_views(case: Case, cam: int, keys=None):
    """objectPoints / imagePoints lists of one camera in key order (float32 objects, float64 pixels as cv2 takes them)."""
    sel = case.obs_cam == cam
    ks = np.unique(case.obs_key[sel]) if keys is None else keys
    objs, imgs = [], []
    for k in ks:
        rows = np.flatnonzero(case.obs_key == k)
        objs.append(case.obs_obj[rows].astype(np.float32))
        imgs.append(case.obs_px[rows].reshape(-1, 1, 2).astype(np.float32))
    return objs, imgs, ks


def camera_status_case():
    """Three cameras of a 1920 x 1080 pinhole lens without distortion, one per camera status the rule can reach before
    the loop: camera 0 has one view (status 1); cameras 1 and 2 see the board fronto-parallel in four views, where
    Zhang's system is singular (camera 1, no guess: status 2) and, from a guess, S loses rank at the solution (camera 2:
    status 3).  Returns (case, cam_flags in the oracle's convention, guess)."""
    from oracle.intrinsics import USE_GUESS

    X = board()
    th = WEBCAM[2].copy()
    th[4:] = 0.0

    def view(t):
        Xc = X + t
        return np.c_[th[0] * Xc[:, 0] / Xc[:, 2] + th[2], th[1] * Xc[:, 1] / Xc[:, 2] + th[3]]

    one = [view(np.array([-0.1, -0.08, 0.6]))]
    par = [view(np.array([-0.1 + 0.02 * k, -0.08, 0.5 + 0.1 * k])) for k in range(4)]
    rows = [(0, 0, one[0])] + [(1, 1 + k, u) for k, u in enumerate(par)] + [(2, 10 + k, u) for k, u in enumerate(par)]
    case = Case(np.concatenate([np.full(len(X), c, np.int32) for c, _, _ in rows]),
                np.concatenate([np.full(len(X), k, np.int64) for _, k, _ in rows]), np.concatenate([X] * len(rows)),
                np.concatenate([u for _, _, u in rows]), np.array([[1920, 1080]] * 3, np.int32), np.array([th] * 3))
    guess = np.full((3, 9), np.nan)
    guess[2] = th
    return case, np.array([0, 0, USE_GUESS]), guess
