"""Sparse scenes for the gP3P tests: rigid bodies whose markers are mostly seen by one camera each, and random ray
configurations for the solver alone."""
from __future__ import annotations

import numpy as np

from oracle.ba_oracle import rodrigues
from tests._rigid_cases import Bodies, make_bodies

__all__ = ["one_view", "mixed", "sparse_bodies", "ray_case", "on_rays"]


def one_view(b: Bodies, seed, keys=None) -> Bodies:
    """b with every (frame, marker) of the frames `keys` (None: all) kept in one random camera's row only; b must hold
    every (frame, marker, camera) row (make_bodies with visible=1)."""
    rng = np.random.default_rng(seed)
    n_cams = int(b.obs_cam.max()) + 1
    n_model = len(b.model)
    pick = rng.integers(0, n_cams, size=(int(b.obs_key.max()) + 1, n_model))
    sel = b.obs_cam == pick[b.obs_key, b.obs_pt]
    if keys is not None:
        sel |= ~np.isin(b.obs_key, keys)
    return Bodies(b.flags, b.const, b.cam_x, b.model, b.truth, b.obs_cam[sel], b.obs_key[sel], b.obs_pt[sel],
                  b.obs_px[sel])  # fmt: skip


def mixed(b: Bodies, seed, single_keys, keep) -> Bodies:
    """b (every row present) with the frames `single_keys` seen as ``one_view`` sees them and every row of the other
    frames kept with probability `keep`."""
    v = one_view(b, seed, keys=single_keys)
    rng = np.random.default_rng(seed + 1)
    sel = np.isin(v.obs_key, single_keys) | (rng.random(len(v.obs_key)) < keep)
    return Bodies(v.flags, v.const, v.cam_x, v.model, v.truth, v.obs_cam[sel], v.obs_key[sel], v.obs_pt[sel],
                  v.obs_px[sel])  # fmt: skip


def sparse_bodies(seed, n_cams=6, n_frames=40, n_model=8, *, noise=0.3, visible=0.22, **kw) -> Bodies:
    """A 0.2 m cluster of n_model markers on a ring of n_cams cameras, each (frame, marker, camera) row kept with
    probability `visible`: with 6 cameras and 8 markers at 0.22 about a quarter of the frames have fewer than three
    markers seen by two cameras."""
    return make_bodies(seed, n_cams=n_cams, n_frames=n_frames, n_model=n_model, noise=noise, visible=visible, **kw)


def ray_case(rng, kind):
    """(c, d, M, R, t): three rays through the true world points R M_i + t of a 0.1-scale triangle about 3 units from
    the cameras.  kind: "wide" (each camera anywhere on a sphere of radius 3 about its point), "near" (centres within
    0.1 of one another) or "central" (one centre)."""
    M = rng.uniform(-0.05, 0.05, (3, 3))
    R = rodrigues(rng.normal(size=3))[0]
    t = rng.normal(size=3) * 0.2
    X = M @ R.T + t
    dirs = rng.normal(size=(3, 3))
    dirs /= np.linalg.norm(dirs, axis=1)[:, None]
    if kind == "wide":
        c = X + 3.0 * dirs
    else:
        c = np.tile(X.mean(axis=0) + 3.0 * dirs[0], (3, 1))
        if kind == "near":
            c = c + 0.1 * rng.normal(size=(3, 3))
    d = X - c
    d /= np.linalg.norm(d, axis=1)[:, None]
    return c, d, M, R, t


def on_rays(c, d, M, R, t):
    """Largest distance of R M_i + t from ray i."""
    X = M @ R.T + t - c
    return max(np.linalg.norm(X[i] - (X[i] @ d[i]) * d[i]) for i in range(3))
