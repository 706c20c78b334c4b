"""Sparse scenes for the gP3P tests: rigid bodies whose markers are mostly seen by one camera each, and random ray
configurations for the solver alone."""
from __future__ import annotations

import numpy as np

from oracle.ba_oracle import rodrigues
from oracle.resection_robust import cameras, project, rot_log
from tests._rigid_cases import Bodies, make_bodies

__all__ = ["one_view", "mixed", "sparse_bodies", "ray_case", "on_rays", "ambiguous_three", "branches"]


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


def ambiguous_three(fourth=False, key=0, lone_cam=3):
    """(b, model, obs, truth): one noise-free body of three markers on the rig of make_bodies(5, n_cams=6): A in cameras
    0-2, B in 1, 2, 4 (both triangulated, n_q = 2), C in camera `lone_cam` alone.  Camera lone_cam's centre lies in
    the plane through C at right angles to the line AB, so the circle on which C turns about AB and C's ray lie in one
    plane: the ray meets the circle twice, both times in front of the camera, and the body has two poses that fit every
    row exactly.  fourth: a marker D in camera 5 alone as well, which only the true pose fits."""
    b = make_bodies(5, n_cams=6, n_frames=1, n_model=4, noise=0.0, visible=1.0)
    cams = cameras(*b.rig())
    centre = np.array([-rodrigues(c.q[:3])[0].T @ c.q[3:6] for c in cams])
    O = np.array([0.01, -0.02, 0.015])  # the foot of C on AB
    v = centre[lone_cam] - O
    u = np.cross(v, [0.3, 0.2, 1.0])
    u /= np.linalg.norm(u)  # AB's direction, at right angles to v
    w0 = v / np.linalg.norm(v)
    w1 = np.cross(u, w0)
    a = np.deg2rad(50.0)
    X = np.array([O + 0.09 * u, O - 0.06 * u, O + 0.07 * (np.cos(a) * w0 + np.sin(a) * w1),
                  O + np.array([0.05, 0.06, -0.04])])  # fmt: skip
    R0, t0 = rodrigues(np.array([0.4, -0.3, 0.8]))[0], np.array([0.02, 0.01, -0.03])
    model = (X - t0) @ R0  # R0^T (X - t0)
    rows = [(0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (1, 4), (2, lone_cam)] + ([(3, 5)] if fourth else [])
    oc = np.array([c for _, c in rows], np.int32)
    op = np.array([m for m, _ in rows], np.int32)
    px = np.array([project(cams[c], rodrigues(cams[c].q[:3])[0], cams[c].q[3:6], X[m : m + 1])[0][0] for m, c in rows])
    return b, model, (oc, np.full(len(rows), key, np.int64), op, px), np.r_[rot_log(R0), t0]


def branches(b, model, obs, gate_px=1e-4):
    """The two exact poses (r, t) of ambiguous_three's rows: over the samples (A row, B row, C), gP3P's hypotheses that
    put every row within gate_px of its pixel and in front of its camera, raw (before any refinement), grouped by
    branch; per branch the most exact one, then refined on every row.  The polish of oracle/gp3p.py (at most three
    Newton steps) leaves these hypotheses 3e-5 px from exact: C's ray lies in the plane of its circle, where the two
    branches are roots of one pair."""
    from oracle.gp3p import gp3p
    from oracle.rigid_pose_gp3p import rays
    from oracle.rigid_pose_robust import refine_body
    from oracle.triangulation_robust import row_errors

    oc, _, op, px = obs
    c, d = rays(*b.rig(), oc, px)
    lone = int(np.flatnonzero(op == 2)[0])
    best = []  # [(error px, q)] one per branch
    for ia in np.flatnonzero(op == 0):
        for ib in np.flatnonzero(op == 1):
            s = [int(ia), int(ib), lone]
            for R, t in gp3p(c[s], d[s], model[op[s]]):
                e2, z = row_errors(*b.rig(), oc, px, np.arange(len(oc)), model[op] @ R.T + t)
                err = float(np.sqrt(e2.max()))
                if not (err <= gate_px and (z > 0).all()):
                    continue
                q = np.r_[rot_log(R), t]
                for j, (e0, q0) in enumerate(best):
                    if np.abs(q - q0).max() < 1e-2:
                        if err < e0:
                            best[j] = (err, q)
                        break
                else:
                    best.append((err, q))
    return [refine_body(*b.rig(), oc, px, model[op], q)[0] for _, q in best]
