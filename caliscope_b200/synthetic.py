"""Seeded array-level rigs of the shapes BASELINE.json names (SURVEY.md section 8d).

Cameras follow the reference's ``CameraSynthesizer().add_ring`` geometry
(/root/reference/src/caliscope/synthetic/camera_synthesizer.py:134-198, inward
facing, Z-up look-at) with the ``WEBCAM`` lens profile (``:23-26``): fx = fy =
1394.6 px, 1920x1080, dist = [0.115, -0.219, 0.0012, 0.0086, 0.113].  Points are
uniform in a cylinder r <= 0.5 m, z in [0, 1.2] m; observations are exact
projections of in-frame points plus N(0, noise_px) noise; the start vector is the
truth perturbed by N(0, 0.005 rad) / N(0, 0.01 m) / N(0, 0.005 m).

This is data synthesis for benchmarks and tests, not part of the solve path.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

WEBCAM_F = 1394.6
WEBCAM_DIST = (0.115, -0.219, 0.0012, 0.0086, 0.113)
WEBCAM_SIZE = (1920, 1080)


@dataclass
class SyntheticRig:
    cam_flags: np.ndarray  # (n_cams,) int32
    cam_const: np.ndarray  # (n_cams, 9) float64
    n_pts: int
    obs_cam: np.ndarray  # (n_obs,) int32
    obs_pt: np.ndarray  # (n_obs,) int32
    obs_xy: np.ndarray  # (n_obs, 2) float64
    x0: np.ndarray  # (n_params,) start vector (BundleParameterization.pack layout)
    x_true: np.ndarray
    outlier_mask: np.ndarray  # (n_obs,) bool
    name: str = ""

    @property
    def n_cams(self) -> int:
        return len(self.cam_flags)

    @property
    def n_obs(self) -> int:
        return len(self.obs_cam)


def _rodrigues_vec(R: np.ndarray) -> np.ndarray:
    """Rotation matrix -> rotation vector (angles here are far from pi)."""
    c = np.clip((np.trace(R) - 1.0) / 2.0, -1.0, 1.0)
    th = np.arccos(c)
    w = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    s = np.linalg.norm(w)
    if s < 1e-12:
        return np.zeros(3)
    return w / s * th


def _rot(r: np.ndarray) -> np.ndarray:
    th = np.linalg.norm(r)
    if th < 1e-12:
        return np.eye(3)
    k = r / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * (K @ K)


def _ring_cameras(n_cams: int):
    per_ring = min(16, n_cams)
    rings = (n_cams + per_ring - 1) // per_ring
    rv, tv = [], []
    for r in range(rings):
        n = min(per_ring, n_cams - r * per_ring)
        radius, height = 2.5 + 0.3 * r, 0.3 + 0.5 * r
        off = np.radians(360.0 / 16.0 / rings * r)
        for i in range(n):
            ang = 2 * np.pi * i / n + off
            pos = np.array([radius * np.cos(ang), radius * np.sin(ang), height])
            fwd = np.array([0.0, 0.0, height]) - pos
            fwd /= np.linalg.norm(fwd)
            right = np.cross(fwd, [0.0, 0.0, 1.0])
            right /= np.linalg.norm(right)
            down = np.cross(fwd, right)
            R = np.stack([right, down, fwd])  # world -> camera
            rv.append(_rodrigues_vec(R))
            tv.append(-R @ pos)
    return np.array(rv), np.array(tv)


def _dome_cameras(n_cams: int):
    """Cameras spread evenly (golden-angle spiral, equal area) over a spherical cap of radius 3 m between 10 and 60
    degrees of elevation around the centre of the point cylinder, each looking at that centre: every camera sees nearly
    every point, so the camera count can grow without cameras that see nothing."""
    centre = np.array([0.0, 0.0, 0.6])
    lo, hi = np.sin(np.radians(10.0)), np.sin(np.radians(60.0))
    rv, tv = [], []
    for i in range(n_cams):
        sz = lo + (hi - lo) * (i + 0.5) / n_cams
        az = i * np.pi * (3.0 - np.sqrt(5.0))
        pos = centre + 3.0 * np.array([np.sqrt(1.0 - sz * sz) * np.cos(az), np.sqrt(1.0 - sz * sz) * np.sin(az), sz])
        fwd = centre - pos
        fwd /= np.linalg.norm(fwd)
        right = np.cross(fwd, [0.0, 0.0, 1.0])
        right /= np.linalg.norm(right)
        down = np.cross(fwd, right)
        R = np.stack([right, down, fwd])  # world -> camera
        rv.append(_rodrigues_vec(R))
        tv.append(-R @ pos)
    return np.array(rv), np.array(tv)


def _project_pinhole(X, rvec, tvec, fx, fy, cx, cy, dist):
    k1, k2, p1, p2, k3 = dist
    Xc = X @ _rot(rvec).T + tvec
    a, b = Xc[:, 0] / Xc[:, 2], Xc[:, 1] / Xc[:, 2]
    r2 = a * a + b * b
    cd = 1 + r2 * (k1 + r2 * (k2 + r2 * k3))
    xd = a * cd + 2 * p1 * a * b + p2 * (r2 + 2 * a * a)
    yd = b * cd + p1 * (r2 + 2 * b * b) + 2 * p2 * a * b
    return np.stack([fx * xd + cx, fy * yd + cy], axis=1), Xc[:, 2]


def make_rig(
    n_cams: int,
    n_pts: int,
    n_obs: int,
    *,
    refine_intrinsics: bool = False,
    seed: int = 0,
    noise_px: float = 0.5,
    outlier_frac: float = 0.0,
    outlier_px: float = 50.0,
    name: str = "",
    cams_per_point: int | None = None,
    layout: str = "ring",
) -> SyntheticRig:
    """``layout``: "ring" -- rings of 16 inward-facing cameras stacked upward (above the fifth ring the cameras see
    almost no points); "dome" -- cameras over a spherical cap, each seeing nearly every point (``_dome_cameras``).
    ``cams_per_point``: local visibility -- every point faces a random azimuth and is seen only by the
    ``cams_per_point`` in-frame cameras nearest to that direction (a marker on a subject inside a ring rig: the
    realistic Caliscope shape, 2-8 cameras per point), instead of by a uniform random subset of all cameras."""
    if layout not in ("ring", "dome"):
        raise ValueError(f"layout must be 'ring' or 'dome', got {layout!r}")
    rng = np.random.default_rng(seed)
    rvec, tvec = _ring_cameras(n_cams) if layout == "ring" else _dome_cameras(n_cams)
    w, h = WEBCAM_SIZE
    cx, cy = w / 2.0, h / 2.0

    rad = 0.5 * np.sqrt(rng.uniform(0, 1, n_pts))
    ang = rng.uniform(0, 2 * np.pi, n_pts)
    X = np.stack([rad * np.cos(ang), rad * np.sin(ang), rng.uniform(0, 1.2, n_pts)], axis=1)

    # all in-frame (cam, pt) pairs, camera-major
    pair_cam, pair_pt, pair_uv = [], [], []
    for c in range(n_cams):
        uv, z = _project_pinhole(X, rvec[c], tvec[c], WEBCAM_F, WEBCAM_F, cx, cy, WEBCAM_DIST)
        ok = (z > 0) & (uv[:, 0] >= 0) & (uv[:, 0] < w) & (uv[:, 1] >= 0) & (uv[:, 1] < h)
        idx = np.nonzero(ok)[0]
        pair_cam.append(np.full(len(idx), c, np.int32))
        pair_pt.append(idx.astype(np.int32))
        pair_uv.append(uv[idx])
    pair_cam = np.concatenate(pair_cam)
    pair_pt = np.concatenate(pair_pt)
    pair_uv = np.concatenate(pair_uv)
    if cams_per_point is not None:
        cam_pos = np.array([-_rot(rvec[c]).T @ tvec[c] for c in range(n_cams)])
        cam_az = np.arctan2(cam_pos[:, 1], cam_pos[:, 0])
        facing = rng.uniform(-np.pi, np.pi, n_pts)
        d = np.abs(np.angle(np.exp(1j * (cam_az[pair_cam] - facing[pair_pt]))))
        order = np.lexsort((d, pair_pt))  # by point, nearest camera first
        pt_sorted = pair_pt[order]
        first = np.searchsorted(pt_sorted, np.arange(n_pts))
        rank_in_pt = np.arange(len(order)) - first[pt_sorted]
        keep = np.sort(order[rank_in_pt < cams_per_point])  # back to camera-major order
        pair_cam, pair_pt, pair_uv = pair_cam[keep], pair_pt[keep], pair_uv[keep]
    n_pairs = len(pair_cam)
    if n_obs <= n_pairs:
        sel = np.sort(rng.permutation(n_pairs)[:n_obs])
    else:  # repeated (cam, pt) rows: static-object style observations
        sel = np.sort(np.concatenate([np.arange(n_pairs), rng.integers(0, n_pairs, n_obs - n_pairs)]))
    obs_cam, obs_pt = pair_cam[sel], pair_pt[sel]
    obs_xy = pair_uv[sel] + rng.normal(0, noise_px, (n_obs, 2))
    outlier = np.zeros(n_obs, bool)
    if outlier_frac > 0:
        outlier = rng.uniform(0, 1, n_obs) < outlier_frac
        obs_xy[outlier] += rng.uniform(-outlier_px, outlier_px, (int(outlier.sum()), 2))

    f0 = WEBCAM_F * (1.02 if refine_intrinsics else 1.0)
    const = np.tile(np.array([f0, f0, cx, cy, *WEBCAM_DIST]), (n_cams, 1))
    flags = np.full(n_cams, 1 if refine_intrinsics else 0, np.int32)
    cam_true, cam0 = [], []
    for c in range(n_cams):
        r0 = rvec[c] + rng.normal(0, 0.005, 3)
        t0 = tvec[c] + rng.normal(0, 0.01, 3)
        if refine_intrinsics:
            cam_true.append(np.concatenate([rvec[c], tvec[c], [1 / 1.02, WEBCAM_DIST[0], WEBCAM_DIST[1]]]))
            cam0.append(np.concatenate([r0, t0, [1.0, WEBCAM_DIST[0], WEBCAM_DIST[1]]]))
        else:
            cam_true.append(np.concatenate([rvec[c], tvec[c]]))
            cam0.append(np.concatenate([r0, t0]))
    X0 = X + rng.normal(0, 0.005, X.shape)
    return SyntheticRig(
        cam_flags=flags,
        cam_const=const,
        n_pts=n_pts,
        obs_cam=obs_cam,
        obs_pt=obs_pt,
        obs_xy=obs_xy,
        x0=np.concatenate(cam0 + [X0.ravel()]),
        x_true=np.concatenate(cam_true + [X.ravel()]),
        outlier_mask=outlier,
        name=name,
    )


# BASELINE.json configs 2..5
def cfg2(seed: int = 0) -> SyntheticRig:
    return make_rig(8, 2000, 40_000, seed=seed, name="cfg2 8-cam/2k-pt/40k-obs extrinsics-only")


def cfg3(seed: int = 0) -> SyntheticRig:
    return make_rig(16, 10_000, 400_000, refine_intrinsics=True, seed=seed,
                    name="cfg3 16-cam/10k-pt/400k-obs extrinsics+intrinsics+distortion")  # fmt: skip


def cfg4(seed: int = 0, refine_intrinsics: bool = False) -> SyntheticRig:
    return make_rig(64, 50_000, 2_000_000, refine_intrinsics=refine_intrinsics, seed=seed,
                    name="cfg4 64-cam/50k-pt/2M-obs" + (" +intrinsics" if refine_intrinsics else " extrinsics-only"))  # fmt: skip


def cfg5(seed: int = 0) -> SyntheticRig:
    return make_rig(64, 50_000, 2_000_000, seed=seed, outlier_frac=0.02,
                    name="cfg5 64-cam/50k-pt/2M-obs + 2% outliers (filter + re-solve loop)")  # fmt: skip


def sparse64(seed: int = 0) -> SyntheticRig:
    """64 cameras / 250 000 points / 2 000 000 observations with 8 cameras per point (local visibility): the same
    observation count as cfg4 at the camera-per-point density of real Caliscope sessions."""
    return make_rig(64, 250_000, 2_000_000, seed=seed, cams_per_point=8,
                    name="sparse64 64-cam/250k-pt/2M-obs, 8 cameras per point (local visibility)")  # fmt: skip


def exact_normalized_observations(rig: SyntheticRig):
    """Inputs of the triangulation step for a rig: normalised projection matrices ``[R|t]`` of the TRUE
    poses, (n_cams,3,4), and the exact normalised image coordinates ``(Xc.x/Xc.z, Xc.y/Xc.z)`` of every
    observation row (what undistortion of noise-free pixels would give)."""
    P = np.where(rig.cam_flags & 1, 9, 6)
    off = np.concatenate([[0], np.cumsum(P)])
    proj = np.empty((rig.n_cams, 3, 4))
    for c in range(rig.n_cams):
        blk = rig.x_true[off[c] : off[c] + 6]
        proj[c, :, :3] = _rot(blk[:3])
        proj[c, :, 3] = blk[3:6]
    X = rig.x_true[off[-1] :].reshape(-1, 3)
    Xc = np.einsum("nij,nj->ni", proj[rig.obs_cam, :, :3], X[rig.obs_pt]) + proj[rig.obs_cam, :, 3]
    return proj, np.ascontiguousarray(Xc[:, :2] / Xc[:, 2:3])


@dataclass
class BoardSession:
    """Synthetic input of the extrinsic bootstrap: a planar calibration board seen by a ring rig over many frames --
    the columns of ``ImagePoints`` (reference core/point_data.py) as arrays, plus the camera tables."""

    cam_ids: np.ndarray  # (n_cams,)
    cam_k: np.ndarray  # (n_cams, 5) fx fy cx cy skew
    cam_dist: np.ndarray  # (n_cams, 12)
    cam_fisheye: np.ndarray  # (n_cams,) int32
    rvec: np.ndarray  # true world -> camera poses
    tvec: np.ndarray
    sync_index: np.ndarray
    cam_id: np.ndarray
    object_id: np.ndarray
    keypoint_id: np.ndarray
    img_xy: np.ndarray  # (n, 2) distorted pixels + noise
    obj_xyz: np.ndarray  # (n, 3) board-frame coordinates, z = 0

    @property
    def n_obs(self) -> int:
        return len(self.cam_id)


def make_board_session(n_cams: int = 64, n_frames: int = 1000, grid=(7, 5), square: float = 0.06, seed: int = 0,
                       noise_px: float = 0.3) -> BoardSession:  # fmt: skip
    """A ``grid`` of corners on a board of ``square`` metres moves through the capture volume; in every frame the cameras
    that look at its front side (normal within 70 degrees of the viewing ray) and have every corner in frame observe all
    corners.  Pinhole WEBCAM lens (Brown-Conrady), 0.3 px noise."""
    rng = np.random.default_rng(seed)
    rvec, tvec = _ring_cameras(n_cams)
    w, h = WEBCAM_SIZE
    cx, cy = w / 2.0, h / 2.0
    gx, gy = np.meshgrid(np.arange(grid[0]), np.arange(grid[1]), indexing="ij")
    corners = np.stack([gx.ravel() * square, gy.ravel() * square, np.zeros(gx.size)], axis=1)
    centre = corners.mean(axis=0)
    Rc = np.array([_rot(r) for r in rvec])
    cam_pos = np.array([-Rc[c].T @ tvec[c] for c in range(n_cams)])
    cols = {k: [] for k in ("sync", "cam", "kp", "xy", "obj")}
    for f in range(n_frames):
        pos = np.array([rng.uniform(-0.35, 0.35), rng.uniform(-0.35, 0.35), rng.uniform(0.2, 1.0)])
        az = rng.uniform(0, 2 * np.pi)
        tilt = rng.normal(0, 0.35, 2)
        # board z axis roughly horizontal, pointing at azimuth az
        zb = np.array([np.cos(az), np.sin(az), 0.0])
        xb = np.cross([0.0, 0.0, 1.0], zb)
        xb /= np.linalg.norm(xb)
        yb = np.cross(zb, xb)
        Rb = np.stack([xb, yb, zb], axis=1) @ _rot(np.array([tilt[0], tilt[1], rng.uniform(-0.5, 0.5)]))
        Xw = (corners - centre) @ Rb.T + pos
        normal = Rb[:, 2]
        for c in range(n_cams):
            view = cam_pos[c] - pos
            if normal @ view / np.linalg.norm(view) < np.cos(np.radians(70)):
                continue
            uv, z = _project_pinhole(Xw, rvec[c], tvec[c], WEBCAM_F, WEBCAM_F, cx, cy, WEBCAM_DIST)
            if not ((z > 0).all() and (uv[:, 0] >= 0).all() and (uv[:, 0] < w).all() and (uv[:, 1] >= 0).all() and (uv[:, 1] < h).all()):
                continue
            n = len(corners)
            cols["sync"].append(np.full(n, f, np.int64)); cols["cam"].append(np.full(n, c, np.int64))
            cols["kp"].append(np.arange(n, dtype=np.int64)); cols["xy"].append(uv + rng.normal(0, noise_px, uv.shape))
            cols["obj"].append(corners.copy())
    k = np.tile([WEBCAM_F, WEBCAM_F, cx, cy, 0.0], (n_cams, 1))
    dist = np.zeros((n_cams, 12))
    dist[:, :5] = WEBCAM_DIST
    cat = {kk: np.concatenate(v) for kk, v in cols.items()}
    return BoardSession(np.arange(n_cams, dtype=np.int64), k, dist, np.zeros(n_cams, np.int32), rvec, tvec, cat["sync"], cat["cam"],
                        np.zeros(len(cat["cam"]), np.int64), cat["kp"], cat["xy"], cat["obj"])  # fmt: skip
