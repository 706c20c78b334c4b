"""Relative pose of every camera pair from 2-D correspondences alone: five-point consensus on the Sampson distance,
refinement to its optimum and a covariance on the GPU (``cb_relative_pose_robust``, DESIGN.md section 4.11).  The route
to a first extrinsic calibration when no board is in view (wand or body keypoints with ``obj_loc_*`` all NaN)."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import _lib as L
from .triangulation import _calibrated_inputs, _ptr
from .uncertainty import PoseUncertainty, pose_from_extrinsics


@dataclass
class PairPoses:
    """Per camera pair with a correspondence, in ascending (cam_a, cam_b).  pose = (r, t): X_b = R X_a + t with |t| = 1
    (the baseline's direction; its length is not observable from 2-D correspondences).  status: 0 ok, 1 fewer than
    min_inliers correspondences, 2 not positive definite (pose is the winning hypothesis, cov NaN), 3 iteration limit,
    4 a consensus correspondence behind a camera at the solution, 5 no consensus (pose, cov, rmse, parallax NaN)."""

    cam_a: np.ndarray  # (P,) int32
    cam_b: np.ndarray  # (P,) int32
    pose: np.ndarray  # (P, 6)
    cov: np.ndarray  # (P, 6, 6), rank 5
    rmse_px: np.ndarray  # (P,) Sampson distance over the consensus set
    parallax_deg: np.ndarray  # (P,) mean angle between R x_a and x_b over the consensus set
    count: np.ndarray  # (P,) int32, every correspondence of the pair
    n_inliers: np.ndarray  # (P,) int32
    status: np.ndarray  # (P,) int32

    def uncertainty(self) -> list[PoseUncertainty | None]:
        """Position and orientation uncertainty of camera b in camera a's frame (``uncertainty.pose_from_extrinsics``),
        None where the covariance is NaN."""
        out: list[PoseUncertainty | None] = []
        for p, c in zip(self.pose, self.cov):
            out.append(None if not np.isfinite(c).all() else pose_from_extrinsics(p[:3], p[3:], c))
        return out


@dataclass
class RelPoseStats:
    group_ms: float = 0.0
    consensus_ms: float = 0.0
    refine_ms: float = 0.0
    cov_ms: float = 0.0
    total_ms: float = 0.0
    kernel_launches: int = 0
    n_pairs: int = 0


def relative_poses_robust(cam_flags, cam_const, obs_cam, obs_key, obs_px, *, cam_x=None, threshold_px: float,
                          min_inliers: int = 15, max_samples: int = 64, pixel_sigma: float = 1.0, max_iter: int = 20,
                          xtol: float = 1e-12, device: int = 0, stream: int = 0,
                          stats: RelPoseStats | None = None) -> PairPoses:  # fmt: skip
    """Relative pose of every camera pair that shares observations (``cb_relative_pose_robust``, DESIGN.md 4.11).

    The cameras are ``BAProblem.cam_flags`` and ``BAProblem.cam_const``; ``cam_x`` (the camera section of x) supplies
    the scale and k1, k2 of free-intrinsics cameras, and its poses are ignored.  Without it those come from the
    constants (s = 1).  Rows with equal ``obs_key`` are one world point; ``obs_px`` are raw pixels.  The observations may
    be host arrays or CUDA tensors on ``device`` (obs_cam int32, obs_key int64, obs_px float64 (n, 2)), read in place.

    Two rows of one key from different cameras are a correspondence of their pair.  Inside each pair, the five-point
    essential matrices of up to ``max_samples`` 5-samples are scored by MSAC on the Sampson distance in undistorted
    pixels, sum min(e^2, threshold_px^2); the lowest score wins.  The correspondences within ``threshold_px`` and in front
    of both cameras are the consensus set (fewer than ``min_inliers``: status 5); the pose is refined on them alone and
    its covariance is ``pixel_sigma^2 H^-1`` in a chart of the unit baseline, returned over (r, t)."""
    if not (np.isfinite(threshold_px) and threshold_px > 0):
        raise ValueError(f"threshold_px must be finite and > 0, got {threshold_px}")
    if int(min_inliers) < 5:
        raise ValueError(f"min_inliers must be >= 5, got {min_inliers}")
    if not 1 <= int(max_samples) <= 4096:
        raise ValueError(f"max_samples must be in 1..4096, got {max_samples}")
    if not (np.isfinite(pixel_sigma) and pixel_sigma >= 0):
        raise ValueError(f"pixel_sigma must be finite and >= 0, got {pixel_sigma}")
    if int(max_iter) < 1:
        raise ValueError(f"max_iter must be >= 1, got {max_iter}")
    if not (np.isfinite(xtol) and xtol >= 0):
        raise ValueError(f"xtol must be finite and >= 0, got {xtol}")
    if cam_x is None:
        flags = np.asarray(cam_flags, np.int32).ravel()
        const = np.asarray(cam_const, np.float64).reshape(len(flags), 9)
        blocks = [np.r_[np.zeros(6), 1.0, const[c, 4], const[c, 5]] if f & L.CB_CAM_FREE_INTRINSICS else np.zeros(6)
                  for c, f in enumerate(flags)]  # fmt: skip
        cam_x = np.concatenate(blocks) if blocks else np.zeros(0)
    lib = L.load()
    nc, flags, const, cx, _, n, on_dev, (cam_p, key_p, px_p), _keep = _calibrated_inputs(
        cam_flags, cam_const, cam_x, None, obs_cam, obs_key, obs_px, device)
    m = max(nc * (nc - 1) // 2, 1)  # at most one output per camera pair
    pose, cov, rmse, par = np.empty((m, 6)), np.empty((m, 6, 6)), np.empty(m), np.empty(m)
    ca, cb, count, nin, status = (np.empty(m, np.int32) for _ in range(5))
    npairs = C.c_int32(0)
    st = L.RelPoseStats()
    L.check(
        lib.cb_relative_pose_robust(nc, _ptr(flags), _ptr(const), _ptr(cx), n, cam_p, key_p, px_p, 1 if on_dev else 0,
                                    float(threshold_px), int(min_inliers), int(max_samples), float(pixel_sigma),
                                    int(max_iter), float(xtol), m, C.byref(npairs), _ptr(ca), _ptr(cb), _ptr(pose),
                                    _ptr(cov), _ptr(rmse), _ptr(par), _ptr(count), _ptr(nin), _ptr(status), C.byref(st),
                                    int(device), C.c_void_p(stream)),
        "relative_poses_robust",
    )  # fmt: skip
    p = npairs.value
    if stats is not None:
        stats.group_ms, stats.consensus_ms, stats.refine_ms = st.group_ms, st.consensus_ms, st.refine_ms
        stats.cov_ms, stats.total_ms, stats.kernel_launches, stats.n_pairs = st.cov_ms, st.total_ms, st.kernel_launches, p
    return PairPoses(cam_a=ca[:p], cam_b=cb[:p], pose=pose[:p], cov=cov[:p], rmse_px=rmse[:p], parallax_deg=par[:p],
                     count=count[:p], n_inliers=nin[:p], status=status[:p])  # fmt: skip


def _rot(r) -> np.ndarray:
    r = np.asarray(r, np.float64)
    th = float(np.sqrt(r @ r))
    K = np.array([[0.0, -r[2], r[1]], [r[2], 0.0, -r[0]], [-r[1], r[0], 0.0]])
    if th < 1e-12:
        return np.eye(3) + K
    return np.eye(3) + np.sin(th) / th * K + (1.0 - np.cos(th)) / th**2 * (K @ K)


def _log(R) -> np.ndarray:
    """Rotation vector of R, theta in [0, pi]."""
    c = float(np.clip((np.trace(R) - 1.0) * 0.5, -1.0, 1.0))
    th = float(np.arccos(c))
    v = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    s = 0.5 * float(np.linalg.norm(v))
    if s > 1e-7:
        return v * (th / (2.0 * s))
    if c > 0:
        return 0.5 * v
    w, V = np.linalg.eigh(0.5 * (R + R.T))  # theta near pi: the axis is R's +1 eigenvector
    a = V[:, np.argmax(w)]
    if a @ v < 0:
        a = -a
    return a * th


@dataclass
class EpipolarStart:
    """A posed rig from 2-D correspondences alone, in the gauge camera seed_a = identity at the origin and a distance
    of 1 between the centres of seed_a and seed_b.  ``x`` is in the bundle-adjustment layout (every camera's block, then
    the points); cameras never posed keep a zero pose and ``posed`` False.  ``obs_cam`` / ``obs_pt`` / ``obs_xy`` are the
    consensus rows of the last bundle adjustment (rows of unposed cameras dropped), ready for ``BAProblem`` with
    ``n_pts = len(pt_key)``; ``pt_key[p]`` is the obs_key of point p and ``obs_row`` the caller row of each row."""

    x: np.ndarray
    posed: np.ndarray  # (n_cams,) bool
    obs_cam: np.ndarray  # (m,) int32
    obs_pt: np.ndarray  # (m,) int32
    obs_xy: np.ndarray  # (m, 2)
    obs_row: np.ndarray  # (m,) int64, caller row
    pt_key: np.ndarray  # (n_pts,) int64
    seed: tuple  # (a, b)
    rounds: list  # cameras added by each resection round
    rmse_px: float  # RMSE of the last bundle adjustment
    pairs: PairPoses


def epipolar_start(cam_flags, cam_const, obs_cam, obs_key, obs_px, *, threshold_px: float, min_inliers: int = 15,
                   min_parallax_deg: float = 1.0, max_samples: int = 64, device: int = 0) -> EpipolarStart:  # fmt: skip
    """A first calibration of the extrinsics from 2-D correspondences alone (rows with equal obs_key are one world
    point), every step on the GPU through the existing device calls:
      1. ``relative_poses_robust`` of every camera pair.
      2. Seed pair: among the pairs with status 0 and parallax_deg >= min_parallax_deg, the most n_inliers (ties to the
         lowest (a, b)); ValueError when there is none.  Camera a is the identity, b the pair's (r, t).
      3. ``triangulation.triangulate_robust`` on the rows of the posed cameras, over keys with at least two posed rows;
         then one bundle adjustment (``BAProblem``, linear loss) of the posed cameras and the status-0 points on those
         points' consensus rows.
      4. Each round, ``resection.resect_robust`` (key = camera, no prior) of every unposed camera against the status-0
         points; a camera with status 0 and at least min_inliers inliers is posed.  None: stop; else step 3 again.
      5. The gauge: camera a at the origin with the identity rotation, |C_a - C_b| = 1.
    The scale is the seed baseline's: Caliscope's scale and origin tools apply afterwards."""
    from .problem import BAProblem
    from .resection import resect_robust
    from .triangulation import triangulate_robust

    flags = np.asarray(cam_flags, np.int32).ravel()
    nc = len(flags)
    const = np.asarray(cam_const, np.float64).reshape(nc, 9)
    cam = np.ascontiguousarray(obs_cam, dtype=np.int32)
    key = np.ascontiguousarray(obs_key, dtype=np.int64)
    px = np.ascontiguousarray(obs_px, dtype=np.float64).reshape(-1, 2)
    pairs = relative_poses_robust(flags, const, cam, key, px, threshold_px=threshold_px, min_inliers=min_inliers,
                                  max_samples=max_samples, device=device)  # fmt: skip
    ok = np.flatnonzero((pairs.status == 0) & (pairs.parallax_deg >= min_parallax_deg))
    if len(ok) == 0:
        raise ValueError("no camera pair with status 0 and enough parallax to seed the rig")
    s = int(ok[np.argmax(pairs.n_inliers[ok])])  # argmax keeps the first of equal counts: the lowest (a, b)
    a, b = int(pairs.cam_a[s]), int(pairs.cam_b[s])
    width = np.where(flags & L.CB_CAM_FREE_INTRINSICS, 9, 6)
    off = np.r_[0, np.cumsum(width)]
    cx = np.zeros(off[-1])
    for c in range(nc):
        if flags[c] & L.CB_CAM_FREE_INTRINSICS:
            cx[off[c] + 6 : off[c] + 9] = (1.0, const[c, 4], const[c, 5])
    cx[off[b] : off[b] + 6] = pairs.pose[s]
    posed = np.zeros(nc, bool)
    posed[[a, b]] = True
    rounds: list = []
    while True:
        # step 3: points from the posed cameras' rows, then one bundle adjustment
        rows = np.flatnonzero(posed[cam])
        uk, inv, cnt = np.unique(key[rows], return_inverse=True, return_counts=True)
        rows = rows[cnt[inv] >= 2]
        tri = triangulate_robust(flags, const, cx, cam[rows], key[rows], px[rows], threshold_px=threshold_px,
                                 device=device)  # fmt: skip
        gkeys, ginv = np.unique(key[rows], return_inverse=True)
        good = tri.status == 0
        keep = tri.inlier & good[ginv]
        pt_key = gkeys[good]
        pt_of_group = np.cumsum(good) - 1
        brows = rows[keep]
        bpt = pt_of_group[ginv[keep]].astype(np.int32)
        sub = np.flatnonzero(posed)
        slot = np.full(nc, -1)
        slot[sub] = np.arange(len(sub))
        sflags = flags[sub]
        x0 = np.concatenate([cx[off[c] : off[c + 1]] for c in sub] + [tri.xyz[good].ravel()])
        with BAProblem(sflags, const[sub], len(pt_key), slot[cam[brows]].astype(np.int32), bpt, px[brows],
                       device=device) as prob:  # fmt: skip
            res = prob.solve(x0)
            rmse = prob.overall_rmse_px(res.x)
        o = 0
        for c in sub:
            cx[off[c] : off[c + 1]] = res.x[o : o + width[c]]
            o += width[c]
        pts = res.x[o:].reshape(-1, 3)
        # step 4: resection of the unposed cameras against the points
        unposed = ~posed
        pos = np.searchsorted(pt_key, key)
        pos = np.minimum(pos, len(pt_key) - 1)
        hit = unposed[cam] & (pt_key[pos] == key) if len(pt_key) else np.zeros(len(key), bool)
        rrows = np.flatnonzero(hit)
        added = []
        if len(rrows):
            rs = resect_robust(flags, const, cx, pts, cam[rrows], cam[rrows].astype(np.int64), pos[rrows].astype(np.int32),
                               px[rrows], threshold_px=threshold_px, min_inliers=max(4, min_inliers), use_prior=False,
                               device=device)  # fmt: skip
            for g in range(len(rs.cam)):
                if rs.status[g] == 0 and rs.n_inliers[g] >= min_inliers:
                    c = int(rs.cam[g])
                    cx[off[c] : off[c] + 6] = rs.pose[g]
                    added.append(c)
        if not added:
            break
        posed[added] = True
        rounds.append(sorted(added))
    # step 5: the gauge, X' = k (R_a X + t_a) with k = 1 / |C_a - C_b|
    Ra, ta = _rot(cx[off[a] : off[a] + 3]), cx[off[a] + 3 : off[a] + 6]
    Rb, tb = _rot(cx[off[b] : off[b] + 3]), cx[off[b] + 3 : off[b] + 6]
    k = 1.0 / float(np.linalg.norm(Ra.T @ ta - Rb.T @ tb))
    for c in np.flatnonzero(posed):
        Rc, tc = _rot(cx[off[c] : off[c] + 3]), cx[off[c] + 3 : off[c] + 6]
        Rn = Rc @ Ra.T
        cx[off[c] : off[c] + 3] = _log(Rn)
        cx[off[c] + 3 : off[c] + 6] = k * (tc - Rn @ ta)
    pts = k * (pts @ Ra.T + ta)
    return EpipolarStart(x=np.concatenate([cx, pts.ravel()]), posed=posed, obs_cam=cam[brows], obs_pt=bpt,
                         obs_xy=px[brows], obs_row=brows.astype(np.int64), pt_key=pt_key, seed=(a, b), rounds=rounds,
                         rmse_px=rmse, pairs=pairs)  # fmt: skip
