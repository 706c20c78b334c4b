"""CPU restatement of the reference's extrinsic bootstrap, stage by stage.  TEST INFRASTRUCTURE ONLY.

Follows /root/reference/src/caliscope/core/bootstrap_pose/pose_network_builder.py:
  compute_camera_to_object_poses_pnp :211-330, compute_relative_poses :488-534, reject_outliers :333-411,
  quaternion_average :414-437, rotation_error :441-455, aggregate_poses :537-575,
  _precompute_common_observations :576-603, calculate_stereo_rmse_for_pair :638-685
and paired_pose_network.py:26-99 (gap filling).  OpenCV calls are replaced by oracle.ippe (planar PnP) and the
two-view DLT below; everything is plain loops over small fixtures.  Pinned by tests/golden/bootstrap_*.npz, produced by
the unmodified reference (tests/golden/make_bootstrap_golden.py).
"""
from __future__ import annotations

from itertools import combinations, permutations

import numpy as np

from . import ippe
from .triangulation import undistort_points


def undistort_all(cam_ids, cam_k, cam_dist, cam_fisheye, obs_cam_id, img_xy) -> np.ndarray:
    """Normalised, float32-rounded coordinates of every row (camera_array.py:135-174)."""
    out = np.full((len(obs_cam_id), 2), np.nan)
    for i, c in enumerate(cam_ids):
        sel = obs_cam_id == c
        if not sel.any():
            continue
        K = np.array([[cam_k[i, 0], cam_k[i, 4], cam_k[i, 2]], [0, cam_k[i, 1], cam_k[i, 3]], [0, 0, 1.0]])
        d = cam_dist[i, :4] if cam_fisheye[i] else cam_dist[i, :5]
        out[sel] = undistort_points(img_xy[sel], K, d, bool(cam_fisheye[i]), "normalized")
    return out


def pnp_poses(cam_ids, norm_xy, sync_index, obs_cam_id, object_id, obj_xyz, min_points: int = 4, fallback_keys: list | None = None):
    """dict (cam_id, sync_index, object_id) -> (R, t, rmse), in sorted key order (pandas groupby order)."""
    keys = sorted(set(zip(obs_cam_id.tolist(), sync_index.tolist(), object_id.tolist())))
    poses = {}
    known = set(int(c) for c in cam_ids)
    for c, s, o in keys:
        if c not in known:
            continue
        sel = (obs_cam_id == c) & (sync_index == s) & (object_id == o)
        obj = obj_xyz[sel].copy()
        obj[:, 2] = np.nan_to_num(obj[:, 2], nan=0.0)
        if not np.ptp(obj[:, 2]) < 1e-6:
            raise NotImplementedError("non-planar PnP group (the reference switches to SQPNP)")
        if sel.sum() < min_points:
            continue
        R, t, fb = ippe.solve_pnp_planar(obj, norm_xy[sel])
        poses[(c, s, o)] = (R, t, ippe.pnp_reprojection_rmse(obj, norm_xy[sel], R, t) if np.isfinite(R).all() else np.nan)
        if fallback_keys is not None and fb:
            fallback_keys.append((c, s, o))
    return poses


def relative_poses(poses: dict, cam_ids, cam_ignore):
    """dict ((a, b), sync, object) -> (R_rel, t_rel): T_B_A = T_B_obj inv(T_A_obj).
    `cam_ids` in the camera array's dict order: the reference forms combinations in that order and keeps a pair only if
    a < b (:505-506), so a pair whose larger id comes first in the dict is never formed."""
    ids = [int(c) for c, ig in zip(cam_ids, cam_ignore) if not ig]
    out = {}
    for a, b in combinations(ids, 2):
        if not a < b:
            continue
        so_a = {(s, o) for c, s, o in poses if c == a}
        so_b = {(s, o) for c, s, o in poses if c == b}
        for s, o in so_a & so_b:
            Ra, ta, _ = poses[(a, s, o)]
            Rb, tb, _ = poses[(b, s, o)]
            out[((a, b), s, o)] = (Rb @ Ra.T, Rb @ (-Ra.T @ ta) + tb)
    return out


def quat_wxyz(R: np.ndarray) -> np.ndarray:
    """Unit quaternion (w, x, y, z) of a rotation matrix (sign as scipy's Rotation.as_quat; immaterial downstream)."""
    from scipy.spatial.transform import Rotation

    return np.roll(Rotation.from_matrix(R).as_quat(), 1)


def quaternion_average(quats: np.ndarray) -> np.ndarray:
    if len(quats) == 1:
        return quats[0]
    M = quats.T @ quats
    _, V = np.linalg.eigh(M)
    q = V[:, -1]
    if q[0] < 0:
        q = -q
    return q / np.linalg.norm(q)


def quat_to_matrix(q: np.ndarray) -> np.ndarray:
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])  # fmt: skip


def rotation_error_deg(R1, R2) -> float:
    tr = np.clip(np.trace(R1 @ R2.T), -1.0, 3.0)
    return float(np.degrees(np.arccos((tr - 1) / 2)))


def reject_outliers(rel: dict, threshold: float = 1.5):
    by_pair: dict = {}
    for (pair, _s, _o), v in rel.items():
        by_pair.setdefault(pair, []).append(v)
    out = {}
    for pair, lst in by_pair.items():
        valid = [v for v in lst if not (np.any(np.isnan(v[0])) or np.any(np.isnan(v[1])))]
        if len(valid) < 5:
            out[pair] = valid
            continue
        quats = np.array([quat_wxyz(v[0]) for v in valid])
        tm = np.array([np.linalg.norm(v[1]) for v in valid])
        q1, q3 = np.percentile(tm, [25, 75])
        lo, hi = q1 - threshold * (q3 - q1), q3 + threshold * (q3 - q1)
        Rm = quat_to_matrix(quaternion_average(quats))
        ang = np.array([rotation_error_deg(v[0], Rm) for v in valid])
        r1, r3 = np.percentile(ang, [25, 75])
        rhi = r3 + threshold * (r3 - r1)
        out[pair] = [v for v, t, a in zip(valid, tm, ang) if not (t < lo or t > hi or a > rhi)]
    return out


def aggregate(filt: dict):
    out = {}
    for pair, lst in filt.items():
        if not lst:
            continue
        if len(lst) == 1:
            out[pair] = lst[0]
            continue
        q = quaternion_average(np.array([quat_wxyz(v[0]) for v in lst]))
        out[pair] = (quat_to_matrix(q), np.mean([v[1] for v in lst], axis=0))
    return out


def triangulate_two_view(R, t, na, nb) -> np.ndarray:
    """cv2.triangulatePoints(P1 = [I|0], P2 = [R|t], ...) for one point, float32 output like the reference's call."""
    P1 = np.eye(3, 4)
    P2 = np.hstack([R, t.reshape(3, 1)])
    A = np.array([na[0] * P1[2] - P1[0], na[1] * P1[2] - P1[1], nb[0] * P2[2] - P2[0], nb[1] * P2[2] - P2[1]])
    _, _, Vt = np.linalg.svd(A)
    X4 = Vt[3].astype(np.float32)
    return (X4[:3] / X4[3]).astype(np.float64)


def stereo_rmse(agg: dict, cam_ids, cam_ignore, norm_xy, sync_index, obs_cam_id, object_id, keypoint_id, min_common=4):
    """dict pair -> rmse (None when fewer than min_common common observations).  The common observations are keyed by
    the dict-order combinations (:589-598) and looked up with the aggregated pair's (a < b) key (:655)."""
    ids = [int(c) for c, ig in zip(cam_ids, cam_ignore) if not ig]
    key = list(zip(sync_index.tolist(), object_id.tolist(), keypoint_id.tolist()))
    out = {p: None for p in agg}
    for a, b in combinations(ids, 2):
        if (a, b) not in agg:
            continue
        ia = {k: i for i, k in enumerate(key) if obs_cam_id[i] == a}
        common = [(ia[k], i) for i, k in enumerate(key) if obs_cam_id[i] == b and k in ia]
        if len(common) < min_common:
            out[(a, b)] = None
            continue
        R, t = agg[(a, b)]
        tot = 0.0
        for i, j in common:
            X = triangulate_two_view(R, t, norm_xy[i], norm_xy[j])
            pa = (X[:2] / X[2]).astype(np.float32)
            Xb = R @ X + t
            pb = (Xb[:2] / Xb[2]).astype(np.float32)
            ea = norm_xy[i].astype(np.float32) - pa
            eb = norm_xy[j].astype(np.float32) - pb
            tot += float(np.sum(ea * ea)) + float(np.sum(eb * eb))
        out[(a, b)] = float(np.sqrt(tot / (2 * len(common))))
    return out


def fill_network(raw: dict):
    """paired_pose_network.py:26-99: pairs -> all ordered pairs reachable by bridging; values (R, t, err)."""

    def inv(v):
        R, t, e = v
        return (R.T, -R.T @ t, e)

    def link(v1, v2):  # (A->B).link(B->C)
        return (v2[0] @ v1[0], v2[0] @ v1[1] + v2[1], v1[2] + v2[2])

    allp = dict(raw)
    for (a, b), v in list(raw.items()):
        allp[(b, a)] = inv(v)
    cams = sorted({c for p in allp for c in p})
    last = -1
    while True:
        missing = [p for p in permutations(cams, 2) if p not in allp]
        if len(missing) == last or not missing:
            break
        last = len(missing)
        for a, c in missing:
            best = None
            for x in cams:
                if (a, x) in allp and (x, c) in allp:
                    cand = link(allp[(a, x)], allp[(x, c)])
                    if best is None or best[2] > cand[2]:
                        best = cand
            if best is not None:
                allp[(a, c)] = best
                allp[(c, a)] = inv(best)
    return allp


# ----------------------------------------------------------------------------------------------------------------
# The reference's own OpenCV calls, for the CPU baseline of bench.py (test infrastructure; needs cv2).  Same call
# sequence as pose_network_builder.py:241-321 (undistort per camera, solvePnP + Rodrigues + projectPoints per group) and
# :638-685 (triangulatePoints + projectPoints per pair), on arrays instead of DataFrames (which only makes it faster).
# ----------------------------------------------------------------------------------------------------------------
def reference_calls_cv2(cam_ids, cam_k, cam_dist, cam_fisheye, sync_index, obs_cam_id, object_id, keypoint_id, img_xy, obj_xyz):
    import cv2

    norm = np.full((len(obs_cam_id), 2), np.nan, np.float32)
    for i, c in enumerate(cam_ids):
        sel = obs_cam_id == c
        if not sel.any():
            continue
        K = np.array([[cam_k[i, 0], cam_k[i, 4], cam_k[i, 2]], [0, cam_k[i, 1], cam_k[i, 3]], [0, 0, 1.0]])
        pts = np.ascontiguousarray(img_xy[sel], dtype=np.float32).reshape(-1, 1, 2)
        norm[sel] = cv2.undistortPoints(pts, K, cam_dist[i, :5], P=np.identity(3)).reshape(-1, 2)
    order = np.lexsort((keypoint_id, object_id, sync_index, obs_cam_id))
    key = np.stack([obs_cam_id[order], sync_index[order], object_id[order]], axis=1)
    brk = np.flatnonzero(np.any(np.diff(key, axis=0) != 0, axis=1)) + 1
    starts = np.concatenate([[0], brk, [len(order)]])
    Kp, Dp = np.identity(3), np.zeros(5)
    poses = {}
    for s, e in zip(starts[:-1], starts[1:]):
        rows = order[s:e]
        if len(rows) < 4:
            continue
        obj = obj_xyz[rows].astype(np.float32)
        img = norm[rows]
        ok, rvec, tvec = cv2.solvePnP(obj, img, cameraMatrix=Kp, distCoeffs=Dp, flags=cv2.SOLVEPNP_IPPE)
        if not ok:
            ok, rvec, tvec = cv2.solvePnP(obj, img, cameraMatrix=Kp, distCoeffs=Dp, flags=cv2.SOLVEPNP_ITERATIVE)
        if ok:
            R, _ = cv2.Rodrigues(rvec)
            proj, _ = cv2.projectPoints(obj, rvec, tvec, Kp, Dp)
            rmse = np.sqrt(np.mean(np.sum((img - proj.reshape(-1, 2)) ** 2, axis=1)))
            poses[tuple(int(v) for v in key[s])] = (R, tvec.flatten(), float(rmse))
    rel = relative_poses(poses, cam_ids, np.zeros(len(cam_ids), bool))
    agg = aggregate(reject_outliers(rel, 1.5))
    # stereo RMSE with cv2, pair by pair
    kk = sync_index * (int(object_id.max()) + 1) * (int(keypoint_id.max()) + 1) + object_id * (int(keypoint_id.max()) + 1) + keypoint_id
    by_cam = {int(c): (kk[obs_cam_id == c], np.flatnonzero(obs_cam_id == c)) for c in cam_ids}
    out = {}
    for (a, b), (R, t) in agg.items():
        ka, ia = by_cam[a]
        kb, ib = by_cam[b]
        common, xa, xb = np.intersect1d(ka, kb, return_indices=True)
        if len(common) < 4:
            continue
        na, nb = norm[ia[xa]], norm[ib[xb]]
        P2 = np.hstack((R, t.reshape(3, 1)))
        p4 = cv2.triangulatePoints(np.eye(3, 4), P2, na.T, nb.T)
        p3 = p4[:3] / p4[3]
        pa, _ = cv2.projectPoints(p3.T, np.zeros(3), np.zeros(3), np.eye(3), np.zeros(5))
        pb, _ = cv2.projectPoints(p3.T, cv2.Rodrigues(R)[0], t, np.eye(3), np.zeros(5))
        err = np.vstack([na - pa.reshape(-1, 2), nb - pb.reshape(-1, 2)])
        out[(a, b)] = (R, t, float(np.sqrt(np.mean(np.sum(err**2, axis=1)))))
    return poses, out


# ----------------------------------------------------------------------------------------------------------------
# The same OpenCV calls stage by stage, on normalised coordinates the caller supplies (test infrastructure; needs cv2).
# Given the device's own undistortion output, which is pinned to cv2.undistortPoints separately, a comparison with these
# isolates the PnP and stereo kernels from the undistortion.
# ----------------------------------------------------------------------------------------------------------------
PNP_OK, PNP_TOO_FEW, PNP_DEGENERATE, PNP_OK_FALLBACK = 0, 1, 3, 4  # caliscope_b200.bootstrap's status codes


def pnp_cv2(norm_xy, cam_id, sync_index, object_id, obj_xyz, min_points: int = 4):
    """pose_network_builder.py:272-321 per (camera, sync, object) group, in sorted key order: cv2.solvePnP(IPPE) on
    float32 normalised points and float32 model points (NaN z counted as 0), SOLVEPNP_ITERATIVE where IPPE fails, the
    RMSE through cv2.projectPoints in float32.  Returns (keys (g, 3), R (g, 3, 3), t (g, 3), rmse (g,), status (g,)):
    PNP_TOO_FEW below min_points (NaN pose), PNP_DEGENERATE for a non-finite pose, PNP_OK_FALLBACK where ITERATIVE ran."""
    import cv2

    cam_id, sync_index, object_id = (np.asarray(a, np.int64) for a in (cam_id, sync_index, object_id))
    order = np.lexsort((object_id, sync_index, cam_id))
    key = np.stack([cam_id[order], sync_index[order], object_id[order]], axis=1)
    brk = np.flatnonzero(np.any(np.diff(key, axis=0) != 0, axis=1)) + 1
    starts = np.concatenate([[0], brk, [len(order)]])
    g = len(starts) - 1
    R = np.full((g, 3, 3), np.nan)
    t = np.full((g, 3), np.nan)
    rmse = np.full(g, np.nan)
    status = np.full(g, PNP_TOO_FEW, np.int32)
    Kp, Dp = np.identity(3), np.zeros(5)
    for i, (s, e) in enumerate(zip(starts[:-1], starts[1:])):
        if e - s < min_points:
            continue
        rows = order[s:e]
        obj = np.asarray(obj_xyz, np.float64)[rows].copy()
        obj[:, 2] = np.nan_to_num(obj[:, 2], nan=0.0)
        if not np.ptp(obj[:, 2]) < 1e-6:
            raise NotImplementedError("non-planar PnP group (the reference switches to SQPNP)")
        obj = obj.astype(np.float32)
        img = np.ascontiguousarray(np.asarray(norm_xy)[rows], dtype=np.float32)
        ok, rvec, tvec = cv2.solvePnP(obj, img, cameraMatrix=Kp, distCoeffs=Dp, flags=cv2.SOLVEPNP_IPPE)
        status[i] = PNP_OK
        if not ok:
            ok, rvec, tvec = cv2.solvePnP(obj, img, cameraMatrix=Kp, distCoeffs=Dp, flags=cv2.SOLVEPNP_ITERATIVE)
            status[i] = PNP_OK_FALLBACK
        if not ok or not (np.isfinite(rvec).all() and np.isfinite(tvec).all()):
            status[i] = PNP_DEGENERATE
            continue
        R[i] = cv2.Rodrigues(rvec)[0]
        t[i] = tvec.ravel()
        proj, _ = cv2.projectPoints(obj, rvec, tvec, Kp, Dp)
        rmse[i] = float(np.sqrt(np.mean(np.sum((img - proj.reshape(-1, 2)) ** 2, axis=1))))
    return key[starts[:-1]], R, t, rmse, status


def stereo_rmse_cv2(pairs, R, t, cam_ids, cam_ignore, norm_xy, cam_id, sync_index, object_id, keypoint_id, min_common: int = 4):
    """calculate_stereo_rmse_for_pair (:638-685) for each (a, b) pair with pose [R | t]: cv2.triangulatePoints on the
    float32 normalised points of the common (sync, object, keypoint) observations, cv2.projectPoints into both views,
    float32 RMSE over the 2N stacked residuals.  Returns (rmse (p,), common count (p,)).  The reference's lookup quirk
    (:589-598 with :655) is kept: a pair whose cameras come in (b, a) order in the dict ``cam_ids``, or that includes an
    ignored camera, has no common observations (count 0, NaN); fewer than ``min_common`` gives NaN with its count."""
    import cv2

    pos = {int(c): i for i, c in enumerate(cam_ids) if not cam_ignore[i]}
    cam_id = np.asarray(cam_id, np.int64)
    key = np.zeros(len(cam_id), np.int64)
    for col in (sync_index, object_id, keypoint_id):  # one integer per (sync, object, keypoint)
        col = np.asarray(col, np.int64) - int(np.min(col))
        key = key * (int(col.max()) + 1) + col
    by_cam = np.argsort(cam_id, kind="stable")
    cams, first = np.unique(cam_id[by_cam], return_index=True)
    bounds = dict(zip(cams.tolist(), zip(first.tolist(), np.append(first[1:], len(by_cam)).tolist())))
    norm = np.asarray(norm_xy, np.float32)
    p = len(pairs)
    rmse = np.full(p, np.nan)
    cnt = np.zeros(p, np.int64)
    for i, (a, b) in enumerate(np.asarray(pairs, np.int64).reshape(-1, 2)):
        a, b = int(a), int(b)
        if a not in pos or b not in pos or not pos[a] < pos[b]:
            continue
        ia, ib = (by_cam[slice(*bounds.get(c, (0, 0)))] for c in (a, b))
        _, xa, xb = np.intersect1d(key[ia], key[ib], return_indices=True)
        cnt[i] = len(xa)
        if len(xa) < min_common:
            continue
        na, nb = norm[ia[xa]], norm[ib[xb]]
        Ri, ti = np.asarray(R[i], np.float64), np.asarray(t[i], np.float64).reshape(3)
        p4 = cv2.triangulatePoints(np.eye(3, 4), np.hstack((Ri, ti.reshape(3, 1))), na.T, nb.T)
        p3 = p4[:3] / p4[3]
        pa, _ = cv2.projectPoints(p3.T, np.zeros(3), np.zeros(3), np.eye(3), np.zeros(5))
        pb, _ = cv2.projectPoints(p3.T, cv2.Rodrigues(Ri)[0], ti, np.eye(3), np.zeros(5))
        err = np.vstack([na - pa.reshape(-1, 2), nb - pb.reshape(-1, 2)])
        rmse[i] = float(np.sqrt(np.mean(np.sum(err**2, axis=1))))
    return rmse, cnt
