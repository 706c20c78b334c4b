"""Stage times of cb_relative_pose_robust (DESIGN.md 4.11), one JSON line per workload.

    python profiles/relative_pose_timing.py [ring8] [rig64] [--steps 3] [--warmup 1] [--no-cpu]

Workloads (caliscope_b200.synthetic.make_rig, observation key = point, 0.5 px noise): ring8 = Caliscope's usual shape,
8 cameras in a ring, ~150k observations, each point seen by the 5 nearest cameras (local visibility), 2 % outliers;
rig64 = make_rig(64, 50_000, 2_000_000), ~3.9e7 correspondences.  Times are the CUDA events recorded inside the call
(CbRelPoseStats), the median over --steps timed calls after --warmup.  "sampson_evals" counts the scoring kernel's
Sampson distances (correspondences x hypothesis slots of every pair, empty slots included); the pose error is the worst
status-0 pair's rotation angle and baseline-direction angle against the truth.  For context only, cv2.findEssentialMat
(RANSAC) + cv2.recoverPose run on the same undistorted correspondences of each pair of ring8 on one host core (a CPU
library, not a baseline of the same computation).  The card's name and power limit are read in the same run.
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from caliscope_b200 import synthetic  # noqa: E402
from caliscope_b200.epipolar import RelPoseStats, relative_poses_robust  # noqa: E402

WORKLOADS = {
    "ring8": lambda: synthetic.make_rig(8, 30_000, 150_000, seed=0, noise_px=0.5, outlier_frac=0.02, cams_per_point=5),
    "rig64": lambda: synthetic.make_rig(64, 50_000, 2_000_000, seed=0, noise_px=0.5),
}


def card() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()  # fmt: skip
        return out[0] if out else "unknown card"
    except (OSError, subprocess.SubprocessError):
        return "unknown card"


def _rot(r):
    import cv2

    return cv2.Rodrigues(np.asarray(r, np.float64))[0]


def _angle(R):
    return float(np.degrees(np.arccos(np.clip((np.trace(R) - 1) / 2, -1, 1))))


def pose_errors(rig, res):
    nc = rig.n_cams
    xt = rig.x_true[: 6 * nc].reshape(nc, 6)
    rot, bas = 0.0, 0.0
    for p in np.flatnonzero(res.status == 0):
        a, b = res.cam_a[p], res.cam_b[p]
        Ra, Rb = _rot(xt[a, :3]), _rot(xt[b, :3])
        R = Rb @ Ra.T
        t = xt[b, 3:] - R @ xt[a, 3:]
        t /= np.linalg.norm(t)
        rot = max(rot, _angle(_rot(res.pose[p, :3]) @ R.T))
        bas = max(bas, float(np.degrees(np.arccos(np.clip(res.pose[p, 3:] @ t, -1, 1)))))
    return rot, bas


def cv2_pairs(rig, seconds_cap=120.0):
    """findEssentialMat (RANSAC, 1 px on the normalised plane scaled by f) + recoverPose per pair, one core."""
    import cv2

    cv2.setNumThreads(1)
    K = np.array([[rig.cam_const[0, 0], 0, rig.cam_const[0, 2]], [0, rig.cam_const[0, 1], rig.cam_const[0, 3]], [0, 0, 1]])
    by_cam = {}
    for c in range(rig.n_cams):
        m = rig.obs_cam == c
        und = cv2.undistortPoints(rig.obs_xy[m].reshape(-1, 1, 2).astype(np.float32), K, rig.cam_const[c, 4:9]).reshape(-1, 2)
        by_cam[c] = dict(zip(rig.obs_pt[m].tolist(), und.astype(np.float64)))
    t0, n = time.perf_counter(), 0
    for a in range(rig.n_cams):
        for b in range(a + 1, rig.n_cams):
            common = sorted(set(by_cam[a]) & set(by_cam[b]))
            if len(common) < 15:
                continue
            xa = np.array([by_cam[a][k] for k in common])
            xb = np.array([by_cam[b][k] for k in common])
            E, mask = cv2.findEssentialMat(xa, xb, np.eye(3), method=cv2.RANSAC, prob=0.999,
                                           threshold=3.0 / rig.cam_const[a, 0])  # fmt: skip
            cv2.recoverPose(E[:3], xa, xb, np.eye(3), mask=mask)
            n += 1
            if time.perf_counter() - t0 > seconds_cap:
                break
    return (time.perf_counter() - t0) * 1e3, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workloads", nargs="*", default=list(WORKLOADS))
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--max-samples", type=int, default=64)
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    name = card()
    for w in a.workloads:
        rig = WORKLOADS[w]()
        key = rig.obs_pt.astype(np.int64)
        kw = dict(threshold_px=3.0, max_samples=a.max_samples)
        for _ in range(a.warmup):
            relative_poses_robust(rig.cam_flags, rig.cam_const, rig.obs_cam, key, rig.obs_xy, **kw)
        stats, walls, res = [], [], None
        for _ in range(a.steps):
            st = RelPoseStats()
            t0 = time.perf_counter()
            res = relative_poses_robust(rig.cam_flags, rig.cam_const, rig.obs_cam, key, rig.obs_xy, stats=st, **kw)
            walls.append((time.perf_counter() - t0) * 1e3)
            stats.append(st)
        med = lambda f: float(np.median([getattr(s, f) for s in stats]))  # noqa: E731
        corr = int(res.count.sum())
        evals = corr * 10 * a.max_samples
        rot, bas = pose_errors(rig, res)
        out = dict(workload=w, card=name, n_obs=int(rig.n_obs), n_cams=int(rig.n_cams), pairs=int(len(res.status)),
                   pairs_ok=int((res.status == 0).sum()), correspondences=corr, max_samples=a.max_samples,
                   group_ms=med("group_ms"), consensus_ms=med("consensus_ms"), refine_ms=med("refine_ms"),
                   cov_ms=med("cov_ms"), total_ms=med("total_ms"), wall_ms=float(np.median(walls)),
                   kernel_launches=stats[-1].kernel_launches, sampson_evals=evals,
                   sampson_evals_per_s=evals / (med("consensus_ms") * 1e-3), max_rot_err_deg=rot,
                   max_baseline_err_deg=bas)  # fmt: skip
        if w == "ring8" and not a.no_cpu:
            ms, n = cv2_pairs(rig)
            out["cv2_one_core_ms"] = ms
            out["cv2_pairs"] = n
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
