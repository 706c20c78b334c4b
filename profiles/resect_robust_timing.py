"""Stage times of cb_resect_robust (DESIGN.md 4.9), one JSON line per (workload, point covariance) pair.

    python profiles/resect_robust_timing.py [rig64] [track] [--steps 5] [--warmup 2] [--cpu-groups 200]
        [--dump-outputs DIR]

rig64: cfg4's 64 cameras and 50 000 points (synthetic.make_rig(64, 50_000, 2_000_000)), key = camera: 64 groups of about
31 000 rows (the long shape), 5 % of the rows moved by up to +-200 px, priors 0.02 rad / 2 cm off the truth; run without
and with a point covariance (a seeded SPD 3x3 per point).  track: a rigid cluster of 12 markers seen by 8 pinhole
cameras over 50 000 frames, key = (camera, frame): 400 000 groups of 12 rows (the short shape, 8 lanes), each group's
pose the camera-from-cluster transform of its frame, 5 % outliers of up to +-200 px, no prior.  Stage times are the CUDA
events recorded inside the call (CbResectStats).  Scoring evaluations are counted from the shapes: sum over the groups of
(1 + 4 min(C(k, 3), max_samples)) x k, an upper bound (samples with fewer than 4 solutions score fewer hypotheses).
The pose error against the truth is over the groups with status 0.  For context only, cv2.solvePnPRansac (P3P, then
solvePnPRefineLM on its inliers) runs on a sample of the groups on one host core: a different algorithm on the CPU, not
a baseline of the same computation.  The card's name and power limit are printed with the numbers.  --dump-outputs
writes every output array of the last timed call of each variant to DIR/<workload>_<variant>.npz.
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from caliscope_b200 import synthetic  # noqa: E402
from caliscope_b200.resection import ResectStats, resect_robust  # noqa: E402
from dump_outputs import dump_outputs  # noqa: E402

TAU = 4.0
MAX_SAMPLES = 64


def card() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()  # fmt: skip
        return out[0] if out else "unknown card"
    except (OSError, subprocess.SubprocessError):
        return "unknown card"


def rodrigues(r):
    """(n, 3) rotation vectors -> (n, 3, 3)"""
    r = np.asarray(r, np.float64).reshape(-1, 3)
    th = np.linalg.norm(r, axis=1)
    k = r / np.where(th > 0, th, 1.0)[:, None]
    K = np.zeros((len(r), 3, 3))
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 2] = -k[:, 2], k[:, 1], -k[:, 0]
    K -= np.transpose(K, (0, 2, 1))
    s, c = np.sin(th)[:, None, None], np.cos(th)[:, None, None]
    return np.eye(3) + s * K + (1 - c) * (K @ K)


def _outliers(rng, px, frac=0.05, amp=200.0):
    px = px.copy()
    m = rng.random(len(px)) < frac
    px[m] += rng.uniform(-amp, amp, (m.sum(), 2))
    return px, m


def _rot_log(R):
    """rotation vectors of (n, 3, 3) matrices (theta in [0, pi), away from pi)"""
    c = np.clip((np.trace(R, axis1=1, axis2=2) - 1) / 2, -1, 1)
    th = np.arccos(c)
    v = np.stack([R[:, 2, 1] - R[:, 1, 2], R[:, 0, 2] - R[:, 2, 0], R[:, 1, 0] - R[:, 0, 1]], axis=1)
    s = np.sin(th)
    return v * np.where(s > 1e-12, th / (2 * np.where(s > 1e-12, s, 1.0)), 0.5)[:, None]


def make(name: str):
    """(inputs, truth pose per group in key order, outlier mask, K per camera for the CPU comparison or None)"""
    rng = np.random.default_rng(7)
    if name == "rig64":
        rig = synthetic.make_rig(64, 50_000, 2_000_000, seed=0, name="cfg4")
        ncp = int(np.where(rig.cam_flags & 1, 9, 6).sum())
        truth = rig.x_true[:ncp].reshape(64, 6)
        prior = truth + np.concatenate([rng.normal(0, 0.02, (64, 3)), rng.normal(0, 0.02, (64, 3))], axis=1)
        pts = rig.x_true[ncp:].reshape(-1, 3)
        px, moved = _outliers(rng, rig.obs_xy)
        args = (rig.cam_flags, rig.cam_const, prior.ravel(), pts, rig.obs_cam, rig.obs_cam.astype(np.int64), rig.obs_pt, px)
        return args, truth, moved, dict(use_prior=True)
    if name == "track":
        n_cams, n_frames, n_mk = 8, 50_000, 12
        mk = rng.uniform(-0.1, 0.1, (n_mk, 3))  # the cluster, in its own frame (metres)
        ang = 2 * np.pi * np.arange(n_cams) / n_cams
        centers = np.stack([3 * np.cos(ang), 3 * np.sin(ang), np.full(n_cams, 1.0)], axis=1)
        Rc = []
        for c in centers:  # look at (0, 0, 1)
            z = np.array([0.0, 0.0, 1.0]) - c
            z /= np.linalg.norm(z)
            x = np.cross([0.0, 0.0, -1.0], z)
            x /= np.linalg.norm(x)
            Rc.append(np.stack([x, np.cross(z, x), z]))
        Rc = np.array(Rc)
        tc = -np.einsum("cij,cj->ci", Rc, centers)
        # cluster motion per frame: a wandering position and orientation
        pos = np.cumsum(rng.normal(0, 0.003, (n_frames, 3)), axis=0) + [0.0, 0.0, 1.0]
        pos -= (pos.mean(axis=0) - [0.0, 0.0, 1.0])
        Rm = rodrigues(rng.normal(0, 0.5, (n_frames, 3)))
        const = np.zeros((n_cams, 9))
        const[:, :4] = [1000.0, 1000.0, 640.0, 360.0]
        flags = np.zeros(n_cams, np.int32)
        # camera-from-cluster pose of every (camera, frame)
        Rg = np.einsum("cij,fjk->cfik", Rc, Rm).reshape(-1, 3, 3)
        tg = (np.einsum("cij,fj->cfi", Rc, pos) + tc[:, None]).reshape(-1, 3)
        Xc = np.einsum("gij,mj->gmi", Rg, mk) + tg[:, None]
        uv = Xc[..., :2] / Xc[..., 2:] * 1000.0 + [640.0, 360.0]
        px = (uv + rng.normal(0, 0.5, uv.shape)).reshape(-1, 2)
        px, moved = _outliers(rng, px)
        G = n_cams * n_frames
        obs_cam = np.repeat(np.arange(n_cams), n_frames * n_mk).astype(np.int32)
        key = np.repeat(np.arange(G, dtype=np.int64), n_mk)
        obs_pt = np.tile(np.arange(n_mk, dtype=np.int32), G)
        cam_x = np.concatenate([_rot_log(Rc), tc], axis=1).ravel()
        truth = np.concatenate([_rot_log(Rg), tg], axis=1)
        return (flags, const, cam_x, mk, obs_cam, key, obs_pt, px), truth, moved, dict(use_prior=False)
    raise SystemExit(f"unknown workload {name}")


def _pose_err(pose, truth, m):
    if not m.any():
        return None
    dR = np.einsum("nji,njk->nik", rodrigues(pose[m, :3]), rodrigues(truth[m, :3]))
    ang = np.degrees(np.arccos(np.clip((np.trace(dR, axis1=1, axis2=2) - 1) / 2, -1, 1)))
    # camera centres
    C = -np.einsum("nji,nj->ni", rodrigues(pose[m, :3]), pose[m, 3:])
    Ct = -np.einsum("nji,nj->ni", rodrigues(truth[m, :3]), truth[m, 3:])
    d = np.linalg.norm(C - Ct, axis=1)
    return {"center_median_m": float(np.median(d)), "center_p99_m": float(np.percentile(d, 99)),
            "angle_median_deg": float(np.median(ang)), "angle_p99_deg": float(np.percentile(ang, 99))}  # fmt: skip


def cpu_context(args, n_groups_sample: int):
    """cv2.solvePnPRansac (P3P) + solvePnPRefineLM on a sample of groups, one host core: ms per group."""
    try:
        import cv2
    except ImportError:
        return None
    cv2.setNumThreads(1)
    flags, const, cam_x, pts, obs_cam, key, obs_pt, px = args
    order = np.argsort(key, kind="stable")
    ks = key[order]
    starts = np.flatnonzero(np.r_[True, ks[1:] != ks[:-1]])
    bounds = np.r_[starts, len(ks)]
    pick = np.linspace(0, len(starts) - 1, min(n_groups_sample, len(starts))).astype(int)
    t0 = time.perf_counter()
    for g in pick:
        rows = order[bounds[g] : bounds[g + 1]]
        c = obs_cam[rows[0]]
        K = np.array([[const[c, 0], 0, const[c, 2]], [0, const[c, 1], const[c, 3]], [0, 0, 1.0]])
        dist = const[c, 4:9] if not flags[c] & 2 else None
        obj = np.ascontiguousarray(pts[obs_pt[rows]])
        img = np.ascontiguousarray(px[rows])
        ok, r, t, inl = cv2.solvePnPRansac(obj, img, K, dist, iterationsCount=MAX_SAMPLES, reprojectionError=TAU,
                                           flags=cv2.SOLVEPNP_P3P)  # fmt: skip
        if ok and inl is not None and len(inl) >= 4:
            cv2.solvePnPRefineLM(obj[inl[:, 0]], img[inl[:, 0]], K, dist, r, t)
    return {"groups": int(len(pick)), "ms_per_group": 1e3 * (time.perf_counter() - t0) / len(pick)}


def run(name: str, steps: int, warmup: int, cpu_groups: int, dump_dir=None):
    args, truth, moved, kw = make(name)
    key = args[5]
    _, k = np.unique(key, return_counts=True)
    T = k * (k - 1) * (k - 2) // 6
    evals = float(np.sum((1 + 4 * np.minimum(T, MAX_SAMPLES)) * k))
    rng = np.random.default_rng(3)
    n_pts = len(args[3])
    A = rng.normal(0, 3e-4, (n_pts, 3, 3))
    pcov = A @ np.transpose(A, (0, 2, 1)) + 1e-8 * np.eye(3)
    cpu = cpu_context(args, cpu_groups)
    for cov in ((None, pcov) if name == "rig64" else (None,)):
        for _ in range(warmup):
            resect_robust(*args, threshold_px=TAU, max_samples=MAX_SAMPLES, points_cov=cov, **kw)
        acc = np.zeros(5)
        launches = 0
        for _ in range(steps):
            st = ResectStats()
            out = resect_robust(*args, threshold_px=TAU, max_samples=MAX_SAMPLES, points_cov=cov, stats=st, **kw)
            acc += [st.group_ms, st.consensus_ms, st.refine_ms, st.cov_ms, st.total_ms]
            launches = st.kernel_launches
        acc /= steps
        dump_outputs(dump_dir, f"{name}_{'pcov' if cov is not None else 'nopcov'}", out)
        ok = out.status == 0
        print(json.dumps({
            "workload": name, "card": card(), "points_cov": cov is not None, "n_obs": int(len(key)),
            "n_groups": int(len(k)), "rows_per_group": float(np.mean(k)),
            "group_ms": acc[0], "consensus_ms": acc[1], "refine_ms": acc[2], "cov_ms": acc[3], "total_ms": acc[4],
            "kernel_launches": launches, "score_evals_upper": evals, "score_evals_per_s": evals / (acc[1] * 1e-3),
            "status_counts": {int(s): int(c) for s, c in zip(*np.unique(out.status, return_counts=True))},
            "outlier_rows": int(moved.sum()), "outliers_rejected": int((moved & ~out.inlier).sum()),
            "clean_rows_rejected": int((~moved & ~out.inlier).sum()), "pose_err": _pose_err(out.pose, truth, ok),
            "cpu_context_opencv_ransac_one_core": cpu,
        }), flush=True)  # fmt: skip


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workloads", nargs="*", default=["rig64", "track"])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--cpu-groups", type=int, default=200)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    a = ap.parse_args()
    for w in a.workloads:
        run(w, a.steps, a.warmup, a.cpu_groups, a.dump_outputs)


if __name__ == "__main__":
    main()
