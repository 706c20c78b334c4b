"""Timing and accuracy of rigid-body layout refinement (``rigid.refine_rigid_model``, DESIGN.md section 4.15).

Workloads (synthetic, seeded):
  track  one body of 10 markers, 8 cameras, 20 000 frames, 0.5 px noise; start poses from pose_rigid_robust on a
         nominal layout 2 mm (per coordinate) off the truth; the refinement takes that call's inlier rows
  multi  32 bodies of 6 markers, 2 000 frames each, otherwise as track

Reports per workload: the card and its power limit, the call's stage times (median of --reps after a warm-up call),
iterations, the layout error against the truth (Kabsch-aligned RMS per coordinate) before and after, the mean
e^T cov^+ e over the bodies (e the refined layout minus the aligned truth; about 3K - 6 when the covariance is right),
and the RMS world error of the markers predicted by a second pose_rigid_robust pass with the refined layout against the
first pass with the nominal one.

    python profiles/rigid_model_timing.py track multi [--reps 5] [--out results.json]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]  # fmt: skip
        name, power = (x.strip() for x in out.split(","))
        return name, power
    except (OSError, subprocess.CalledProcessError, IndexError, ValueError):
        return "unknown", "unknown"


def _scene(bodies, K, frames, seed):
    """make_scene's track for one body; for several, bodies on disjoint model ranges and keys seen by make_scene's rig,
    generated per (body, camera) in one projection call."""
    from oracle.ba_oracle import rodrigues
    from oracle.resection_robust import cameras, project
    from tests._rigid_cases import Bodies
    from tests._rigid_model_cases import Scene, make_scene, perturb_pose

    if bodies == 1:
        return make_scene(seed, n_model=K, n_frames=frames, n_cams=8, noise=0.5, model_off=2e-3, visible=0.7)
    base = make_scene(seed, n_model=K, n_frames=1, n_cams=8).bodies
    cams = cameras(base.flags, base.const, base.cam_x)
    rng = np.random.default_rng(seed)
    model = rng.uniform(-0.1, 0.1, (bodies * K, 3))
    truth = np.zeros((bodies * frames, 6))
    ax = rng.normal(size=(len(truth), 3))
    truth[:, :3] = ax / np.linalg.norm(ax, axis=1, keepdims=True) * rng.uniform(0, np.pi * 0.8, (len(truth), 1))
    truth[:, 3:] = rng.uniform(-0.3, 0.3, (len(truth), 3))
    Rs = np.stack([rodrigues(q[:3])[0] for q in truth])
    oc, ok, op, px = [], [], [], []
    for bb in range(bodies):
        fr = np.arange(bb * frames, (bb + 1) * frames)
        Xw = np.einsum("fij,kj->fki", Rs[fr], model[bb * K : (bb + 1) * K]) + truth[fr, None, 3:]
        for c, cam in enumerate(cams):
            uv, _ = project(cam, rodrigues(cam.q[:3])[0], cam.q[3:6], Xw.reshape(-1, 3))
            keep = rng.random(len(uv)) < 0.7
            f_idx, k_idx = np.divmod(np.flatnonzero(keep), K)
            oc.append(np.full(len(f_idx), c)); ok.append(fr[f_idx]); op.append(bb * K + k_idx)
            px.append(uv[keep] + rng.normal(0, 0.5, (len(f_idx), 2)))
    order = np.lexsort((np.concatenate(op), np.concatenate(ok)))
    b = Bodies(base.flags, base.const, base.cam_x, model, truth, np.concatenate(oc).astype(np.int32)[order],
               np.concatenate(ok).astype(np.int64)[order], np.concatenate(op).astype(np.int32)[order],
               np.concatenate(px)[order])  # fmt: skip
    nominal = model + rng.normal(0, 2e-3, model.shape)
    start = np.array([perturb_pose(rng, q, 1.0, 2e-3) for q in truth])
    return Scene(b, model.copy(), nominal, np.arange(len(truth)), start, np.arange(0, bodies * K + 1, K))


def _world_rms(sc, layout, keys, poses):
    from oracle.ba_oracle import rodrigues

    b = sc.bodies
    fk = np.unique(b.obs_key)
    idx = np.searchsorted(fk, keys)
    # the frame's body: the model range of the key's first row
    first = np.searchsorted(b.obs_key[np.argsort(b.obs_key, kind="stable")], keys)
    pts = b.obs_pt[np.argsort(b.obs_key, kind="stable")][first]
    body = np.searchsorted(sc.body_start, pts, side="right") - 1
    err = []
    for q, i, bb in zip(poses, idx, body):
        lo, hi = sc.body_start[bb], sc.body_start[bb + 1]
        t = b.truth[i]
        pred = layout[lo:hi] @ rodrigues(q[:3])[0].T + q[3:]
        true = sc.truth_model[lo:hi] @ rodrigues(t[:3])[0].T + t[3:]
        err.append(pred - true)
    return float(np.sqrt(np.nanmean(np.square(np.concatenate(err)))))


def run(name, bodies, K, frames, reps):
    from caliscope_b200 import rigid
    from tests._rigid_model_cases import kabsch_error

    sc = _scene(bodies, K, frames, 11)
    b = sc.bodies
    p1 = rigid.pose_rigid_robust(b.flags, b.const, b.cam_x, sc.nominal, b.obs_cam, b.obs_key, b.obs_pt, b.obs_px,
                                 threshold_px=4.0)  # fmt: skip
    use = p1.inlier
    obs = [x[use] for x in (b.obs_cam, b.obs_key, b.obs_pt, b.obs_px)]
    args = (b.flags, b.const, b.cam_x, sc.nominal, *obs, (p1.key, p1.pose))
    rigid.refine_rigid_model(*args, bodies=sc.body_start, pixel_sigma=0.5)  # warm-up
    stats = []
    for _ in range(reps):
        st = rigid.RigidModelStats()
        res = rigid.refine_rigid_model(*args, bodies=sc.body_start, pixel_sigma=0.5, stats=st)
        stats.append(st)
    med = {k: float(np.median([getattr(s, k) for s in stats])) for k in ("group_ms", "solve_ms", "cov_ms", "total_ms")}
    before, after, chi = [], [], []
    for bb in range(len(sc.body_start) - 1):
        lo, hi = sc.body_start[bb], sc.body_start[bb + 1]
        e0 = kabsch_error(sc.nominal[lo:hi], sc.truth_model[lo:hi])
        e1 = kabsch_error(res.model[lo:hi], sc.truth_model[lo:hi])
        before.append(np.sqrt(np.mean(e0 * e0)))
        after.append(np.sqrt(np.mean(e1 * e1)))
        if res.status[bb] == 0:
            chi.append(float(e1 @ np.linalg.pinv(res.cov[bb], rcond=1e-10) @ e1))
    p2 = rigid.pose_rigid_robust(b.flags, b.const, b.cam_x, res.model, *obs, threshold_px=4.0,
                                 prior=(res.key, res.pose))  # fmt: skip
    card, power = _card()
    return {
        "workload": name, "card": card, "power_limit": power, "bodies": bodies, "markers": K, "frames": frames,
        "rows": int(use.sum()), "stage_ms": med, "kernel_launches": stats[-1].kernel_launches,
        "iterations_max": int(res.iterations.max()), "status_0_bodies": int((res.status == 0).sum()),
        "layout_rms_mm_before": 1e3 * float(np.mean(before)), "layout_rms_mm_after": 1e3 * float(np.mean(after)),
        "mean_chi2": float(np.mean(chi)) if chi else None, "chi2_dof": 3 * K - 6,
        "world_rms_mm_first_pass": 1e3 * _world_rms(sc, sc.nominal, p1.key, p1.pose),
        "world_rms_mm_second_pass": 1e3 * _world_rms(sc, res.model, p2.key, p2.pose),
    }  # fmt: skip


WORKLOADS = {"track": (1, 10, 20000), "multi": (32, 6, 2000)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workloads", nargs="+", choices=sorted(WORKLOADS))
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rows = [run(w, *WORKLOADS[w], a.reps) for w in a.workloads]
    text = json.dumps(rows, indent=1)
    print(text)
    if a.out:
        Path(a.out).write_text(text)


if __name__ == "__main__":
    main()
