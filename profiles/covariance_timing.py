"""Stage times of BAProblem.covariance (DESIGN.md 4.6) at the solution of a bench workload, one JSON line per workload.

    python profiles/covariance_timing.py [cfg4] [sparse64] [--steps 10] [--warmup 3]

Solves once, then times `steps` covariance calls (camera block and every point block, host buffers out).  The stage
times are CUDA events recorded inside the call (cb_ba_problem_stat 4 / 5 / 6); the stage flops are counted from the
shapes.  The card's name and power limit are printed with the numbers.
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import caliscope_b200 as cb  # noqa: E402
from bench import make_workload  # noqa: E402


def card() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()  # fmt: skip
        return out[0] if out else "unknown card"
    except (OSError, subprocess.SubprocessError):
        return "unknown card"


def run(name: str, steps: int, warmup: int) -> dict:
    import torch

    rig = make_workload(name)
    with cb.BAProblem(rig.cam_flags, rig.cam_const, rig.n_pts, rig.obs_cam, rig.obs_pt, rig.obs_xy) as p:
        sol = p.solve(rig.x0)
        P, nP = p.cam_stride, p.n_cams * p.cam_stride
        for _ in range(warmup):
            cov = p.covariance(sol.x)
        torch.cuda.synchronize()
        stages = np.zeros(3)
        t0 = time.perf_counter()
        for _ in range(steps):
            cov = p.covariance(sol.x)
            stages += [p.stat(4), p.stat(5), p.stat(6)]
        wall = time.perf_counter() - t0
        schur_flop = p.stat(1)
    stages /= steps
    # unique cameras per point: the marginal pass forms Z_c^T Sigma_cd Z_d for every unordered pair (c, d) of them
    k = np.bincount(np.unique(rig.obs_pt.astype(np.int64) * rig.n_cams + rig.obs_cam) // rig.n_cams, minlength=rig.n_pts)
    n_sw = -(-nP // 32) * 32
    names = ("linearisation_schur", "dense_inverse", "point_marginals")
    flops = (
        float(schur_flop),  # the Schur product; the point pass is latency bound and not counted
        float(4 * n_sw**3),  # block sweep: n/32 steps of an n x n x 32 x 2 update
        float(np.sum(k * (k + 1) / 2 * (2 * 3 * P * P + 2 * 9 * P))),
    )
    return {
        "workload": name, "card": card(), "n_cams": rig.n_cams, "n_pts": rig.n_pts, "n_obs": rig.n_obs,
        "n_camera_params": int(nP), "mean_cameras_per_point": float(k.mean()), "steps": steps,
        "ms_per_call": 1e3 * wall / steps,
        "stages_ms": dict(zip(names, map(float, stages))),
        "stage_flops": dict(zip(names, flops)),
        "stage_gflops_per_s": {n: f / (t * 1e-3) / 1e9 if t > 0 else None for n, f, t in zip(names, flops, stages)},
        "dof": int(cov.dof), "variance_factor": float(cov.variance_factor),
    }  # fmt: skip


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("workloads", nargs="*", default=["cfg4", "sparse64"])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    for name in args.workloads:
        print(json.dumps(run(name, args.steps, args.warmup)), flush=True)


if __name__ == "__main__":
    main()
