"""Cost of fixed parameters in the LM trial (DESIGN.md 4.12), one JSON line per variant.

    python profiles/fixed_params_timing.py [--steps 5] [--warmup 1] [--trials 10]

Workload: cfg4 (caliscope_b200.synthetic.cfg4: 64 cameras, 50 k points, 2 M observations, extrinsics only), solved from
its start vector with three fixed sets: nothing fixed (a problem created without fixed lists, today's kernels), 8 whole
cameras fixed (the masked reduced system), and every tenth point fixed (the FIXP point pass and back-substitution).
Every solve runs exactly --trials LM trials (tolerances 0, max_nfev = trials + 1), so the three variants do the same
number of trials; "ms_per_trial" is the engine's CUDA-event time of the LM loop (SolveResult.solve_ms) over the trials,
the median over --steps solves after --warmup.  The card's name and power limit are read in the same run.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import caliscope_b200 as cb  # noqa: E402
from caliscope_b200 import synthetic  # noqa: E402


def card() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()  # fmt: skip
        return out[0] if out else "unknown card"
    except (OSError, subprocess.SubprocessError):
        return "unknown card"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--trials", type=int, default=10)
    args = ap.parse_args()
    r = synthetic.cfg4()
    ncp = 6 * r.n_cams
    variants = {
        "nothing fixed": {},
        "8 cameras fixed": dict(fixed_cam_params=np.arange(8 * 6)),
        "10% of points fixed": dict(fixed_points=np.arange(0, r.n_pts, 10)),
    }
    gpu = card()
    for name, kw in variants.items():
        with cb.BAProblem(r.cam_flags, r.cam_const, r.n_pts, r.obs_cam, r.obs_pt, r.obs_xy, **kw) as p:
            times, res = [], None
            for i in range(args.warmup + args.steps):
                res = p.solve(r.x0, ftol=0.0, xtol=0.0, gtol=0.0, max_nfev=args.trials + 1)
                if i >= args.warmup:
                    times.append(res.solve_ms / max(res.nfev - 1, 1))
            free = np.ones(len(r.x0), bool)
            free[kw.get("fixed_cam_params", [])] = False
            for j in kw.get("fixed_points", []):
                free[ncp + 3 * j : ncp + 3 * j + 3] = False
            print(json.dumps({
                "workload": "cfg4", "variant": name, "trials": res.nfev - 1, "nit": res.nit,
                "ms_per_trial": float(np.median(times)), "ms_per_trial_all": [round(t, 4) for t in times],
                "cost": res.cost, "fixed_entries_unchanged": bool(np.array_equal(res.x[~free], r.x0[~free])),
                "gpu": gpu,
            }), flush=True)  # fmt: skip


if __name__ == "__main__":
    main()
