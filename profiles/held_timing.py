"""Cost of held parameters -- fixed sets (DESIGN.md 4.12) and Gaussian priors (4.13) -- in the LM trial, one JSON line
per workload and variant.

    python profiles/held_timing.py [--steps 7] [--warmup 1] [--trials 10]

Workloads: cfg4 (caliscope_b200.synthetic.cfg4: 64 cameras, 50 k points, 2 M observations, extrinsics only; PCG reduced
solve) and cfg2 (8 cameras, 2 k points, 40 k observations; the one-CTA small_rig_step_kernel), solved from their start
vectors with five held sets: nothing held (a problem created without fixed sets or priors, the kernels it ran before
either existed); 8 whole cameras fixed and every tenth point fixed (the HELD camera-side and point-pass variants with an
empty prior table, and the FIXP back-substitution for the points); a full 6 x 6 information on every camera and a full
3 x 3 information on every tenth point (the same HELD variants, plus the prior-cost kernel in every camera pass).  Every
solve runs exactly --trials LM trials (tolerances 0, max_nfev = trials + 1), so the variants do the same number of
trials; "ms_per_trial" is the engine's CUDA-event time of the LM loop (SolveResult.solve_ms) over the trials, the median
over --steps solves after --warmup, the variants alternating solve by solve so that drift on a shared card hits them
alike.  "fixed_entries_unchanged" checks that a solve returns the fixed entries of x as given.  The card's name and power
limit are read in the same run.
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


def variants(r):
    """name -> BAProblem keyword arguments.  Information of the data's order (1e3), means at the start values plus 1e-3."""
    rng = np.random.default_rng(0)
    nc, ncp = r.n_cams, 6 * r.n_cams
    A = rng.standard_normal((nc, 6, 6))
    info = np.zeros((nc, 9, 9))
    info[:, :6, :6] = 1e3 * (np.einsum("kij,klj->kil", A, A) / 6 + np.eye(6))
    mean = np.zeros((nc, 9))
    mean[:, :6] = r.x0[:ncp].reshape(nc, 6) + 1e-3
    pts = np.arange(0, r.n_pts, 10)
    B = rng.standard_normal((len(pts), 3, 3))
    pinfo = 1e3 * (np.einsum("kij,klj->kil", B, B) / 3 + np.eye(3))
    pmean = r.x0[ncp:].reshape(-1, 3)[pts] + 1e-3
    return {
        "nothing held": {},
        "8 cameras fixed": dict(fixed_cam_params=np.arange(8 * 6)),
        "every tenth point fixed": dict(fixed_points=pts),
        f"full camera priors on all {nc} cameras": dict(camera_priors=(np.arange(nc), mean, info)),
        "point priors on every tenth point": dict(point_priors=(pts, pmean, pinfo)),
    }


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--trials", type=int, default=10)
    args = ap.parse_args()
    gpu = card()
    for wl, r in (("cfg4", synthetic.cfg4()), ("cfg2", synthetic.cfg2())):
        ncp = 6 * r.n_cams
        kws = variants(r)
        probs = {name: cb.BAProblem(r.cam_flags, r.cam_const, r.n_pts, r.obs_cam, r.obs_pt, r.obs_xy, **kw)
                 for name, kw in kws.items()}  # fmt: skip
        times = {name: [] for name in probs}
        last = {}
        for i in range(args.warmup + args.steps):
            for name, p in probs.items():
                res = p.solve(r.x0, ftol=0.0, xtol=0.0, gtol=0.0, max_nfev=args.trials + 1)
                last[name] = res
                if i >= args.warmup:
                    times[name].append(res.solve_ms / max(res.nfev - 1, 1))
        base = float(np.median(times["nothing held"]))
        for name, p in probs.items():
            res, med = last[name], float(np.median(times[name]))
            free = np.ones(len(r.x0), bool)
            free[kws[name].get("fixed_cam_params", [])] = False
            for j in kws[name].get("fixed_points", []):
                free[ncp + 3 * j : ncp + 3 * j + 3] = False
            print(json.dumps({
                "workload": wl, "variant": name, "trials": res.nfev - 1, "nit": res.nit,
                "ms_per_trial": med, "vs_nothing_held": med / base, "ms_per_trial_all": [round(t, 4) for t in times[name]],
                "cost": res.cost, "fixed_entries_unchanged": bool(np.array_equal(res.x[~free], r.x0[~free])),
                "direct_solve": int(p.stat(2)), "gpu": gpu,
            }), flush=True)  # fmt: skip
            p.close()


if __name__ == "__main__":
    main()
