"""Stage times of cb_triangulate_refine (DESIGN.md 4.7), one JSON line per (workload, camera covariance) pair.

    python profiles/triangulate_refine_timing.py [cfg4] [mocap] [--steps 5] [--warmup 2] [--dump-outputs DIR]

cfg4: 64 cameras, 50 000 groups, 2 000 000 observations (synthetic.cfg4).  mocap: 8 cameras, 500 000 groups of 2-8 rows
(make_rig with cams_per_point=8).  Cameras at the rig's true poses, noisy pixels.  Each workload runs without and with a
camera covariance (a seeded SPD matrix in x's camera layout).  Stage times are the CUDA events recorded inside the call
(CbTriRefineStats).  The mean LM step count comes from the oracle on a 2000-group sample (same rule, so the same counts
up to rounding at the convergence floor); refine-stage row evaluations are (steps + 2) x rows per group: the start, one
evaluation per step, and the behind-camera pass.  Covariance flops are counted from the shapes: pairs x 2 (3 P^2 + 9 P)
over the unordered pairs of each group's distinct cameras.  The card's name and power limit are printed with the numbers.
--dump-outputs writes every output array of the last timed call of each variant to DIR/<workload>_<variant>.npz.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from caliscope_b200 import synthetic  # noqa: E402
from caliscope_b200.triangulation import RefineStats, triangulate_refined  # noqa: E402
from dump_outputs import dump_outputs  # noqa: E402


def card() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()  # fmt: skip
        return out[0] if out else "unknown card"
    except (OSError, subprocess.SubprocessError):
        return "unknown card"


def make(name: str):
    if name == "cfg4":
        return synthetic.cfg4(seed=0)
    if name == "mocap":
        return synthetic.make_rig(8, 500_000, 2_500_000, cams_per_point=8, seed=0, name="mocap")
    raise SystemExit(f"unknown workload {name}")


def mean_steps(rig, ncp: int, sample: int = 2000) -> float:
    from oracle import triangulation_refine as T

    pts = np.random.default_rng(0).choice(rig.n_pts, sample, replace=False)
    rows = np.flatnonzero(np.isin(rig.obs_pt, pts))
    grp, G = T.group_rows(rig.obs_pt[rows])
    args = (rig.cam_flags, rig.cam_const, rig.x_true[:ncp], rig.obs_cam[rows], rig.obs_xy[rows], grp)
    x0 = T.dlt_start(*args, G)
    _, _, status, steps = T.refine_points(*args, x0)
    live = status != T.STATUS_FEW_ROWS
    return float(steps[live].mean())


def run(name: str, steps: int, warmup: int, dump_dir=None):
    import torch

    rig = make(name)
    ncp = int(np.where(rig.cam_flags & 1, 9, 6).sum())
    P = 9 if (rig.cam_flags & 1).any() else 6
    cx = rig.x_true[:ncp]
    key = rig.obs_pt.astype(np.int64)
    rng = np.random.default_rng(1)
    L = 1e-4 * (np.eye(ncp) + 0.3 * rng.normal(size=(ncp, ncp)) / np.sqrt(ncp))
    n_rows = np.bincount(rig.obs_pt, minlength=rig.n_pts)
    k = np.bincount(np.unique(key * rig.n_cams + rig.obs_cam) // rig.n_cams, minlength=rig.n_pts)
    live = n_rows >= 2
    pairs = float(np.sum((k * (k + 1) / 2)[live]))
    m_steps = mean_steps(rig, ncp)
    for cov in (None, L @ L.T):
        for _ in range(warmup):
            triangulate_refined(rig.cam_flags, rig.cam_const, cx, rig.obs_cam, key, rig.obs_xy, camera_cov=cov)
        torch.cuda.synchronize()
        acc = np.zeros(5)
        for _ in range(steps):
            st = RefineStats()
            out = triangulate_refined(rig.cam_flags, rig.cam_const, cx, rig.obs_cam, key, rig.obs_xy, camera_cov=cov,
                                      stats=st)  # fmt: skip
            acc += [st.group_ms, st.dlt_ms, st.refine_ms, st.cov_ms, st.total_ms]
        acc /= steps
        dump_outputs(dump_dir, f"{name}_{'cov' if cov is not None else 'nocov'}", out)
        cov_flop = pairs * 2 * (3 * P * P + 9 * P) if cov is not None else 0.0
        row_evals = (m_steps + 2) * float(n_rows[live].sum())
        print(json.dumps({
            "workload": name, "camera_cov": cov is not None, "card": card(), "n_cams": rig.n_cams, "P": P,
            "n_groups": int(len(out.status)), "n_obs": rig.n_obs, "mean_rows_per_group": float(n_rows[live].mean()),
            "status_counts": np.bincount(out.status, minlength=5).tolist(), "steps": steps,
            "stages_ms": {"group": acc[0], "dlt": acc[1], "refine": acc[2], "cov": acc[3], "total": acc[4]},
            "mean_lm_steps_sampled": m_steps, "refine_row_evals_per_s": row_evals / (acc[2] * 1e-3),
            "cov_pairs": pairs, "cov_flop": cov_flop,
            "cov_gflop_per_s": cov_flop / (acc[3] * 1e-3) / 1e9 if cov is not None and acc[3] > 0 else None,
            "kernel_launches": st.kernel_launches,
        }), flush=True)  # fmt: skip


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("workloads", nargs="*", default=["cfg4", "mocap"])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    args = ap.parse_args()
    for name in args.workloads:
        run(name, args.steps, args.warmup, args.dump_outputs)


if __name__ == "__main__":
    main()
