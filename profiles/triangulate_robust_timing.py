"""Stage times of cb_triangulate_robust (DESIGN.md 4.8) next to cb_triangulate_refine on the same input, one JSON line per
(workload, camera covariance) pair.

    python profiles/triangulate_robust_timing.py [cfg4] [mocap] [--steps 5] [--warmup 2] [--dump-outputs DIR]

cfg4: 64 cameras, 50 000 groups, 2 000 000 observations.  mocap: 8 cameras, 500 000 groups of 2-8 rows (make_rig with
cams_per_point=8).  Cameras at the rig's true poses, noisy pixels, and 5 % of the rows moved by up to +-200 px in each
coordinate (make_rig's outlier_frac / outlier_px).  Each workload runs without and with a camera covariance (a seeded SPD
matrix in x's camera layout).  Stage times are the CUDA events recorded inside the calls (CbTriRobustStats,
CbTriRefineStats).  Consensus row evaluations are counted from the shapes: sum over the groups of min(T, max_pairs) x k
(T = k (k - 1) / 2 pairs of a group of k rows; same-camera pairs are counted although they skip the scoring).  The
distance to the true point is over the groups both calls report with status 0.  The card's name and power limit are
printed with the numbers.  --dump-outputs writes every output array of the last timed call of each variant to
DIR/<workload>_<call>_<variant>.npz.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from caliscope_b200 import synthetic  # noqa: E402
from caliscope_b200.triangulation import RefineStats, RobustStats, triangulate_refined, triangulate_robust  # noqa: E402
from dump_outputs import dump_outputs  # noqa: E402

TAU = 4.0
MAX_PAIRS = 64


def card() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()  # fmt: skip
        return out[0] if out else "unknown card"
    except (OSError, subprocess.SubprocessError):
        return "unknown card"


def make(name: str):
    if name == "cfg4":
        return synthetic.make_rig(64, 50_000, 2_000_000, seed=0, outlier_frac=0.05, outlier_px=200.0, name="cfg4")
    if name == "mocap":
        return synthetic.make_rig(8, 500_000, 2_500_000, cams_per_point=8, seed=0, outlier_frac=0.05, outlier_px=200.0,
                                  name="mocap")  # fmt: skip
    raise SystemExit(f"unknown workload {name}")


def _err(xyz, truth, m):
    d = np.linalg.norm(xyz[m] - truth[m], axis=1)
    return {"median": float(np.median(d)), "p99": float(np.percentile(d, 99))} if len(d) else None


def run(name: str, steps: int, warmup: int, dump_dir=None):
    import torch

    rig = make(name)
    ncp = int(np.where(rig.cam_flags & 1, 9, 6).sum())
    cx = rig.x_true[:ncp]
    key = rig.obs_pt.astype(np.int64)
    truth = rig.x_true[ncp:].reshape(-1, 3)[np.unique(key)]  # groups are the observed points in ascending key order
    rng = np.random.default_rng(1)
    L = 1e-4 * (np.eye(ncp) + 0.3 * rng.normal(size=(ncp, ncp)) / np.sqrt(ncp))
    k = np.bincount(rig.obs_pt, minlength=rig.n_pts).astype(np.int64)
    row_evals = float(np.sum(np.minimum(k * (k - 1) // 2, MAX_PAIRS) * k))
    args = (rig.cam_flags, rig.cam_const, cx, rig.obs_cam, key, rig.obs_xy)
    for cov in (None, L @ L.T):
        for _ in range(warmup):
            triangulate_robust(*args, threshold_px=TAU, max_pairs=MAX_PAIRS, camera_cov=cov)
            triangulate_refined(*args, camera_cov=cov)
        torch.cuda.synchronize()
        acc, ref_acc = np.zeros(5), np.zeros(5)
        for _ in range(steps):  # the two calls alternate
            st = RobustStats()
            out = triangulate_robust(*args, threshold_px=TAU, max_pairs=MAX_PAIRS, camera_cov=cov, stats=st)
            acc += [st.group_ms, st.consensus_ms, st.refine_ms, st.cov_ms, st.total_ms]
            rst = RefineStats()
            ref = triangulate_refined(*args, camera_cov=cov, stats=rst)
            ref_acc += [rst.group_ms, rst.dlt_ms, rst.refine_ms, rst.cov_ms, rst.total_ms]
        acc /= steps
        ref_acc /= steps
        variant = "cov" if cov is not None else "nocov"
        dump_outputs(dump_dir, f"{name}_robust_{variant}", out)
        dump_outputs(dump_dir, f"{name}_refined_{variant}", ref)
        both = (out.status == 0) & (ref.status == 0)
        print(json.dumps({
            "workload": name, "camera_cov": cov is not None, "card": card(), "n_cams": rig.n_cams,
            "n_groups": int(len(out.status)), "n_obs": rig.n_obs, "outlier_rows": int(rig.outlier_mask.sum()),
            "threshold_px": TAU, "max_pairs": MAX_PAIRS, "steps": steps,
            "robust_stages_ms": {"group": acc[0], "consensus": acc[1], "refine": acc[2], "cov": acc[3], "total": acc[4]},
            "robust_status_counts": np.bincount(out.status, minlength=6).tolist(),
            "consensus_row_evals": row_evals, "consensus_row_evals_per_s": row_evals / (acc[1] * 1e-3),
            "inlier_rows": int(out.inlier.sum()),
            "outliers_rejected": float((~out.inlier[rig.outlier_mask]).mean()),
            "refined_stages_ms": {"group": ref_acc[0], "dlt": ref_acc[1], "refine": ref_acc[2], "cov": ref_acc[3],
                                  "total": ref_acc[4]},
            "refined_status_counts": np.bincount(ref.status, minlength=5).tolist(),
            "groups_both_ok": int(both.sum()),
            "err_m_robust": _err(out.xyz, truth, both), "err_m_refined": _err(ref.xyz, truth, both),
            "robust_kernel_launches": st.kernel_launches, "refined_kernel_launches": rst.kernel_launches,
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
