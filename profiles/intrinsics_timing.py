"""Stage times of cb_calibrate_intrinsics (DESIGN.md 4.10), one JSON line per workload.

    python profiles/intrinsics_timing.py [one3000] [eight1000] [sixtyfour300] [--steps 3] [--warmup 1] [--no-cpu]
        [--dump-outputs DIR]

Workloads, all of a 54-corner (9 x 6) chessboard seen with 0.5 px noise (tests/_intrinsics_cases.py): one3000 = one
1920 x 1080 camera with 3000 views; eight1000 = 8 cameras (two lenses alternating) with 1000 views each;
sixtyfour300 = 64 cameras with 300 views each.  Times are the CUDA events recorded inside the call
(CbIntrinsicsStats), the median over --steps timed calls after --warmup; the parameter error is |theta_hat - truth| /
std, worst over cameras and parameters.  For context only, cv2.calibrateCamera runs on 30 / 100 / 300 views of the first
camera on one host core (a CPU library, not a baseline of the same computation).  The card's name and power limit are
read in the same run and printed with the numbers.  --dump-outputs writes every output array of the last timed call of
each workload to DIR/<workload>.npz.
"""
import argparse
import json
import os
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from caliscope_b200.intrinsics import IntrinsicsStats, calibrate_cameras  # noqa: E402
from dump_outputs import dump_outputs  # noqa: E402
from tests._intrinsics_cases import STRONG, WEBCAM, cv2_views, make_case  # noqa: E402

WORKLOADS = {"one3000": ([WEBCAM], 3000), "eight1000": ([WEBCAM, STRONG] * 4, 1000),
             "sixtyfour300": ([WEBCAM, STRONG] * 32, 300)}  # fmt: skip


def card() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()  # fmt: skip
        return out[0] if out else "unknown card"
    except (OSError, subprocess.SubprocessError):
        return "unknown card"


def cv2_context(case) -> dict:
    try:
        import cv2
    except ImportError:
        return {}
    cv2.setNumThreads(1)
    out = {}
    keys = np.unique(case.obs_key[case.obs_cam == 0])
    for nv in (30, 100, 300):
        if nv > len(keys):
            break
        objs, imgs, _ = cv2_views(case, 0, keys[:nv])
        t = time.perf_counter()
        cv2.calibrateCamera(objs, imgs, tuple(int(v) for v in case.image_size[0]), None, None)
        out[f"cv2_{nv}_views_s"] = round(time.perf_counter() - t, 3)
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("workloads", nargs="*", default=list(WORKLOADS))
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    a = ap.parse_args()
    name = card()
    for w in a.workloads:
        lenses, nv = WORKLOADS[w]
        case = make_case(31, lenses, nv)
        times = []
        for i in range(a.warmup + a.steps):
            st = IntrinsicsStats()
            t = time.perf_counter()
            res = calibrate_cameras(case.obs_cam, case.obs_key, case.obs_obj, case.obs_px, case.image_size, stats=st)
            wall = (time.perf_counter() - t) * 1e3
            if i >= a.warmup:
                times.append((st.total_ms, st.group_ms, st.start_ms, st.lm_ms, st.cov_ms, wall))
        dump_outputs(a.dump_outputs, w, res)
        med = np.median(np.array(times), axis=0)
        line = {"workload": w, "cameras": len(lenses), "views_per_camera": nv, "rows": int(len(case.obs_cam)),
                "total_ms": round(med[0], 3), "group_ms": round(med[1], 3), "start_ms": round(med[2], 3),
                "lm_ms": round(med[3], 3), "cov_ms": round(med[4], 3), "wall_ms": round(med[5], 3),
                "lm_iterations_max": int(res.iterations.max()), "lm_iterations_median": float(np.median(res.iterations)),
                "statuses": {int(s): int(c) for s, c in zip(*np.unique(res.status, return_counts=True))},
                "views_used": int(res.n_views.sum()), "kernel_launches": st.kernel_launches,
                "max_err_over_std": float(np.nanmax(np.abs(res.params - case.truth) / res.std)),
                "card": name, "host_cores": os.cpu_count()}  # fmt: skip
        if not a.no_cpu:
            line.update(cv2_context(case))
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
