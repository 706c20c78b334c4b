"""Where the time of one resident solve goes, outside and inside the point pass and the Schur product (DESIGN.md 7).

    python profiles/solve_tail.py [cfg4] [cfg4_shard8] [--steps 20] [--warmup 5] [--trace-dir DIR]

For each bench workload the problem is created and solved exactly as bench.py's timed region does it (device-resident
observations, the device-loop graph, the same solve options, the 256 MB L2 flush between steps when
bench.needs_l2_flush says so), in two runs of `steps` solves each:

* a plain run: the step time from a CUDA-event pair around each `solve` on the solve stream, as bench.py measures it,
  the host spans the engine times inside the call (cb_ba_problem_stat 14-17: bounds, start state, upload of x, LM loop
  and download of x up to the one synchronisation) and the host time of the whole `solve` call (Python included);
* a run under torch.profiler with CUDA activities: device time per solve of every kernel, copy and memset the engine
  issues (the graph's kernels keep their names; the flush is left out).

`idle_ms` is the step time minus the device-busy time: the solve stream runs one thing at a time, so that is the sum of
the gaps in which the GPU waits on the host.  One JSON line per workload; the card's name and power limit are read in
the same run.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time
from collections import defaultdict
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import caliscope_b200 as cb  # noqa: E402
import bench  # noqa: E402

HOST_SPANS = ("set_bounds", "init_state", "upload_x", "loop_and_download_until_sync")


def card() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()  # fmt: skip
        return out[0] if out else "unknown card"
    except (OSError, subprocess.SubprocessError):
        return "unknown card"


def short(name: str) -> str:
    """`void cb::resjac_kernel<6, 0>(cb::LmState const*, ...)` -> `resjac_kernel<6, 0>`"""
    name = re.sub(r"^void\s+", "", name)
    depth, cut = 0, len(name)
    for i, ch in enumerate(name):  # the first '(' outside template brackets starts the parameter list
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            cut = i
            break
    return name[:cut].replace("cb::", "")


def run(name: str, steps: int, warmup: int, trace_dir: str | None) -> dict:
    import torch

    rig = bench.make_workload(name)
    n_c, n_p, n_o, refine = bench.WORKLOADS[name]
    stream = torch.cuda.current_stream().cuda_stream
    solve_kw = dict(ftol=1e-8, rank=0, world_size=1, stream=stream)
    d_cam = torch.from_numpy(rig.obs_cam).cuda()
    d_pt = torch.from_numpy(rig.obs_pt).cuda()
    d_xy = torch.from_numpy(np.ascontiguousarray(rig.obs_xy)).cuda()
    flush = None
    if bench.needs_l2_flush(n_c, n_p, n_o, 9 if refine else 6, 1):
        flush = torch.empty(bench.FLUSH_BYTES, dtype=torch.uint8, device="cuda")
    out: dict = {"workload": name, "card": card(), "steps": steps, "l2_flush": flush is not None}
    with cb.BAProblem(rig.cam_flags, rig.cam_const, rig.n_pts, d_cam, d_pt, d_xy, stream=stream) as prob:

        def steps_run(k: int, host: np.ndarray | None = None):
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(k)]
            res = None
            for i in range(k):
                if flush is not None:
                    flush.fill_(i & 0x7F)
                ev[i][0].record()
                t0 = time.perf_counter()
                res = prob.solve(rig.x0, **solve_kw)
                t1 = time.perf_counter()
                ev[i][1].record()
                if host is not None:
                    host += [prob.stat(14 + j) for j in range(len(HOST_SPANS))] + [1e6 * (t1 - t0)]
            torch.cuda.synchronize()
            return res, [a.elapsed_time(b) for a, b in ev]

        steps_run(warmup)
        host = np.zeros(len(HOST_SPANS) + 1)
        res, ms = steps_run(steps, host)
        host /= steps
        l0 = cb._lib.load().cb_ba_launch_count()
        steps_run(1)
        launches = cb._lib.load().cb_ba_launch_count() - l0

        acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
        with torch.profiler.profile(activities=acts) as prof:
            steps_run(steps)
        with tempfile.TemporaryDirectory() as tmp:
            path = os.path.join(trace_dir or tmp, f"solve_tail_{name}.pt.trace.json")
            if trace_dir:
                os.makedirs(trace_dir, exist_ok=True)
            prof.export_chrome_trace(path)
            trace = json.loads(Path(path).read_text())

    per = defaultdict(lambda: [0.0, 0])  # name -> [µs, count] over all profiled steps
    for e in trace.get("traceEvents", []):
        if e.get("ph") != "X" or e.get("cat") not in ("kernel", "gpu_memcpy", "gpu_memset"):
            continue
        n = short(e["name"]) if e["cat"] == "kernel" else e["name"]
        if "at::native" in n:  # the L2 flush between steps
            continue
        per[n][0] += float(e["dur"])
        per[n][1] += 1
    kernels = {n: {"us_per_solve": v[0] / steps, "launches_per_solve": v[1] / steps}
               for n, v in sorted(per.items(), key=lambda kv: -kv[1][0])}  # fmt: skip
    busy_ms = sum(v["us_per_solve"] for v in kernels.values()) / 1e3
    big = sum(v["us_per_solve"] for n, v in kernels.items() if n.startswith(("pt_pass_kernel", "schur_syrk_kernel"))) / 1e3
    step_ms = float(np.mean(ms))
    out.update({
        "nfev": int(res.nfev), "nit": int(res.nit), "status": int(res.status), "gpu_launches_per_solve": int(launches),
        "step_ms": step_ms, "step_ms_min": float(np.min(ms)), "step_ms_max": float(np.max(ms)),
        "device_busy_ms": busy_ms, "idle_ms": step_ms - busy_ms,
        "point_pass_and_schur_ms": big, "tail_ms": step_ms - big,
        "trials_per_solve": sum(v["launches_per_solve"] for n, v in kernels.items() if n.startswith("pt_pass_kernel")),
        "host_us": dict(zip(HOST_SPANS + ("whole_solve_call",), map(float, host))),
        "device_us_per_solve": kernels,
    })  # fmt: skip
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("workloads", nargs="*", default=["cfg4", "cfg4_shard8"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--trace-dir", default=None, help="keep the chrome traces here (default: a temporary directory)")
    args = ap.parse_args()
    import torch

    # start CUPTI before any graph is instantiated: a graph built before the first profiling session reports only
    # some of its kernels in the trace
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]):
        torch.zeros(1, device="cuda")
    for name in args.workloads:
        print(json.dumps(run(name, args.steps, args.warmup, args.trace_dir)), flush=True)


if __name__ == "__main__":
    main()
