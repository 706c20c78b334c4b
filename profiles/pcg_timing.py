"""Per-iteration cost of the PCG cluster kernel: time launches forced to k iterations, fit a line."""
import ctypes as C
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import caliscope_b200 as cb  # noqa: E402
from bench import make_workload  # noqa: E402
from caliscope_b200 import _lib  # noqa: E402

lib = _lib.load()
# cfg2 (48 camera parameters) is solved directly, without PCG
for name in sys.argv[1:] or ["cfg3", "cfg4", "cfg4_intrinsics"]:
    rig = make_workload(name)
    with cb.BAProblem(rig.cam_flags, rig.cam_const, rig.n_pts, rig.obs_cam, rig.obs_pt, rig.obs_xy) as p:
        p.normal_equations(rig.x0, 1e-4)
        out = []
        for k in (1, 20, 100, 200):
            ms = C.c_double()
            _lib.check(lib.cb_ba_debug_pcg_time(p._h, k, 20, C.addressof(ms), None), "pcg_time")
            out.append((k, ms.value * 1e3))
        slope = (out[-1][1] - out[1][1]) / (out[-1][0] - out[1][0])
        print(f"{name}: nP={p.n_cams * p.cam_stride} " + " ".join(f"it{k}:{us:.1f}us" for k, us in out) + f" -> {slope:.2f} us/iteration")
