"""ctypes binding of ``libcaliscope_b200.so`` (C ABI in ``include/caliscope_b200.h``).

The library is the product: if it is missing or cannot be loaded this module raises --
there is no CPU fallback anywhere in ``caliscope_b200``.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
LIB_NAME = "libcaliscope_b200.so"

CB_CAM_FREE_INTRINSICS = 1
CB_CAM_FISHEYE = 2
LOSS_IDS = {"linear": 0, "soft_l1": 1, "huber": 2, "cauchy": 3, "arctan": 4}


class EngineUnavailable(RuntimeError):
    """libcaliscope_b200.so is missing / unloadable, or no CUDA device is usable."""


class EngineError(RuntimeError):
    def __init__(self, code: int, what: str, detail: str):
        super().__init__(f"{what} failed: {detail} (code {code})")
        self.code = code


class ProblemDesc(C.Structure):
    _fields_ = [
        ("n_cams", C.c_int32),
        ("n_pts", C.c_int32),
        ("n_obs", C.c_int64),
        ("cam_flags", C.c_void_p),
        ("cam_const", C.c_void_p),
        ("obs_cam", C.c_void_p),
        ("obs_pt", C.c_void_p),
        ("obs_xy", C.c_void_p),
        ("obs_on_device", C.c_int32),
        ("obs_cam_bits", C.c_int32),
        ("cam_order", C.c_void_p),
        ("n_constraints", C.c_int64),
        ("groups_a", C.c_void_p),
        ("groups_b", C.c_void_p),
        ("distances", C.c_void_p),
        ("weights", C.c_void_p),
    ]


class Priors(C.Structure):  # CbBaPriors
    _fields_ = [
        ("n_cams", C.c_int32),
        ("cams", C.c_void_p),
        ("cam_mean", C.c_void_p),
        ("cam_info", C.c_void_p),
        ("n_pts", C.c_int32),
        ("pts", C.c_void_p),
        ("pt_mean", C.c_void_p),
        ("pt_info", C.c_void_p),
    ]


ALLREDUCE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p)


class Options(C.Structure):
    _fields_ = [
        ("ftol", C.c_double),
        ("xtol", C.c_double),
        ("gtol", C.c_double),
        ("max_nfev", C.c_int64),
        ("loss", C.c_int32),
        ("f_scale", C.c_double),
        ("verbose", C.c_int32),
        ("use_bounds", C.c_int32),
        ("lambda0", C.c_double),
        ("pcg_tol", C.c_double),
        ("pcg_max_iter", C.c_int32),
        ("allreduce", ALLREDUCE_FN),
        ("allreduce_user", C.c_void_p),
        ("nccl_comm", C.c_void_p),
        ("peer_group", C.c_void_p),
        ("rank", C.c_int32),
        ("world_size", C.c_int32),
        ("time_kernels", C.c_int32),
        ("pad_", C.c_int32),
    ]


class Result(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("nfev", C.c_int64),
        ("njev", C.c_int64),
        ("nit", C.c_int64),
        ("cost", C.c_double),
        ("initial_cost", C.c_double),
        ("optimality", C.c_double),
        ("lambda_final", C.c_double),
        ("pcg_iterations", C.c_int64),
        ("kernel_launches", C.c_int64),
        ("solve_ms", C.c_double),
        ("rj_ms", C.c_double),
        ("rj_launches", C.c_int64),
        ("syrk_ms", C.c_double),
        ("syrk_launches", C.c_int64),
        ("trials_queued", C.c_int64),
        ("used_graph", C.c_int32),
        ("pad_", C.c_int32),
    ]


class TriStats(C.Structure):
    _fields_ = [
        ("group_ms", C.c_double),
        ("dlt_ms", C.c_double),
        ("total_ms", C.c_double),
        ("kernel_launches", C.c_int32),
        ("pad_", C.c_int32),
    ]


class TriRefineStats(C.Structure):
    _fields_ = [
        ("group_ms", C.c_double),
        ("dlt_ms", C.c_double),
        ("refine_ms", C.c_double),
        ("cov_ms", C.c_double),
        ("total_ms", C.c_double),
        ("kernel_launches", C.c_int32),
        ("pad_", C.c_int32),
    ]


class TriRobustStats(C.Structure):
    _fields_ = [
        ("group_ms", C.c_double),
        ("consensus_ms", C.c_double),
        ("refine_ms", C.c_double),
        ("cov_ms", C.c_double),
        ("total_ms", C.c_double),
        ("kernel_launches", C.c_int32),
        ("pad_", C.c_int32),
    ]


class ResectStats(C.Structure):
    _fields_ = [
        ("group_ms", C.c_double),
        ("consensus_ms", C.c_double),
        ("refine_ms", C.c_double),
        ("cov_ms", C.c_double),
        ("total_ms", C.c_double),
        ("kernel_launches", C.c_int32),
        ("pad_", C.c_int32),
    ]


class RigidStats(C.Structure):
    _fields_ = [
        ("group_ms", C.c_double),
        ("points_ms", C.c_double),
        ("consensus_ms", C.c_double),
        ("refine_ms", C.c_double),
        ("cov_ms", C.c_double),
        ("total_ms", C.c_double),
        ("kernel_launches", C.c_int32),
        ("pad_", C.c_int32),
    ]


class RigidModelStats(C.Structure):
    _fields_ = [
        ("group_ms", C.c_double),
        ("solve_ms", C.c_double),
        ("cov_ms", C.c_double),
        ("total_ms", C.c_double),
        ("kernel_launches", C.c_int32),
        ("pad_", C.c_int32),
    ]


class RelPoseStats(C.Structure):
    _fields_ = [
        ("group_ms", C.c_double),
        ("consensus_ms", C.c_double),
        ("refine_ms", C.c_double),
        ("cov_ms", C.c_double),
        ("total_ms", C.c_double),
        ("kernel_launches", C.c_int32),
        ("pad_", C.c_int32),
    ]


class IntrinsicsStats(C.Structure):
    _fields_ = [
        ("group_ms", C.c_double),
        ("start_ms", C.c_double),
        ("lm_ms", C.c_double),
        ("cov_ms", C.c_double),
        ("total_ms", C.c_double),
        ("iterations", C.c_int32),
        ("kernel_launches", C.c_int32),
    ]


# every symbol include/caliscope_b200.h declares: name -> (restype, argtypes)
_P = C.c_void_p
_D = C.POINTER(C.c_double)
SYMBOLS = {
    "cb_ba_abi_version": (C.c_int, []),
    "cb_ba_error_string": (C.c_char_p, [C.c_int]),
    "cb_ba_last_error": (C.c_char_p, []),
    "cb_ba_default_options": (None, [C.POINTER(Options)]),
    "cb_ba_problem_create": (C.c_int, [C.POINTER(ProblemDesc), C.c_int, _P, C.POINTER(_P)]),
    "cb_ba_problem_create_fixed": (
        C.c_int,
        [C.POINTER(ProblemDesc), C.c_int32, _P, C.c_int32, _P, C.c_int, _P, C.POINTER(_P)],
    ),
    "cb_ba_problem_create_priors": (
        C.c_int,
        [C.POINTER(ProblemDesc), C.c_int32, _P, C.c_int32, _P, C.POINTER(Priors), C.c_int, _P, C.POINTER(_P)],
    ),
    "cb_ba_problem_destroy": (C.c_int, [_P]),
    "cb_ba_problem_n_params": (C.c_int64, [_P]),
    "cb_ba_problem_stat": (C.c_double, [_P, C.c_int]),
    "cb_ba_constraint_rows": (C.c_int, [_P, _P, _P, _P, _P]),
    "cb_ba_solve": (C.c_int, [_P, C.POINTER(Options), _P, C.POINTER(Result), _P]),
    "cb_ba_solve_from": (C.c_int, [_P, C.POINTER(Options), _P, _P, C.POINTER(Result), _P]),
    "cb_ba_residuals": (C.c_int, [_P, _P, _P, _P]),
    "cb_ba_jacobian_blocks": (C.c_int, [_P, _P, _P, _P, _P]),
    "cb_ba_reproj_errors_px": (C.c_int, [_P, _P, _P, _P]),
    "cb_ba_cam_stride": (C.c_int, [_P]),
    "cb_ba_normal_equations": (
        C.c_int,
        [_P, _P, C.c_double, C.c_int32, C.c_double, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P],
    ),
    "cb_ba_covariance": (
        C.c_int,
        [_P, _P, C.c_int32, C.c_double, C.c_int32, _P, C.c_double, _P, _P, _P, _P, _P, _P],
    ),
    "cb_ba_error_order_stats": (C.c_int, [_P, _P, C.c_double, _P, _P, _P, _P, _P]),
    "cb_ba_rmse_px": (C.c_int, [_P, _P, _P, _P, _P]),
    "cb_ba_cull": (C.c_int, [_P, _P, _P, C.c_int32, C.POINTER(_P), _P, _P, _P]),
    "cb_ba_debug_pcg_time": (C.c_int, [_P, C.c_int, C.c_int, _P, _P]),
    "cb_debug_fp64_peak": (C.c_int, [C.c_int, _P, _P]),
    "cb_shard_select": (C.c_int, [C.c_int64, _P, _P, _P, C.c_int32, C.c_int32, C.c_int64, _P, _P, _P, _P, _P, C.c_int32]),
    "cb_csv_write_numeric": (C.c_int, [C.c_char_p, C.c_char_p, C.c_int64, C.c_int32, _P, _P, C.c_int32]),
    "cb_csv_scan": (C.c_int, [C.c_char_p, _P, _P]),
    "cb_csv_parse_numeric": (C.c_int, [C.c_char_p, C.c_int64, C.c_int32, _P, _P, _P, C.c_int32]),
    "cb_pnp_ippe": (C.c_int, [C.c_int32, _P, _P, _P, C.c_int64, _P, _P, _P, _P, C.c_int32, C.c_int32, _P, _P, _P, _P, _P, _P, _P,
                              _P, C.c_int, _P]),
    "cb_stereo_rmse": (C.c_int, [C.c_int32, _P, _P, _P, C.c_int32, _P, _P, _P, C.c_int64, _P, _P, _P, C.c_int32, _P, _P, _P,
                                 C.c_int, _P]),
    "cb_relative_pose_network": (C.c_int, [C.c_int32, C.c_int32, _P, _P, _P, _P, _P, C.c_double, C.c_double, C.c_int32, _P, _P, _P, _P,
                                           _P, _P, C.c_int64, _P, _P, _P, C.c_int, _P]),
    "cb_undistort_points": (C.c_int, [C.c_int32, _P, _P, _P, C.c_int64, _P, _P, C.c_int, C.c_int, _P, C.c_int, _P]),
    "cb_triangulate_dlt": (
        C.c_int,
        [C.c_int32, _P, C.c_int64, _P, _P, _P, C.c_int, C.c_int32, C.POINTER(C.c_int32), _P, _P, _P, _P,
         C.POINTER(TriStats), C.c_int, _P],
    ),
    "cb_undistort_triangulate": (
        C.c_int,
        [C.c_int32, _P, _P, _P, _P, C.c_int64, _P, _P, _P, C.c_int, C.c_int32, C.POINTER(C.c_int32), _P, _P, _P, _P,
         C.POINTER(TriStats), C.c_int, _P],
    ),
    "cb_triangulate_refine": (
        C.c_int,
        [C.c_int32, _P, _P, _P, _P, C.c_int64, _P, _P, _P, C.c_int, C.c_double, C.c_int32, C.c_double, C.c_int32,
         C.POINTER(C.c_int32), _P, _P, _P, _P, _P, _P, C.POINTER(TriRefineStats), C.c_int, _P],
    ),
    "cb_triangulate_robust": (
        C.c_int,
        [C.c_int32, _P, _P, _P, _P, C.c_int64, _P, _P, _P, C.c_int, C.c_double, C.c_int32, C.c_int32, C.c_double,
         C.c_int32, C.c_double, C.c_int32, C.POINTER(C.c_int32), _P, _P, _P, _P, _P, _P, _P, _P,
         C.POINTER(TriRobustStats), C.c_int, _P],
    ),
    "cb_resect_robust": (
        C.c_int,
        [C.c_int32, _P, _P, _P, C.c_int32, _P, _P, C.c_int64, _P, _P, _P, _P, C.c_int, C.c_double, C.c_int32, C.c_int32,
         C.c_int32, C.c_double, C.c_int32, C.c_double, C.c_int32, C.POINTER(C.c_int32), _P, _P, _P, _P, _P, _P, _P, _P,
         _P, C.POINTER(ResectStats), C.c_int, _P],
    ),
    "cb_rigid_pose_robust": (
        C.c_int,
        [C.c_int32, _P, _P, _P, _P, C.c_int32, _P, C.c_int64, _P, _P, _P, _P, C.c_int, C.c_double, C.c_int32, C.c_int32,
         C.c_int32, C.c_int32, _P, _P, C.c_double, C.c_int32, C.c_double, C.c_int32, C.POINTER(C.c_int32), _P, _P, _P,
         _P, _P, _P, _P, _P, _P, C.POINTER(RigidStats), C.c_int, _P],
    ),
    "cb_rigid_pose_robust_gp3p": (
        C.c_int,
        [C.c_int32, _P, _P, _P, _P, C.c_int32, _P, C.c_int64, _P, _P, _P, _P, C.c_int, C.c_double, C.c_int32, C.c_int32,
         C.c_int32, C.c_int32, C.c_int32, _P, _P, C.c_double, C.c_int32, C.c_double, C.c_int32, C.POINTER(C.c_int32),
         _P, _P, _P, _P, _P, _P, _P, _P, _P, C.POINTER(RigidStats), C.c_int, _P],
    ),
    "cb_rigid_model_refine": (
        C.c_int,
        [C.c_int32, _P, _P, _P, _P, C.c_int32, _P, C.c_int32, _P, C.c_int64, _P, _P, _P, _P, C.c_int, C.c_int32, _P, _P,
         C.c_double, C.c_int32, C.c_double, C.c_int32, C.POINTER(C.c_int32), _P, _P, _P, _P, _P, _P, _P, _P, _P, _P,
         _P, _P, C.POINTER(RigidModelStats), C.c_int, _P],
    ),
    "cb_relative_pose_robust": (
        C.c_int,
        [C.c_int32, _P, _P, _P, C.c_int64, _P, _P, _P, C.c_int, C.c_double, C.c_int32, C.c_int32, C.c_double, C.c_int32,
         C.c_double, C.c_int32, C.POINTER(C.c_int32), _P, _P, _P, _P, _P, _P, _P, _P, _P,
         C.POINTER(RelPoseStats), C.c_int, _P],
    ),
    "cb_calibrate_intrinsics": (
        C.c_int,
        [C.c_int32, _P, _P, _P, _P, C.c_int64, _P, _P, _P, _P, C.c_int, C.c_int32, C.c_int32, C.c_int32, C.c_double,
         C.c_int32,
         C.POINTER(C.c_int32), _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P,
         C.POINTER(IntrinsicsStats), C.c_int, _P],
    ),
    "cb_peer_create": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int64, C.POINTER(_P), _P]),
    "cb_peer_connect": (C.c_int, [_P, _P]),
    "cb_peer_destroy": (C.c_int, [_P]),
    "cb_nccl_unique_id": (C.c_int, [_P]),
    "cb_nccl_comm_create": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.POINTER(_P)]),
    "cb_nccl_comm_destroy": (C.c_int, [_P]),
    "cb_ba_launch_count": (C.c_int64, []),
}

_lib = None


def lib_path() -> Path:
    return Path(os.environ.get("CALISCOPE_B200_LIB", PKG_DIR / LIB_NAME))


def load() -> C.CDLL:
    """Load the shared library (once) and type every exported entry point."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if not path.exists():
        raise EngineUnavailable(
            f"{path} not found -- build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a).  caliscope_b200 has no CPU fallback."
        )
    try:
        lib = C.CDLL(str(path))
    except OSError as e:  # pragma: no cover - depends on the box
        raise EngineUnavailable(f"cannot load {path}: {e}") from e
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(code: int, what: str) -> None:
    if code == 0:
        return
    lib = load()
    detail = (lib.cb_ba_last_error() or b"").decode() or (lib.cb_ba_error_string(code) or b"").decode()
    if code == -3:
        raise EngineUnavailable(f"{what}: {detail}")
    raise EngineError(code, what, detail)
