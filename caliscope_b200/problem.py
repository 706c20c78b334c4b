"""Device-resident bundle-adjustment problem: the arrays ``CaptureVolume.optimize`` hands to
scipy (/root/reference/src/caliscope/core/capture_volume.py:346-365, 390-399) flattened for the
C ABI, plus thin wrappers over the evaluation entry points."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import _lib as L


def _ptr(a: np.ndarray) -> int:
    return a.ctypes.data


def _prior_arrays(priors, w: int, name: str) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(index, mean, info) as contiguous int32 (k,), float64 (k, w), float64 (k, w, w); None: no priors."""
    if priors is None:
        return np.zeros(0, np.int32), np.zeros((0, w)), np.zeros((0, w, w))
    idx, mean, info = priors
    idx = np.ascontiguousarray(idx, dtype=np.int32).ravel()
    mean = np.ascontiguousarray(mean, dtype=np.float64)
    info = np.ascontiguousarray(info, dtype=np.float64)
    k = len(idx)
    if mean.shape != (k, w) or info.shape != (k, w, w):
        raise ValueError(f"{name}: mean must have shape ({k}, {w}) and info ({k}, {w}, {w}), got {mean.shape} and "
                         f"{info.shape}")  # fmt: skip
    return idx, mean, info


def _check_device_obs(obs_cam, obs_pt, obs_xy, device: int) -> int:
    """Validate a device-resident observation list, which the engine reads in place: CUDA tensors on ``device``,
    contiguous, equal lengths; obs_cam int32 or int16, obs_pt int32, obs_xy float64 (n, 2).  Returns obs_cam's width in
    bits.  Nothing is converted: a conversion would be a copy the caller did not ask for."""
    dtypes = {"obs_cam": ("torch.int32", "torch.int16"), "obs_pt": ("torch.int32",), "obs_xy": ("torch.float64",)}
    arrays = {"obs_cam": obs_cam, "obs_pt": obs_pt, "obs_xy": obs_xy}
    for name, a in arrays.items():
        dev = getattr(a, "device", None)
        if getattr(dev, "type", None) != "cuda" or dev.index != device:
            raise ValueError(f"{name} must be a CUDA tensor on cuda:{device}, got device {dev}")
        if str(getattr(a, "dtype", None)) not in dtypes[name]:
            raise ValueError(f"{name} must have dtype {' or '.join(dtypes[name])}, got {getattr(a, 'dtype', None)}")
        if not a.is_contiguous():
            raise ValueError(f"{name} must be contiguous")
    n = int(obs_cam.shape[0])
    if tuple(obs_cam.shape) != (n,) or tuple(obs_pt.shape) != (n,):
        raise ValueError(f"obs_cam and obs_pt must be 1-D of the same length, got {tuple(obs_cam.shape)}, {tuple(obs_pt.shape)}")
    if tuple(obs_xy.shape) != (n, 2):
        raise ValueError(f"obs_xy must have shape ({n}, 2), got {tuple(obs_xy.shape)}")
    return 16 if str(obs_cam.dtype) == "torch.int16" else 32


def blocks_to_arrays(blocks) -> tuple[np.ndarray, np.ndarray]:
    """``BundleParameterization.blocks`` (bundle_parameterization.py:36-51) -> (cam_flags, cam_const)."""
    flags = np.zeros(len(blocks), np.int32)
    const = np.zeros((len(blocks), 9), np.float64)
    for i, b in enumerate(blocks):
        fixed = tuple(float(v) for v in b.dist_fixed)
        if b.fisheye:
            if len(fixed) != 4:
                raise ValueError(f"Fisheye projection requires 4 distortion coefficients, got {len(fixed)}")
            flags[i] = L.CB_CAM_FISHEYE
            const[i] = [b.fx_initial, b.fy_initial, b.cx, b.cy, *fixed, 0.0]
        else:
            fixed = (fixed + (0.0, 0.0, 0.0))[:3]
            flags[i] = L.CB_CAM_FREE_INTRINSICS if b.free_intrinsics else 0
            const[i] = [b.fx_initial, b.fy_initial, b.cx, b.cy, b.k1_initial, b.k2_initial, *fixed]
    return flags, const


@dataclass
class Covariance:
    """``BAProblem.covariance``: parameter covariance at x, relative to the gauge ``fixed`` (DESIGN.md section 4.6).

    ``cameras``: (n_camera_params, n_camera_params) in x's camera layout; rows and columns of fixed parameters are 0,
    those of cameras without observations NaN.  ``points``: (n_pts, 3, 3), NaN where ``point_rank`` is not 3 (points
    seen by one camera, unobserved points, points of rigid-constraint components, rank -1); the problem's fixed points
    have zero blocks and rank -2.  ``variance_factor``: the s2
    the inverse was scaled by; ``dof``: m - rank of the gauge-fixed Jacobian."""

    cameras: np.ndarray
    points: np.ndarray | None
    point_rank: np.ndarray
    variance_factor: float
    dof: int
    fixed: np.ndarray


@dataclass
class SolveResult:
    """Fields of scipy's OptimizeResult that the reference reads (capture_volume.py:413-433) plus counters."""

    x: np.ndarray
    status: int
    nfev: int
    njev: int
    nit: int
    cost: float
    initial_cost: float
    optimality: float
    lambda_final: float
    pcg_iterations: int
    kernel_launches: int
    solve_ms: float
    rj_ms: float
    rj_launches: int
    syrk_ms: float = 0.0
    syrk_launches: int = 0
    trials_queued: int = 0
    used_graph: bool = False
    used_graph_mode: int = 0  # 0 direct launches, 1 one graph per trial, 2 device loop (WHILE graph)
    success: bool = True
    message: str = ""

    _MESSAGES = {
        -1: "Improper input parameters status returned from the engine.",
        0: "The maximum number of function evaluations is exceeded.",
        1: "`gtol` termination condition is satisfied.",
        2: "`ftol` termination condition is satisfied.",
        3: "`xtol` termination condition is satisfied.",
        4: "Both `ftol` and `xtol` termination conditions are satisfied.",
    }

    def __post_init__(self):
        self.success = self.status > 0
        self.message = self._MESSAGES.get(self.status, "")


class BAProblem:
    """One observation list + camera table on one GPU.

    ``obs_*`` may be NumPy arrays (copied host->device inside the constructor) or contiguous CUDA tensors on ``device``
    (used in place, no copy): obs_cam int32 or int16, obs_pt int32, obs_xy float64 of shape (n, 2).  Tensors of any
    other dtype, device, layout or length raise ValueError.
    """

    def __init__(self, cam_flags, cam_const, n_pts, obs_cam, obs_pt, obs_xy, *, constraints=None, device: int = 0,
                 stream: int = 0, cam_order=None, fixed_cam_params=None, fixed_points=None, camera_priors=None,
                 point_priors=None):
        """``constraints``: optional ``(groups_a (n_c,4), groups_b (n_c,4), distances (n_c,), weights (n_c,))`` --
        the rigid-distance rows of capture_volume.py:373-383 / reprojection.py:112-117.

        ``fixed_cam_params``: indices into x's camera section (the layout ``covariance``'s ``fixed`` uses) and
        ``fixed_points``: point indices, held at their values in x0 by every solve (DESIGN.md section 4.12): a solve is
        the solve over the free parameters alone, and the fixed entries of its x are x0's, bit for bit.  A calibrated rig
        held while a new camera is adjusted, surveyed points that set scale and frame, or partly known intrinsics.

        ``camera_priors``: ``(cams (k,), mean (k, 9), info (k, 9, 9))`` and ``point_priors``: ``(points (k,), mean (k, 3),
        info (k, 3, 3))``: Gaussian priors (DESIGN.md section 4.13), ``1/2 (x - mean)^T info (x - mean)`` added to the
        objective whatever the loss.  A camera's mean is its slice of x (6 or 9 values, padded to 9); a 6-parameter
        camera's info is zero outside its 6 x 6 block.  ``info`` is positive semi-definite, in the objective's units:
        ``uncertainty.prior_information`` makes it from a covariance.  Fixed parameters and priors may share a camera."""
        lib = L.load()
        self._lib = lib
        self._h = None
        self.cam_flags = np.ascontiguousarray(cam_flags, dtype=np.int32)
        self.cam_const = np.ascontiguousarray(cam_const, dtype=np.float64).reshape(-1, 9)
        self.n_cams = len(self.cam_flags)
        self.n_pts = int(n_pts)
        self.device = int(device)
        on_dev = hasattr(obs_cam, "data_ptr")
        cam_bits = 32
        if on_dev:
            cam_bits = _check_device_obs(obs_cam, obs_pt, obs_xy, self.device)
            keep = (obs_cam, obs_pt, obs_xy)
            n_obs = int(obs_cam.shape[0])
            ptrs = (obs_cam.data_ptr(), obs_pt.data_ptr(), obs_xy.data_ptr())
        else:
            if isinstance(obs_cam, np.ndarray) and obs_cam.dtype == np.int16:
                oc = np.ascontiguousarray(obs_cam)  # the reference's camera_indices dtype: widened on the device
                cam_bits = 16
            else:
                oc = np.ascontiguousarray(obs_cam, dtype=np.int32)
            op = np.ascontiguousarray(obs_pt, dtype=np.int32)
            ox = np.ascontiguousarray(obs_xy, dtype=np.float64).reshape(-1, 2)
            if not (len(oc) == len(op) == len(ox)):
                raise ValueError("obs_cam, obs_pt and obs_xy must have the same length")
            keep = (oc, op, ox)
            n_obs = len(oc)
            ptrs = (_ptr(oc), _ptr(op), _ptr(ox))
        self._keep = keep
        self.n_obs = n_obs
        widths = np.where(self.cam_flags & L.CB_CAM_FREE_INTRINSICS, 9, 6)
        self.cam_offsets = np.concatenate([[0], np.cumsum(widths)]).astype(np.int64)
        self.n_camera_params = int(self.cam_offsets[-1])
        self.n_params = self.n_camera_params + 3 * self.n_pts
        order = None if cam_order is None else np.ascontiguousarray(cam_order, dtype=np.int32)
        if order is not None and order.shape != (self.n_cams,):
            raise ValueError(f"cam_order must have shape ({self.n_cams},)")
        self.n_constraints = 0
        cons_ptrs = (None,) * 4
        if constraints is not None and constraints[0] is not None and len(constraints[0]) > 0:
            ga = np.ascontiguousarray(constraints[0], dtype=np.int32).reshape(-1, 4)
            gb = np.ascontiguousarray(constraints[1], dtype=np.int32).reshape(-1, 4)
            dist = np.ascontiguousarray(constraints[2], dtype=np.float64)
            w = np.ascontiguousarray(constraints[3], dtype=np.float64)
            if not (len(ga) == len(gb) == len(dist) == len(w)):
                raise ValueError("constraint arrays must have the same length")
            self.n_constraints = len(ga)
            self.constraints = (ga, gb, dist, w)
            cons_ptrs = tuple(_ptr(a) for a in self.constraints)
        desc = L.ProblemDesc(
            self.n_cams, self.n_pts, n_obs, _ptr(self.cam_flags), _ptr(self.cam_const), ptrs[0], ptrs[1], ptrs[2],
            1 if on_dev else 0, cam_bits, _ptr(order) if order is not None else None, self.n_constraints, *cons_ptrs,
        )  # fmt: skip
        self.fixed_cam_params = np.unique(np.asarray([] if fixed_cam_params is None else fixed_cam_params, np.int64))
        self.fixed_points = np.unique(np.asarray([] if fixed_points is None else fixed_points, np.int64))
        fc = np.ascontiguousarray(fixed_cam_params if fixed_cam_params is not None else [], dtype=np.int32).ravel()
        fp = np.ascontiguousarray(fixed_points if fixed_points is not None else [], dtype=np.int32).ravel()
        self.camera_priors = _prior_arrays(camera_priors, 9, "camera_priors")
        self.point_priors = _prior_arrays(point_priors, 3, "point_priors")
        h = C.c_void_p()
        pri = None
        if self.has_priors:
            (ci, cm, cl), (pi, pm, pl) = self.camera_priors, self.point_priors
            pri = C.byref(L.Priors(len(ci), _ptr(ci), _ptr(cm), _ptr(cl), len(pi), _ptr(pi), _ptr(pm), _ptr(pl)))
        rc = lib.cb_ba_problem_create_priors(C.byref(desc), len(fc), _ptr(fc) if len(fc) else None, len(fp),
                                             _ptr(fp) if len(fp) else None, pri, self.device, C.c_void_p(stream),
                                             C.byref(h))  # fmt: skip
        L.check(rc, "problem_create")
        self._h = h
        self.cam_stride = int(lib.cb_ba_cam_stride(h))

    @property
    def has_priors(self) -> bool:
        return len(self.camera_priors[0]) > 0 or len(self.point_priors[0]) > 0

    # -- lifetime -----------------------------------------------------------------------------
    def close(self) -> None:
        if self._h is not None:
            self._lib.cb_ba_problem_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def stat(self, what: int) -> float:
        """``cb_ba_problem_stat``: 0 sparse Schur lists in use, 1 flops per Schur-product launch, 2 direct reduced solve,
        3 Schur CTAs, 4-6 stage milliseconds of the last ``covariance`` call, 7 lanes per point (8 or 32), 8 repeated
        (camera, point) rows, 9 camera table in shared memory, 10 reduced solve (0 direct, 1 L2-streamed PCG, 2 register
        PCG), 11 PCG cluster CTAs, 12 register-PCG columns per lane (0 otherwise), 13 internal camera order differs from
        the caller's numbering, 14-17 host microseconds of the last ``solve`` in the bounds, the start state, the upload
        of x, and the LM loop with the download of x up to its synchronisation.  -1 for an unknown key."""
        return float(self._lib.cb_ba_problem_stat(self._h, int(what)))

    def _x(self, x) -> np.ndarray:
        x = np.ascontiguousarray(x, dtype=np.float64)
        if x.shape != (self.n_params,):
            raise ValueError(f"x must have shape ({self.n_params},), got {x.shape}")
        return x

    # -- evaluation ---------------------------------------------------------------------------
    def residuals(self, x, stream: int = 0) -> np.ndarray:
        """== joint_residuals: 2*n_obs reprojection rows, then the n_c constraint rows."""
        x = self._x(x)
        out = np.empty(2 * self.n_obs + self.n_constraints)
        L.check(self._lib.cb_ba_residuals(self._h, _ptr(x), _ptr(out), C.c_void_p(stream)), "residuals")
        if self.n_constraints:
            tail = out[2 * self.n_obs :]
            L.check(self._lib.cb_ba_constraint_rows(self._h, _ptr(x), _ptr(tail), None, C.c_void_p(stream)), "constraint_rows")
        return out

    def constraint_rows(self, x, stream: int = 0) -> tuple[np.ndarray, np.ndarray]:
        """(r (n_c,), dir (n_c,3)): constraint residuals and weight * unit direction (Jacobian entries are +-dir/4)."""
        x = self._x(x)
        r = np.empty(self.n_constraints)
        d = np.empty((self.n_constraints, 3))
        L.check(self._lib.cb_ba_constraint_rows(self._h, _ptr(x), _ptr(r), _ptr(d), C.c_void_p(stream)), "constraint_rows")
        return r, d

    def jacobian_blocks(self, x, stream: int = 0) -> tuple[np.ndarray, np.ndarray]:
        x = self._x(x)
        Jc = np.empty((self.n_obs, 2, 9))
        Jp = np.empty((self.n_obs, 2, 3))
        L.check(
            self._lib.cb_ba_jacobian_blocks(self._h, _ptr(x), _ptr(Jc), _ptr(Jp), C.c_void_p(stream)), "jacobian_blocks"
        )
        return Jc, Jp

    def reproj_errors_px(self, x, stream: int = 0) -> np.ndarray:
        x = self._x(x)
        out = np.empty((self.n_obs, 2))
        L.check(self._lib.cb_ba_reproj_errors_px(self._h, _ptr(x), _ptr(out), C.c_void_p(stream)), "reproj_errors_px")
        return out

    def rmse_px(self, x, stream: int = 0) -> tuple[float, np.ndarray]:
        """(overall RMSE, per-camera RMSE) in pixels, reduced on the device
        (ReprojectionReport.overall_rmse / by_camera, capture_volume.py:197-202)."""
        x = self._x(x)
        overall = C.c_double()
        per_cam = np.empty(self.n_cams)
        L.check(self._lib.cb_ba_rmse_px(self._h, _ptr(x), C.addressof(overall), _ptr(per_cam), C.c_void_p(stream)), "rmse_px")
        return overall.value, per_cam

    def overall_rmse_px(self, x) -> float:
        return self.rmse_px(x)[0]

    def cull(self, x, thresholds, min_per_camera: int = 10, want_mask: bool = True, stream: int = 0):
        """Device-side ``_filter_by_reprojection_thresholds`` (capture_volume.py:607-646): returns
        (filtered BAProblem on the same cameras / point numbering, keep mask in this problem's observation
        order or None).  The observation list never leaves the device."""
        x = self._x(x)
        thr = np.ascontiguousarray(thresholds, dtype=np.float64)
        if thr.shape != (self.n_cams,):
            raise ValueError(f"thresholds must have shape ({self.n_cams},)")
        if min_per_camera < 0:
            raise ValueError(f"min_per_camera must be >= 0 (0: thresholds only), got {min_per_camera}")
        mask = np.empty(self.n_obs, np.uint8) if want_mask else None
        h = C.c_void_p()
        n_kept = C.c_int64()
        L.check(
            self._lib.cb_ba_cull(self._h, _ptr(x), _ptr(thr), int(min_per_camera), C.byref(h), C.addressof(n_kept),
                                 _ptr(mask) if want_mask else None, C.c_void_p(stream)),
            "cull",
        )  # fmt: skip
        new = BAProblem.__new__(BAProblem)
        new._lib, new._h, new._keep = self._lib, h, ()
        new.cam_flags, new.cam_const = self.cam_flags, self.cam_const
        new.n_cams, new.n_pts, new.device, new.n_obs = self.n_cams, self.n_pts, self.device, int(n_kept.value)
        new.cam_offsets, new.n_camera_params, new.n_params = self.cam_offsets, self.n_camera_params, self.n_params
        new.cam_stride = self.cam_stride
        new.fixed_cam_params, new.fixed_points = self.fixed_cam_params, self.fixed_points  # the engine keeps both sets
        new.camera_priors, new.point_priors = self.camera_priors, self.point_priors  # and the priors
        new.n_constraints = self.n_constraints
        if self.n_constraints:
            new.constraints = self.constraints
        return new, (mask.astype(bool) if want_mask else None)

    def normal_equations(self, x, lam: float, loss: str = "linear", f_scale: float = 1.0, stream: int = 0) -> dict:
        """One damped linearisation, every stage returned (test / diagnostic)."""
        x = self._x(x)
        P, nc, npt = self.cam_stride, self.n_cams, self.n_pts
        nP = nc * P
        out = {
            "U": np.empty((nc, P, P)), "gc": np.empty((nc, P)), "V": np.empty((npt, 3, 3)), "gp": np.empty((npt, 3)),
            "S": np.empty((nP, nP)), "b": np.empty(nP), "dc": np.empty((nc, P)), "dp": np.empty((npt, 3)),
        }  # fmt: skip
        cost = C.c_double()
        L.check(
            self._lib.cb_ba_normal_equations(
                self._h, _ptr(x), float(lam), L.LOSS_IDS[loss], float(f_scale), C.addressof(cost),
                _ptr(out["U"]), _ptr(out["gc"]), _ptr(out["V"]), _ptr(out["gp"]), _ptr(out["S"]), _ptr(out["b"]),
                _ptr(out["dc"]), _ptr(out["dp"]), C.c_void_p(stream),
            ),
            "normal_equations",
        )  # fmt: skip
        out["cost"] = cost.value
        return out

    def covariance(self, x, *, loss: str = "linear", f_scale: float = 1.0, fixed=None, variance_factor=None,
                   points: bool = True, stream: int = 0) -> Covariance:
        """Covariance of the parameters at x (normally a solution of the same loss), ``cb_ba_covariance``.
        ``fixed``: indices into x's camera section held fixed to remove the gauge; None: ``uncertainty.default_gauge``,
        or nothing on a problem with fixed parameters (``fixed_cam_params`` / ``fixed_points``), which join ``fixed``,
        or with priors, whose information enters the inverse (the result is then the posterior covariance).
        ``variance_factor``: s2 (e.g. ``(pixel_sigma / fx) ** 2``); None: 2 cost / dof.  The problem must hold every
        observation (not one rank's shard)."""
        from . import uncertainty

        if loss not in L.LOSS_IDS:
            raise ValueError(f"`loss` must be one of {list(L.LOSS_IDS)}")
        x = self._x(x)
        if fixed is None and (len(self.fixed_cam_params) or len(self.fixed_points) or self.has_priors):
            fixed = []  # the problem's fixed parameters and priors set the gauge; if they do not, the pivot check refuses
        elif fixed is None:
            observed = self.error_order_stats(x, 50.0, stream, want_err=False)[3] > 0
            fixed = uncertainty.default_gauge(x, self.cam_offsets, observed, self.n_constraints > 0)
        fixed = np.ascontiguousarray(fixed, dtype=np.int32).ravel()
        cam = np.empty((self.n_camera_params, self.n_camera_params))
        pts = np.empty((self.n_pts, 3, 3)) if points else None
        rank = np.empty(self.n_pts, np.int32)
        s2 = C.c_double()
        dof = C.c_int64()
        L.check(
            self._lib.cb_ba_covariance(
                self._h, _ptr(x), L.LOSS_IDS[loss], float(f_scale), len(fixed), _ptr(fixed) if len(fixed) else None,
                float(variance_factor) if variance_factor is not None else 0.0, _ptr(cam), _ptr(pts) if points else None,
                C.addressof(s2), C.addressof(dof), _ptr(rank), C.c_void_p(stream),
            ),
            "covariance",
        )  # fmt: skip
        return Covariance(cameras=cam, points=pts, point_rank=rank, variance_factor=s2.value, dof=int(dof.value),
                          fixed=fixed)  # fmt: skip

    def error_order_stats(self, x, q_percent: float, stream: int = 0, want_err: bool = True):
        x = self._x(x)
        err = np.empty(self.n_obs) if want_err else None
        lo = np.empty(self.n_cams)
        hi = np.empty(self.n_cams)
        cnt = np.empty(self.n_cams, np.int64)
        L.check(
            self._lib.cb_ba_error_order_stats(
                self._h, _ptr(x), float(q_percent), _ptr(err) if want_err else None, _ptr(lo), _ptr(hi), _ptr(cnt),
                C.c_void_p(stream)
            ),
            "error_order_stats",
        )
        return err, lo, hi, cnt

    # -- solve --------------------------------------------------------------------------------
    def solve(
        self,
        x0,
        *,
        ftol: float = 1e-8,
        xtol: float = 1e-8,
        gtol: float = 1e-8,
        max_nfev: int | None = None,
        loss: str = "linear",
        f_scale: float = 1.0,
        verbose: int = 0,
        use_bounds: bool = True,
        lambda0: float = 1e-4,
        pcg_tol: float = 1e-6,
        allreduce=None,
        nccl_comm=None,
        peer_group=None,
        rank: int = 0,
        world_size: int = 1,
        stream: int = 0,
        time_kernels: bool = False,
    ) -> SolveResult:
        if loss not in L.LOSS_IDS:
            raise ValueError(f"`loss` must be one of {list(L.LOSS_IDS)}")
        x0 = self._x(x0)
        x = np.empty_like(x0)  # the engine reads x0 and writes the result here: x0 stays untouched, x is a fresh array
        opt = L.Options()
        self._lib.cb_ba_default_options(C.byref(opt))
        opt.ftol, opt.xtol, opt.gtol = float(ftol), float(xtol), float(gtol)
        opt.max_nfev = 0 if max_nfev is None else int(max_nfev)
        opt.loss = L.LOSS_IDS[loss]
        opt.f_scale = float(f_scale)
        opt.verbose = int(verbose)
        opt.use_bounds = 1 if use_bounds else 0
        opt.lambda0 = float(lambda0)
        opt.pcg_tol = float(pcg_tol)
        cb = None
        if allreduce is not None:
            cb = L.ALLREDUCE_FN(allreduce)
            opt.allreduce = cb
        if nccl_comm is not None:
            opt.nccl_comm = C.c_void_p(getattr(nccl_comm, "handle", nccl_comm))
        if peer_group is not None:
            opt.peer_group = C.c_void_p(getattr(peer_group, "handle", peer_group))
        opt.rank, opt.world_size = int(rank), int(world_size)
        opt.time_kernels = 1 if time_kernels else 0
        res = L.Result()
        try:
            L.check(self._lib.cb_ba_solve_from(self._h, C.byref(opt), _ptr(x0), _ptr(x), C.byref(res), C.c_void_p(stream)),
                    "solve")
        except Exception:
            # a sharded solve that fails part-way leaves the ranks' reduction sequence numbers out of step: the engine
            # refuses further solves on this peer group; make the Python cache re-create it (collectively) next time
            if peer_group is not None and hasattr(peer_group, "poisoned"):
                peer_group.poisoned = True
            raise
        del cb
        return SolveResult(
            x=x, status=res.status, nfev=res.nfev, njev=res.njev, nit=res.nit, cost=res.cost,
            initial_cost=res.initial_cost, optimality=res.optimality, lambda_final=res.lambda_final,
            pcg_iterations=res.pcg_iterations, kernel_launches=res.kernel_launches, solve_ms=res.solve_ms,
            rj_ms=res.rj_ms, rj_launches=res.rj_launches, syrk_ms=res.syrk_ms, syrk_launches=res.syrk_launches,
            trials_queued=res.trials_queued, used_graph=bool(res.used_graph), used_graph_mode=int(res.used_graph),
        )  # fmt: skip
