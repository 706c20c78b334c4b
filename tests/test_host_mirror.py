"""Host-side logic (no GPU): the parameterization mirror against the unmodified reference class
(only with a reference checkout, see tests/_util.py), flattening of blocks for the C ABI,
the least_squares seam's call recognition, and the C-ABI library's exported symbols."""
from __future__ import annotations

import ctypes
import re
import sys
from pathlib import Path

import numpy as np
import pytest

from tests._util import REFERENCE_SKIP, reference_checkout

ROOT = Path(__file__).resolve().parent.parent
REF_ROOT = reference_checkout()
REF = REF_ROOT / "src" if REF_ROOT else None

needs_reference = pytest.mark.skipif(REF is None, reason=REFERENCE_SKIP)


@pytest.fixture(scope="module")
def ref_modules():
    for p in (str(ROOT / "tests" / "golden" / "_refshim"), str(REF)):
        if p not in sys.path:
            sys.path.insert(0, p)
    from caliscope.core.bundle_parameterization import BundleParameterization as RefBP
    from caliscope.core.capture_volume import CaptureVolume
    from caliscope.synthetic.scene_factories import default_ring_scene

    ring = default_ring_scene()
    cv = CaptureVolume(ring.camera_array, ring.image_points_noisy, ring.world_points)
    return RefBP, cv


@needs_reference
@pytest.mark.parametrize("refine", [False, True])
def test_parameterization_mirror_equals_reference(ref_modules, refine):
    from caliscope_b200.bundle_parameterization import BundleParameterization as MyBP

    RefBP, cv = ref_modules
    n = len(cv.world_points.points)
    a = RefBP.from_camera_array(cv.camera_array, n_points=n, refine_intrinsics=refine)
    b = MyBP.from_camera_array(cv.camera_array, n_points=n, refine_intrinsics=refine)
    assert a.camera_param_offsets == b.camera_param_offsets
    assert a.n_camera_params == b.n_camera_params
    assert [x.n_params for x in a.blocks] == [x.n_params for x in b.blocks]
    xa = a.pack(cv.camera_array, cv.world_points.points)
    assert np.array_equal(xa, b.pack(cv.camera_array, cv.world_points.points))
    for p, q in zip(a.bounds(), b.bounds()):
        assert np.array_equal(p, q)
    for i in range(len(a.blocks)):
        for p, q in zip(a.trial_projection_inputs(xa, i), b.trial_projection_inputs(xa, i)):
            assert np.array_equal(p, q)
    cam = np.repeat(np.arange(4), 5).astype(np.int16)
    obj = np.arange(20).astype(np.int32)
    ga = np.array([[0, 0, 0, 0], [0, 1, 2, 3]], dtype=np.int32)
    gb = np.array([[5, 5, 5, 5], [8, 9, 10, 11]], dtype=np.int32)
    assert (a.sparsity(cam, obj, 0, None, None).toarray() == b.sparsity(cam, obj, 0, None, None).toarray()).all()
    assert (a.sparsity(cam, obj, 2, ga, gb).toarray() == b.sparsity(cam, obj, 2, ga, gb).toarray()).all()
    x2 = xa.copy()
    if refine:
        x2[6], x2[16], x2[17 + 9] = 0.502, 0.995, 1.995
    wa = [(w.cam_id, w.parameter, w.bound, w.value) for w in a.bound_warnings(x2)]
    wb = [(w.cam_id, w.parameter, w.bound, w.value) for w in b.bound_warnings(x2)]
    assert wa == wb and (len(wa) == 3 if refine else wa == [])
    from copy import deepcopy

    ca, cb_ = deepcopy(cv.camera_array), deepcopy(cv.camera_array)
    pa, pb = a.unpack_into(ca, x2), b.unpack_into(cb_, x2)
    assert np.array_equal(pa, pb)
    for cid in ca.cameras:
        assert np.array_equal(ca.cameras[cid].matrix, cb_.cameras[cid].matrix)
        assert np.array_equal(ca.cameras[cid].distortions, cb_.cameras[cid].distortions)
        assert np.array_equal(ca.cameras[cid].rotation, cb_.cameras[cid].rotation)


@needs_reference
def test_blocks_flatten_like_golden_generator(ref_modules):
    from caliscope_b200 import blocks_to_arrays
    from tests._util import load_golden

    RefBP, cv = ref_modules
    par = RefBP.from_camera_array(cv.camera_array, n_points=3, refine_intrinsics=True)
    flags, const = blocks_to_arrays(par.blocks)
    g, rig = load_golden("ring_noisy_refine1.npz")
    assert np.array_equal(flags, g["cam_flags"]) and np.array_equal(const, g["cam_const"])


def test_fisheye_requires_four_coefficients():
    from caliscope_b200.bundle_parameterization import BundleParameterization, CalibrationError

    class Cam:
        matrix = np.eye(3)
        distortions = np.zeros(5)
        fisheye = True

    class Arr:
        posed_index_to_cam_id = {0: 7}
        cameras = {7: Cam()}

    with pytest.raises(Exception) as e:
        BundleParameterization.from_camera_array(Arr(), n_points=1, refine_intrinsics=True)
    assert "4 distortion coefficients" in str(e.value)
    Cam.matrix = None
    with pytest.raises(Exception) as e:
        BundleParameterization.from_camera_array(Arr(), n_points=1, refine_intrinsics=False)
    assert "no intrinsics" in str(e.value)
    assert issubclass(CalibrationError, Exception)


def test_least_squares_seam_recognises_only_the_ba_call():
    from caliscope_b200 import solver
    from caliscope_b200.bundle_parameterization import BundleParameterization

    def joint_residuals(x, *a):
        return x

    par = BundleParameterization(blocks=(), n_points=0)
    assert solver.is_bundle_adjustment_call(joint_residuals, (par, 1, 2, 3))
    assert not solver.is_bundle_adjustment_call(lambda x: x, (par, 1, 2, 3))
    assert not solver.is_bundle_adjustment_call(joint_residuals, (1, 2))
    with pytest.raises(NotImplementedError):
        solver.least_squares(lambda x: x, np.zeros(2))


def test_shared_library_exports_every_declared_symbol():
    """No compute calls here (no GPU): load the C-ABI library and resolve each name in the header."""
    from caliscope_b200 import _lib

    header = (ROOT / "include" / "caliscope_b200.h").read_text()
    declared = set(re.findall(r"\b(cb_[a-z_0-9]+)\s*\(", header))
    assert declared, "header parse failed"
    assert declared == set(_lib.SYMBOLS), f"binding table out of sync: {declared ^ set(_lib.SYMBOLS)}"
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.cb_ba_abi_version() == 3
    opt = _lib.Options()
    lib.cb_ba_default_options(ctypes.byref(opt))
    assert opt.ftol == 1e-8 and opt.xtol == 1e-8 and opt.gtol == 1e-8 and opt.use_bounds == 1
    assert lib.cb_ba_error_string(-3) == b"no CUDA device"


def test_product_package_never_imports_the_oracle():
    for f in (ROOT / "caliscope_b200").rglob("*.py"):
        src = f.read_text()
        assert "import oracle" not in src and "from oracle" not in src, f


@pytest.mark.skipif(__import__("torch").cuda.is_available(), reason="CPU-only behaviour")
def test_engine_fails_loudly_without_a_gpu():
    import caliscope_b200 as cb
    from tests._util import load_golden

    g, rig = load_golden("small_pinhole_refine0.npz")
    with pytest.raises(cb.EngineUnavailable):
        cb.BAProblem(rig.cam_flags, rig.cam_const, rig.n_pts, rig.obs_cam, rig.obs_pt, rig.obs_xy)


def test_filter_keep_mask_and_percentile_rule_on_reference_errors():
    """Host half of the percentile filter against the reference's own filter output (golden)."""
    from caliscope_b200 import filtering
    from tests._util import load_golden

    g, rig = load_golden("session4_refine0.npz")
    keep = filtering.keep_mask(g["filt_err"], g["filt_cam"], g["filt_thresholds"], int(g["filt_min_per_camera"]))
    assert np.array_equal(keep, g["filt_keep"])
    q = 100.0 - float(g["filt_percentile"])
    for c in range(rig.n_cams):
        e = np.sort(g["filt_err"][g["filt_cam"] == c])
        v = (len(e) - 1) * (q / 100.0)
        lo, hi = e[int(np.floor(v))], e[min(int(np.floor(v)) + 1, len(e) - 1)]
        t = filtering._numpy_linear_interp(np.array([lo]), np.array([hi]), np.array([v - np.floor(v)]))[0]
        assert t == np.percentile(e, q) == g["filt_thresholds"][c]
    rng = np.random.default_rng(0)
    for n in (1, 2, 7, 100, 1001):
        e = np.sort(rng.uniform(0, 5, n))
        for q in (0.0, 2.5, 50.0, 97.5, 100.0, 33.3):
            v = (n - 1) * (q / 100.0)
            lo, hi = e[int(np.floor(v))], e[min(int(np.floor(v)) + 1, n - 1)]
            t = filtering._numpy_linear_interp(np.array([lo]), np.array([hi]), np.array([v - np.floor(v)]))[0]
            assert t == np.percentile(e, q)


def test_every_device_entry_point_refuses_to_run_without_a_gpu():
    """The triangulation / undistortion mirrors and the peer-memory transport go through the same C ABI: on a
    box without a device they raise EngineUnavailable (CB_E_NO_DEVICE), they do not compute on the CPU."""
    import caliscope_b200 as cb
    from caliscope_b200 import _lib
    from caliscope_b200 import triangulation as T

    try:
        import torch

        if torch.cuda.is_available():
            pytest.skip("CUDA device present")
    except ImportError:
        pass
    proj = np.tile(np.hstack([np.eye(3), np.zeros((3, 1))]), (2, 1, 1))
    with pytest.raises(cb.EngineUnavailable):
        T.triangulate_groups(proj, np.array([0, 1], np.int32), np.array([0, 0], np.int64), np.zeros((2, 2)))
    with pytest.raises(cb.EngineUnavailable):
        T.undistort_points(np.zeros((3, 2)), None, np.eye(3)[None], [np.zeros(5)], [False])
    lib = _lib.load()
    h = ctypes.c_void_p()
    buf = (ctypes.c_char * 64)()
    assert lib.cb_peer_create(0, 2, 0, 1024, ctypes.byref(h), buf) == -3  # CB_E_NO_DEVICE
    assert lib.cb_peer_create(5, 2, 0, 1024, ctypes.byref(h), buf) == -1  # CB_E_INVALID: rank >= world_size


def test_least_squares_rejects_bounds_it_does_not_implement():
    """The engine implements exactly BundleParameterization.bounds(); anything else must fail loudly instead of being
    silently replaced (ADVICE round 1)."""
    from caliscope_b200 import solver
    from caliscope_b200.bundle_parameterization import BundleParameterization, CameraBlock

    blocks = tuple(CameraBlock(cam_id=c, free_intrinsics=(c != 1), fx_initial=1000.0, fy_initial=1000.0, cx=640.0, cy=360.0,
                               fisheye=False, dist_fixed=(0.0, 0.0, 0.0)) for c in range(3))  # fmt: skip
    par = BundleParameterization(blocks=blocks, n_points=5)
    lo, hi = par.bounds()
    n = len(lo)
    solver._check_supported(par, lo, hi, True, "jac", None, n)  # the reference's own bounds pass
    solver._check_supported(par, -np.inf, np.inf, False, "jac", "lsmr", n)
    bad_hi = hi.copy()
    bad_hi[6] = 3.0
    with pytest.raises(NotImplementedError, match="bounds"):
        solver._check_supported(par, lo, bad_hi, True, "jac", None, n)
    bad_lo = lo.copy()
    bad_lo[-1] = 0.0  # a bound on a world point
    with pytest.raises(NotImplementedError, match="bounds"):
        solver._check_supported(par, bad_lo, hi, True, "jac", None, n)
    with pytest.raises(NotImplementedError, match="x_scale"):
        solver._check_supported(par, lo, hi, True, 1.0, None, n)
    with pytest.raises(NotImplementedError, match="tr_solver"):
        solver._check_supported(par, lo, hi, True, "jac", "exact", n)
