"""caliscope_b200 -- H100-native sparse bundle adjustment behind Caliscope's
``CaptureVolume.optimize()`` / ``calibrate_extrinsics()`` seam.

Hand-written sm_90a CUDA (``csrc/``) behind a C ABI (``include/caliscope_b200.h``);
this package is the host-side mirror of the reference's interface for that path.
"""
from ._lib import EngineError, EngineUnavailable  # noqa: F401
from .problem import BAProblem, Covariance, SolveResult, blocks_to_arrays  # noqa: F401
from .uncertainty import PoseUncertainty, camera_poses, default_gauge, pose_from_extrinsics  # noqa: F401

__all__ = ["BAProblem", "Covariance", "SolveResult", "EngineError", "EngineUnavailable", "blocks_to_arrays",
           "PoseUncertainty", "camera_poses", "default_gauge", "pose_from_extrinsics"]
