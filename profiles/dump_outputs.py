"""--dump-outputs of the triangulation, resection and intrinsics timing scripts: every output array of one call to an
.npz, so the outputs of two builds can be compared bit for bit."""
import dataclasses
from pathlib import Path

import numpy as np


def dump_outputs(out_dir, tag: str, out) -> None:
    """every array field of the result dataclass `out` to out_dir/tag.npz (nothing when out_dir is None)"""
    if out_dir:
        Path(out_dir).mkdir(parents=True, exist_ok=True)
        arrays = {f.name: getattr(out, f.name) for f in dataclasses.fields(out) if getattr(out, f.name) is not None}
        np.savez(Path(out_dir) / f"{tag}.npz", **arrays)
