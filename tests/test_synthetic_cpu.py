"""The synthetic rig generator (caliscope_b200/synthetic.py): the dome layout reaches camera counts the ring layout cannot."""
from __future__ import annotations

import numpy as np
import pytest

from caliscope_b200 import synthetic


def _seen_fraction(r) -> np.ndarray:
    """Per camera: share of the points it has at least one observation of."""
    seen = np.zeros((r.n_cams, r.n_pts), bool)
    seen[r.obs_cam, r.obs_pt] = True
    return seen.mean(axis=1)


def test_dome_cameras_each_see_nearly_every_point():
    # more observations than in-frame pairs: every pair is kept (plus repeats), so the rows show the full visibility
    r = synthetic.make_rig(240, 300, 200_000, seed=1, layout="dome")
    frac = _seen_fraction(r)
    print(f"240-camera dome: every camera sees at least {frac.min():.3f} of the points")
    assert frac.min() >= 0.9
    ring = synthetic.make_rig(240, 300, 200_000, seed=1)
    assert (_seen_fraction(ring) < 0.1).any()  # the stacked rings: the top cameras see (almost) nothing


def test_layout_is_checked():
    with pytest.raises(ValueError, match="layout"):
        synthetic.make_rig(8, 10, 10, layout="sphere")
