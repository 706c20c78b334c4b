"""Synthetic rigs with rigid-distance constraint rows, and the engine variant each must reach (test infrastructure).

``tie`` turns a ``synthetic.make_rig`` rig into constraint arrays in the reference's format (``groups_a`` / ``groups_b``
(n_c, 4), ``distances``, ``weights``): each component is a chain of point-to-point rows (the point repeated four times,
as in the board and truss fixtures) plus, for components of eight or more points, centroid rows between two groups of
four distinct points.  Distances come from the true points, weights are the fixtures' (pixel sigma / f) / sigma.

Components are chosen "local" (points seen by the same few cameras, like the corners of one board) or "spread" (drawn
across the whole rig, so that one component reaches cameras in several 96-column Schur tiles).  With ``degenerate``, the
first component holds a point that no camera sees and the last one a point seen by a single camera."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from oracle import ba_oracle as O
from tests import _engine_cases as EC

WEIGHT = 0.35852574  # the fixtures' weight: (0.5 px / 1394.6 px) / 0.001 m


def pick_components(r, sizes, mode: str, rng) -> list[np.ndarray]:
    taken = np.zeros(r.n_pts, bool)
    comps = []
    for m in sizes:
        if mode == "spread":
            c = rng.choice(np.nonzero(~taken)[0], m, replace=False)
        elif mode == "local":  # points of one camera, then of the cameras after it, until m are found
            start = int(rng.integers(r.n_cams))
            got: list[int] = []
            for cam in np.roll(np.arange(r.n_cams), -start):
                seen = np.unique(r.obs_pt[r.obs_cam == cam])
                seen = seen[~taken[seen] & ~np.isin(seen, got)]
                got.extend(rng.permutation(seen)[: m - len(got)].tolist())
                if len(got) == m:
                    break
            c = np.array(got)
        else:
            raise ValueError(mode)
        assert len(c) == m, (mode, m)
        taken[c] = True
        comps.append(c)
    return comps


def tie(x_true, n_camera_params: int, comps, rng):
    """Constraint rows that make each point set of ``comps`` one component (order within a set: the chain order)."""
    pts = x_true[n_camera_params:].reshape(-1, 3)
    ga, gb = [], []
    for c in comps:
        for i in range(len(c) - 1):
            ga.append([c[i]] * 4)
            gb.append([c[i + 1]] * 4)
        for _ in range(len(c) // 8):
            q = rng.choice(c, 8, replace=False)
            ga.append(q[:4])
            gb.append(q[4:])
    ga = np.asarray(ga, np.int32)
    gb = np.asarray(gb, np.int32)
    dist = np.linalg.norm(pts[ga].mean(axis=1) - pts[gb].mean(axis=1), axis=1)
    return ga, gb, dist, np.full(len(ga), WEIGHT)


@dataclass
class ConstrainedCase:
    id: str
    base: EC.Case
    sizes: tuple
    mode: str
    stats: dict = field(default_factory=dict)  # stat key -> value the problem must report
    degenerate: bool = False
    min_cams: int = 0  # some component must be seen by more than this many cameras

    def make(self, degenerate: bool | None = None):
        """(synthetic rig, oracle rig with its constraint rows, components)."""
        r = self.base.make()
        rng = np.random.default_rng(len(self.id))
        comps = pick_components(r, self.sizes, self.mode, rng)
        keep = np.ones(r.n_obs, bool)
        if self.degenerate if degenerate is None else degenerate:
            keep &= r.obs_pt != comps[0][0]  # no camera sees it
            single = np.nonzero(r.obs_pt == comps[-1][-1])[0]
            keep[single[1:]] = False  # one camera sees it
        base = EC.oracle_rig(r, keep)
        ga, gb, dist, w = tie(r.x_true, base.n_camera_params, comps, rng)
        rig = O.Rig(base.cam_flags, base.cam_const, base.n_pts, base.obs_cam, base.obs_pt, base.obs_xy, ga, gb, dist, w)
        if self.min_cams:
            seen = max(len(np.unique(rig.obs_cam[np.isin(rig.obs_pt, c)])) for c in comps)
            assert seen > self.min_cams, f"{self.id}: the widest component is seen by {seen} cameras"
        return r, rig, comps


def constraints_of(rig: O.Rig):
    return (rig.groups_a, rig.groups_b, rig.distances, rig.weights)


_s = EC._s
SPARSE = EC.Case("ring40-local-1500", 40, 1500, 9000, seed=5, cams_per_point=6)
SPARSE_REFINE = EC.Case("ring40-refine-local-1500", 40, 1500, 9000, True, seed=5, cams_per_point=6)
CASES = {c.id: c for c in [
    # one 60-point component: n = 180 > CC_SMEM_DIM, E factored in global memory; one 96-column tile, direct solve
    ConstrainedCase("ring16-direct-comp60", EC.CASES["ring16-direct-nP96"], (60,), "local", EC.CASES["ring16-direct-nP96"].stats),
    # 3 column tiles, local visibility, 40 components of 8 points drawn across the rig: every component reaches several
    # tiles.  Run with the Schur row lists forced on and forced off.
    ConstrainedCase("ring40-sparse-spread", SPARSE, (8,) * 40, "spread", {EC.SOLVE: EC.PCG_REG, EC.PCG_CTAS: 5, EC.PCG_CL: 12},
                    degenerate=True),
    # P = 9: cameras whose 9 columns straddle a tile edge
    ConstrainedCase("ring40-refine-sparse-spread", SPARSE_REFINE, (8,) * 40, "spread",
                    {EC.SOLVE: EC.PCG_REG, EC.PCG_CTAS: 8, EC.PCG_CL: 12}, degenerate=True),
    # register PCG with cl = 18; components of 43 (n = 129, just past shared memory) and 128 points, each seen by more
    # than 64 cameras (a camera bitmap of three words)
    ConstrainedCase("dome80-pcg-cl18-comp43-128", EC.CASES["dome80-pcg-cl18-nP480"], (43, 128), "spread",
                    EC.CASES["dome80-pcg-cl18-nP480"].stats, min_cams=64),
    # the L2-streamed PCG at P = 9
    ConstrainedCase("dome70-refine-pcg-l2-comps", EC.CASES["dome70-refine-pcg-l2-nP630"], (20, 20, 20), "spread",
                    EC.CASES["dome70-refine-pcg-l2-nP630"].stats),
    # static object seen in every frame (repeated (camera, point) rows, 32 lanes per point), all 100 points one truss
    ConstrainedCase("static-ring12-dups-truss100", EC.CASES["static-ring12-lanes32-dups"], (100,), "local",
                    EC.CASES["static-ring12-lanes32-dups"].stats),
]}  # fmt: skip
# The largest component the engine takes: 400 points, n = 1200, the Cholesky of E in global memory by one CTA.  At P = 9
# the component kernel's shared memory is 227 072 B plus the camera bitmap, next to the 227 KB a CTA may opt in to.
LARGEST = {c.id: c for c in [
    ConstrainedCase("ring16-comp400", EC.Case("ring16-900", 16, 900, 9000), (400,), "spread", {EC.SOLVE: EC.DIRECT}),
    ConstrainedCase("ring10-refine-comp400", EC.Case("ring10-refine-900", 10, 900, 9000, True), (400,), "spread",
                    {EC.SOLVE: EC.DIRECT}),
]}  # fmt: skip
