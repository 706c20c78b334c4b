"""Rigs that reach each shape-selected engine variant, with the variant the engine must report for them (test
infrastructure).  The engine picks kernel instantiations and the reduced solve from the problem's shape alone, so a
path is tested only if some rig has its shape; ``BAProblem.stat`` keys 7-13 say which path a problem took (DESIGN.md §4,
"Where the variants are chosen"), and ``check_stats`` pins them so that a moved threshold cannot silently send a case
back to an already covered path."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from oracle import ba_oracle as O

# BAProblem.stat keys
LANES, DUPS, CAM_SMEM, SOLVE, PCG_CTAS, PCG_CL, REORDERED = 7, 8, 9, 10, 11, 12, 13
DIRECT, PCG_L2, PCG_REG = 0, 1, 2


@dataclass
class Case:
    id: str
    n_cams: int
    n_pts: int
    n_obs: int
    refine: bool = False
    layout: str = "ring"
    seed: int | None = None  # None: n_cams
    stats: dict = field(default_factory=dict)  # stat key -> value the problem must report
    cams_per_point: int | None = None  # local visibility (synthetic.make_rig)

    def make(self):
        from caliscope_b200 import synthetic

        seed = self.n_cams if self.seed is None else self.seed
        return synthetic.make_rig(self.n_cams, self.n_pts, self.n_obs, seed=seed, refine_intrinsics=self.refine,
                                  layout=self.layout, cams_per_point=self.cams_per_point)  # fmt: skip


def _s(lanes, dups, smem, solve, ctas, cl, reordered=0):
    return {LANES: lanes, DUPS: dups, CAM_SMEM: smem, SOLVE: solve, PCG_CTAS: ctas, PCG_CL: cl, REORDERED: reordered}


# 30, 102, 198, 360, 384 reduced parameters; 600 takes the PCG with the slab streamed from L2, over 7 column tiles
TILE_SHAPES = [Case("5-False", 5, 700, 9000), Case("17-False", 17, 700, 9000), Case("33-False", 33, 700, 9000),
               Case("40-True", 40, 700, 9000, True), Case("64-False", 64, 700, 9000), Case("100-False", 100, 700, 9000)]  # fmt: skip
# Each new case names the variant it exists for.  Register PCG: cluster CTAs = ceil(nP / 48), columns per lane cl = 2 / 6
# / 12 / 18 up to nP = 64 / 192 / 384 / 576; a direct problem still reports the register configuration it would use.
VARIANTS = [
    Case("ring16-direct-nP96", 16, 700, 9000, stats=_s(8, 0, 1, DIRECT, 2, 6)),
    # 10 and 11 cameras see fewer than 9000 (camera, point) pairs of 700 points: some rows repeat
    Case("ring10-refine-direct-nP90", 10, 700, 9000, True, stats=_s(8, 1, 1, DIRECT, 2, 6)),
    Case("ring11-refine-pcg-cl6-nP99", 11, 700, 9000, True, stats=_s(8, 1, 1, PCG_REG, 3, 6)),
    Case("ring64-refine-pcg-cl18-nP576", 64, 700, 9000, True, stats=_s(8, 0, 1, PCG_REG, 12, 18)),
    Case("dome80-pcg-cl18-nP480", 80, 700, 9000, layout="dome", stats=_s(8, 0, 1, PCG_REG, 10, 18)),
    Case("dome70-refine-pcg-l2-nP630", 70, 700, 9000, True, "dome", stats=_s(8, 0, 1, PCG_L2, 8, 0)),
    # static object: 100 points in every frame, 120 rows per point, repeated (camera, point) rows
    Case("static-ring12-lanes32-dups", 12, 100, 12000, stats=_s(32, 1, 1, DIRECT, 2, 6)),
    Case("static-ring12-refine-lanes32-dups", 12, 100, 12000, True, stats=_s(32, 1, 1, PCG_REG, 3, 6)),
    Case("dome128-lanes32", 128, 300, 33000, layout="dome", stats=_s(32, 0, 1, PCG_L2, 8, 0)),
    # camera table of 180 x 37 doubles = 52 KB: shared memory above the 48 KB default, by opt-in
    Case("dome180-smem-optin", 180, 700, 12000, layout="dome", stats=_s(8, 0, 1, PCG_L2, 8, 0)),
    # 240 x 37 doubles = 69 KB: the camera table stays in global memory
    Case("dome240-global-table-lanes32", 240, 300, 60000, layout="dome", stats=_s(32, 0, 0, PCG_L2, 8, 0)),
]
CASES = {c.id: c for c in TILE_SHAPES + VARIANTS}
COVARIANCE_CASES = [c.id for c in TILE_SHAPES] + [c.id for c in VARIANTS if c.stats[LANES] == 32 or c.n_cams == 240]


def oracle_rig(r, keep=None) -> O.Rig:
    if keep is None:
        keep = np.ones(r.n_obs, bool)
    return O.Rig(r.cam_flags, r.cam_const, r.n_pts, r.obs_cam[keep], r.obs_pt[keep], r.obs_xy[keep])


def problem(rig: O.Rig, pr=None, **kw):
    """The engine's BAProblem of an oracle rig, with its constraints, the priors ``pr`` (``_held_oracle.Priors``) and
    BAProblem's keywords ``kw``."""
    import caliscope_b200 as cb

    cons = (rig.groups_a, rig.groups_b, rig.distances, rig.weights) if rig.n_constraints else None
    kw.update(pr.kwargs() if pr is not None else {})
    return cb.BAProblem(rig.cam_flags, rig.cam_const, rig.n_pts, rig.obs_cam, rig.obs_pt, rig.obs_xy, constraints=cons,
                        **kw)  # fmt: skip


def free_mask(rig: O.Rig, cam_params=(), points=()) -> np.ndarray:
    """Boolean over x: False at the camera-parameter indices and the coordinates of the points given."""
    free = np.ones(rig.n_params, bool)
    free[np.asarray(cam_params, np.int64)] = False
    for j in points:
        free[rig.n_camera_params + 3 * j : rig.n_camera_params + 3 * j + 3] = False
    return free


def relabelled_sparse_case():
    """48 cameras with local visibility, two in three with free intrinsics: compacted Schur lists, a camera order the
    engine chooses itself (test_gpu_engine_paths.py's rig) and 6-parameter cameras inside a P = 9 problem.  Returns the
    rig, its start vector and its true x."""
    from caliscope_b200 import synthetic

    r = synthetic.make_rig(48, 4000, 24000, seed=7, cams_per_point=6, refine_intrinsics=True)
    wide = np.arange(r.n_cams) % 3 != 0
    const = r.cam_const.copy()
    const[~wide, :2] = synthetic.WEBCAM_F

    def layout(x):
        blocks = x[: 9 * r.n_cams].reshape(r.n_cams, 9)
        return np.concatenate([blocks[c] if wide[c] else blocks[c, :6] for c in range(r.n_cams)] + [x[9 * r.n_cams :]])

    rig = O.Rig(wide.astype(np.int32), const, r.n_pts, r.obs_cam, r.obs_pt, r.obs_xy)
    return rig, layout(r.x0), layout(r.x_true)


def stats(p) -> dict:
    return {k: int(p.stat(k)) for k in (LANES, DUPS, CAM_SMEM, SOLVE, PCG_CTAS, PCG_CL, REORDERED)}


def check_stats(p, case: Case) -> dict:
    got = stats(p)
    print(f"{case.id}: P {p.cam_stride} nP {p.n_cams * p.cam_stride} stat keys {got}")
    want = case.stats
    assert {k: got[k] for k in want} == want, f"{case.id}: expected stat keys {want}, got {got}"
    return got


def check_step(S, b, dc, solve_mode, tag=""):
    """The camera step against the engine's own reduced system S dc = -b.  Direct (LDL^T): normwise backward error
    ||S dc + b|| / (||S|| ||dc|| + ||b||) <= 1e-12.  PCG: the engine's stopping rule, the block-Jacobi preconditioned
    residual sqrt(r^T M^-1 r / b^T M^-1 b) <= 1e-6 (M: the P x P diagonal blocks of S), with 10 % slack because the
    kernel tests its recursively updated residual, which drifts from the true one by rounding."""
    x = dc.ravel()
    n = len(b)
    P = n // dc.shape[0]
    if solve_mode == DIRECT:
        be = np.linalg.norm(S @ x + b) / (np.linalg.norm(S, 2) * np.linalg.norm(x) + np.linalg.norm(b))
        print(f"{tag} direct step backward error {be:.2e} (bound 1e-12, margin {1e-12 / max(be, 1e-300):.1f}x)")
        assert be <= 1e-12
    else:
        r = -b - S @ x
        Minv = np.zeros((n // P, P, P))
        for c in range(n // P):
            Minv[c] = np.linalg.inv(S[c * P : (c + 1) * P, c * P : (c + 1) * P])

        def mnorm2(v):
            v = v.reshape(-1, P)
            return float(np.einsum("cp,cpq,cq->", v, Minv, v))

        rel = np.sqrt(mnorm2(r) / mnorm2(b))
        bound = 1.1e-6
        print(f"{tag} PCG preconditioned relative residual {rel:.3e} (bound {bound:.1e}, margin {bound / max(rel, 1e-300):.2f}x)")
        assert rel <= bound
