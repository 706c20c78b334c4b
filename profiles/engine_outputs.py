"""Every output of the bundle-adjustment engine on the shape-selected test rigs, for comparing two builds bit for bit.

    CALISCOPE_B200_LIB=<build A>/libcaliscope_b200.so python profiles/engine_outputs.py dump runs/a
    CALISCOPE_B200_LIB=<build B>/libcaliscope_b200.so python profiles/engine_outputs.py dump runs/b
    python profiles/engine_outputs.py compare runs/a runs/b

``dump`` writes one .npz per rig of ``tests/_engine_cases.CASES`` and one rig with rigid-distance constraints: the solve (x,
cost, nfev, kernel_launches), every array of ``normal_equations`` and, where ``COVARIANCE_CASES`` lists the rig, the
covariance.  ``compare`` exits non-zero unless every array of every file is equal (NaNs in the same places)."""
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from caliscope_b200._lib import EngineError  # noqa: E402

CONSTRAINED = "dome80-pcg-cl18-comp43-128"


def outputs(p, x0, covariance: bool) -> dict:
    res = p.solve(x0)
    out = {"x": res.x, "cost": res.cost, "nfev": res.nfev, "kernel_launches": res.kernel_launches}
    out.update({f"ne_{k}": v for k, v in p.normal_equations(x0, 1e-3).items()})
    if covariance:
        try:
            c = p.covariance(res.x)
        except EngineError as e:  # e.g. the default gauge leaves the rig's reduced system singular: the refusal is the output
            return {**out, "cov_error": str(e)}
        out.update(cov_cameras=c.cameras, cov_points=c.points, cov_rank=c.point_rank, cov_s2=c.variance_factor, cov_dof=c.dof)
    return out


def dump(out_dir: Path) -> None:
    import caliscope_b200 as cb
    from tests import _constraint_cases as CCS
    from tests import _engine_cases as EC

    out_dir.mkdir(parents=True, exist_ok=True)
    rigs = [(c.id, EC.oracle_rig(r), r.x0, None, c.id in EC.COVARIANCE_CASES) for c in EC.CASES.values() for r in [c.make()]]
    r, rig, _ = CCS.CASES[CONSTRAINED].make()
    rigs.append(("constrained-" + CONSTRAINED, rig, r.x0, CCS.constraints_of(rig), False))
    for name, rig, x0, cons, cov in rigs:
        with cb.BAProblem(rig.cam_flags, rig.cam_const, rig.n_pts, rig.obs_cam, rig.obs_pt, rig.obs_xy, constraints=cons) as p:
            out = outputs(p, x0, cov)
        np.savez(out_dir / f"{name}.npz", **out)
        print(f"{name}: nfev {out['nfev']} cost {out['cost']:.15e} launches {out['kernel_launches']}" + (", covariance" if cov else ""))


def compare(a: Path, b: Path) -> int:
    names = sorted(f.name for f in a.glob("*.npz"))
    bad = int(names != sorted(f.name for f in b.glob("*.npz")) or not names)
    for n in names:
        fa, fb = np.load(a / n), np.load(b / n)
        diff = [k for k in set(fa.files) | set(fb.files)
                if k not in fa.files or k not in fb.files or not np.array_equal(fa[k], fb[k], equal_nan=fa[k].dtype.kind == "f")]  # fmt: skip
        print(f"{n}: {len(fa.files)} arrays, " + (f"DIFFERENT: {sorted(diff)}" if diff else "identical"))
        bad += len(diff)
    return 1 if bad else 0


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "dump":
        dump(Path(sys.argv[2]))
    elif len(sys.argv) == 4 and sys.argv[1] == "compare":
        sys.exit(compare(Path(sys.argv[2]), Path(sys.argv[3])))
    else:
        sys.exit(__doc__)
