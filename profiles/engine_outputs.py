"""Every output of the bundle-adjustment engine on the shape-selected test rigs, for comparing two builds bit for bit.

    CALISCOPE_B200_LIB=<build A>/libcaliscope_b200.so python profiles/engine_outputs.py dump runs/a
    CALISCOPE_B200_LIB=<build B>/libcaliscope_b200.so python profiles/engine_outputs.py dump runs/b
    python profiles/engine_outputs.py compare runs/a runs/b

``dump`` writes one .npz per rig of ``tests/_engine_cases.CASES`` and one rig with rigid-distance constraints: the solve (x,
cost, nfev, kernel_launches), every array of ``normal_equations`` and, where ``COVARIANCE_CASES`` lists the rig, the
covariance.  Each rig of ``CASES`` is dumped twice more with held parameters, as ``tests/test_gpu_priors.py`` holds them:
its fixed sets alone (``-fixed``) and its priors beside fixed sets (``-priors+fixed``), from the start vector with the
true values at the fixed entries.  ``compare`` exits non-zero unless every array of every file is equal (NaNs in the same places)."""
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


def held_problems(rig, x0, xt):
    """(suffix, priors, BAProblem keywords, start vector) of the rig's two held problems."""
    from tests import _engine_cases as EC
    from tests.test_gpu_priors import _case_fixed_sets, _case_priors

    fc, fp = _case_fixed_sets(rig)
    pr, pfc, pfp = _case_priors(rig, x0)
    out = []
    for suffix, pri, c, p in (("-fixed", None, fc, fp), ("-priors+fixed", pr, pfc, pfp)):
        x = np.where(EC.free_mask(rig, c, p), x0, xt)
        out.append((suffix, pri, dict(fixed_cam_params=c, fixed_points=p), x))
    return out


def dump(out_dir: Path) -> None:
    from tests import _constraint_cases as CCS
    from tests import _engine_cases as EC

    out_dir.mkdir(parents=True, exist_ok=True)
    rigs = []
    for c in EC.CASES.values():
        r = c.make()
        rig, cov = EC.oracle_rig(r), c.id in EC.COVARIANCE_CASES
        rigs.append((c.id, rig, r.x0, None, {}, cov))
        rigs += [(c.id + s, rig, x, pr, kw, cov) for s, pr, kw, x in held_problems(rig, r.x0, r.x_true)]
    r, rig, _ = CCS.CASES[CONSTRAINED].make()
    rigs.append(("constrained-" + CONSTRAINED, rig, r.x0, None, {}, False))
    for name, rig, x0, pr, kw, cov in rigs:
        with EC.problem(rig, pr, **kw) as p:
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
