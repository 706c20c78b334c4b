"""Stage times and accuracy of cb_rigid_pose_robust (DESIGN.md 4.14), one JSON line per workload.

    python profiles/rigid_pose_timing.py [track] [board64] [sparse] [--steps 5] [--warmup 2] [--gp3p-samples G]

track: section 4.9's scene (resect_robust_timing.make("track")) keyed by frame: a 0.2 m cluster of 12 markers seen by 8
pinhole cameras 3 m away over 50 000 frames, 50 000 groups of 96 rows, 5 % of the rows moved by up to +-200 px, no
prior.  The same input keyed by (camera, frame) goes through resect_robust, and each camera's pose of the cluster is
turned into a body pose (X_w = R_c^T (X_cam - t_c)) for the per-camera error beside the rig's.  board64: 64 pinhole
cameras on a ring of 3 m around a 10 x 7 ChArUco-like board (0.04 m squares, 70 corners) at 2 000 random poses, a
corner seen by the cameras on its front side (about 2 200 rows per frame), 5 % outliers, with the camera covariance
term (a block-diagonal 1 mrad / 1 mm camera covariance, the cameras perturbed by one draw of it).  Stage times are the
CUDA events recorded inside the call (CbRigidStats), the median over --steps timed calls after --warmup.  Pose errors
are over the groups with status 0: the angle of R_true^T R and the distance of the body origins; chi2 is the mean of
e^T Sigma^-1 e over those groups (6 when the covariance is calibrated).  The card's name and power limit are printed with
the numbers.

sparse: 6 pinhole cameras on a ring of 3 m around a 0.2 m cluster of 8 markers, each (marker,
camera) row kept with probability 0.25 (about a fifth of the frames have fewer than three markers seen by two cameras),
0.5 px noise, 3 % of the rows moved by up to 200 px, no prior, 20 000 frames.  --gp3p-samples G (default 0: off) is passed to every
workload; with G > 0 the line also holds the same call with gP3P off: the share of groups with status 0 both ways, and
the pose errors and chi2 of the groups only gP3P poses.
"""
import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE))
from caliscope_b200.resection import resect_robust  # noqa: E402
from caliscope_b200.rigid import RigidStats, pose_rigid_robust  # noqa: E402
from resect_robust_timing import _outliers, card, make, rodrigues  # noqa: E402
from scipy.spatial.transform import Rotation  # noqa: E402

TAU = 4.0


def _rotvec(R):
    """rotation vectors of (n, 3, 3) matrices, NaN where R is not finite"""
    R = np.asarray(R, np.float64)
    ok = np.isfinite(R).all(axis=(-2, -1))
    out = np.full(R.shape[:-1], np.nan)
    out[ok] = Rotation.from_matrix(R[ok]).as_rotvec()
    return out


def _ring(centers, target=(0.0, 0.0, 1.0)):
    """(R, t) of cameras at `centers` looking at `target` (z forward, y down)"""
    Rc = []
    for c in centers:
        z = np.asarray(target) - c
        z /= np.linalg.norm(z)
        x = np.cross([0.0, 0.0, -1.0], z)
        x /= np.linalg.norm(x)
        Rc.append(np.stack([x, np.cross(z, x), z]))
    Rc = np.array(Rc)
    return Rc, -np.einsum("cij,cj->ci", Rc, centers)


def _errors(pose, truth, m):
    if not m.any():
        return {}
    dR = np.einsum("nji,njk->nik", rodrigues(pose[m, :3]), rodrigues(truth[m, :3]))
    ang = np.degrees(np.arccos(np.clip((np.trace(dR, axis1=1, axis2=2) - 1) / 2, -1, 1)))
    d = np.linalg.norm(pose[m, 3:] - truth[m, 3:], axis=1) * 1e3
    return {"pos_median_mm": float(np.median(d)), "pos_p99_mm": float(np.percentile(d, 99)),
            "angle_median_deg": float(np.median(ang)), "angle_p99_deg": float(np.percentile(ang, 99))}  # fmt: skip


def _chi2_each(pose, cov, truth, m):
    e = pose[m] - truth[m]
    return np.einsum("gi,gi->g", e, np.linalg.solve(cov[m], e[:, :, None])[:, :, 0])


def _chi2(pose, cov, truth, m):
    return float(np.mean(_chi2_each(pose, cov, truth, m)))


def _distinct_markers(r, obs_key, obs_pt, groups):
    """the distinct model points of each group's consensus rows"""
    g_of_row = np.searchsorted(r.key, obs_key)
    return [int(len(np.unique(obs_pt[(g_of_row == g) & r.inlier]))) for g in groups]


def track():
    """(rigid inputs, body truth per frame, moved rows, kwargs, per-camera body errors from resect_robust)"""
    (flags, const, cam_x, mk, obs_cam, key, obs_pt, px), truth_g, moved, _ = make("track")
    n_cams = len(flags)
    n_frames = len(truth_g) // n_cams
    # the scene's cameras (make's look-at ring), with rotation vectors that hold near theta = pi too
    ang = 2 * np.pi * np.arange(n_cams) / n_cams
    Rc, tc = _ring(np.stack([3 * np.cos(ang), 3 * np.sin(ang), np.full(n_cams, 1.0)], axis=1))
    cam_x = np.concatenate([_rotvec(Rc), tc], axis=1).ravel()
    # body pose from camera 0's camera-from-cluster truth: R_b = R_c^T R_g, t_b = R_c^T (t_g - t_c)
    Rb = np.einsum("ji,fjk->fik", Rc[0], rodrigues(truth_g[:n_frames, :3]))
    tb = np.einsum("ji,fj->fi", Rc[0], truth_g[:n_frames, 3:] - tc[0])
    truth = np.concatenate([_rotvec(Rb), tb], axis=1)
    frame = key % n_frames
    t0 = time.perf_counter()
    r = resect_robust(flags, const, cam_x, mk, obs_cam, key, obs_pt, px, threshold_px=TAU, use_prior=False)
    res_s = time.perf_counter() - t0
    g = np.arange(len(r.pose))
    c, f = g // n_frames, g % n_frames
    Rw = np.einsum("gji,gjk->gik", Rc[c], rodrigues(r.pose[:, :3]))
    tw = np.einsum("gji,gj->gi", Rc[c], r.pose[:, 3:] - tc[c])
    per_cam = _errors(np.concatenate([_rotvec(Rw), tw], axis=1), truth[f], r.status == 0)
    per_cam["wall_s"] = res_s
    return (flags, const, cam_x, mk, obs_cam, frame.astype(np.int64), obs_pt, px), truth, moved, {}, per_cam


def board64(n_frames=2000):
    rng = np.random.default_rng(11)
    n_cams = 64
    ang = 2 * np.pi * np.arange(n_cams) / n_cams
    centers = np.stack([3 * np.cos(ang), 3 * np.sin(ang), 1.0 + 0.3 * np.sin(3 * ang)], axis=1)
    Rc, tc = _ring(centers)
    gx, gy = np.meshgrid(np.arange(10) * 0.04, np.arange(7) * 0.04)
    model = np.stack([gx.ravel() - 0.18, gy.ravel() - 0.12, np.zeros(70)], axis=1)
    rv = rng.normal(size=(n_frames, 3))
    rv *= (rng.uniform(0, 0.8 * np.pi, n_frames) / np.linalg.norm(rv, axis=1))[:, None]
    truth = np.concatenate([rv, rng.uniform(-0.3, 0.3, (n_frames, 3)) + [0.0, 0.0, 1.0]], axis=1)
    Rb = rodrigues(rv)
    Xw = np.einsum("fij,mj->fmi", Rb, model) + truth[:, None, 3:]  # (f, m, 3)
    normal = Rb[:, :, 2]  # board z in the world
    Xc = np.einsum("cij,fmj->cfmi", Rc, Xw) + tc[:, None, None]
    facing = np.einsum("fi,cfi->cf", normal, centers[:, None] - truth[None, :, 3:]) > 0
    vis = facing[:, :, None] & (Xc[..., 2] > 0.1)
    uv = Xc[..., :2] / Xc[..., 2:] * 1000.0 + [640.0, 360.0]
    c, f, m = np.nonzero(vis)
    order = np.lexsort((c, m, f))
    c, f, m = c[order], f[order], m[order]
    px = uv[c, f, m] + rng.normal(0, 0.5, (len(c), 2))
    px, moved = _outliers(rng, px)
    flags = np.zeros(n_cams, np.int32)
    const = np.zeros((n_cams, 9))
    const[:, :4] = [1000.0, 1000.0, 640.0, 360.0]
    cam_x = np.concatenate([_rotvec(Rc), tc], axis=1).ravel()
    cc = np.diag(np.tile([1e-3**2] * 3 + [1e-3**2] * 3, n_cams))
    x_cal = cam_x + np.sqrt(np.diag(cc)) * rng.normal(size=len(cam_x))
    args = (flags, const, x_cal, model, c.astype(np.int32), f.astype(np.int64), m.astype(np.int32), px)
    return args, truth, moved, {"camera_cov": cc}, None


def sparse(n_frames=20000):
    """make_bodies' ring scene thinned to visibility 0.25 (tests/_rigid_cases.py), with outliers"""
    from tests._rigid_cases import make_bodies, plant_outliers

    b = make_bodies(51, n_cams=6, n_frames=n_frames, n_model=8, noise=0.5, visible=0.25)
    b.obs_px, moved = plant_outliers(52, b.obs_px, 0.03, lo=10.0, hi=200.0)
    args = (b.flags, b.const, b.cam_x, b.model, b.obs_cam, b.obs_key, b.obs_pt, b.obs_px)
    return args, b.truth, moved, {}, None


def _timed(args, kw, steps, warmup):
    runs = []
    for i in range(warmup + steps):
        st = RigidStats()
        r = pose_rigid_robust(*args, threshold_px=TAU, pixel_sigma=0.5, stats=st, **kw)
        if i >= warmup:
            runs.append(st)
    return r, runs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workloads", nargs="*", default=["track", "board64"])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--gp3p-samples", type=int, default=0)
    a = ap.parse_args()
    who = card()
    for name in a.workloads:
        args, truth, moved, kw, per_cam = {"track": track, "board64": board64, "sparse": sparse}[name]()
        kw = dict(kw, gp3p_samples=a.gp3p_samples)
        r, runs = _timed(args, kw, a.steps, a.warmup)
        med = lambda f: float(np.median([getattr(s, f) for s in runs]))  # noqa: E731
        ok = r.status == 0
        out = {"workload": name, "card": who, "gp3p_samples": a.gp3p_samples, "groups": int(len(r.status)),
               "rows": int(len(args[4])), "n_points_below_3": float((r.n_points < 3).mean()),
               "stage_ms": {f: med(f) for f in ("group_ms", "points_ms", "consensus_ms", "refine_ms", "cov_ms",
                                                "total_ms")},
               "kernel_launches": runs[-1].kernel_launches, "status0": float(ok.mean()),
               "moved_rows": int(moved.sum()), "moved_rejected": float((~r.inlier[moved]).mean()),
               "clean_kept": float(r.inlier[~moved].mean()), "rig": _errors(r.pose, truth, ok),
               "chi2_mean": _chi2(r.pose, r.cov, truth, ok)}  # fmt: skip
        if per_cam is not None:
            out["per_camera_resect"] = per_cam
        if a.gp3p_samples > 0:
            r0, runs0 = _timed(args, dict(kw, gp3p_samples=0), a.steps, a.warmup)
            new = (r0.status != 0) & ok
            out["gp3p_off"] = {"status0": float((r0.status == 0).mean()),
                               "consensus_ms": float(np.median([s.consensus_ms for s in runs0])),
                               "total_ms": float(np.median([s.total_ms for s in runs0])),
                               "rig": _errors(r0.pose, truth, r0.status == 0),
                               "chi2_mean": _chi2(r0.pose, r0.cov, truth, r0.status == 0)}  # fmt: skip
            d = _chi2_each(r.pose, r.cov, truth, new)
            far = np.flatnonzero(new)[d > 22.46]  # beyond chi-square(6)'s 0.999 quantile
            amb = (r0.status != 0) & (r.status == 6)
            out["newly_posed"] = {"groups": int(new.sum()), "rig": _errors(r.pose, truth, new),
                                  "chi2_mean": float(d.mean()) if new.any() else None,
                                  "chi2_median": float(np.median(d)) if new.any() else None,
                                  "chi2_above_22_46": int(len(far)), "status6_groups": int(amb.sum()),
                                  "above_22_46": [{"key": int(r.key[g]), "chi2": float(x),
                                                   "distinct_markers": n} for g, x, n in
                                                  zip(far, d[d > 22.46], _distinct_markers(r, args[5], args[6], far))]}  # fmt: skip
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
