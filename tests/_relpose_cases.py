"""Seeded 2-D-only inputs for the relative-pose tests and their comparison with the oracle.

``scene``: cameras on a ring looking at the origin, points near it, every point seen by every camera (key = point), with
pixel noise, planted outliers and NaN rows.  ``pair_bank``: many independent camera pairs in one call, one geometry
family and lens per pair.  ``oracle_bank`` runs the oracle on each pair alone in a process pool; ``compare`` checks a
device result against it pair by pair."""
from __future__ import annotations

import multiprocessing as mp
import os
from concurrent.futures import ProcessPoolExecutor
from dataclasses import dataclass, fields

import cv2
import numpy as np


def look_at(c):
    """World-to-camera R, t of a camera at c looking at the origin (y down)."""
    z = -np.asarray(c, np.float64) / np.linalg.norm(c)
    x = np.cross([0.0, -1.0, 0.0], z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z])
    return R, -R @ c


def scene(n_cams=4, n_pts=60, seed=0, noise_px=0.0, outlier_frac=0.0, nan_rows=0, fisheye=(), free=(), repeat=0):
    """(cam_flags, cam_const, cam_x, obs_cam, obs_key, obs_px, truth R (n, 3, 3), truth t (n, 3), outlier mask)."""
    rng = np.random.default_rng(seed)
    flags = np.zeros(n_cams, np.int32)
    const = np.zeros((n_cams, 9))
    Rs, ts, xs = [], [], []
    for c in range(n_cams):
        ang = 2 * np.pi * c / n_cams + rng.uniform(-0.1, 0.1)
        R, t = look_at(np.array([3.0 * np.cos(ang), rng.uniform(-0.3, 0.3), 3.0 * np.sin(ang)]))
        Rs.append(R)
        ts.append(t)
        f = rng.uniform(700, 900)
        const[c] = [f, f * rng.uniform(0.98, 1.02), 640 + rng.uniform(-5, 5), 360 + rng.uniform(-5, 5),
                    rng.uniform(-0.05, 0.05), rng.uniform(-0.01, 0.01), 0.0, 0.0, 0.0]  # fmt: skip
        if c in fisheye:
            flags[c] |= 2
            const[c, 4:8] = [0.01, -0.005, 0.001, 0.0]
        if c in free:
            flags[c] |= 1
        q = np.r_[cv2.Rodrigues(R)[0].ravel(), t]
        xs.append(np.r_[q, 1.0, const[c, 4], const[c, 5]] if c in free else q)
    X = rng.uniform(-0.8, 0.8, (n_pts, 3))
    cam, key, px = [], [], []
    for p in range(n_pts):
        for c in range(n_cams):
            K = np.array([[const[c, 0], 0, const[c, 2]], [0, const[c, 1], const[c, 3]], [0, 0, 1.0]])
            rv = cv2.Rodrigues(Rs[c])[0]
            if flags[c] & 2:
                uv = cv2.fisheye.projectPoints(X[p][None, None], rv, ts[c], K, const[c, 4:8])[0].reshape(2)
            else:
                uv = cv2.projectPoints(X[p][None], rv, ts[c], K, const[c, [4, 5, 6, 7, 8]])[0].reshape(2)
            for _ in range(1 + (repeat if p % 7 == 0 and c == 0 else 0)):
                cam.append(c)
                key.append(p)
                px.append(uv + rng.normal(0, noise_px, 2))
    cam, key, px = np.array(cam, np.int32), np.array(key, np.int64), np.array(px)
    out = rng.random(len(px)) < outlier_frac
    px[out] = rng.uniform([0, 0], [1280, 720], (out.sum(), 2))
    if nan_rows:
        px[rng.choice(len(px), nan_rows, replace=False)] = np.nan
    perm = rng.permutation(len(px))
    return flags, const, np.concatenate(xs), cam[perm], key[perm], px[perm], np.array(Rs), np.array(ts), out[perm]


def relative_truth(Rs, ts, a, b):
    """R, unit t of camera b relative to camera a (X_b = R X_a + t)."""
    R = Rs[b] @ Rs[a].T
    t = ts[b] - R @ ts[a]
    return R, t / np.linalg.norm(t)


# ---- a bank of independent camera pairs ------------------------------------------------------------------------------
# Every family is a relative pose (R, camera b's centre C in camera a's frame, so t = -R C) and a point set in camera a's
# frame around (0, 0, 5):
#   general         R within ~0.25 rad, C within ~0.6
#   sideways        R = I, t = (-b, 0, 0): t_z = 0 exactly, so the sign of the estimate's t_z (the Householder chart's
#                   reflection) is set by rounding
#   forward         C = (0, 0, 1) with a small rotation: the epipole inside the image
#   planar          every point on one tilted plane
#   tiny            |t| = 5e-4, 1e-4 of the depth
#   rotation        t = 0 (truth t NaN): the baseline's direction is unobservable
#   facing-y        R = diag(-1, 1, -1), an exact rotation by pi about y, camera b at (0, 0, 10) looking back
#   facing-oblique  R = 2 n n^T - I with n = (0, 3, -1) / sqrt(10): pi about an axis with n_x = 0
#   wild            a rotation of 1.2-2.0 rad about a random axis (use with 40 % outliers)
FAMILIES = ("general", "sideways", "forward", "planar", "tiny", "rotation", "facing-y", "facing-oblique", "wild")
# lenses: pinhole (Brown-Conrady k1 k2), fisheye (mild equidistant), sentinel (camera b is _undistort_cases' fish_wild,
# and `sentinel` of its rows are pixels that cv2.fisheye.undistortPoints returns as (-1e6, -1e6)), free (both cameras
# with free intrinsics, s != 1 and k1, k2 taken from x)
LENSES = ("pinhole", "fisheye", "sentinel", "free")
FACING_OBLIQUE_AXIS = np.array([0.0, 3.0, -1.0]) / np.sqrt(10.0)


def _rot(r):
    return cv2.Rodrigues(np.asarray(r, np.float64))[0]


def _family_pose(fam, rng):
    """(R, C) of camera b and the point sampler of family `fam`."""
    cube = lambda n: rng.uniform(-1.0, 1.0, (n, 3)) + [0.0, 0.0, 5.0]  # noqa: E731
    if fam == "general":
        return _rot(rng.normal(0, 0.25, 3)), rng.normal(0, 0.6, 3), cube
    if fam == "sideways":
        return np.eye(3), np.array([rng.uniform(0.3, 0.8), 0.0, 0.0]), cube
    if fam == "forward":
        return _rot(rng.normal(0, 0.05, 3)), np.array([0.0, 0.0, 1.0]), cube
    if fam == "planar":
        nrm = np.r_[rng.uniform(-0.3, 0.3, 2), 1.0]

        def plane(n):
            xy = rng.uniform(-1.5, 1.5, (n, 2))
            return np.c_[xy, 5.0 - (nrm[0] * xy[:, 0] + nrm[1] * xy[:, 1]) / nrm[2]]

        return _rot(rng.normal(0, 0.25, 3)), rng.normal(0, 0.6, 3), plane
    if fam == "tiny":
        d = rng.normal(0, 1, 3)
        return _rot(rng.normal(0, 0.25, 3)), 5e-4 * d / np.linalg.norm(d), cube
    if fam == "rotation":
        return _rot(rng.normal(0, 0.3, 3)), np.zeros(3), cube
    if fam == "facing-y":
        return np.diag([-1.0, 1.0, -1.0]), np.array([0.0, 0.0, 10.0]), cube
    if fam == "facing-oblique":
        n = FACING_OBLIQUE_AXIS
        R = 2.0 * np.outer(n, n) - np.eye(3)
        return R, np.array([0.0, 0.0, 5.0]) - 5.0 * R[2], cube
    if fam == "wild":
        ax = rng.normal(0, 1, 3)
        R = _rot(ax / np.linalg.norm(ax) * rng.uniform(1.2, 2.0))
        return R, np.array([0.0, 0.0, 5.0]) - 5.0 * R[2], cube
    raise ValueError(fam)


def _lens(lens, rng):
    """(flags, const (9,), the camera's block of x, projector of points in the camera's frame) of one camera."""
    f = rng.uniform(700, 900)
    const = np.array([f, f * rng.uniform(0.98, 1.02), 640 + rng.uniform(-5, 5), 360 + rng.uniform(-5, 5),
                      rng.uniform(-0.05, 0.05), rng.uniform(-0.01, 0.01), 0.0, 0.0, 0.0])  # fmt: skip
    flags, x, s, k12 = 0, np.zeros(6), 1.0, const[4:6]
    if lens == "fisheye":
        flags, const[4:8] = 2, [0.01, -0.005, 0.001, 0.0]
    elif lens == "wild":
        from tests._undistort_cases import cameras

        cam = next(c for c in cameras() if c.name == "fish_wild")
        flags, const = 2, np.r_[cam.K[0, 0], cam.K[1, 1], cam.K[0, 2], cam.K[1, 2], cam.d, 0.0]
    elif lens == "free":
        s, k12 = rng.choice([-1, 1]) * rng.uniform(0.02, 0.1) + 1.0, rng.uniform([-0.05, -0.01], [0.05, 0.01])
        flags, x = 1, np.r_[np.zeros(6), s, k12]
    K = np.array([[s * const[0], 0, const[2]], [0, s * const[1], const[3]], [0, 0, 1.0]])

    def project(X):
        if flags & 2:
            return cv2.fisheye.projectPoints(X[:, None], np.zeros(3), np.zeros(3), K, const[4:8])[0].reshape(-1, 2)
        return cv2.projectPoints(X, np.zeros(3), np.zeros(3), K, np.r_[k12, const[6:9]])[0].reshape(-1, 2)

    return flags, const, x, project


def sentinel_pixels(const, n, rng):
    """n pixels that cv2.fisheye.undistortPoints maps to its (-1e6, -1e6) failure sentinel for the fisheye camera const."""
    K = np.array([[const[0], 0, const[2]], [0, const[1], const[3]], [0, 0, 1.0]])
    out = np.zeros((0, 2))
    while len(out) < n:
        p = rng.uniform([-3000.0, -3000.0], [4000.0, 4000.0], (4 * n + 64, 2)).astype(np.float32)
        u = cv2.fisheye.undistortPoints(p[:, None], K, const[4:8]).reshape(-1, 2)
        out = np.r_[out, p[(u == np.float32(-1e6)).all(axis=1)].astype(np.float64)]
    return out[:n]


@dataclass
class Bank:
    """Pair i is cameras (2 i, 2 i + 1); the device reports the pairs in that order."""

    flags: np.ndarray
    const: np.ndarray
    x: np.ndarray
    cam: np.ndarray
    key: np.ndarray
    px: np.ndarray
    R: np.ndarray  # (P, 3, 3) truth
    t: np.ndarray  # (P, 3) unit truth (NaN for pure rotation)
    family: list
    specs: list

    def pair_args(self, i):
        """The oracle's inputs of pair i alone, its cameras renumbered (0, 1)."""
        rows = np.flatnonzero((self.cam == 2 * i) | (self.cam == 2 * i + 1))
        nx = [9 if f & 1 else 6 for f in self.flags]
        o = sum(nx[: 2 * i])
        x = self.x[o : o + nx[2 * i] + nx[2 * i + 1]]
        return (self.flags[2 * i : 2 * i + 2], self.const[2 * i : 2 * i + 2], x, self.cam[rows] - 2 * i, self.key[rows],
                self.px[rows])  # fmt: skip

    def args(self):
        return self.flags, self.const, self.x, self.cam, self.key, self.px


def pair_bank(specs, seed=0) -> Bank:
    """P independent camera pairs in one call.  Spec i = dict(family, k, noise_px=0, outlier_frac=0, nan_rows=0,
    lens="pinhole", sentinel=3, far_frac=0): its own cameras 2 i, 2 i + 1 and k keys of its own, each seen once by both
    cameras; outliers replace camera b's pixel of a key, NaN rows either camera's; a far_frac share of the points is
    moved 1000 times farther along camera a's rays.  Rows are shuffled across the whole call."""
    rng = np.random.default_rng(seed)
    flags, const, xs, cam, key, px, Rs, ts, fams = [], [], [], [], [], [], [], [], []
    k0 = 0
    for i, sp in enumerate(specs):
        fam, k, lens = sp["family"], int(sp["k"]), sp.get("lens", "pinhole")
        assert fam in FAMILIES and lens in LENSES, sp
        R, C, points = _family_pose(fam, rng)
        t = -R @ C
        X = np.zeros((0, 3))
        while len(X) < k:  # in front of both cameras and inside a 100-degree cone of each
            Y = points(4 * k)
            Yb = Y @ R.T + t
            ok = (Y[:, 2] > 0.3) & (Yb[:, 2] > 0.3) & (np.abs(Y[:, :2]).max(1) < 1.2 * Y[:, 2])
            ok &= np.abs(Yb[:, :2]).max(1) < 1.2 * Yb[:, 2]
            X = np.r_[X, Y[ok]]
        X = X[:k]
        X[: int(round(sp.get("far_frac", 0.0) * k))] *= 1000.0  # along camera a's rays, ~1e4 baselines away
        lenses = {"sentinel": ("fisheye", "wild"), "free": ("free", "free")}.get(lens, (lens, lens))
        uv = []
        for c, (ln, Xc) in enumerate(zip(lenses, (X, X @ R.T + t))):
            fl, co, xc, project = _lens(ln, rng)
            flags.append(fl)
            const.append(co)
            xs.append(xc)
            uv.append(project(Xc) + rng.normal(0, sp.get("noise_px", 0.0), (k, 2)))
        out = rng.random(k) < sp.get("outlier_frac", 0.0)
        uv[1][out] = rng.uniform([0, 0], [1280, 720], (out.sum(), 2))
        if lens == "sentinel":
            ns = sp.get("sentinel", 3)
            uv[1][rng.choice(k, ns, replace=False)] = sentinel_pixels(const[-1], ns, rng)
        p = np.concatenate(uv)
        if sp.get("nan_rows", 0):
            p[rng.choice(2 * k, sp["nan_rows"], replace=False)] = np.nan
        cam += [2 * i] * k + [2 * i + 1] * k
        key.append(np.r_[np.arange(k), np.arange(k)] + k0)
        px.append(p)
        k0 += k
        Rs.append(R)
        ts.append(t / np.linalg.norm(t) if fam != "rotation" else np.full(3, np.nan))
        fams.append(fam)
    cam, key, px = np.array(cam, np.int32), np.concatenate(key).astype(np.int64), np.concatenate(px)
    perm = rng.permutation(len(px))
    return Bank(np.array(flags, np.int32), np.array(const), np.concatenate(xs), cam[perm], key[perm], px[perm],
                np.array(Rs), np.array(ts), fams, list(specs))  # fmt: skip


# ---- the oracle of every pair alone, in parallel -----------------------------------------------------------------------
FLOOR_RTOL = 1e-10  # a trial cost this close to the current cost is accepted or rejected by rounding
SPREAD_ORDERS = 6  # row orders of the consensus set re-evaluated per pair: reversed and five seeded permutations


def _oracle_job(job):
    """The oracle on one pair, and how far rounding alone moves its refinement: (result, spread).

    The rule does not depend on the order of the consensus set, but its sums do, so the refinement (step 6), the
    parallax and the covariance (step 7) are evaluated again from the same winner on SPREAD_ORDERS other row orders.
    spread (None without a refinement): the statuses reached, the largest differences from the oracle's pose, rmse,
    parallax and cov, and `floor`: whether a trial's cost came within FLOOR_RTOL of the current cost, so that an accept
    decision, and with it the path, the iteration at which |d| <= xtol (|q| + xtol) holds and the status 0, 3 or 4, is
    decided by rounding."""
    from oracle import relative_pose as O

    args, kw = job
    calls, costs = [], []
    refine, normal_eq = O.refine, O._normal_eq

    def recording_refine(*a, **k):
        calls.append((a, k))
        return refine(*a, **k)

    def recording_normal_eq(q, a):
        out = normal_eq(q, a)
        costs.append(out[0])
        return out

    O.refine, O._normal_eq = recording_refine, recording_normal_eq
    try:
        res = O.relative_poses_robust(*args, **kw)
    finally:
        O.refine, O._normal_eq = refine, normal_eq
    if not calls:
        return res, None
    (R0, t0, xa, xb, fa, fb), k = calls[0]
    cur, floor = costs[0], False
    for ct in costs[1:]:
        floor |= abs(ct - cur) <= FLOOR_RTOL * cur
        cur = min(cur, ct)
    rng = np.random.default_rng(0)
    orders = [np.arange(len(xa))[::-1]] + [rng.permutation(len(xa)) for _ in range(SPREAD_ORDERS - 1)]
    spread = dict(statuses={int(res.status[0])}, pose=0.0, rmse_px=0.0, parallax_deg=0.0, cov=0.0, floor=floor)
    for o in orders:
        r, t, rmse, st = refine(R0, t0, xa[o], xb[o], fa, fb, **k)
        spread["statuses"].add(int(st))
        pose = np.r_[r, t]
        if not np.isfinite(res.pose[0]).all():
            continue
        spread["pose"] = max(spread["pose"], np.abs(pose - res.pose[0]).max())
        spread["rmse_px"] = max(spread["rmse_px"], abs(rmse - res.rmse_px[0]))
        par = O.parallax_deg(O.rodrigues(r), xa[o], xb[o])
        spread["parallax_deg"] = max(spread["parallax_deg"], abs(par - res.parallax_deg[0]))
        if st != O.STATUS_NOT_PD and res.status[0] != O.STATUS_NOT_PD:
            cov = O.covariance(r, t, xa[o], xb[o], fa, fb, kw.get("pixel_sigma", 1.0))[0]
            spread["cov"] = max(spread["cov"], np.abs(cov - res.cov[0]).max())
    return res, spread


def merge_results(parts):
    """One RelPoseResult of the per-pair results `parts` (in order)."""
    from oracle.relative_pose import RelPoseResult

    out = {}
    for f in fields(RelPoseResult):
        vals = [getattr(r, f.name) for r in parts]
        out[f.name] = sum(vals, []) if f.name == "inlier" else np.concatenate(vals)
    return RelPoseResult(**out)


def oracle_bank(bank: Bank, **kw):
    """The oracle on every pair of `bank` alone (cameras renumbered (0, 1)), in a process pool of at most 8 workers,
    merged and given the bank's camera numbers back; `spread` holds each pair's rounding spread (_oracle_job).  The pool
    starts its workers from a fresh interpreter (forkserver), never by forking the caller, which may hold a CUDA
    context."""
    jobs = [(bank.pair_args(i), kw) for i in range(len(bank.family))]
    order = sorted(range(len(jobs)), key=lambda i: -len(jobs[i][0][3]))  # largest pairs first
    with ProcessPoolExecutor(max_workers=min(8, os.cpu_count() or 1), mp_context=mp.get_context("forkserver")) as ex:
        done = dict(zip(order, ex.map(_oracle_job, [jobs[i] for i in order])))
    res = merge_results([done[i][0] for i in range(len(jobs))])
    res.cam_a = 2 * np.arange(len(jobs), dtype=np.int32)
    res.cam_b = res.cam_a + 1
    res.spread = [done[i][1] for i in range(len(jobs))]
    return res


# ---- the device against the oracle -------------------------------------------------------------------------------------
TIE_RTOL = 1e-9  # best and second scores within this (relative to max(1, best)): the winner is not determined
# a tie is checked against the truth instead: the coordinates are float32-rounded (6e-8 relative), so even noise-free
# pairs reach the truth only to ~1e-6 (general pairs of 30 points: up to 1.4e-6 in t)
TRUTH_ATOL = 1e-5


def is_tie(orc, p) -> bool:
    return bool(np.isfinite(orc.second[p]) and orc.second[p] - orc.best[p] <= TIE_RTOL * max(1.0, orc.best[p]))


def tied(orc, p) -> bool:
    """A tie whose winner shows in the outputs: without a consensus (status 5) every output is NaN or 0 whichever wins."""
    return is_tie(orc, p) and orc.status[p] != 5


def _rodrigues(r):
    return cv2.Rodrigues(np.asarray(r, np.float64))[0]


@dataclass
class Report:
    pairs: int
    ties: dict  # family -> tied pairs
    statuses: dict  # status -> pairs (device)
    failures: list
    widened: dict  # family -> pairs compared at their rounding spread rather than 1e-8

    def __str__(self):
        return (f"{self.pairs} pairs, statuses {dict(sorted(self.statuses.items()))}, ties per family {self.ties}, "
                f"compared at their rounding spread per family {self.widened}")


SPREAD_FACTOR = 10.0  # the device sums in yet another order: allow ten times the spread the oracle's own orders show
WIDENED_SHARE = 0.25  # at most this share of the refined pairs may be compared at their spread


def compare(dev, orc, *, family=None, noise_free=None, bounded=None, truth_R=None, truth_t=None) -> Report:
    """Every pair of the device result `dev` against the oracle `orc`.

    Not a tie: status, count and n_inliers equal; pose within 1e-8; rmse and parallax within a relative 1e-8; cov within
    1e-8 of max |cov|.  With the oracle's rounding spread (`orc.spread`, oracle_bank), a pair whose refinement rounding
    alone moves further is compared at SPREAD_FACTOR times that spread instead, and a pair at the rounding floor (a
    trial's cost within FLOOR_RTOL of the current cost) may end at 3 where the oracle converged (0 or 4), or converge
    where the oracle stopped at 3.  In a call of 40 or more refined pairs, at most WIDENED_SHARE of them may be compared
    at their spread.  Pure rotation: t is unobservable and t, -t give the same Sampson distances, so t is compared up to
    its sign.
    A tie (best and second scores within TIE_RTOL, and an oracle status other than 5, whose outputs do not depend on the
    winner): the winner may differ, so status equal to the oracle's; for a `noise_free` pair with a truth, Rodrigues(r)
    within TRUTH_ATOL of R and, at status 0, t within TRUTH_ATOL of the truth's (where it is finite), and n_inliers
    equal except for pure rotation, whose depth test is arbitrary.  At most 2 % of the `bounded` pairs may tie.
    Failures are collected, not raised, so that one report lists them all."""
    P = len(orc.status)
    fam = list(family) if family is not None else ["scene"] * P
    noise_free = np.zeros(P, bool) if noise_free is None else np.asarray(noise_free, bool)
    bounded = np.ones(P, bool) if bounded is None else np.asarray(bounded, bool)
    spreads = getattr(orc, "spread", [None] * P)
    fails, ties, statuses, widened = [], {}, {}, {}
    assert len(dev.status) == P, (len(dev.status), P)
    assert (dev.cam_a == orc.cam_a).all() and (dev.cam_b == orc.cam_b).all()

    def bad(p, what):
        fails.append(f"pair {p} ({fam[p]}, oracle status {orc.status[p]}): {what}")

    for p in range(P):
        statuses[int(dev.status[p])] = statuses.get(int(dev.status[p]), 0) + 1
        if dev.count[p] != orc.count[p]:
            bad(p, f"count {dev.count[p]} != {orc.count[p]}")
        sp = spreads[p]
        allowed = {int(orc.status[p])}
        tol = dict(pose=1e-8, rmse_px=0.0, parallax_deg=0.0, cov=0.0)
        if sp is not None:
            allowed |= sp["statuses"]
            if sp["floor"]:
                allowed |= {0, 3, 4} if orc.status[p] == 3 else {3} if orc.status[p] in (0, 4) else set()
            for f in tol:
                tol[f] = max(tol[f], SPREAD_FACTOR * sp[f])
            scale = np.abs(orc.cov[p]).max() if orc.status[p] in (0, 3, 4) else np.inf
            if (sp["pose"] > 1e-8 or sp["cov"] > 1e-8 * scale
                    or any(sp[f] > 1e-8 * abs(getattr(orc, f)[p]) for f in ("rmse_px", "parallax_deg"))):  # fmt: skip
                widened[fam[p]] = widened.get(fam[p], 0) + 1
        if dev.status[p] not in allowed:
            bad(p, f"status {dev.status[p]} not in {sorted(allowed)}")
        if tied(orc, p):
            ties[fam[p]] = ties.get(fam[p], 0) + 1
            if noise_free[p] and fam[p] != "rotation" and dev.n_inliers[p] != orc.n_inliers[p]:
                bad(p, f"tie: n_inliers {dev.n_inliers[p]} != {orc.n_inliers[p]}")
            if noise_free[p] and truth_R is not None and orc.status[p] in (0, 2, 3, 4):
                e = np.abs(_rodrigues(dev.pose[p, :3]) - truth_R[p]).max()
                if not e <= TRUTH_ATOL:
                    bad(p, f"tie: |Rodrigues(r) - R_truth| {e:.2e}")
                if orc.status[p] == 0 and np.isfinite(truth_t[p]).all():
                    e = np.abs(dev.pose[p, 3:] - truth_t[p]).max()
                    if not e <= TRUTH_ATOL:
                        bad(p, f"tie: |t - t_truth| {e:.2e}")
            continue
        if dev.n_inliers[p] != orc.n_inliers[p]:
            bad(p, f"n_inliers {dev.n_inliers[p]} != {orc.n_inliers[p]}")
        if orc.status[p] in (0, 2, 3, 4):
            d = np.abs(dev.pose[p] - orc.pose[p])
            if fam[p] == "rotation":
                d[3:] = np.minimum(d[3:], np.abs(dev.pose[p, 3:] + orc.pose[p, 3:]).max())
            if not d.max() <= tol["pose"]:
                sig = np.sqrt(np.diag(orc.cov[p]))
                bad(p, f"pose differs by {d.max():.2e} ({np.nanmax(d / sig):.2e} oracle standard deviations): "
                       f"{dev.pose[p]} vs {orc.pose[p]}")  # fmt: skip
            for name in ("rmse_px", "parallax_deg"):
                a, b = getattr(dev, name)[p], getattr(orc, name)[p]
                if not abs(a - b) <= max(1e-8 * abs(b) + 1e-10, tol[name]):
                    bad(p, f"{name} {a!r} vs {b!r}")
        if orc.status[p] in (0, 3, 4):
            scale = np.abs(orc.cov[p]).max()
            e = np.abs(dev.cov[p] - orc.cov[p]).max()
            if not e <= max(1e-8 * scale, tol["cov"]):
                bad(p, f"cov differs by {e / scale:.2e} of max |cov|")
        elif not np.isnan(dev.cov[p]).all():
            bad(p, "cov not NaN")
        if orc.status[p] in (1, 5) and not (np.isnan(dev.pose[p]).all() and np.isnan(dev.rmse_px[p])):
            bad(p, "pose or rmse not NaN")
    n_ties = sum(tied(orc, p) for p in range(P) if bounded[p])
    if n_ties > 0.02 * bounded.sum():
        fails.append(f"{n_ties} of {bounded.sum()} bounded pairs tie (at most 2 % may)")
    refined = sum(s is not None for s in spreads)
    if refined >= 40 and sum(widened.values()) > WIDENED_SHARE * refined:
        fails.append(f"{sum(widened.values())} of {refined} refined pairs compared at their spread (at most "
                     f"{WIDENED_SHARE:.0%} may)")  # fmt: skip
    return Report(P, ties, statuses, fails, widened)


def assert_report(rep: Report, name: str):
    print(f"{name}: {rep}")
    assert not rep.failures, f"{name}: {len(rep.failures)} failures\n" + "\n".join(rep.failures[:40])
