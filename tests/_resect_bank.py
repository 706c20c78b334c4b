"""Banks of independent robust-resection groups and their comparison with the oracle.

``make_bank`` puts many independent groups in one ``cb_resect_robust`` call: each group has its own camera slot (its own
intrinsics and prior), its own points and its own key, and the rows of the call are shuffled across groups with the
caller order inside each key kept.  ``oracle_bank`` runs ``oracle/resection_robust.resect_robust`` on each group alone
in a process pool and merges the results in the call's group order; ``check`` / ``inlier_check`` compare a device
result with it.

A group is a spec dict:
  family  general (2-6 m from a 1 m cloud), planar (board corners, frontal or oblique), far (50 m away), wide (fisheye,
          points out to 80 degrees off axis), identity (R = I exactly), down (R = diag(1, -1, -1) exactly, or
          pi - 1e-7 about a tilted axis with ``tilted``), behind (some rows' points behind the camera), decisive (below),
          pad (1-3 rows: status 1), and the status recipes collinear and near_collinear (2), far_px (5), two_cams (6),
          behind_axis (4)
  lens    pinhole (P = 6), free (P = 9: s, k1, k2 in x) or fisheye
  k       rows; noise_px; outlier_frac; nan_pts (points set to NaN); repeat (rows repeated, jittered 0.2 px)
  prior   near (0.02 rad, 0.05 m off), far (0.5 rad, 1 m off) or truth
Decisive groups: every row is an exact projection under pose A or pose B (A's rows with 0.01 px of noise, so that A's
hypotheses do not tie with each other); A has one more row than B (an even k adds one row far from both), B is the
prior, and the rows at ``at`` are A's.  A's best hypothesis then wins by tau^2 less A's small residual sum, and a score
that drops or misplaces one of A's rows ties B's at best, which the prior (slot 0) wins."""
from __future__ import annotations

import multiprocessing as mp
import os
from concurrent.futures import ProcessPoolExecutor
from dataclasses import dataclass, fields

import numpy as np

from oracle.ba_oracle import rodrigues
from oracle.resection_robust import ResectResult, cameras, project, resect_robust, rot_log
from tests._resect_cases import look_at, make_rig

TAU = 4.0
LENSES = ("pinhole", "free", "fisheye")
FAMILIES = ("general", "planar", "far", "wide", "identity", "down", "behind")
RES_CHUNK = 512  # rows per scoring chunk of the long shape (cb_resect.cuh)
RES_LONG_ROWS = 512  # the long shape needs more rows per group than this, on average over the call (cb_engine.cu)
RES_TABLE_BYTES = 1 << 30  # ... and a hypothesis table of at most this many bytes
RES_HYP_BYTES = 96  # one hypothesis in the table: R and t in fp64
LONG_EXTRA_LAUNCHES = 6  # res_hyp, res_chunks, the scan's two, res_score, res_select, res_classify for res_consensus


# ---- the call's shape ----------------------------------------------------------------------------------------------------
def slots(max_samples):
    return 1 + 4 * max_samples


def is_long(counts, max_samples):
    n, g = int(np.sum(counts)), len(counts)
    return n // g > RES_LONG_ROWS and g * slots(max_samples) * RES_HYP_BYTES <= RES_TABLE_BYTES


def lanes(counts, max_samples):
    """Lanes per group of the short-shape consensus, the refinement and the covariance (tri_lanes; 32 in the long shape)."""
    if is_long(counts, max_samples):
        return 32
    return 32 if int(np.sum(counts)) // len(counts) > 96 else 8


def chunks(counts):
    return int(np.maximum(1, (np.asarray(counts) + RES_CHUNK - 1) // RES_CHUNK).sum())


def tiles(max_samples):
    return -(-slots(max_samples) // 128)


def shape_name(counts, max_samples):
    return "long" if is_long(counts, max_samples) else f"short{lanes(counts, max_samples)}"


# ---- one group -----------------------------------------------------------------------------------------------------------
def _lens(lens, rng):
    if lens == "fisheye":
        return 2, np.array([600.0, 600.0, 640.0, 480.0, 0.02, -0.01, 0.003, -0.001, 0.0]), []
    f = rng.uniform(850, 950)
    const = np.array([f, f * rng.uniform(0.99, 1.01), 640.0 + rng.uniform(-5, 5), 480.0 + rng.uniform(-5, 5), -0.08, 0.02,
                      0.001, -0.0005, 0.001])  # fmt: skip
    if lens == "free":
        return 1, const, [1.01, const[4] * 1.1, const[5] * 0.9]
    return 0, const, []


def _random_pose(rng, dist):
    d = rng.normal(0, 1, 3)
    d /= np.linalg.norm(d)
    r, t = look_at(dist * d)
    R = rodrigues(np.asarray(r))[0]
    roll = rodrigues(np.array([0.0, 0.0, rng.uniform(-np.pi, np.pi)]))[0]
    R = roll @ R
    return R, roll @ t


def _points_for(family, spec, rng, R, t, n):
    """World points of a family: in front of the camera (R, t)."""
    if family == "planar":
        g = int(np.ceil(np.sqrt(n * 1.5)))
        gx, gy = np.meshgrid(np.arange(g), np.arange(g))
        P = np.stack([gx.ravel() * 0.04, gy.ravel() * 0.04, np.zeros(g * g)], axis=1)
        P[:, :2] -= P[:, :2].mean(axis=0)
        return P[np.sort(rng.choice(len(P), n, replace=False))]
    if family == "wide":  # directions out to 80 degrees off the optical axis, depths 1-4 m
        th = np.radians(rng.uniform(0, 80, n))
        th[0] = np.radians(80.0)
        ph = rng.uniform(0, 2 * np.pi, n)
        dep = rng.uniform(1.0, 4.0, n)
        Xc = np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)], axis=1) * dep[:, None]
        return (Xc - t) @ R
    if family in ("identity", "down"):  # a 1 m cloud 3 m in front
        Xc = rng.uniform(-1, 1, (n, 3)) + np.array([0.0, 0.0, 3.0])
        return (Xc - t) @ R
    return rng.uniform(-0.5, 0.5, (n, 3))


def _pose_for(spec, rng):
    fam = spec["family"]
    if fam in ("general", "behind", "decisive"):
        return _random_pose(rng, rng.uniform(2.0, 6.0))
    if fam == "far":
        return _random_pose(rng, 50.0)
    if fam == "wide":
        return _random_pose(rng, 0.5)
    if fam == "planar":  # the board in z = 0; frontal (camera on its normal) or 50 degrees oblique
        tilt = np.radians(50.0) if spec.get("oblique") else rng.uniform(-0.05, 0.05)
        R = rodrigues(np.array([np.pi + tilt, 0.0, rng.uniform(-0.3, 0.3)]))[0]
        return R, np.array([0.0, 0.0, 0.6]) + rng.uniform(-0.05, 0.05, 3)
    if fam == "identity":
        return np.eye(3), rng.uniform(-0.3, 0.3, 3)
    if fam == "down":
        if spec.get("tilted"):
            a = np.array([1.0, 0.6, -0.4])
            return rodrigues(a / np.linalg.norm(a) * (np.pi - 1e-7))[0], rng.uniform(-0.3, 0.3, 3)
        return np.diag([1.0, -1.0, -1.0]), rng.uniform(-0.3, 0.3, 3)
    raise ValueError(fam)


def _q_of(R):
    """The rotation vector the prior and the truth use: exactly 0 at I, exactly (pi, 0, 0) at diag(1, -1, -1)."""
    if np.array_equal(R, np.eye(3)):
        return np.zeros(3)
    if np.array_equal(R, np.diag([1.0, -1.0, -1.0])):
        return np.array([np.pi, 0.0, 0.0])
    return rot_log(R)


@dataclass
class Group:
    flags: list  # per camera slot of the group (two for two_cams)
    const: list
    x: list  # each slot's block of x (the prior)
    pts: np.ndarray  # (m, 3) the group's own points
    cam: np.ndarray  # (k,) slot within the group
    pt: np.ndarray  # (k,) point within the group
    px: np.ndarray  # (k, 2)
    R: np.ndarray  # truth (NaN for the status recipes that have none)
    t: np.ndarray
    role: np.ndarray | None = None  # decisive groups: "A", "B" or "N" per row
    RB: np.ndarray | None = None  # decisive groups: pose B (the prior)
    tB: np.ndarray | None = None


def _prior(spec, rng, r, t):
    kind = spec.get("prior", "near")
    if kind == "truth":
        return np.r_[r, t]
    s_r, s_t = (0.5, 1.0) if kind == "far" else (0.02, 0.05)
    return np.r_[r + rng.normal(0, s_r, 3), t + rng.normal(0, s_t, 3)]


def _project_R(flag, const, extra, R, t, X):
    cam = cameras(np.array([flag]), const[None], np.r_[rot_log(R), t, extra])[0]
    return project(cam, R, t, X)


def make_group(spec, seed) -> Group:
    rng = np.random.default_rng(seed)
    fam, k = spec["family"], int(spec.get("k", 12))
    if fam == "pad":
        flag, const, extra = _lens("pinhole", rng)
        R, t = _random_pose(rng, 4.0)
        X = rng.uniform(-0.5, 0.5, (k, 3))
        uv, _ = _project_R(flag, const, extra, R, t, X)
        return Group([flag], [const], [np.r_[_q_of(R), t, extra]], X, np.zeros(k, np.int32), np.arange(k, dtype=np.int32),
                     uv, R, t)  # fmt: skip
    if fam in ("collinear", "near_collinear", "behind_axis"):
        return _status_recipe(fam)
    if fam == "far_px":  # pixels unrelated to the points: no consensus
        flag, const, extra = _lens(spec.get("lens", "pinhole"), rng)
        R, t = _random_pose(rng, 4.0)
        X = rng.uniform(-0.5, 0.5, (k, 3))
        px = rng.uniform(-5e4, 5e4, (k, 2))
        return Group([flag], [const], [np.r_[_q_of(R), t, extra]], X, np.zeros(k, np.int32), np.arange(k, dtype=np.int32),
                     px, np.full((3, 3), np.nan), np.full(3, np.nan))  # fmt: skip
    if fam == "two_cams":
        g = make_group(dict(spec, family="general"), seed)
        g2 = make_group(dict(spec, family="general"), seed + 1)
        cam = np.zeros(len(g.pt), np.int32)
        cam[1::2] = 1
        return Group(g.flags + g2.flags, g.const + g2.const, g.x + g2.x, g.pts, cam, g.pt, g.px, g.R, g.t)
    if fam == "decisive":
        return _decisive(spec, rng)
    flag, const, extra = _lens(spec.get("lens", "pinhole"), rng)
    R, t = _pose_for(spec, rng)
    n_pts = k
    X = _points_for(fam, spec, rng, R, t, n_pts)
    uv, _ = _project_R(flag, const, extra, R, t, X)
    px = uv + rng.normal(0, spec.get("noise_px", 0.0), uv.shape)
    if spec.get("outlier_frac"):
        m = rng.random(k) < spec["outlier_frac"]
        ang = rng.uniform(0, 2 * np.pi, m.sum())
        px[m] += np.stack([np.cos(ang), np.sin(ang)], axis=1) * rng.uniform(20, 200, (m.sum(), 1))
    if fam == "behind":  # a fifth of the rows see points behind the camera (their pixels: where the point's mirror is)
        m = np.zeros(k, bool)
        m[rng.choice(k, max(1, k // 5), replace=False)] = True
        Xc = X @ R.T + t
        Xc[m, 2] = -Xc[m, 2]
        X = (Xc - t) @ R
    pt = np.arange(k, dtype=np.int32)
    if spec.get("nan_pts"):
        X = X.copy()
        X[rng.choice(k, spec["nan_pts"], replace=False)] = np.nan
    if spec.get("repeat"):
        r = np.sort(rng.choice(k, spec["repeat"], replace=False))
        pt = np.r_[pt, pt[r]]
        px = np.r_[px, px[r] + rng.normal(0, 0.2, (len(r), 2))]
    q = np.r_[_prior(spec, rng, _q_of(R), t), extra]
    return Group([flag], [const], [q], X, np.zeros(len(pt), np.int32), pt, px, R, t)


def _decisive(spec, rng) -> Group:
    k = int(spec["k"])
    at = sorted({a for a in spec.get("at", ()) if a < k})
    flag, const, extra = _lens(spec.get("lens", "pinhole"), rng)
    RA, tA = _random_pose(rng, 4.0)
    dR = rodrigues(np.array([0.0, 0.15, 0.05]))[0]
    RB, tB = dR @ RA, dR @ tA + np.array([0.1, -0.05, 0.0])
    X = np.empty((0, 3))
    while len(X) < k:  # points whose two projections are far apart (> 4 tau) and in front of both poses
        P = rng.uniform(-0.6, 0.6, (2 * k, 3))
        ua, za = _project_R(flag, const, extra, RA, tA, P)
        ub, zb = _project_R(flag, const, extra, RB, tB, P)
        ok = (np.linalg.norm(ua - ub, axis=1) > 4 * TAU) & (za > 0.1) & (zb > 0.1)
        X = np.r_[X, P[ok]]
    X = X[:k]
    ua, _ = _project_R(flag, const, extra, RA, tA, X)
    ub, _ = _project_R(flag, const, extra, RB, tB, X)
    n_b = (k - 1) // 2
    n_a = n_b + 1
    role = np.full(k, "B", object)
    role[at] = "A"
    free = np.flatnonzero(role == "B")
    if k % 2 == 0:  # one row far from both poses
        role[rng.choice(free)] = "N"
        free = np.flatnonzero(role == "B")
    role[rng.choice(free, n_a - len(at), replace=False)] = "A"
    a = role == "A"
    px = np.where(a[:, None], ua + rng.normal(0, 0.01, ua.shape), ub)
    px[role == "N"] = ua[role == "N"] + 8 * TAU
    assert a.sum() == n_a and (role == "B").sum() == n_b
    q = np.r_[_q_of(RB), tB, extra]
    return Group([flag], [const], [q], X, np.zeros(k, np.int32), np.arange(k, dtype=np.int32), px, RA, tA, role, RB, tB)


def _status_recipe(fam) -> Group:
    """tests/test_resect_robust_cpu.py::test_status_codes' groups: 12 exact collinear points (status 2), and the status-4
    group (tau = 50 and max_samples = 1: the prior, 0.1 m behind the truth, wins, and a point on the optical axis 0.05 m
    behind the true camera is in the consensus set)."""
    if fam in ("collinear", "near_collinear"):
        flags, const, cam_x, _, _, _, _ = make_rig(8, 3, 30, noise=0.3)
        P = np.stack([np.linspace(-1, 1, 12), np.zeros(12), np.zeros(12)], axis=1)
        if fam == "near_collinear":  # 1e-7 m off the line: the scaled H's last pivot ~1e-14, below PD_RTOL but not 0
            P[:, 1:] = np.random.default_rng(3).normal(0, 1e-7, (12, 2))
        cam = cameras(flags, const, cam_x)[0]
        R = rodrigues(cam.q[:3])[0]
        uv, _ = project(cam, R, cam.q[3:6], P)
        return Group([int(flags[0])], [const[0]], [cam_x[:6].copy()], P, np.zeros(12, np.int32),
                     np.arange(12, dtype=np.int32), uv, R, cam.q[3:6].copy())  # fmt: skip
    flags, const, cam_x, pts, _, _, _ = make_rig(10, 1, 20, noise=0.0)
    cam = cameras(flags, const, cam_x)[0]
    R, t = rodrigues(cam.q[:3])[0], cam.q[3:6]
    P = np.r_[pts, [R.T @ (np.array([0.0, 0.0, -0.05]) - t)]]
    uv, _ = project(cam, R, t, P)
    uv[-1] = [const[0, 2], const[0, 3]]
    prior = cam_x.copy()
    prior[5] += 0.1
    n = len(P)
    return Group([int(flags[0])], [const[0]], [prior], P, np.zeros(n, np.int32), np.arange(n, dtype=np.int32), uv, R,
                 t.copy())  # fmt: skip


# ---- a bank of groups in one call ----------------------------------------------------------------------------------------
@dataclass
class Bank:
    flags: np.ndarray
    const: np.ndarray
    x: np.ndarray
    pts: np.ndarray
    pts_cov: np.ndarray
    cam: np.ndarray
    key: np.ndarray
    pt: np.ndarray
    px: np.ndarray
    specs: list
    groups: list  # Group per spec
    rows: list  # caller rows of each spec's group, in the group's order
    slot0: np.ndarray  # first camera slot of each spec's group
    pt0: np.ndarray  # first point of each spec's group

    @property
    def order(self):
        """Spec index of the call's group g (groups come out in ascending key order)."""
        return np.argsort([self.key[r[0]] for r in self.rows], kind="stable")

    def args(self):
        return self.flags, self.const, self.x, self.pts, self.cam, self.key, self.pt, self.px

    def counts(self):
        return np.array([len(r) for r in self.rows])

    def group_args(self, i):
        """Group i alone: its camera slots renumbered from 0, its points from 0, one key."""
        g = self.groups[i]
        k = len(g.cam)
        pcov = self.pts_cov[self.pt0[i] : self.pt0[i] + len(g.pts)]
        return (np.array(g.flags, np.int32), np.stack(g.const), np.concatenate(g.x), g.pts, g.cam, np.zeros(k, np.int64),
                g.pt, g.px, pcov)  # fmt: skip


def make_bank(specs, seed, *, n_shuffled=None, nan_cov=()) -> Bank:
    """Every spec's group in one call: group i has key 3 i + 1 (so that relabelled banks can take other keys), its own
    camera slots and points; pts_cov is random SPD (NaN at the points listed in nan_cov as (spec, point)).  The rows of
    the first n_shuffled groups (default all) are shuffled across those groups; the later groups' rows follow in order,
    so that appending groups keeps the earlier groups' row numbers."""
    groups = [make_group(sp, seed * 100003 + i) for i, sp in enumerate(specs)]
    flags, const, xs, pts, cam, key, pt, px, slot0, pt0, lab = [], [], [], [], [], [], [], [], [], [], []
    ns = npt = 0
    for i, g in enumerate(groups):
        slot0.append(ns)
        pt0.append(npt)
        flags += g.flags
        const += g.const
        xs += g.x
        pts.append(g.pts)
        cam.append(g.cam + ns)
        pt.append(g.pt + npt)
        px.append(g.px)
        key.append(np.full(len(g.cam), 3 * i + 1, np.int64))
        lab.append(np.full(len(g.cam), i))
        ns += len(g.flags)
        npt += len(g.pts)
    cam, pt, px, key, lab = (np.concatenate(v) for v in (cam, pt, px, key, lab))
    rng = np.random.default_rng(seed)
    pcov_a = rng.normal(0, 1e-3, (npt, 3, 3))
    pts_cov = pcov_a @ np.transpose(pcov_a, (0, 2, 1)) + 1e-7 * np.eye(3)
    for i, p in nan_cov:
        pts_cov[pt0[i] + p] = np.nan
    n_sh = len(groups) if n_shuffled is None else n_shuffled
    head = int((lab < n_sh).sum())
    perm = np.r_[_interleave(lab[:head], np.random.default_rng(seed + 1)), np.arange(head, len(lab))]
    inv = np.empty_like(perm)
    inv[perm] = np.arange(len(perm))
    rows = [inv[lab == i] for i in range(len(groups))]  # caller rows of group i, in the group's order
    return Bank(np.array(flags, np.int32), np.stack(const), np.concatenate(xs), np.concatenate(pts), pts_cov,
                cam[perm].astype(np.int32), key[perm], pt[perm].astype(np.int32), px[perm], list(specs), groups, rows,
                np.array(slot0), np.array(pt0))  # fmt: skip


def _interleave(lab, rng):
    """A permutation of the rows that shuffles them across groups and keeps each group's rows in order."""
    shuf = lab[rng.permutation(len(lab))]
    perm = np.empty(len(lab), np.int64)
    for i in np.unique(lab):
        perm[shuf == i] = np.flatnonzero(lab == i)
    return perm


def relabelled(bank: Bank, seed) -> tuple[Bank, np.ndarray]:
    """The same groups with the keys permuted and the rows shuffled again (caller order within each key kept); returns
    the new bank and, for each of its output groups, the output group of `bank` it is."""
    rng = np.random.default_rng(seed)
    G = len(bank.groups)
    newpos = rng.permutation(G)  # spec i becomes the newpos[i]-th key
    lab = np.empty(len(bank.cam), np.int64)
    for i, r in enumerate(bank.rows):
        lab[r] = i
    old_rows_in_order = np.concatenate(bank.rows)
    lab_o = np.concatenate([np.full(len(r), i) for i, r in enumerate(bank.rows)])
    perm = _interleave(lab_o, rng)
    src = old_rows_in_order[perm]  # new caller row j takes old caller row src[j]
    inv = np.empty_like(perm)
    inv[perm] = np.arange(len(perm))
    rows = [inv[lab_o == i] for i in range(G)]
    key = (3 * newpos[lab_o] + 2)[perm].astype(np.int64)
    nb = Bank(bank.flags, bank.const, bank.x, bank.pts, bank.pts_cov, bank.cam[src], key, bank.pt[src], bank.px[src],
              bank.specs, bank.groups, rows, bank.slot0, bank.pt0)  # fmt: skip
    old_out = np.empty(G, np.int64)
    old_out[bank.order] = np.arange(G)
    return nb, old_out[nb.order]


# ---- the oracle per group --------------------------------------------------------------------------------------------------
def _oracle_job(job):
    args, kw = job
    pcov = args[-1] if kw.pop("with_cov", False) else None
    return resect_robust(*args[:-1], points_cov=pcov, **kw)


def oracle_bank(bank: Bank, idx=None, *, workers=8, **kw) -> ResectResult:
    """The oracle on every group of `bank` (or on the specs `idx`) alone, in a process pool started from a fresh
    interpreter (forkserver, never a fork of a caller that may hold a CUDA context), merged in the call's group order
    (restricted to idx when given) with the call's camera slots and row numbers."""
    order = [int(i) for i in bank.order if idx is None or i in set(idx)]
    jobs = [(bank.group_args(i), dict(kw)) for i in order]
    big = sorted(range(len(jobs)), key=lambda j: -len(jobs[j][0][4]))  # largest groups first
    with ProcessPoolExecutor(max_workers=min(workers, os.cpu_count() or 1), mp_context=mp.get_context("forkserver")) as ex:
        done = dict(zip(big, ex.map(_oracle_job, [jobs[j] for j in big])))
    parts = [done[j] for j in range(len(jobs))]
    out = {}
    for f in fields(ResectResult):
        if f.name == "inlier":
            continue
        out[f.name] = np.concatenate([getattr(p, f.name) for p in parts])
    out["cam"] = np.array([bank.slot0[i] + p.cam[0] for i, p in zip(order, parts)], np.int32)
    out["rep_row"] = np.array([bank.rows[i][p.rep_row[0]] for i, p in zip(order, parts)], np.int32)
    inl = np.zeros(len(bank.cam), bool)
    for i, p in zip(order, parts):
        inl[bank.rows[i]] = p.inlier
    out["inlier"] = inl
    return ResectResult(**out)


def take(res, g):
    """Groups g of a device result (a new object; inlier left whole)."""
    from copy import copy

    o = copy(res)
    for f in ("cam", "pose", "cov", "rmse_px", "count", "n_inliers", "rep_row", "status"):
        setattr(o, f, getattr(res, f)[g])
    return o


# ---- the device against the oracle -----------------------------------------------------------------------------------------
def tie_mask(orc):
    """Groups whose two best hypothesis scores are a near-tie (the winner is not determined); a group without consensus
    has the same outputs whichever wins.  Exactly equal scores are one hypothesis twice (a hashed sample that repeats a
    triple), which the lowest slot settles: not a tie."""
    with np.errstate(invalid="ignore"):
        gap = orc.second - orc.best
        tie = np.isfinite(orc.second) & (gap > 0) & (gap <= 1e-9 * np.maximum(1.0, np.abs(orc.best)))
    return tie & ~np.isin(orc.status, (1, 5, 6))


def at_floor(dev, orc):
    """Refined groups where the device ends at 0 and the oracle at 3 (the iteration limit) or the reverse: a refinement
    that crawls (nearly affine far groups) reaches the limit on one side of the stop test and not on the other when
    rounding moves its last steps.  Their poses must still agree to 1e-6."""
    return (dev.status != orc.status) & np.isin(dev.status, (0, 3)) & np.isin(orc.status, (0, 3))


def check(dev, orc, *, near_tie_max=0.1, cov_rtol=1e-8, crawl=False):
    """Exact count / rep_row / status / inlier equality away from near-tie scores; poses, rmse and cov to 1e-8.

    crawl (for banks with nearly degenerate groups): a refinement that ends at 0 on one side and at the iteration limit
    on the other (at_floor, at most 2 % of the groups) and any refinement stopped by the limit compare poses to 1e-6;
    rmse takes an absolute 1e-10 px (exact pixels leave ~1e-12 px of rounding); cov takes cond(cov) x 1e-12 where that
    exceeds cov_rtol (H summed in another order differs in its last bits, ~1e-13 relative, and its inverse moves by
    cond(H) times that)."""
    np.testing.assert_array_equal(dev.count, orc.count)
    np.testing.assert_array_equal(dev.rep_row, orc.rep_row)
    np.testing.assert_array_equal(dev.cam, orc.cam)
    tie = tie_mask(orc)
    assert tie.mean() <= near_tie_max
    ok = ~tie
    floor = ok & at_floor(dev, orc) if crawl else np.zeros_like(ok)
    assert floor.sum() <= max(1, 0.02 * len(floor)), np.flatnonzero(floor)
    if floor.any():
        print(f"refinements at the rounding floor (status 0 against 3): groups {np.flatnonzero(floor).tolist()}")
        sc = np.maximum(1.0, np.abs(orc.pose[floor]))
        assert np.all(np.abs(dev.pose[floor] - orc.pose[floor]) <= 1e-6 * sc)
    diff = np.flatnonzero(ok & ~floor & (dev.status != orc.status))
    assert not len(diff), [(int(g), int(dev.status[g]), int(orc.status[g]), int(dev.n_inliers[g]), int(orc.n_inliers[g]),
                            float(orc.second[g] - orc.best[g])) for g in diff]  # fmt: skip
    np.testing.assert_array_equal(dev.n_inliers[ok], orc.n_inliers[ok])
    both = ok & ~floor & np.isin(orc.status, (0, 3, 4)) & np.isin(dev.status, (0, 3, 4))
    scale = np.maximum(1.0, np.abs(orc.pose[both]))
    tol = np.where((orc.status[both] == 3) & crawl, 1e-6, 1e-8)[:, None]
    bad = np.flatnonzero(both)[np.any(np.abs(dev.pose[both] - orc.pose[both]) > tol * scale, axis=1)]
    assert not len(bad), (bad, dev.status[bad], orc.status[bad], dev.pose[bad] - orc.pose[bad])
    np.testing.assert_allclose(dev.rmse_px[both], orc.rmse_px[both], rtol=1e-8, atol=1e-10 if crawl else 1e-12)
    c_o, c_d = orc.cov[both], dev.cov[both]
    np.testing.assert_array_equal(np.isnan(c_d), np.isnan(c_o))  # a NaN point covariance in the consensus set
    fin = np.isfinite(c_o).all(axis=(1, 2))
    c_o, c_d = c_o[fin], c_d[fin]
    cs = np.maximum(np.abs(c_o).max(axis=(1, 2), keepdims=True), 1e-300)
    rel = (np.abs(c_d - c_o) / cs).max(axis=(1, 2))
    tol = np.maximum(cov_rtol, 1e-12 * np.linalg.cond(c_o)) if crawl else np.full(len(c_o), cov_rtol)
    assert np.all(rel <= tol), [(int(g), float(r), float(np.linalg.cond(c))) for g, r, c, t in
                                zip(np.flatnonzero(both)[fin], rel, c_o, tol) if r > t]  # fmt: skip
    at_hyp = ok & (orc.status == 2)  # status 2: the hypothesis as pose, cov NaN
    assert np.isnan(dev.cov[at_hyp]).all() and np.isfinite(dev.pose[at_hyp]).all()
    nan_o = ~np.isin(orc.status, (0, 2, 3, 4)) & ok
    assert np.isnan(dev.pose[nan_o]).all() and np.isnan(dev.cov[nan_o]).all()
    return tie


def inlier_check(dev, orc, keys, tie):
    _, grp = np.unique(keys, return_inverse=True)
    rows_ok = ~tie[grp.ravel()]
    np.testing.assert_array_equal(dev.inlier[rows_ok], orc.inlier[rows_ok])


def same_across_shapes(a, b, tie):
    """Two device results for the same groups in calls of different shapes: the integer outputs equal away from the
    oracle's near-ties, pose, rmse and cov to 1e-8 (the long shape sums scores per chunk, the short one row by row)."""
    for f in ("cam", "count", "rep_row"):
        np.testing.assert_array_equal(getattr(a, f), getattr(b, f), err_msg=f)
    ok = ~tie
    for f in ("status", "n_inliers"):
        np.testing.assert_array_equal(getattr(a, f)[ok], getattr(b, f)[ok], err_msg=f)
    r = ok & np.isin(a.status, (0, 2, 3, 4))
    np.testing.assert_allclose(a.pose[r], b.pose[r], rtol=0, atol=1e-8 * max(1.0, float(np.abs(a.pose[r]).max(initial=0))))
    np.testing.assert_allclose(a.rmse_px[r], b.rmse_px[r], rtol=1e-8, atol=1e-10)
    c = r & np.isfinite(a.cov).all(axis=(1, 2))
    np.testing.assert_array_equal(np.isfinite(a.cov[r]).all(axis=(1, 2)), np.isfinite(b.cov[r]).all(axis=(1, 2)))
    if c.any():
        s = np.abs(a.cov[c]).max(axis=(1, 2), keepdims=True)
        assert np.all(np.abs(a.cov[c] - b.cov[c]) <= 1e-8 * s)
