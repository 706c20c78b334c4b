"""Constructed groups for the rigid-body pose edge tests: every status on one rig (make_bodies(5, n_cams=6)'s), put
together in one call with disjoint point ranges of one model table; groups with one decisive sample at a chosen task,
on the Horn and the gP3P path; and single groups of many repeated rows."""
from __future__ import annotations

import numpy as np

from oracle.ba_oracle import rodrigues
from oracle.resection_robust import cameras, project
from tests._gp3p_cases import ambiguous_three
from tests._rigid_cases import Bodies, make_bodies

__all__ = ["compose", "status_scene", "project_rows"]


def project_rows(b, X, rows, noise=0.0, seed=0):
    """obs_cam, obs_pt, obs_px of (marker, camera) rows of world points X on b's rig."""
    cams = cameras(*b.rig())
    rng = np.random.default_rng(seed)
    px = np.array([project(cams[c], rodrigues(cams[c].q[:3])[0], cams[c].q[3:6], X[m : m + 1])[0][0] for m, c in rows])
    px = px + rng.normal(0, noise, px.shape)
    return np.array([c for _, c in rows], np.int32), np.array([m for m, _ in rows], np.int32), px


def compose(b, parts):
    """parts: (model, (obs_cam, obs_pt, obs_px), key, prior pose or None) -> Bodies on b's rig with one model table,
    and the priors (keys ascending)."""
    models, oc, ok, op, px, pk, pp = [], [], [], [], [], [], []
    off = 0
    for model, (c, p, x), key, prior in parts:
        models.append(model)
        oc.append(c)
        ok.append(np.full(len(c), key, np.int64))
        op.append(p + off)
        px.append(x)
        if prior is not None:
            pk.append(key)
            pp.append(prior)
        off += len(model)
    order = np.argsort(pk, kind="stable")
    out = Bodies(b.flags, b.const, b.cam_x, np.concatenate(models), None, np.concatenate(oc), np.concatenate(ok),
                 np.concatenate(op), np.concatenate(px))  # fmt: skip
    return out, (np.asarray(pk, np.int64)[order], np.asarray(pp).reshape(-1, 6)[order])


def _body(b, model, q):
    R = rodrigues(q[:3])[0]
    return model @ R.T + q[3:]


def status_scene(gp3p, filler=0):
    """Groups meant for status 0 (key 0), 1 (key 1), 2 (key 2: collinear markers, the true pose as the prior; key 3
    holds the same markers 1e-7 off their line, where H is positive definite again: status 0 from the prior), 4 (key 4: a marker the refinement carries behind camera 0), 5 (key 5: without
    gP3P every marker in one camera; with it two markers only, so that every sample repeats one) and, with gP3P, 6
    (key 6: tests/_gp3p_cases.ambiguous_three).  filler > 0 adds a group (key 7) of `filler` markers seen by every
    camera, which moves the mean rows per group.  Threshold 50 px and min_inliers 4 suit every group."""
    b = make_bodies(5, n_cams=6, n_frames=1, n_model=10, noise=0.0, visible=1.0)
    bn = make_bodies(5, n_cams=6, n_frames=1, n_model=10, noise=0.3, visible=1.0)
    q = b.truth[0]
    parts = [(bn.model, (bn.obs_cam, bn.obs_pt, bn.obs_px), 0, None)]
    parts.append((b.model[:3], (b.obs_cam[:3], b.obs_pt[:3], b.obs_px[:3]), 1, None))
    line = np.outer(np.linspace(-0.1, 0.1, 5), [0.3, -0.5, 0.8])
    for key, off in ((2, 0.0), (3, 1e-7)):
        m = line.copy()
        m[2] += off * np.array([0.8, 0.0, -0.3]) / np.linalg.norm([0.8, 0.0, -0.3])
        rows = [(i, c) for i in range(5) for c in range(6)]
        parts.append((m, project_rows(b, _body(b, m, q), rows), key, q))
    # 4: tests/test_rigid_pose_cpu.py's _behind_case with every row in camera 0, so that the prior, whose pixels are
    # within a few of the truth's, outscores every gP3P pose at the truth, where the marker's row costs tau^2
    cams = cameras(*b.rig())
    R0, t0 = rodrigues(cams[0].q[:3])[0], cams[0].q[3:6]
    Rb, tb = rodrigues(q[:3])[0], q[3:]
    Xw = R0.T @ (np.array([0.0, 0.0, -0.05]) - t0)
    model = np.r_[b.model, [Rb.T @ (Xw - tb)]]
    keep = b.obs_cam == 0
    c, p, x = b.obs_cam[keep], b.obs_pt[keep], b.obs_px[keep]
    c, p = np.r_[c, 0].astype(np.int32), np.r_[p, len(model) - 1].astype(np.int32)
    x = np.r_[x, [[b.const[0, 2], b.const[0, 3]]]]
    prior = q.copy()
    prior[3:] += 0.1 * R0[2]
    parts.append((model, (c, p, x), 4, prior))
    # 5
    if gp3p:
        sel = b.obs_pt < 2
    else:
        sel = b.obs_cam == (b.obs_pt % 6)
    parts.append((b.model, (b.obs_cam[sel], b.obs_pt[sel], b.obs_px[sel]), 5, None))
    if gp3p:
        _, m6, (c6, _, p6, x6), _ = ambiguous_three()
        parts.append((m6, (c6, p6, x6), 6, None))
    if filler:
        bf = make_bodies(6, n_cams=6, n_frames=1, n_model=filler, noise=0.3, visible=1.0)
        # the same rig (seed 5's) seeing seed 6's body
        cf, pf, xf = project_rows(b, _body(bf, bf.model, bf.truth[0]),
                                  [(i, c) for i in range(filler) for c in range(6)], noise=0.3, seed=7)  # fmt: skip
        parts.append((bf.model, (cf, pf, xf), 7, None))
    return compose(b, parts)


def _triples(n):
    return [(i, j, l) for i in range(n) for j in range(i + 1, n) for l in range(j + 1, n)]


def decisive_horn(n_cams, tasks, n_q=7, seed=71):
    """One group per task t of `tasks` (keys 0, 1, ...): n_q markers seen by every one of n_cams cameras, noise-free, all
    qualified, C(n_q, 3) <= 64 samples in lexicographic order.  Only the markers of sample t - 1 sit at the true pose;
    every other marker's rows are those of a point 5-9 cm off it, so sample t - 1 is the one Horn pose at the truth.
    Returns the scene, the truth and the decisive sample of every group."""
    b = make_bodies(seed, n_cams=n_cams, n_frames=1, n_model=n_q, noise=0.0, visible=1.0)
    rng = np.random.default_rng(seed)
    q = b.truth[0]
    X = _body(b, b.model, q)
    parts, good = [], []
    for key, t in enumerate(tasks):
        trip = _triples(n_q)[t - 1]
        Xk = X.copy()
        rows = [(i, c) for i in range(n_q) for c in range(n_cams)]
        _, _, true_px = project_rows(b, X, rows)
        for i in range(n_q):
            while i not in trip:  # a displacement that moves every one of the marker's pixels by 10 px or more
                v = rng.normal(size=3)
                Xk[i] = X[i] + v / np.linalg.norm(v) * rng.uniform(0.05, 0.09)
                d = np.linalg.norm(project_rows(b, Xk, rows)[2] - true_px, axis=1)
                if d[np.array([m for m, _ in rows]) == i].min() >= 10.0:
                    break
        parts.append((b.model, project_rows(b, Xk, rows), key, None))
        good.append(trip)
    s, _ = compose(b, parts)
    return s, q, good


def decisive_gp3p(tasks, gp3p_samples=40, k=12, filler=0, seed=81):
    """One group per task t of `tasks` (keys 0, 1, ...) of k rows on make_bodies(seed, 6 cameras)'s rig, without a
    triangulated triple: marker A in two cameras (qualified), B, C and D in one camera each, and k - 5 rows of markers
    seen once at 40-80 px from their true pixels.  C(k, 3) > gp3p_samples, so the samples are the hashed draw; the rows
    are placed so that sample t - 1 is (A, B, C), that no other drawn sample is three of the true rows with distinct
    markers or repeats it, and that the true pose is hypothesis c >= 1 of that sample (ascending roots).  The consensus
    then holds four distinct markers (status 0).  Rows within a key are in position order.  filler
    > 0 adds a group (key len(tasks)) of `filler` markers in every camera.  Returns the scene, the truth and (m, c)."""
    from oracle.gp3p import gp3p as solve
    from oracle.resection_robust import candidate_samples
    from oracle.rigid_pose_gp3p import rays

    n_cams = 6
    b = make_bodies(seed, n_cams=n_cams, n_frames=1, n_model=k - 1, noise=0.0, visible=1.0)
    _triples_of = lambda v: [(v[i], v[j], v[l]) for i, j, l in _triples(len(v))]  # noqa: E731
    q = b.truth[0]
    X = _body(b, b.model, q)
    cs = candidate_samples(k, gp3p_samples)
    rng = np.random.default_rng(seed)
    parts, which = [], []
    for key, t in enumerate(tasks):
        m = t - 1
        S = cs[m]
        assert S is not None and cs.index(S) == m, (t, S)
        found = None
        for _ in range(400):
            pa, pb, pc = rng.permutation(S)
            ca, ca2, cb, cc, cd = rng.choice(n_cams, 5, replace=False)
            free = [p for p in range(k) if p not in S]
            q2, qd = (int(x) for x in rng.choice(free, 2, replace=False))
            pos = {pa: (0, ca), q2: (0, ca2), pb: (1, cb), pc: (2, cc), qd: (3, cd)}
            true3 = [tuple(sorted(x)) for x in _triples_of(list(pos)) if len({pos[p][0] for p in x}) == 3]
            if any(x in cs and x != tuple(S) for x in true3):
                continue
            bad = [p for p in range(k) if p not in pos]
            for j, p in enumerate(bad):
                pos[p] = (4 + j, int(rng.integers(n_cams)))
            rows = [pos[p] for p in range(k)]
            oc, op, px = project_rows(b, X, rows)
            for j in range(len(bad)):
                ang = rng.uniform(0, 2 * np.pi)
                px[bad[j]] += rng.uniform(40, 80) * np.array([np.cos(ang), np.sin(ang)])
            cen, ray = rays(*b.rig(), oc, px)
            s3 = list(S)
            hyp = solve(cen[s3], ray[s3], b.model[op[s3]])
            at = [h for h, (R, tt) in enumerate(hyp) if np.abs(R - rodrigues(q[:3])[0]).max() < 1e-6 and
                  np.abs(tt - q[3:]).max() < 1e-6]  # fmt: skip
            if len(at) == 1 and at[0] >= 1:
                found = (oc, op, px, (m, at[0]))
                break
        assert found is not None, t
        parts.append((b.model, found[:3], key, None))
        which.append(found[3])
    if filler:
        bf = make_bodies(seed + 1, n_cams=n_cams, n_frames=1, n_model=filler, noise=0.0, visible=1.0)
        parts.append((bf.model, project_rows(b, _body(bf, bf.model, q), [(i, c) for i in range(filler)
                                                                         for c in range(n_cams)], noise=0.3),
                      len(tasks), None))  # fmt: skip
    s, _ = compose(b, parts)
    return s, q, which


def huge(n_rows, kind, seed=91):
    """One group of exactly n_rows rows, its rows repeated with fresh 0.3 px noise: kind "horn" (8 markers in each of 8
    cameras, all triangulated), "gp3p" (10 markers each in one of 6 cameras, none triangulated) or "ambiguous"
    (tests/_gp3p_cases.ambiguous_three's seven rows, noise-free, so that lane 0's scan for a fourth distinct marker
    reads every consensus flag)."""
    rng = np.random.default_rng(seed)
    if kind == "ambiguous":
        b, model, (oc, _, op, px), _ = ambiguous_three()
        noise = 0.0
    else:
        n_cams, n_model = (8, 8) if kind == "horn" else (6, 10)
        b = make_bodies(seed, n_cams=n_cams, n_frames=1, n_model=n_model, noise=0.0, visible=1.0)
        if kind == "gp3p":
            keep = b.obs_cam == (b.obs_pt % n_cams)
            b = Bodies(b.flags, b.const, b.cam_x, b.model, b.truth, *(a[keep] for a in b.obs()))
        model, oc, op, px, noise = b.model, b.obs_cam, b.obs_pt, b.obs_px, 0.3
    idx = np.resize(np.arange(len(oc)), n_rows)
    out = Bodies(b.flags, b.const, b.cam_x, model, b.truth, oc[idx].astype(np.int32), np.zeros(n_rows, np.int64),
                 op[idx].astype(np.int32), px[idx] + rng.normal(0, noise, (n_rows, 2)))  # fmt: skip
    return out
