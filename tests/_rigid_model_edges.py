"""Constructed scenes for the rigid-body layout refinement edge tests, on top of ``_rigid_model_cases.make_scene``: used-
frame counts at the cluster and round edges, frames with gaps in their marker masks, frames at the frame-use boundary,
bodies of every status in one call, camera-term runs of many and of one row, extreme keys and far starts; and a mirror
of the host's cluster rule (rmod_impl in cb_engine.cu)."""
from __future__ import annotations

import numpy as np

from oracle.ba_oracle import rodrigues
from oracle.resection_robust import cameras, project, rot_log
from oracle.rigid_model import frame_table
from tests._rigid_cases import Bodies
from tests._rigid_model_cases import Scene, make_scene

__all__ = ["RMOD_WARPS", "cluster_size", "rounds", "used_frames", "run_sizes", "keep_rows", "drop_start", "join",
           "body_alone", "cluster_scene", "mixed_cluster_scene", "marker_scene", "boundary_scene", "BOUNDARY_KEYS",
           "status_mix", "MIX_STATUS", "MIX_MAX_ITER", "camterm_scene", "key_scene", "EXTREME_KEYS",
           "far_scene"]  # fmt: skip

RMOD_WARPS, MAX_CLUSTER, FRAMES_PER_WARP = 8, 8, 4


def cluster_size(max_nf):
    """CTAs per body's cluster: about four frames per warp, 1 to 8 CTAs, from the call's largest used-frame count."""
    return max(1, min(MAX_CLUSTER, -(-max_nf // (FRAMES_PER_WARP * RMOD_WARPS))))


def rounds(nf, cs):
    """rmod_pass's rounds over a body's nf used frames on a cluster of cs CTAs (8 cs warps)."""
    return -(-nf // (RMOD_WARPS * cs))


def used_frames(sc):
    """Used frames per body by the oracle's frame table."""
    b = sc.bodies
    _, rows, _, used = frame_table(b.obs_key, b.obs_pt, sc.start_key, sc.start_pose)
    out = np.zeros(len(sc.body_start) - 1, np.int64)
    for r, u in zip(rows, used):
        if u:
            out[np.searchsorted(sc.body_start, b.obs_pt[r[0]], side="right") - 1] += 1
    return out


def run_sizes(sc):
    """Rows per (key, camera) run."""
    b = sc.bodies
    _, n = np.unique(np.stack([b.obs_key, b.obs_cam.astype(np.int64)]), axis=1, return_counts=True)
    return n


def keep_rows(sc, keep):
    b = sc.bodies
    for name in ("obs_cam", "obs_key", "obs_pt", "obs_px"):
        setattr(b, name, getattr(b, name)[keep])


def drop_start(sc, keys):
    keep = ~np.isin(sc.start_key, keys)
    sc.start_key, sc.start_pose = sc.start_key[keep], sc.start_pose[keep]


def _duplicate(sc, sel):
    b = sc.bodies
    for name in ("obs_cam", "obs_key", "obs_pt", "obs_px"):
        v = getattr(b, name)
        setattr(b, name, np.concatenate([v, v[sel]]))


def _at_truth(sc):
    """The start layout and start poses at the truth."""
    sc.nominal = sc.truth_model.copy()
    sc.start_pose = sc.bodies.truth[np.searchsorted(sc.frame_keys, sc.start_key)].copy()


def join(parts, seed, noise):
    """Scenes on disjoint keys as one call on parts[0]'s rig: every part's rows re-projected from its truth layout and
    poses with that rig, plus N(0, noise[i]) pixel noise; the bodies in part order."""
    base = parts[0].bodies
    cams = cameras(base.flags, base.const, base.cam_x)
    rng = np.random.default_rng(seed)
    sizes = [len(p.truth_model) for p in parts]
    off = np.concatenate([[0], np.cumsum(sizes)])
    oc, ok, op, px = [], [], [], []
    for i, p in enumerate(parts):
        b = p.bodies
        for r in range(len(b.obs_cam)):
            q = b.truth[np.searchsorted(p.frame_keys, b.obs_key[r])]
            Xw = p.truth_model[b.obs_pt[r]] @ rodrigues(q[:3])[0].T + q[3:]
            c = cams[b.obs_cam[r]]
            px.append(project(c, rodrigues(c.q[:3])[0], c.q[3:6], Xw[None])[0][0] + rng.normal(0, noise[i], 2))
        oc.append(b.obs_cam)
        ok.append(b.obs_key)
        op.append(b.obs_pt + off[i])
    model = np.concatenate([p.truth_model for p in parts])
    bodies = Bodies(base.flags, base.const, base.cam_x, model, np.concatenate([p.bodies.truth for p in parts]),
                    np.concatenate(oc).astype(np.int32), np.concatenate(ok).astype(np.int64),
                    np.concatenate(op).astype(np.int32), np.array(px))  # fmt: skip
    sk = np.concatenate([p.start_key for p in parts])
    sp = np.concatenate([p.start_pose.reshape(-1, 6) for p in parts])
    order = np.argsort(sk, kind="stable")
    return Scene(bodies, model.copy(), np.concatenate([p.nominal for p in parts]), sk[order], sp[order],
                 off.astype(np.int64), np.concatenate([p.frame_keys for p in parts]))  # fmt: skip


def body_alone(sc, i):
    """Body i of a joined scene as a call of its own (same rows, rig, start layout and start poses)."""
    b = sc.bodies
    lo, hi = int(sc.body_start[i]), int(sc.body_start[i + 1])
    sel = (b.obs_pt >= lo) & (b.obs_pt < hi)
    nb = Bodies(b.flags, b.const, b.cam_x, b.model[lo:hi], b.truth, b.obs_cam[sel], b.obs_key[sel],
                (b.obs_pt[sel] - lo).astype(np.int32), b.obs_px[sel])  # fmt: skip
    return Scene(nb, sc.truth_model[lo:hi], sc.nominal[lo:hi], sc.start_key, sc.start_pose, np.array([0, hi - lo]),
                 sc.frame_keys)  # fmt: skip


def cluster_scene(nf, seed=101):
    """One body of 4 markers, every (frame, marker, camera) row kept, so all nf frames are used."""
    return make_scene(seed, n_model=4, n_frames=nf, visible=1.0)


MIXED_FRAMES = (1, 5, 300)


def mixed_cluster_scene(seed=103):
    """Bodies of 1, 5 and 300 used frames (4, 5 and 4 markers) in one call: all three run on 8-CTA clusters."""
    parts = [make_scene(seed + 7 * i, n_model=k, n_frames=nf, visible=1.0, frame_keys=np.arange(nf) + 1000 * i)
             for i, (k, nf) in enumerate(zip((4, 5, 4), MIXED_FRAMES))]  # fmt: skip
    return join(parts, seed, (0.3,) * 3)


def marker_scene(K, seed=None, n_frames=12):
    """One body of K markers seen by every camera; frames 1, 5, 9 drop marker 0, frames 2, 6, 10 marker K-1 and frames
    3, 7, 11 every odd marker, where at least 3 markers stay (so at K = 3 no frame drops one).  Warps of one round hold
    different masks and the marker-to-slot map has gaps."""
    sc = make_scene(200 + K if seed is None else seed, n_model=K, n_frames=n_frames, visible=1.0)
    b = sc.bodies
    drop = np.zeros(len(b.obs_pt), bool)
    for f in range(n_frames):
        out = {1: [0], 2: [K - 1], 3: list(range(1, K, 2))}.get(f % 4, [])
        if K - len(out) >= 3:
            drop |= (b.obs_key == f) & np.isin(b.obs_pt, out)
    keep_rows(sc, ~drop)
    return sc


# key -> what it is: 2 three rows of three markers, 4 four rows of two markers, 6 exactly four rows of three markers
# (the smallest used frame), 8 rows without a start pose, 10 a start pose without rows
BOUNDARY_KEYS = dict(three_rows=2, two_markers=4, minimal=6, no_start=8, no_rows=10)


def boundary_scene(seed=107):
    """One body of 5 markers over keys 0 .. 13, the keys of BOUNDARY_KEYS replaced by frames at the frame-use boundary
    and every other key a full frame, so the gram offsets of later frames shift with each."""
    sc = make_scene(seed, n_model=5, n_frames=14, visible=1.0)
    b = sc.bodies
    k = BOUNDARY_KEYS
    keep = ~np.isin(b.obs_key, [k["three_rows"], k["two_markers"], k["minimal"], k["no_rows"]])
    for key, rows in ((k["three_rows"], [(0, 0), (1, 1), (2, 2)]), (k["two_markers"], [(0, 0), (0, 1), (1, 0), (1, 1)]),
                      (k["minimal"], [(0, 0), (0, 1), (1, 2), (2, 3)])):  # fmt: skip
        for m, c in rows:
            keep |= (b.obs_key == key) & (b.obs_pt == m) & (b.obs_cam == c)
    keep_rows(sc, keep)
    drop_start(sc, [k["no_start"]])
    return sc


MIX_STATUS = (0, 1, 1, 2, 4, 3)
MIX_MAX_ITER = 3


def status_mix(seed=109, free=()):
    """Six bodies of 4, 5, 3, 6, 7 and 8 markers in one call, meant for MIX_STATUS at max_iter = MIX_MAX_ITER:
    0 a noise-free body started at its truth; 1 a body whose marker 4 is seen only in a frame without a start pose (it
    has used frames); 1 a body with no start pose at all; 2 a collinear start layout; 4 a noise-free body started at its
    truth and also seen by a camera at camera 0's centre looking the other way; 3 a noisy body started 1 degree, 2 mm
    and 2 mm (layout) off."""
    kw = dict(free=free)
    p0 = make_scene(seed, n_model=4, n_frames=8, noise=0.0, visible=1.0, frame_keys=np.arange(8), **kw)
    _at_truth(p0)
    p1 = make_scene(seed + 1, n_model=5, n_frames=8, frame_keys=np.arange(8) + 100, **kw)
    keep_rows(p1, (p1.bodies.obs_pt != 4) | (p1.bodies.obs_key == 100))
    drop_start(p1, [100])
    p2 = make_scene(seed + 2, n_model=3, n_frames=4, frame_keys=np.arange(4) + 200, **kw)
    drop_start(p2, p2.start_key)
    p3 = make_scene(seed + 3, n_model=6, n_frames=8, frame_keys=np.arange(8) + 300, **kw)
    p3.nominal = np.outer(np.arange(6) - 2.5, [0.03, -0.02, 0.05])
    p4 = make_scene(seed + 4, n_model=7, n_frames=6, noise=0.0, visible=1.0, frame_keys=np.arange(6) + 400, **kw)
    _at_truth(p4)
    p5 = make_scene(seed + 5, n_model=8, n_frames=8, frame_keys=np.arange(8) + 500, **kw)
    sc = join([p0, p1, p2, p3, p4, p5], seed, (0.0, 0.3, 0.3, 0.3, 0.0, 0.3))
    _add_behind_camera(sc, 4)
    return sc


def _add_behind_camera(sc, i):
    """A camera at camera 0's centre looking the other way, seeing every camera-0 row of body i behind it, with the
    pixels the engine's projection gives there at the truth."""
    b = sc.bodies
    Q = np.diag([-1.0, 1.0, -1.0])  # a half turn about the camera's y axis
    R0 = rodrigues(b.cam_x[:3])[0]
    n_cams = len(b.flags)
    P = np.where(b.flags & 1, 9, 6)
    x_new = np.concatenate([rot_log(Q @ R0), Q @ b.cam_x[3:6], b.cam_x[6:P[0]]])
    lo, hi = sc.body_start[i], sc.body_start[i + 1]
    extra = np.flatnonzero((b.obs_cam == 0) & (b.obs_pt >= lo) & (b.obs_pt < hi))
    b.flags = np.append(b.flags, b.flags[0]).astype(np.int32)
    b.const = np.vstack([b.const, b.const[0]])
    b.cam_x = np.concatenate([b.cam_x[: P.sum()], x_new])
    c = cameras(b.flags, b.const, b.cam_x)[n_cams]
    px = []
    for r in extra:
        q = b.truth[np.searchsorted(sc.frame_keys, b.obs_key[r])]
        Xw = b.model[b.obs_pt[r]] @ rodrigues(q[:3])[0].T + q[3:]
        px.append(project(c, rodrigues(c.q[:3])[0], c.q[3:6], Xw[None])[0][0])
    b.obs_cam = np.concatenate([b.obs_cam, np.full(len(extra), n_cams, np.int32)])
    b.obs_key = np.concatenate([b.obs_key, b.obs_key[extra]])
    b.obs_pt = np.concatenate([b.obs_pt, b.obs_pt[extra]])
    b.obs_px = np.vstack([b.obs_px, np.array(px)])


# camterm_scene's body 0 (32 markers, keys 0 .. 7): key -> (camera, rows of its run)
CAMTERM_RUNS = {1: (0, 33), 2: (1, 64), 3: (2, 1)}
CAMTERM_SINGLE = (4, 3)  # key 4 is seen by camera 3 alone
CAMTERM_UNSEEN = 7  # body 1 has no row of camera 7


def camterm_scene(seed=113, free=()):
    """Body 0: 32 markers, every one seen by every camera, with a camera-0 run of 33 rows (marker 0's row twice) at key 1,
    a camera-1 run of 64 rows (every row twice) at key 2, a one-row camera-2 run at key 3, and key 4 seen by camera 3
    alone.  Body 1: 5 markers, no row of camera 7 (its Ĝ columns of camera 7 are zero).  Duplicated rows are rows like
    any other, each with its own noise."""
    p0 = make_scene(seed, n_model=32, n_frames=8, visible=1.0, free=free)
    b = p0.bodies
    (c1, _), (c2, _), (c3, _) = CAMTERM_RUNS[1], CAMTERM_RUNS[2], CAMTERM_RUNS[3]
    keep = ~((b.obs_key == 3) & (b.obs_cam == c3) & (b.obs_pt != 5))
    keep &= ~((b.obs_key == CAMTERM_SINGLE[0]) & (b.obs_cam != CAMTERM_SINGLE[1]))
    keep_rows(p0, keep)
    _duplicate(p0, np.flatnonzero(((b.obs_key == 1) & (b.obs_cam == c1) & (b.obs_pt == 0)) |
                                  ((b.obs_key == 2) & (b.obs_cam == c2))))  # fmt: skip
    p1 = make_scene(seed + 1, n_model=5, n_frames=6, frame_keys=np.arange(6) + 100, free=free)
    keep_rows(p1, p1.bodies.obs_cam != CAMTERM_UNSEEN)
    return join([p0, p1], seed, (0.3, 0.3))


EXTREME_KEYS = np.array([0, 1, 7, 2**31, 2**32 + 3, 2**62, 2**63 - 2, 2**63 - 1], np.int64)


def key_scene(seed=127):
    """One body over EXTREME_KEYS, start poses for all but keys 7 and 2^32 + 3, rows in a shuffled order."""
    sc = make_scene(seed, n_model=5, n_frames=len(EXTREME_KEYS), frame_keys=EXTREME_KEYS)
    drop_start(sc, [7, 2**32 + 3])
    keep_rows(sc, np.random.default_rng(seed).permutation(len(sc.bodies.obs_cam)))
    return sc


def far_scene(seed=131):
    """One body of 6 markers, 10 frames, started 5 degrees and 2 cm (poses) and 5 mm (layout) off."""
    return make_scene(seed, n_model=6, n_frames=10, rot_deg=5.0, trans=0.02, model_off=5e-3)
