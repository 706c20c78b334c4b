"""Sessions for the extrinsic-bootstrap tests at rig scale, with the kernel shapes each one reaches.

The device stages pick their work split from the data: ``pnp_ippe_kernel`` gives a warp to each (camera, frame, board)
group and walks its rows 32 apart; ``cb_stereo_rmse`` runs ``stereo_pairs_kernel<32>`` instead of ``<8>`` when the
observations per (frame, board, corner) key exceed 12; ``quat_average_kernel`` spreads a camera pair's samples over 128
threads.  Each case names the shapes it exists for (`Case.reaches`) and `reached` measures them from the arrays, so a
generator change that stops reaching a shape fails the CPU suite instead of silently dropping coverage."""
from __future__ import annotations

import functools
from dataclasses import dataclass, field

import numpy as np

from caliscope_b200 import bootstrap as B
from caliscope_b200 import synthetic

PNP_STRIDE_SIZES = (31, 32, 33, 63, 64, 65, 88)  # rows per PnP group on both sides of each 32-row warp stride
PLANTED_SYNC = 10_000  # first sync index of the planted groups (seen by one camera only)


@dataclass
class Case:
    name: str
    tab: B.CameraTables
    cam_id: np.ndarray
    sync_index: np.ndarray
    object_id: np.ndarray
    keypoint_id: np.ndarray
    img_xy: np.ndarray  # (n, 2) distorted pixels
    obj_xyz: np.ndarray  # (n, 3) board coordinates
    truth: dict | None = None  # camera id -> (R, t) world -> camera, where the generator knows it
    reaches: frozenset = field(default_factory=frozenset)

    @property
    def n_obs(self) -> int:
        return len(self.cam_id)

    def calibrated(self) -> np.ndarray:
        """Rows of cameras that have intrinsics (the rows the PnP call uses)."""
        return np.isin(self.cam_id, self.tab.cam_ids[self.tab.has_intrinsics])


def _tab(ids, k, dist, fisheye, ignore=None, has=None) -> B.CameraTables:
    ids = np.asarray(ids, np.int64)
    n = len(ids)
    return B.CameraTables(ids, {int(c): i for i, c in enumerate(ids)}, np.asarray(k, float), np.asarray(dist, float),
                          np.asarray(fisheye, np.int32), np.zeros(n, bool) if ignore is None else np.asarray(ignore, bool),
                          np.ones(n, bool) if has is None else np.asarray(has, bool))  # fmt: skip


def _truth(rvec, tvec, ids) -> dict:
    return {int(c): (synthetic._rot(r), np.asarray(t, float)) for c, r, t in zip(ids, rvec, tvec)}


def _from_session(name, s, reaches, rows=None, img_xy=None) -> Case:
    sel = slice(None) if rows is None else rows
    return Case(name, _tab(s.cam_ids, s.cam_k, s.cam_dist, s.cam_fisheye), s.cam_id[sel], s.sync_index[sel], s.object_id[sel],
                s.keypoint_id[sel], (s.img_xy if img_xy is None else img_xy)[sel], s.obj_xyz[sel], _truth(s.rvec, s.tvec, s.cam_ids),
                frozenset(reaches))  # fmt: skip


@functools.lru_cache(maxsize=None)
def _ring64_session():
    return synthetic.make_board_session(64, 60, seed=1, noise_px=0.3)


def ring64() -> Case:
    return _from_session("ring64", _ring64_session(), {"stereo32", "frame20", "pairs1000", "pnp_gt32"})


def ring64_partial() -> Case:
    """11x8 board; every view keeps a random subset of its corners, some views exactly PNP_STRIDE_SIZES of them."""
    s = synthetic.make_board_session(64, 40, grid=(11, 8), square=0.035, seed=2, noise_px=0.3)
    rng = np.random.default_rng(12)
    view = s.sync_index * 64 + s.cam_id  # rows of a view are contiguous
    starts = np.flatnonzero(np.concatenate([[True], np.diff(view) != 0]))
    ends = np.append(starts[1:], len(view))
    forced = rng.choice(len(starts), 3 * len(PNP_STRIDE_SIZES), replace=False)
    want = {int(v): PNP_STRIDE_SIZES[i % len(PNP_STRIDE_SIZES)] for i, v in enumerate(forced)}
    keep = np.zeros(len(view), bool)
    for v, (b, e) in enumerate(zip(starts, ends)):
        k = want.get(v, int(rng.integers(4, e - b + 1)))
        keep[b + rng.choice(e - b, k, replace=False)] = True
    return _from_session("ring64_partial", s, {"pnp_stride", "pnp_gt32"}, rows=keep)


def ring64_outliers() -> Case:
    """ring64 with every corner of ~3 % of the views shifted by one 20-40 px vector: wrong poses for those views."""
    s = _ring64_session()
    rng = np.random.default_rng(7)
    view = s.sync_index * 64 + s.cam_id
    views = np.unique(view)
    bad = rng.choice(views, int(0.03 * len(views)), replace=False)
    ang = rng.uniform(0, 2 * np.pi, len(bad))
    mag = rng.uniform(20.0, 40.0, len(bad))
    shift = dict(zip(bad.tolist(), np.stack([mag * np.cos(ang), mag * np.sin(ang)], axis=1)))
    xy = s.img_xy.copy()
    hit = np.isin(view, bad)
    xy[hit] += np.array([shift[int(v)] for v in view[hit]])
    return _from_session("ring64_outliers", s, {"stereo32", "iqr_t", "iqr_r"}, img_xy=xy)


def mixed_rig() -> Case:
    """24 cameras with ids 5 + 3 i in a shuffled dict order, every third one fisheye, two ignored, one without intrinsics;
    two boards (object ids 0 and 3) in every frame, sync indices 1000 + 7 f."""
    import cv2

    n_cams, n_frames = 24, 50
    rng = np.random.default_rng(5)
    rvec, tvec = synthetic._ring_cameras(n_cams)
    ids = 5 + 3 * np.arange(n_cams)
    fish = (np.arange(n_cams) % 3 == 0).astype(np.int32)
    w, h = synthetic.WEBCAM_SIZE
    k = np.tile([synthetic.WEBCAM_F, synthetic.WEBCAM_F, w / 2.0, h / 2.0, 0.0], (n_cams, 1))
    k[fish == 1] = [560.0, 557.0, w / 2.0 + 3.1, h / 2.0 - 2.3, 0.0]
    dist = np.zeros((n_cams, 12))
    dist[:, :5] = synthetic.WEBCAM_DIST
    dist[fish == 1] = 0.0
    dist[fish == 1, :4] = [0.05, -0.012, 0.003, -0.0006]
    gx, gy = np.meshgrid(np.arange(7), np.arange(5), indexing="ij")
    corners = np.stack([gx.ravel() * 0.05, gy.ravel() * 0.05, np.zeros(gx.size)], axis=1)
    Rc = np.array([synthetic._rot(r) for r in rvec])
    cam_pos = np.array([-Rc[c].T @ tvec[c] for c in range(n_cams)])
    cols = {kk: [] for kk in ("sync", "cam", "obj", "kp", "xy", "X")}
    for f in range(n_frames):
        for oid in (0, 3):
            pos = np.array([rng.uniform(-0.4, 0.4), rng.uniform(-0.4, 0.4), rng.uniform(0.2, 1.0)])
            az = rng.uniform(0, 2 * np.pi)
            zb = np.array([np.cos(az), np.sin(az), 0.0])
            xb = np.cross([0.0, 0.0, 1.0], zb)
            xb /= np.linalg.norm(xb)
            Rb = np.stack([xb, np.cross(zb, xb), zb], axis=1) @ synthetic._rot(rng.normal(0, 0.3, 3))
            Xw = (corners - corners.mean(axis=0)) @ Rb.T + pos
            for c in range(n_cams):
                view = cam_pos[c] - pos
                if Rb[:, 2] @ view / np.linalg.norm(view) < np.cos(np.radians(65)):
                    continue
                K = np.array([[k[c, 0], 0, k[c, 2]], [0, k[c, 1], k[c, 3]], [0, 0, 1.0]])
                if fish[c]:
                    uv = cv2.fisheye.projectPoints(Xw.reshape(-1, 1, 3), rvec[c], tvec[c], K, dist[c, :4])[0].reshape(-1, 2)
                else:
                    uv = cv2.projectPoints(Xw, rvec[c], tvec[c], K, dist[c, :5])[0].reshape(-1, 2)
                z = (Xw @ Rc[c].T + tvec[c])[:, 2]
                if not ((z > 0).all() and (uv >= 0).all() and (uv[:, 0] < w).all() and (uv[:, 1] < h).all()):
                    continue
                n = len(corners)
                cols["sync"].append(np.full(n, 1000 + 7 * f)); cols["cam"].append(np.full(n, ids[c])); cols["obj"].append(np.full(n, oid))
                cols["kp"].append(np.arange(n)); cols["xy"].append(uv + rng.normal(0, 0.3, uv.shape)); cols["X"].append(corners)
    cat = {kk: np.concatenate(v) for kk, v in cols.items()}
    order = rng.permutation(n_cams)  # dict order
    ignore = np.zeros(n_cams, bool)
    ignore[[4, 13]] = True
    has = np.ones(n_cams, bool)
    has[8] = False
    kt = k.copy()
    kt[~has] = [1.0, 1.0, 0.0, 0.0, 0.0]  # what camera_tables stores for a camera without intrinsics
    tab = _tab(ids[order], kt[order], dist[order] * has[order, None], fish[order], ignore[order], has[order])
    return Case("mixed_rig", tab, cat["cam"], cat["sync"], cat["obj"], cat["kp"], cat["xy"], cat["X"],
                _truth(rvec[order], tvec[order], ids[order]),
                frozenset({"stereo8", "fisheye", "multi_object", "dict_order_drop", "ignored", "no_intrinsics"}))  # fmt: skip


def planted() -> Case:
    """An 8-camera session plus groups that only one camera sees (no pair): 39 collinear points and one off the line (IPPE
    gives up, the fallback runs with 40 rows), 40 collinear points, a 40-row board with NaN z, groups of 3 and 4 rows; and
    two camera pairs that share exactly 3 and 4 corners of one frame."""
    import cv2

    s = synthetic.make_board_session(8, 20, seed=3, noise_px=0.3)
    rng = np.random.default_rng(9)
    K = np.array([[s.cam_k[0, 0], 0, s.cam_k[0, 2]], [0, s.cam_k[0, 1], s.cam_k[0, 3]], [0, 0, 1.0]])
    D = s.cam_dist[0, :5]
    rows = []  # (cam, sync, kp, u, v, X, Y, Z)

    def add(cam, sync, X, rvec, tvec, kps=None):
        uv = cv2.projectPoints(np.nan_to_num(X), np.asarray(rvec, float), np.asarray(tvec, float), K, D)[0].reshape(-1, 2)
        uv = uv + rng.normal(0, 0.3, uv.shape)
        for i, (p, q) in enumerate(zip(uv, X)):
            rows.append((cam, sync, i if kps is None else kps[i], p[0], p[1], q[0], q[1], q[2]))

    pose = ([0.2, -0.1, 0.05], [0.05, -0.02, 1.5])
    line = np.stack([np.linspace(-0.2, 0.2, 40), np.zeros(40), np.zeros(40)], axis=1)
    one_off = line.copy()
    one_off[17] = [0.03, 0.12, 0.0]
    gx, gy = np.meshgrid(np.arange(8), np.arange(5), indexing="ij")
    board = np.stack([gx.ravel() * 0.04, gy.ravel() * 0.04, np.full(gx.size, np.nan)], axis=1)
    add(0, PLANTED_SYNC, one_off, *pose)
    add(0, PLANTED_SYNC + 1, line, *pose)
    add(0, PLANTED_SYNC + 2, board, *pose)
    add(0, PLANTED_SYNC + 3, board[[0, 9, 30]], *pose)
    add(0, PLANTED_SYNC + 4, board[[0, 9, 30, 38]], *pose)
    # cameras 8 .. 11 see one frame each: (8, 9) share corners 3..5, (10, 11) share corners 3..6
    pts = np.concatenate([rng.uniform(-0.15, 0.15, (10, 2)), np.zeros((10, 1))], axis=1)
    for cam, sync, sel, rv, tv in [(8, PLANTED_SYNC + 10, range(0, 6), [0.1, 0.2, 0.0], [0.0, 0.0, 1.4]),
                                   (9, PLANTED_SYNC + 10, range(3, 9), [0.1, -0.2, 0.05], [0.3, 0.0, 1.5]),
                                   (10, PLANTED_SYNC + 11, range(0, 7), [-0.1, 0.15, 0.0], [0.0, 0.05, 1.3]),
                                   (11, PLANTED_SYNC + 11, range(3, 10), [-0.05, -0.25, 0.1], [-0.3, 0.0, 1.6])]:  # fmt: skip
        sel = list(sel)
        add(cam, sync, pts[sel], rv, tv, kps=sel)
    a = np.array(rows)
    n_cams = 12
    k = np.concatenate([s.cam_k, np.tile(s.cam_k[:1], (4, 1))])
    dist = np.concatenate([s.cam_dist, np.tile(s.cam_dist[:1], (4, 1))])
    tab = _tab(np.arange(n_cams), k, dist, np.zeros(n_cams, np.int32))
    cat = lambda base, col: np.concatenate([base, col])  # noqa: E731
    return Case("planted", tab, cat(s.cam_id, a[:, 0].astype(np.int64)), cat(s.sync_index, a[:, 1].astype(np.int64)),
                cat(s.object_id, np.zeros(len(a), np.int64)), cat(s.keypoint_id, a[:, 2].astype(np.int64)), cat(s.img_xy, a[:, 3:5]),
                cat(s.obj_xyz, a[:, 5:8]), None,
                frozenset({"pnp_fallback_gt32", "pnp_collinear", "pnp_nan_z", "pnp_too_few", "pnp_min_rows", "common3", "common4"}))  # fmt: skip


def bench_full() -> Case:
    """The session ``bench.py --workload bootstrap64`` times (696 115 observations)."""
    return _from_session("bench_full", synthetic.make_board_session(64, 1000, seed=0), {"stereo32", "pair_gt128"})


BUILDERS = {f.__name__: f for f in (ring64, ring64_partial, ring64_outliers, mixed_rig, planted, bench_full)}


# ---------------------------------------------------------------------------------------------------------------------
# shapes
# ---------------------------------------------------------------------------------------------------------------------
def _runs(*cols) -> np.ndarray:
    """Sizes of the groups of equal rows of `cols`."""
    order = np.lexsort(cols[::-1])
    k = np.stack([c[order] for c in cols], axis=1)
    brk = np.flatnonzero(np.any(np.diff(k, axis=0) != 0, axis=1)) + 1
    return np.diff(np.concatenate([[0], brk, [len(k)]]))


def stereo_lanes(c: Case) -> int:
    """Lanes per (sync, object, keypoint) group that cb_stereo_rmse picks: 32 when n / n_groups > 12 (integer division)
    over the rows of cameras in the table."""
    known = np.isin(c.cam_id, c.tab.cam_ids)
    n = int(known.sum())
    ng = len(_runs(c.sync_index[known], c.object_id[known], c.keypoint_id[known]))
    return 32 if n // max(ng, 1) > 12 else 8


def pair_samples(c: Case) -> dict:
    """(a, b) -> number of (sync, object) frames in which the reference forms the pair (dict-order rule, ignored cameras
    excluded), counting every group with at least 4 rows (the poses the network receives)."""
    cal = c.calibrated()
    sizes_key = {}
    for cam, s, o in zip(c.cam_id[cal], c.sync_index[cal], c.object_id[cal]):
        sizes_key[(int(cam), int(s), int(o))] = sizes_key.get((int(cam), int(s), int(o)), 0) + 1
    pos = {int(cc): i for i, cc in enumerate(c.tab.cam_ids) if not c.tab.ignore[i]}
    frames: dict = {}
    for (cam, s, o), n in sizes_key.items():
        if n >= 4 and cam in pos:
            frames.setdefault((s, o), []).append(cam)
    out: dict = {}
    for cams in frames.values():
        cams.sort()
        for i in range(len(cams)):
            for j in range(i + 1, len(cams)):
                if pos[cams[i]] < pos[cams[j]]:
                    out[(cams[i], cams[j])] = out.get((cams[i], cams[j]), 0) + 1
    return out


def _dict_order_drops(c: Case) -> bool:
    pos = {int(cc): i for i, cc in enumerate(c.tab.cam_ids) if not c.tab.ignore[i]}
    cal = c.calibrated() & np.isin(c.cam_id, list(pos))
    seen = {}
    for cam, s, o in set(zip(c.cam_id[cal].tolist(), c.sync_index[cal].tolist(), c.object_id[cal].tolist())):
        seen.setdefault((s, o), set()).add(cam)
    return any(a < b and pos[a] > pos[b] for cams in seen.values() for a in cams for b in cams)


def common_counts(c: Case, pairs) -> np.ndarray:
    """Common (sync, object, keypoint) observations of each camera pair (vectorised: one packed key per row)."""
    key = B._pack(c.sync_index, c.object_id, c.keypoint_id)
    by_cam = {int(cc): np.unique(key[c.cam_id == cc]) for cc in np.unique(c.cam_id)}
    empty = np.zeros(0, np.int64)
    return np.array([len(np.intersect1d(by_cam.get(int(a), empty), by_cam.get(int(b), empty), assume_unique=True))
                     for a, b in pairs], np.int64)  # fmt: skip


def reached(c: Case) -> set[str]:
    """The structural shapes of `c` (the IQR-rule shapes need poses: see `iqr_rejections`)."""
    out = set()
    cal = c.calibrated()
    sizes = _runs(c.cam_id[cal], c.sync_index[cal], c.object_id[cal])
    out.add(f"stereo{stereo_lanes(c)}")
    if (sizes > 32).any():
        out.add("pnp_gt32")
    if all((sizes == k).any() for k in PNP_STRIDE_SIZES):
        out.add("pnp_stride")
    if (sizes < 4).any():
        out.add("pnp_too_few")
    if (sizes == 4).any():
        out.add("pnp_min_rows")
    live = np.isin(c.cam_id, c.tab.cam_ids[~c.tab.ignore]) & cal
    views = np.unique(np.stack([c.sync_index[live], c.object_id[live], c.cam_id[live]], axis=1), axis=0)
    if len(views) and _runs(views[:, 0], views[:, 1]).max() >= 20:
        out.add("frame20")
    frames = np.unique(np.stack([c.sync_index, c.object_id], axis=1), axis=0)
    if _runs(frames[:, 0]).max() > 1:
        out.add("multi_object")
    ps = pair_samples(c)
    if len(ps) > 1000:
        out.add("pairs1000")
    if ps and max(ps.values()) > 128:
        out.add("pair_gt128")
    fish_ids = c.tab.cam_ids[c.tab.fisheye == 1]
    if np.isin(c.cam_id, fish_ids).any():
        out.add("fisheye")
    if np.isin(c.cam_id, c.tab.cam_ids[c.tab.ignore]).any():
        out.add("ignored")
    if np.isin(c.cam_id, c.tab.cam_ids[~c.tab.has_intrinsics]).any():
        out.add("no_intrinsics")
    if _dict_order_drops(c):
        out.add("dict_order_drop")
    if c.name == "planted":
        out |= _planted_reaches(c)
    return out


def _planted_reaches(c: Case) -> set[str]:
    from oracle import bootstrap as OB
    from oracle import ippe

    out = set()
    norm = OB.undistort_all(c.tab.cam_ids, c.tab.k, c.tab.dist, c.tab.fisheye, c.cam_id, c.img_xy)
    for s in range(PLANTED_SYNC, PLANTED_SYNC + 3):
        m = (c.cam_id == 0) & (c.sync_index == s)
        R, _, fb = ippe.solve_pnp_planar(c.obj_xyz[m], norm[m])
        if fb and m.sum() > 32 and np.isfinite(R).all():
            out.add("pnp_fallback_gt32")
        if not fb and m.sum() > 32 and not np.isfinite(R).any():
            out.add("pnp_collinear")
        if not fb and np.isnan(c.obj_xyz[m, 2]).all() and np.isfinite(R).all():
            out.add("pnp_nan_z")
    cnt = common_counts(c, [(8, 9), (10, 11)])
    if cnt[0] == 3:
        out.add("common3")
    if cnt[1] == 4:
        out.add("common4")
    return out


def iqr_rejections(c: Case, keys, R, t) -> tuple[int, int]:
    """Rows of pairs with >= 5 samples that the translation rule alone, and the rotation rule alone, rejects (host arrays,
    default multiplier 1.5 on the rule in question, the other one disabled)."""
    rel = B.relative_pose_arrays(keys, R, t, c.tab)
    _, keep_t, *_ = B.filter_and_aggregate(rel, 1.5, rotation_threshold_multiplier=1e30, translation_threshold_multiplier=1.5)
    _, keep_r, *_ = B.filter_and_aggregate(rel, 1.5, rotation_threshold_multiplier=1.5, translation_threshold_multiplier=1e30)
    return int((~keep_t).sum()), int((~keep_r).sum())
