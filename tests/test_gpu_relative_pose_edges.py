"""cb_relative_pose_robust on the GPU against oracle/relative_pose.py at its edges: hundreds of independent pairs of every
geometry family in one call, pairs that span several scoring chunks, the sample table's edges, every status and the
refusals.  The oracle runs per pair in a process pool (tests/_relpose_cases.py)."""
from __future__ import annotations

import ctypes as C
import time
from math import comb

import numpy as np
import pytest

from tests._relpose_cases import FAMILIES, LENSES, Bank, assert_report, compare, is_tie, oracle_bank, pair_bank

pytestmark = pytest.mark.gpu

TAU = 3.0
RES_CHUNK = 512  # correspondences per scoring chunk (cb_resect.cuh)


def _run(bank: Bank, **kw):
    from caliscope_b200.epipolar import relative_poses_robust

    return relative_poses_robust(bank.flags, bank.const, bank.cam, bank.key, bank.px, cam_x=bank.x, threshold_px=TAU,
                                 **kw)  # fmt: skip


def _lanes(res) -> int:
    """The refinement's lanes per pair: 32 when the call's mean correspondences per pair exceed 96 (tri_lanes)."""
    return 32 if int(res.count.sum()) // len(res.count) > 96 else 8


def _noise_free(bank):
    return np.array([sp.get("noise_px", 0.0) == 0 for sp in bank.specs])


def _bounded(bank):
    """The noisy pairs of k >= 8.  At k = 6 or 7 every hypothesis fits its own five correspondences exactly and scores
    only the one or two others; when those fall outside tau for every hypothesis, every score is the same multiple of
    tau^2, so ties there are part of the geometry, not a weakness of the comparison."""
    return ~_noise_free(bank) & np.array([sp["k"] >= 8 for sp in bank.specs])


def _truth_t(bank):
    """The truth's t where it is determined: not for pure rotation or a 1e-4 baseline."""
    t = bank.t.copy()
    t[[f in ("tiny", "rotation") for f in bank.family]] = np.nan
    return t


def _compare(dev, orc, bank, name, t0):
    rep = compare(dev, orc, family=bank.family, noise_free=_noise_free(bank), bounded=_bounded(bank), truth_R=bank.R,
                  truth_t=_truth_t(bank))
    print(f"{name}: {time.perf_counter() - t0:.1f} s")
    assert_report(rep, name)
    return rep


def _geometry_specs():
    """Every family at k in {6, 7, 8, 9, 12, 20, 60} in six variants: noisy (0.5 px, 1 px with 10 % outliers, 0.2 px)
    with the lenses in turn, noise-free (not for the planar, tiny and wild families, whose noise-free pairs tie between
    distinct poses), NaN rows."""
    specs = []
    for k in (6, 7, 8, 9, 12, 20, 60):
        for i, fam in enumerate(FAMILIES):
            for v in range(6):
                sp = dict(family=fam, k=k, lens=LENSES[(i + v) % 4], noise_px=0.5, sentinel=1 if k < 12 else 3)
                if v == 3:
                    if fam in ("planar", "tiny", "wild"):
                        continue
                    sp["noise_px"] = 0.0
                if v == 2 and k >= 12:
                    sp["nan_rows"] = 2
                if v == 4:
                    sp.update(noise_px=1.0, outlier_frac=0.1)
                if v == 5:
                    sp["noise_px"] = 0.2
                if fam == "wild":
                    sp["outlier_frac"] = 0.4
                specs.append(sp)
    return specs


def test_geometry_bank():
    """Every pair of every family, lens and k against the oracle in one call of 357 pairs (max_samples 8: exhaustive
    samples at k = 6, hashed above); mean correspondences per pair below 96, so the refinement runs 8 lanes."""
    t0 = time.perf_counter()
    bank = pair_bank(_geometry_specs(), seed=31)
    kw = dict(min_inliers=6, max_samples=8)
    dev = _run(bank, **kw)
    orc = oracle_bank(bank, threshold_px=TAU, **kw)
    assert len(bank.family) == 357 and _lanes(dev) == 8
    rep = _compare(dev, orc, bank, "geometry bank", t0)
    for fam in FAMILIES:
        assert sum(f == fam for f in bank.family) >= 20, fam
    assert rep.statuses.get(0, 0) >= 100
    _assert_same_axis_sign_at_pi(dev, orc, bank)


def _assert_same_axis_sign_at_pi(dev, orc, bank):
    """Rotation at pi: r and -r are the same rotation, and the rule (rot_log, cv2.Rodrigues' branch for s < 1e-5) picks
    one of them from signs of entries of R near zero.  On every refined facing pair, tie or not, the device's r has the
    oracle's axis sign (compared on r itself, not on Rodrigues(r), which cannot tell them apart)."""
    rows, tied = [], 0
    for p, fam in enumerate(bank.family):
        if fam.startswith("facing") and orc.status[p] in (0, 2, 3, 4) and dev.status[p] in (0, 2, 3, 4):
            rows.append((p, float(dev.pose[p, :3] @ orc.pose[p, :3]), bool(_noise_free(bank)[p])))
            tied += is_tie(orc, p)
    exact = [r for r in rows if r[2]]
    print(f"facing pairs: {len(rows)} refined, {len(exact)} noise-free (rotation exactly pi), {tied} tied")
    assert len(exact) >= 10
    flipped = [p for p, dot, _ in rows if not dot > 0]
    assert not flipped, f"the device and the oracle pick opposite axis signs at pi on pairs {flipped}"


def _chunk_specs():
    """Pairs spanning 1, 2, 3 and 6 chunks (k = 511 ... 3000), each followed by a pair of 4, 5 or 6 correspondences
    (below min_inliers) and a one-chunk pair of 40."""
    specs = []
    for i, k in enumerate((511, 512, 513, 1024, 1025, 3000)):
        specs.append(dict(family="general", k=k, noise_px=0.5, outlier_frac=0.05, nan_rows=3))
        specs.append(dict(family="general", k=4 + i % 3, noise_px=0.5))
        specs.append(dict(family="sideways", k=40, noise_px=0.5))
    return specs


def _reordered(bank: Bank, order, seed) -> Bank:
    """The same pairs as `bank`, new pair j = old pair order[j], rows shuffled again."""
    inv = np.argsort(order)
    nx = np.array([9 if f & 1 else 6 for f in bank.flags])
    off = np.r_[0, np.cumsum(nx)]
    cams = np.ravel([[2 * o, 2 * o + 1] for o in order])
    x = np.concatenate([bank.x[off[c] : off[c + 1]] for c in cams])
    cam = (2 * inv[bank.cam // 2] + bank.cam % 2).astype(np.int32)
    perm = np.random.default_rng(seed).permutation(len(cam))
    return Bank(bank.flags[cams], bank.const[cams], x, cam[perm], bank.key[perm], bank.px[perm], bank.R[order],
                bank.t[order], [bank.family[o] for o in order], [bank.specs[o] for o in order])  # fmt: skip


def test_chunk_edges_and_reordering():
    """Pairs of 511, 512, 513, 1024, 1025 and 3000 correspondences (1, 1, 2, 2, 3 and 6 scoring chunks) interleaved with
    one-chunk pairs, some below min_inliers, against the oracle (max_samples 16; 32 refinement lanes).  The same pairs in
    another order and another row order give bit-identical outputs per pair."""
    t0 = time.perf_counter()
    bank = pair_bank(_chunk_specs(), seed=32)
    kw = dict(min_inliers=15, max_samples=16)
    dev = _run(bank, **kw)
    nchunk = np.maximum(1, -(-dev.count // RES_CHUNK))
    assert nchunk.tolist() == [1, 1, 1, 1, 1, 1, 2, 1, 1, 2, 1, 1, 3, 1, 1, 6, 1, 1]
    assert _lanes(dev) == 32
    orc = oracle_bank(bank, threshold_px=TAU, **kw)
    rep = _compare(dev, orc, bank, "chunk edges", t0)
    assert rep.statuses.get(1, 0) == 6
    order = np.random.default_rng(5).permutation(len(bank.family))
    again = _run(_reordered(bank, order, seed=6), **kw)
    for f in ("pose", "cov", "rmse_px", "parallax_deg", "count", "n_inliers", "status"):
        assert np.array_equal(getattr(again, f), getattr(dev, f)[order], equal_nan=True), f


@pytest.mark.parametrize("k, max_samples, min_inliers, exhaustive", [(9, 126, 6, True),
                                                                     (9, 125, 6, False), (5, 8, 5, True),
                                                                     (11, 4096, 6, True)])  # fmt: skip
def test_sample_table_edges(k, max_samples, min_inliers, exhaustive):
    """T = C(k, 5) against max_samples: C(9, 5) = 126 fills the table exactly, 125 switches to hashed samples, k = 5 has
    one sample, k = 11 with max_samples 4096 puts 462 samples in a 40960-slot table (a score grid 320 blocks tall)."""
    t0 = time.perf_counter()
    assert (comb(k, 5) <= max_samples) == exhaustive
    fams = ["general", "forward", "sideways", "wild"] if k > 5 else ["general", "forward", "sideways"]
    specs = [dict(family=f, k=k, noise_px=0.5, lens=LENSES[i % 4]) for i, f in enumerate(fams)]
    bank = pair_bank(specs, seed=33 + k + max_samples)
    kw = dict(min_inliers=min_inliers, max_samples=max_samples)
    dev = _run(bank, **kw)
    orc = oracle_bank(bank, threshold_px=TAU, **kw)
    assert _lanes(dev) == 8
    if k == 5:
        # one sample: every one of its essential matrices fits all five points, so the scores tie and the winner is
        # whichever rounding prefers; the pose still fits the five points
        rep = compare(dev, orc, family=bank.family, bounded=np.zeros(len(specs), bool))
        assert_report(rep, "k = 5")
        ok = np.isin(dev.status, (0, 3, 4))
        assert ok.any() and (dev.rmse_px[ok] < 1e-6).all(), dev.rmse_px
    else:
        _compare(dev, orc, bank, f"k = {k}, max_samples {max_samples}", t0)


def _status_calls():
    """(name, bank, kwargs) of the calls that reach every status:
    1: k < min_inliers; 5: every row NaN (no hypothesis) and 70 % outliers (consensus below min_inliers); 4: points 1000
    times farther than the rest, whose depths flip at the solution (max_iter 200, so that 3 does not come first);
    2: every family with both plain lenses at k = 30, where the noisy 1e-4 baseline with pinhole lenses fails the
    positive-definiteness test (seed 1; 2 is rare: none of 40 other seeded tiny-baseline pairs reaches it); 3: max_iter
    1 on every family."""
    specs = [dict(family="general", k=10, noise_px=0.5), dict(family="general", k=20, nan_rows=40),
             dict(family="general", k=30, noise_px=0.5, outlier_frac=0.7)]  # fmt: skip
    specs += [dict(family=f, k=40, noise_px=0.5, far_frac=0.3) for f in ("general", "forward", "sideways") * 3]
    return [
        ("statuses 1, 4, 5", pair_bank(specs, seed=34), dict(min_inliers=15, max_samples=16, max_iter=200)),
        ("status 2", pair_bank([dict(family=f, k=30, lens=lens, noise_px=0.5) for f in FAMILIES
                                for lens in ("pinhole", "free")], seed=1), dict(min_inliers=6, max_samples=8)),
        ("max_iter 1", pair_bank([dict(family=f, k=30, noise_px=0.5) for f in FAMILIES], seed=35),
         dict(min_inliers=15, max_samples=8, max_iter=1)),
    ]  # fmt: skip


def test_every_status_is_reached():
    """The device reaches every status on the calls of _status_calls, each where the oracle reaches it."""
    (_, b145, kw145), (_, b2, kw2), (_, b3, kw3) = _status_calls()
    dev = _run(b145, **kw145)
    assert dev.status[:3].tolist() == [1, 5, 5] and (dev.status == 4).sum() >= 3, dev.status
    dev = _run(b2, **kw2)
    assert (dev.status == 2).any(), dev.status
    # the pair that reaches 2 is not at the rounding floor, and the oracle reaches 2 on it too
    orc = oracle_bank(b2, threshold_px=TAU, **kw2)
    for p in np.flatnonzero(dev.status == 2):
        assert orc.status[p] == 2 and orc.spread[p]["statuses"] == {2} and not orc.spread[p]["floor"], p
    dev = _run(b3, **kw3)
    assert (dev.status == 3).sum() >= len(FAMILIES) - 2, dev.status


def test_every_status_matches_the_oracle():
    t0 = time.perf_counter()
    for name, bank, kw in _status_calls():
        _compare(_run(bank, **kw), oracle_bank(bank, threshold_px=TAU, **kw), bank, name, t0)


def _raw_call(lib, flags, const, x, cam, key, px, max_pairs, n_pairs):
    ptr = lambda v: v.ctypes.data_as(C.c_void_p)  # noqa: E731
    m = max(max_pairs, 1)
    out = [np.empty(m, np.int32) for _ in range(2)] + [np.empty(6 * m), np.empty(36 * m), np.empty(m), np.empty(m)]
    out += [np.empty(m, np.int32) for _ in range(3)]
    fl, co, xx, ca, ke, pp = (np.ascontiguousarray(v) for v in (flags, const, x, cam, key, px))
    return lib.cb_relative_pose_robust(len(fl), ptr(fl), ptr(co), ptr(xx), len(ca), ptr(ca), ptr(ke), ptr(pp), 0, TAU,
                                       15, 16, 1.0, 20, 1e-12, max_pairs, C.byref(n_pairs), *[ptr(o) for o in out],
                                       None, 0, None)  # fmt: skip


def test_refusals_of_pair_count_and_slot_count():
    """Room for fewer pairs than the call has: CB_E_INVALID with the number needed in *n_pairs_out.  One key of 65537
    rows (65537 * 65536 / 2 = 2 147 516 416 row pairs, above 2^31 - 1): CB_E_INVALID from the slot count, before any slot
    is allocated or sorted."""
    from caliscope_b200 import _lib as L

    lib = L.load()
    bank = pair_bank([dict(family="general", k=20, noise_px=0.5) for _ in range(5)], seed=36)
    n_pairs = C.c_int32(-7)
    assert _raw_call(lib, *bank.args(), 5, n_pairs) == 0 and n_pairs.value == 5
    for room in (4, 1, 0):
        n_pairs.value = -7
        assert _raw_call(lib, *bank.args(), room, n_pairs) == -1, room  # CB_E_INVALID
        assert n_pairs.value == 5, room
    n = 65537
    cam = (np.arange(n) % 2).astype(np.int32)
    key = np.zeros(n, np.int64)
    px = np.random.default_rng(0).uniform(0, 700, (n, 2))
    n_pairs.value = -7
    t0 = time.perf_counter()
    assert _raw_call(lib, bank.flags[:2], bank.const[:2], bank.x[:12], cam, key, px, 1, n_pairs) == -1
    assert "2^31 - 1" in (lib.cb_ba_last_error() or b"").decode()
    print(f"65537-row key refused in {time.perf_counter() - t0:.2f} s")
