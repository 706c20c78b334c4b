"""cb_resect_robust on the GPU against oracle/resection_robust.py at its edges: hundreds of independent groups of every
geometry family and lens in one call, the same groups in all three consensus shapes (long, 32 and 8 lanes), decisive
rows at the scoring-chunk edges, the slot tiles, the hypothesis-table bound, the sample table's edges, every status in
every shape, point covariances with repeated points, and relabelled calls.  The oracle runs per group in a process pool
(tests/_resect_bank.py).  Every test prints and asserts the path it reaches."""
from __future__ import annotations

import time
from math import comb

import numpy as np
import pytest

from tests._resect_bank import (FAMILIES, LENSES, LONG_EXTRA_LAUNCHES, TAU, check, chunks, inlier_check, is_long, lanes,
                                make_bank, oracle_bank, relabelled, same_across_shapes, shape_name, take, tie_mask,
                                tiles)  # fmt: skip

pytestmark = pytest.mark.gpu


def _run(bank, *, with_cov=False, **kw):
    from caliscope_b200.resection import ResectStats, resect_robust

    st = ResectStats()
    out = resect_robust(*bank.args(), threshold_px=kw.pop("threshold_px", TAU), stats=st,
                        points_cov=bank.pts_cov if with_cov else None, **kw)  # fmt: skip
    return out, st


def _path(name, bank, st, max_samples=64):
    c = bank.counts()
    long_ = is_long(c, max_samples)
    print(f"{name}: {len(c)} groups, {int(c.sum())} rows, shape {shape_name(c, max_samples)}, lanes "
          f"{lanes(c, max_samples)}, chunks {chunks(c) if long_ else '-'}, tiles {tiles(max_samples) if long_ else '-'}, "
          f"launches {st.kernel_launches}")  # fmt: skip
    return long_


def _oracle(bank, idx=None, **kw):
    kw.setdefault("threshold_px", TAU)
    return oracle_bank(bank, idx, **kw)


# ---- geometry bank -------------------------------------------------------------------------------------------------------
def _geometry_specs():
    """Every family at k in {4, 5, 6, 8, 12, 20, 60, 150} in six variants, lenses in turn (wide: fisheye)."""
    specs = []
    for k in (4, 5, 6, 8, 12, 20, 60, 150):
        for i, fam in enumerate(FAMILIES):
            for v in range(6):
                sp = dict(family=fam, k=k, lens="fisheye" if fam == "wide" else LENSES[(i + v) % 3], noise_px=0.3)
                if v == 0:  # noise-free; identity and down with 0.001 px, so that the winner is within 1e-6 of R
                    sp["noise_px"] = 1e-3 if fam in ("identity", "down") else 0.0
                if v == 1:
                    sp["prior"] = "far"
                if v == 2:
                    sp.update(noise_px=1.0, outlier_frac=0.2)
                if v == 3:
                    if k < 12:
                        continue
                    sp.update(noise_px=1.0, outlier_frac=0.5)
                if v == 4:
                    sp.update(prior="truth", nan_pts=1 if k >= 8 else 0, repeat=2 if k >= 8 else 0)
                if v == 5:
                    sp.update(noise_px=1e-3 if fam in ("identity", "down") else 0.3, tilted=True, oblique=True)
                specs.append(sp)
    return specs


def _noise_free(bank):
    return np.array([bank.specs[i].get("noise_px", 0) == 0 for i in bank.order])


def _check_ties_against_truth(dev, orc, bank):
    """A noise-free near-tie: every hypothesis fits, and the refinement reaches the truth whichever wins."""
    tie = tie_mask(orc)
    nf = tie & _noise_free(bank) & np.isin(dev.status, (0, 3))
    for g in np.flatnonzero(nf):
        grp = bank.groups[bank.order[g]]
        from oracle.ba_oracle import rodrigues

        assert np.abs(rodrigues(dev.pose[g, :3])[0] - grp.R).max() < 1e-4, g
        assert np.abs(dev.pose[g, 3:] - grp.t).max() < 1e-4 * max(1.0, np.abs(grp.t).max()), g
    return tie.sum(), nf.sum()


@pytest.mark.parametrize("use_prior", [True, False])
def test_geometry_bank(use_prior):
    t0 = time.perf_counter()
    bank = make_bank(_geometry_specs(), 17)
    dev, st = _run(bank, use_prior=use_prior)
    orc = _oracle(bank, use_prior=use_prior)
    assert not _path("geometry bank", bank, st) and lanes(bank.counts(), 64) == 8
    G = len(bank.groups)
    assert G >= 300
    fam = [bank.specs[i]["family"] for i in bank.order]
    lens = [bank.specs[i]["lens"] for i in bank.order]
    for f in FAMILIES:
        assert fam.count(f) >= 20, f
    for L in LENSES:
        assert lens.count(L) >= 20, L
    tie = check(dev, orc, near_tie_max=0.25, crawl=True)
    inlier_check(dev, orc, bank.key, tie)
    n_tie, n_nf = _check_ties_against_truth(dev, orc, bank)
    sts = {int(s): int((orc.status == s).sum()) for s in np.unique(orc.status)}
    print(f"statuses {sts}, ties {n_tie} ({n_nf} noise-free, checked against the truth), {time.perf_counter() - t0:.1f} s")
    assert sts.get(0, 0) >= 100
    # rotation at 0 and pi: the device's r has the oracle's sign (r itself, not Rodrigues(r))
    edge = np.array([f in ("identity", "down") for f in fam]) & np.isin(orc.status, (0, 3, 4)) & np.isin(dev.status, (0, 3, 4))
    assert edge.sum() >= 40
    dots = np.einsum("gi,gi->g", dev.pose[edge, :3], orc.pose[edge, :3])
    norms = np.linalg.norm(orc.pose[edge, :3], axis=1)
    big = norms > 1.0  # at pi; near 0 the sign of a tiny r carries no axis
    assert np.all(dots[big] > 0), np.flatnonzero(edge)[big][dots[big] <= 0]
    ok = edge & ~tie
    np.testing.assert_allclose(dev.pose[ok, :3], orc.pose[ok, :3], rtol=0, atol=1e-7)


# ---- the same groups in all three shapes, every status --------------------------------------------------------------------
def _core_specs():
    """Long groups (600-3000 rows, one with repeated rows, one with NaN points), short general groups and the status
    recipes 1, 2 (exactly and nearly collinear), 5 and 6."""
    return [dict(family="general", k=600, noise_px=0.5, outlier_frac=0.2, lens="free"),
            dict(family="general", k=1100, noise_px=0.3, repeat=40, lens="pinhole"),
            dict(family="wide", k=1700, noise_px=0.3, nan_pts=5, lens="fisheye"),
            dict(family="decisive", k=3000, at=(0, 511, 512, 1023, 1024, 2999)),
            dict(family="general", k=20, noise_px=0.3, repeat=3, lens="pinhole"),
            dict(family="planar", k=60, noise_px=0.3, lens="free", oblique=True),
            dict(family="pad", k=3),
            dict(family="collinear"),
            dict(family="far_px", k=10),
            dict(family="near_collinear"),
            dict(family="two_cams", k=10, noise_px=0.3)]  # fmt: skip


def _padded(specs, n_pad):
    return specs + [dict(family="pad", k=1 + i % 3) for i in range(n_pad)]


@pytest.mark.parametrize("max_iter", [20, 1])
def test_shape_invariance_and_statuses(max_iter):
    """One set of groups alone (long shape), padded to a mean in (96, 512] (32 lanes) and to a mean <= 96 (8 lanes), with
    a point covariance that is NaN at a point of a long group's consensus set.  max_iter = 20 reaches statuses 0, 1, 2, 5
    and 6 in every shape, max_iter = 1 status 3."""
    t0 = time.perf_counter()
    core = _core_specs()
    G = len(core)
    nan_cov = [(1, 7)]
    res, launches = {}, {}
    for name, n_pad in (("long", 0), ("short32", 10), ("short8", 80)):
        bank = make_bank(_padded(core, n_pad), 5, n_shuffled=G, nan_cov=nan_cov)
        dev, st = _run(bank, with_cov=True, max_iter=max_iter)
        _path(f"{name} (max_iter {max_iter})", bank, st)
        assert shape_name(bank.counts(), 64) == name
        orc = _oracle(bank, max_iter=max_iter, with_cov=True)
        tie = check(dev, orc, crawl=True)
        inlier_check(dev, orc, bank.key, tie)
        assert (orc.status[G:] == 1).all()
        res[name], launches[name] = (take(dev, slice(0, G)), tie[:G]), st.kernel_launches
        want = {1, 2, 5, 6} | ({0} if max_iter == 20 else {3})
        assert want <= set(orc.status[:G].tolist()) and want <= set(dev.status[:G].tolist()), (orc.status[:G], dev.status[:G])
        assert np.isnan(dev.cov[1]).all()  # point 7 of group 1 is a consensus row
    a, tie = res["long"]
    for name in ("short32", "short8"):
        same_across_shapes(a, res[name][0], tie | res[name][1])
    # the long shape makes six more launches than the short one; the ten padding groups of the 32-lane call leave the point
    # sort's key width (and so its passes) as it is
    print(f"launches {launches}, {time.perf_counter() - t0:.1f} s")
    bank32 = make_bank(_padded(core, 10), 5, n_shuffled=G)
    assert _sort_launches(bank32) == _sort_launches(make_bank(core, 5))
    assert launches["long"] - launches["short32"] == LONG_EXTRA_LAUNCHES


def _bits_for(v):  # cb_engine.cu's bits_for
    b = 1
    while b < 64 and (v >> b) != 0:
        b += 1
    return b


def _sort_launches(bank):
    """Launches of the (group, point) radix sort before res_cov_kernel: 2 per 8-bit digit of its key (cb_engine.cu)."""
    key_bits = min(64, max(1, _bits_for(max(len(bank.pts) - 1, 0))) + _bits_for(len(bank.groups)))
    return 2 * ((key_bits + 7) // 8)


def test_status_4_in_every_shape():
    """The status-4 recipe (tau = 50, max_samples = 1) with long groups added for the long shape and padding for 8 and
    32 lanes."""
    base = [dict(family="behind_axis"), dict(family="behind_axis")]
    for name, specs in (("long", base + [dict(family="general", k=1500, noise_px=0.3), dict(family="general", k=1600, noise_px=0.3)]),
                        ("short32", base + [dict(family="general", k=400, noise_px=0.3)]),
                        ("short8", _padded(base, 4))):  # fmt: skip
        bank = make_bank(specs, 8)
        dev, st = _run(bank, threshold_px=50.0, max_samples=1)
        _path(f"status 4 {name}", bank, st, max_samples=1)
        assert shape_name(bank.counts(), 1) == name
        orc = _oracle(bank, threshold_px=50.0, max_samples=1)
        tie = check(dev, orc, crawl=True)
        inlier_check(dev, orc, bank.key, tie)
        assert (orc.status[:2] == 4).all() and (dev.status[:2] == 4).all()


# ---- chunk edges, reordering -----------------------------------------------------------------------------------------------
def _chunk_specs():
    specs = []
    short = [dict(family="general", k=4, noise_px=0.3), dict(family="pad", k=3), dict(family="two_cams", k=6, noise_px=0.3)]
    for i, k in enumerate((511, 512, 513, 1024, 1025, 3000)):
        specs.append(dict(family="decisive", k=k, at=(0, 511, 512, 1023, 1024, k - 1), lens=LENSES[i % 3]))
        specs.append(short[i % 3])
    return specs


@pytest.mark.parametrize("use_prior", [True, False])
def test_chunk_edges(use_prior):
    """Decisive groups of 511 ... 3000 rows with A's rows at 0, 511, 512, 1023, 1024 and the last, interleaved with short
    groups (mean ~ 550 rows: the long shape); with max_iter = 1 as well (the pose is then one step from the winning
    hypothesis); relabelled and reordered, every output is bit-identical."""
    t0 = time.perf_counter()
    bank = make_bank(_chunk_specs(), 23)
    for max_iter in (20, 1):
        dev, st = _run(bank, use_prior=use_prior, max_iter=max_iter, with_cov=True)
        assert _path(f"chunk edges (max_iter {max_iter})", bank, st)
        assert chunks(bank.counts()) == 1 + 1 + 2 + 2 + 3 + 6 + 6
        orc = _oracle(bank, use_prior=use_prior, max_iter=max_iter, with_cov=True)
        tie = check(dev, orc, near_tie_max=0.0, crawl=True)
        inlier_check(dev, orc, bank.key, tie)
        dec = np.array([bank.specs[i]["family"] == "decisive" for i in bank.order])
        n_a = np.array([(bank.groups[i].role == "A").sum() if bank.groups[i].role is not None else 0 for i in bank.order])
        np.testing.assert_array_equal(dev.n_inliers[dec], n_a[dec])
        print("statuses", dev.status.tolist())
    nb, src = relabelled(bank, 4)
    again, st2 = _run(nb, use_prior=use_prior, max_iter=1, with_cov=True)
    assert st2.kernel_launches == st.kernel_launches
    for f in ("cam", "pose", "cov", "rmse_px", "count", "n_inliers", "status"):
        np.testing.assert_array_equal(getattr(again, f), getattr(dev, f)[src], err_msg=f)
    for g_new, g_old in enumerate(src):
        np.testing.assert_array_equal(again.inlier[nb.rows[nb.order[g_new]]], dev.inlier[bank.rows[bank.order[g_old]]])
    print(f"{time.perf_counter() - t0:.1f} s")


# ---- slot tiles, the table bound, the sample table ----------------------------------------------------------------------------
@pytest.mark.parametrize("max_samples", [31, 32, 4096])
@pytest.mark.parametrize("use_prior", [True, False])
def test_slot_tiles(max_samples, use_prior):
    """S = 1 + 4 max_samples = 125, 129 and 16385 slots: 1, 2 and 129 tiles of 128 (at 32 the second tile holds one slot,
    sample 31's fourth solution)."""
    specs = [dict(family="general", k=520 + 60 * i, noise_px=0.5, outlier_frac=0.2, lens=LENSES[i % 3]) for i in range(4)]
    bank = make_bank(specs, 31)
    dev, st = _run(bank, max_samples=max_samples, use_prior=use_prior)
    assert _path(f"slot tiles {max_samples}", bank, st, max_samples)
    assert tiles(max_samples) == {31: 1, 32: 2, 4096: 129}[max_samples]
    orc = _oracle(bank, max_samples=max_samples, use_prior=use_prior, workers=4)
    tie = check(dev, orc, near_tie_max=0.0, crawl=True)
    inlier_check(dev, orc, bank.key, tie)
    assert (orc.status == 0).all()


def test_table_bound():
    """682 groups of 513 rows at max_samples = 4096: a table of 682 x 16385 x 96 B <= 2^30, the long shape; 683 groups
    exceed it and fall back to 32 lanes.  The groups both calls share agree; a seeded subset of 16 matches the oracle."""
    t0 = time.perf_counter()
    specs = [dict(family="general", k=513, noise_px=0.5, outlier_frac=0.1, lens=LENSES[i % 3]) for i in range(683)]
    bank = make_bank(specs, 41)
    small = make_bank(specs[:682], 41)
    d682, s682 = _run(small, max_samples=4096)
    d683, s683 = _run(bank, max_samples=4096)
    assert _path("table bound 682", small, s682, 4096)
    assert not _path("table bound 683", bank, s683, 4096) and lanes(bank.counts(), 4096) == 32
    assert s682.kernel_launches - s683.kernel_launches == LONG_EXTRA_LAUNCHES
    sub = np.sort(np.random.default_rng(5).choice(682, 16, replace=False))
    orc = _oracle(small, sub, max_samples=4096, workers=4)
    a, b = take(d682, sub), take(d683, sub)
    b.rep_row = a.rep_row  # the two calls shuffle their rows differently
    tie = check(a, orc, near_tie_max=0.0, crawl=True)
    assert (orc.status == 0).all()
    # the same groups in both calls: compare the group outputs (row numbers differ between the two banks)
    same_across_shapes(a, b, tie)
    for g in sub:
        i = small.order[g]
        np.testing.assert_array_equal(d682.inlier[small.rows[i]], d683.inlier[bank.rows[i]])
    print(f"{time.perf_counter() - t0:.1f} s")


@pytest.mark.parametrize("k,max_samples", [(10, 120), (10, 119), (4, 4), (4, 3), (30, 4096)])
def test_sample_table_edges(k, max_samples):
    """C(k, 3) against max_samples: k = 10 at 120 (exhaustive, full) and 119 (hashed), k = 4 at 4 and 3, k = 30 at 4096
    (4060 exhaustive samples); eight groups each, noisy with outliers, in an 8-lane call."""
    specs = [dict(family="general", k=k, noise_px=0.5, outlier_frac=0.15 if k > 4 else 0.0, lens=LENSES[i % 3])
             for i in range(8)]  # fmt: skip
    bank = make_bank(specs, 50 + k + max_samples)
    exhaustive = comb(k, 3) <= max_samples
    for use_prior in (True, False):
        dev, st = _run(bank, max_samples=max_samples, use_prior=use_prior, min_inliers=4)
        _path(f"k {k} max_samples {max_samples} ({'exhaustive' if exhaustive else 'hashed'} samples)", bank, st,
              max_samples)  # fmt: skip
        assert lanes(bank.counts(), max_samples) == 8
        orc = _oracle(bank, max_samples=max_samples, use_prior=use_prior, min_inliers=4)
        # four rows give eight residuals for six parameters: H's condition amplifies last-bit differences in the cov
        tie = check(dev, orc, near_tie_max=0.25, cov_rtol=1e-7 if k == 4 else 1e-8, crawl=True)
        inlier_check(dev, orc, bank.key, tie)
