"""The relative-pose oracle (oracle/relative_pose.py) against OpenCV and against the truth of seeded scenes."""
from __future__ import annotations

import cv2
import numpy as np
import pytest

from oracle import relative_pose as O
from tests._relpose_cases import relative_truth, scene


def _config(rng):
    X = rng.uniform(-1, 1, (5, 3)) + [0, 0, 5]
    R = cv2.Rodrigues(rng.normal(0, 0.2, 3))[0]
    t = rng.normal(0, 1, 3)
    Xb = X @ R.T + t
    return X[:, :2] / X[:, 2:], Xb[:, :2] / Xb[:, 2:], R, t


def _canon(E):
    E = E / np.linalg.norm(E)
    return E * np.sign(E.flat[np.argmax(np.abs(E))])


def _constraint_residual(E, xa, xb):
    """Largest epipolar and cubic-constraint residual of E scaled to |E|_F = 1."""
    E = E / np.linalg.norm(E)
    ha, hb = np.c_[xa, np.ones(len(xa))], np.c_[xb, np.ones(len(xb))]
    return max(np.abs(np.einsum("ni,ij,nj->n", hb, E, ha)).max(), np.abs(O.cubic_residuals(E)).max())


def test_five_point_matches_opencv():
    """Same number of real solutions as cv2.findEssentialMat and the same E up to scale and sign within 1e-7, except in
    configurations whose polynomial has two real roots within 1e-6 of each other (at most 1 %).  Where an E differs, the
    oracle's meets the epipolar and cubic constraints to 1e-12 and OpenCV's does not: OpenCV's is the inaccurate one."""
    rng = np.random.default_rng(1)
    near, differ = 0, 0
    for _ in range(1000):
        xa, xb, _, _ = _config(rng)
        mine = O.five_point(xa, xb)
        cv = cv2.findEssentialMat(xa, xb, np.eye(3), method=cv2.LMEDS)[0].reshape(-1, 3, 3)
        N = O.null_basis(xa, xb)
        G = O.constraint_matrix(N)
        O._gauss_jordan(G, 10)
        roots = np.sort(O.real_roots(O.det_poly(O.hidden_matrix(G))))
        if len(roots) > 1 and np.diff(roots).min() < 1e-6:
            near += 1
            continue
        assert len(mine) == len(cv)
        for a in mine:
            assert _constraint_residual(a, xa, xb) <= 1e-12
        ours = [a for a in mine if min(np.abs(_canon(a) - _canon(b)).max() for b in cv) > 1e-7]
        theirs = [b for b in cv if min(np.abs(_canon(a) - _canon(b)).max() for a in mine) > 1e-7]
        differ += bool(ours)
        for b in theirs:
            assert _constraint_residual(b, xa, xb) > 1e-12
    print(f"near-double roots: {near} of 1000; configurations where OpenCV's E is the inaccurate one: {differ}")
    assert near <= 10


def test_decomposition_and_cheirality_match_opencv():
    rng = np.random.default_rng(2)
    for _ in range(50):
        xa, xb, R, t = _config(rng)
        E = O.skew(t / np.linalg.norm(t)) @ R
        R1, R2, tc = cv2.decomposeEssentialMat(E)
        mine = O.decompose(E)
        for Rm, tm in mine:
            assert min(np.abs(Rm - R1).max(), np.abs(Rm - R2).max()) < 1e-9
            assert min(np.abs(tm - tc.ravel()).max(), np.abs(tm + tc.ravel()).max()) < 1e-9
        Rp, tp = _pick(E, xa, xb)
        _, Rr, tr, _ = cv2.recoverPose(E, xa, xb, np.eye(3))
        assert np.abs(Rp - Rr).max() < 1e-9 and np.abs(tp - tr.ravel()).max() < 1e-9


def _pick(E, xa, xb):
    for R, t in O.decompose(E):
        if (O.depths(R, t, xa, xb) > 0).all():
            return R, t
    return None


def test_sampson_matches_opencv():
    rng = np.random.default_rng(3)
    xa, xb = rng.normal(0, 0.3, (20, 2)), rng.normal(0, 0.3, (20, 2))
    E = O.skew(np.array([0.6, 0.0, 0.8])) @ cv2.Rodrigues(np.array([0.1, -0.2, 0.05]))[0]
    Ka = np.array([[800.0, 0, 640], [0, 790, 360], [0, 0, 1]])
    Kb = np.array([[700.0, 0, 620], [0, 710, 350], [0, 0, 1]])
    F = np.linalg.inv(Kb).T @ E @ np.linalg.inv(Ka)
    pa = xa @ Ka[:2, :2].T + Ka[:2, 2]
    pb = xb @ Kb[:2, :2].T + Kb[:2, 2]
    mine = O.sampson(E, xa, xb, (800.0, 790.0), (700.0, 710.0))
    for i in range(20):
        ref = cv2.sampsonDistance(np.r_[pa[i], 1.0][:, None], np.r_[pb[i], 1.0][:, None], F)
        assert abs(mine[i] - ref) <= 1e-9 * abs(ref)


def test_noise_free_rig_recovers_the_truth():
    flags, const, x, cam, key, px, Rs, ts, _ = scene(4, 40, seed=4)
    res = O.relative_poses_robust(flags, const, x, cam, key, px, threshold_px=1.0, max_samples=16)
    assert len(res.status) == 6 and (res.status == 0).all()
    for p in range(6):
        R, t = relative_truth(Rs, ts, res.cam_a[p], res.cam_b[p])
        Rm = O.rodrigues(res.pose[p, :3])
        assert np.linalg.norm(cv2.Rodrigues(Rm @ R.T)[0]) < 1e-6
        assert np.abs(res.pose[p, 3:] - t).max() < 1e-6


def test_noisy_rig_rejects_outliers_and_reaches_the_optimum():
    from scipy.optimize import least_squares

    flags, const, x, cam, key, px, Rs, ts, out = scene(4, 60, seed=5, noise_px=0.5, outlier_frac=0.05)
    res = O.relative_poses_robust(flags, const, x, cam, key, px, threshold_px=3.0, max_samples=32)
    pairs = O.correspondences(cam, key)
    norm = O.usable_coordinates(flags, const, x, cam, px)
    foc = O.focal_lengths(flags, const, x)
    for p, ((a, b), (ra, rb)) in enumerate(pairs.items()):
        assert res.status[p] == 0
        cons = res.inlier[p]
        assert not (out[ra] | out[rb])[cons].any()
        xa, xb = norm[ra][cons], norm[rb][cons]
        t = res.pose[p, 3:]
        u1, u2 = O.householder_basis(t)
        ls = least_squares(lambda q: O.residuals(q, t, u1, u2, xa, xb, foc[a], foc[b]),
                           np.r_[res.pose[p, :3], 0.0, 0.0], method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15)
        assert np.abs(ls.x[:3] - res.pose[p, :3]).max() < 1e-8
        assert np.abs(ls.x[3:]).max() < 1e-8


def test_covariance_is_calibrated():
    """Over at least 200 seeded pairs with 1 px noise, the mean of d^T cov5^-1 d is within 4 standard errors of 5, where
    d = estimate - truth in the chart at the estimate: (r_est - r_true, u1 . (t_est - t_true), u2 . (t_est - t_true))."""
    vals = []
    for seed in range(70):
        flags, const, x, cam, key, px, Rs, ts, _ = scene(3, 40, seed=100 + seed, noise_px=1.0)
        res = O.relative_poses_robust(flags, const, x, cam, key, px, threshold_px=6.0, max_samples=8)
        for p in range(len(res.status)):
            if res.status[p] != 0:
                continue
            R, t = relative_truth(Rs, ts, res.cam_a[p], res.cam_b[p])
            te = res.pose[p, 3:]
            u1, u2 = O.householder_basis(te)
            d = np.r_[res.pose[p, :3] - cv2.Rodrigues(R)[0].ravel(), u1 @ (te - t), u2 @ (te - t)]
            vals.append(d @ np.linalg.solve(res.cov5[p], d))
    vals = np.array(vals)
    assert len(vals) >= 200
    se = vals.std() / np.sqrt(len(vals))
    print(f"{len(vals)} pairs: mean {vals.mean():.3f}, standard error {se:.3f}")
    assert abs(vals.mean() - 5.0) <= 4 * se


@pytest.mark.parametrize("k", [5, 6, 9, 20, 200])
def test_candidate_samples_are_sorted_distinct(k):
    for s in O.candidate_samples(k, 64):
        if s is not None:
            assert list(s) == sorted(set(s)) and len(s) == 5 and max(s) < k


def _split_bank():
    from tests._relpose_cases import pair_bank

    fams = ["general", "sideways", "forward", "planar", "tiny", "rotation", "facing-y", "facing-oblique", "wild",
            "general", "sideways", "general"]  # fmt: skip
    lenses = ["pinhole", "fisheye", "sentinel", "free"]
    specs = [dict(family=f, k=9 + 3 * i, noise_px=0.5 if i % 3 else 0.0, lens=lenses[i % 4], nan_rows=i % 2,
                  outlier_frac=0.4 if f == "wild" else 0.0, sentinel=2) for i, f in enumerate(fams)]  # fmt: skip
    return pair_bank(specs, seed=21)


def test_bank_split_matches_the_whole_call():
    """The oracle of every bank pair alone, cameras renumbered (0, 1) and run in a process pool, equals the oracle of
    the whole call field for field: the pairs of a bank share no correspondence and their order does not matter."""
    from tests._relpose_cases import oracle_bank

    bank = _split_bank()
    kw = dict(threshold_px=3.0, min_inliers=6, max_samples=8)
    whole = O.relative_poses_robust(*bank.args(), **kw)
    split = oracle_bank(bank, **kw)
    assert len(whole.status) == len(bank.family) == 12
    for f in ("cam_a", "cam_b", "pose", "cov", "cov5", "rmse_px", "parallax_deg", "count", "n_inliers", "status", "best",
              "second"):  # fmt: skip
        assert np.array_equal(getattr(whole, f), getattr(split, f), equal_nan=True), f
    assert all(np.array_equal(a, b) for a, b in zip(whole.inlier, split.inlier, strict=True))
    assert len(set(whole.status.tolist())) >= 2


def test_bank_families_reach_their_edges():
    """facing-y / facing-oblique: the five-point hypothesis nearest the truth takes rot_log's s < 1e-5 branch (rotation
    at pi); sideways: the oracle's t_z takes both signs across seeds (the Householder chart's reflection flips);
    sentinel: the planted rows are OpenCV's (-1e6, -1e6) before usable_coordinates and unusable (NaN) after it."""
    from oracle.triangulation_robust import undistorted_coordinates
    from tests._relpose_cases import pair_bank

    for fam in ("facing-y", "facing-oblique"):
        for seed in range(3):
            bank = pair_bank([dict(family=fam, k=12)], seed=seed)
            flags, const, x, cam, key, px = bank.args()
            norm = O.usable_coordinates(flags, const, x, cam, px)
            (ra, rb), = O.correspondences(cam, key).values()
            hyps = [h for h in O.hypothesis(norm[ra[:5]], norm[rb[:5]]) if h is not None]
            R = min(hyps, key=lambda h: np.abs(h[0] - bank.R[0]).max())[0]
            assert np.abs(R - bank.R[0]).max() < 1e-5  # float32 coordinates, five points
            s = np.linalg.norm([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]]) / 2
            assert s < 1e-5 and np.trace(R) < -0.99, (fam, seed, s)
    tz = []
    for seed in range(6):
        bank = pair_bank([dict(family="sideways", k=30, noise_px=0.5)], seed=seed)
        assert bank.t[0, 2] == 0.0
        res = O.relative_poses_robust(*bank.args(), threshold_px=3.0, min_inliers=6, max_samples=8)
        tz.append(res.pose[0, 5])
    assert min(tz) < 0 < max(tz), tz
    bank = pair_bank([dict(family="general", k=40, lens="sentinel", sentinel=5)], seed=4)
    flags, const, x, cam, key, px = bank.args()
    raw = undistorted_coordinates(flags, const, x, cam, px)
    sent = (raw == -1e6).all(axis=1)
    assert sent.sum() == 5 and (cam[sent] == 1).all() and (flags[1] & 2)
    assert np.isnan(O.usable_coordinates(flags, const, x, cam, px)[sent]).all()
