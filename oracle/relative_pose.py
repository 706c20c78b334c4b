"""CPU oracle of the robust relative pose of every camera pair from 2-D correspondences alone: five-point consensus, then
refinement of the pose on the Sampson distance and its covariance (``cb_relative_pose_robust``, DESIGN.md section 4.11).

TEST INFRASTRUCTURE ONLY — the product (caliscope_b200/) never imports this module.

Cameras in the bundle-adjustment layout (cam_flags, cam_const, the camera section of x; only the intrinsics are read);
observations obs_cam, obs_key, obs_px (raw pixels).  Rows with equal obs_key are one world point.  The coordinates are
``cv2.undistortPoints`` of float32 pixels, rounded to float32; a row whose coordinates are not finite, or a fisheye row
that OpenCV returns as its (-1e6, -1e6) failure sentinel, is unusable.
  0. Correspondences: rows i < j of one key (key-sorted, caller order within a key) from different cameras are one
     correspondence of the pair (a, b), a < b, oriented so that its a-row is camera a's.  A pair's correspondences are
     ordered by key, then (i, j); k of them at positions 0..k-1.  Pairs in ascending (a, b).
  1. k < min_inliers: status 1.
  2. Candidate samples, T = C(k, 5): every 5-subset in lexicographic order when T <= max_samples; else sample
     m = 0..max_samples-1 draws positions splitmix64(m 2^32 + t) mod k, t = 0, 1, ..., keeps the first five distinct
     (sorted) and gives up after 16 draws.
  3. Hypotheses of a sample of five usable correspondences: ``five_point`` (Nister) on the normalised coordinates, up
     to 10 essential matrices; each is ``decompose``d into (R1, t), (R1, -t), (R2, t), (R2, -t), |t| = 1, and the first
     that puts the five points at positive depth in both cameras (``depths``) is the hypothesis.  Slot 10 m + c.
  4. Score (MSAC): sum over all k correspondences of min(e^2, tau^2), e the Sampson distance in undistorted pixels
     (``sampson``) with E = [t]x R; an unusable correspondence or a non-finite e adds tau^2.  The lowest score wins, the
     lowest slot on a tie.
  5. Consensus set: the usable correspondences with e^2 <= tau^2 and positive depths at the winner.  No hypothesis or
     fewer than min_inliers: status 5 (pose, cov, rmse, parallax NaN; n_inliers 0).
  6. Levenberg-Marquardt over q = (r, alpha, beta) on the consensus set: r = rot_log(R), t = normalize(t0 + alpha u1 +
     beta u2) with u1, u2 columns 1 and 2 of the Householder reflector taking t0 to -+e3 (fixed at the start); residual
     the signed Sampson distance; resection's loop (lam0 1e-3, /10 *10, |d| <= xtol (|q| + xtol), max_iter).
  7. Covariance at q* (status 0, 3, 4): the chart re-based at t*, cov5 = pixel_sigma^2 H^-1 over (r, du), returned as
     J cov5 J^T with J = diag(I3, [u1 u2](t*)) (6 x 6 over (r, t), rank 5).
  8. Status, first match wins: 1, 5, 2 (H fails pd at the start or at the solution; pose = the hypothesis, cov NaN), 3
     (max_iter reached), 4 (a consensus correspondence has a non-positive depth at q*), 0.
Outputs per pair: cam_a, cam_b, pose (r, t) with X_b = R X_a + t, cov, rmse_px (Sampson, consensus set), parallax_deg
(mean angle between R x_a and x_b over the consensus set), count, n_inliers, status.
"""
from __future__ import annotations

from dataclasses import dataclass
from itertools import combinations
from math import sqrt

import numpy as np

from oracle.resection_robust import DRAWS, rot_log, splitmix64
from oracle.triangulation_refine import PD_RTOL, REFINE_LAMBDA0
from oracle.triangulation_robust import undistorted_coordinates

STATUS_OK, STATUS_FEW, STATUS_NOT_PD, STATUS_MAX_ITER, STATUS_BEHIND, STATUS_NO_CONSENSUS = range(6)
SLOTS_PER_SAMPLE = 10

# ---- monomial tables of the five-point solver --------------------------------------------------------------------------
# linear (x, y, z, 1); quadratic and cubic monomials in (x, y, z); cubic order Nister's, so that after Gauss-Jordan on
# the first ten columns the rows of x^2 z, x^2, y^2 z, y^2, xyz, xy pair up (x^2 z - z x^2, ...)
LIN = [(1, 0, 0), (0, 1, 0), (0, 0, 1), (0, 0, 0)]
QUAD = [(2, 0, 0), (0, 2, 0), (0, 0, 2), (1, 1, 0), (1, 0, 1), (0, 1, 1), (1, 0, 0), (0, 1, 0), (0, 0, 1), (0, 0, 0)]
CUB = [(3, 0, 0), (0, 3, 0), (2, 1, 0), (1, 2, 0), (2, 0, 1), (2, 0, 0), (0, 2, 1), (0, 2, 0), (1, 1, 1), (1, 1, 0),
       (1, 0, 2), (1, 0, 1), (1, 0, 0), (0, 1, 2), (0, 1, 1), (0, 1, 0), (0, 0, 3), (0, 0, 2), (0, 0, 1), (0, 0, 0)]  # fmt: skip


def _add(a, b):
    return tuple(p + q for p, q in zip(a, b))


LL_Q = [[QUAD.index(_add(LIN[i], LIN[j])) for j in range(4)] for i in range(4)]  # lin x lin -> quad index
QL_C = [[CUB.index(_add(QUAD[i], LIN[j])) for j in range(4)] for i in range(10)]  # quad x lin -> cubic index


def _mul_ll(a, b):
    o = np.zeros(10)
    for i in range(4):
        for j in range(4):
            o[LL_Q[i][j]] += a[i] * b[j]
    return o


def _mul_ql(a, b):
    o = np.zeros(20)
    for i in range(10):
        for j in range(4):
            o[QL_C[i][j]] += a[i] * b[j]
    return o


def constraint_matrix(basis):
    """The 10 x 20 cubic constraints (det E = 0, then 2 E E^T E - tr(E E^T) E = 0 row-major) of E = x X + y Y + z Z + W,
    basis (4, 9) = X, Y, Z, W."""
    Ep = [[basis[:, 3 * i + j] for j in range(3)] for i in range(3)]  # linear polynomial of each entry
    M = np.zeros((10, 20))
    M[0] = (_mul_ql(_mul_ll(Ep[1][1], Ep[2][2]) - _mul_ll(Ep[1][2], Ep[2][1]), Ep[0][0])
            - _mul_ql(_mul_ll(Ep[1][0], Ep[2][2]) - _mul_ll(Ep[1][2], Ep[2][0]), Ep[0][1])
            + _mul_ql(_mul_ll(Ep[1][0], Ep[2][1]) - _mul_ll(Ep[1][1], Ep[2][0]), Ep[0][2]))  # fmt: skip
    EEt = [[sum(_mul_ll(Ep[i][k], Ep[j][k]) for k in range(3)) for j in range(3)] for i in range(3)]
    tr = EEt[0][0] + EEt[1][1] + EEt[2][2]
    for i in range(3):
        for j in range(3):
            M[1 + 3 * i + j] = 2.0 * sum(_mul_ql(EEt[i][k], Ep[k][j]) for k in range(3)) - _mul_ql(tr, Ep[i][j])
    return M


def _gauss_jordan(M, ncols):
    """Gauss-Jordan with partial pivoting on the first ncols columns, in place; False when a pivot is zero."""
    n = M.shape[0]
    for c in range(ncols):
        p = c + int(np.argmax(np.abs(M[c:, c])))
        if not abs(M[p, c]) > 0.0:
            return False
        if p != c:
            M[[c, p]] = M[[p, c]]
        M[c] /= M[c, c]
        for r in range(n):
            if r != c:
                M[r] -= M[r, c] * M[c]
    return True


def null_basis(xa, xb):
    """(4, 9) orthonormal basis of the null space of the 5 x 9 epipolar system x_b^T E x_a = 0 (E row-major): columns
    5..8 of the orthogonal factor of the Householder QR of its transpose; None when a reflector's column is zero."""
    Q = np.stack([xb[:, 0] * xa[:, 0], xb[:, 0] * xa[:, 1], xb[:, 0], xb[:, 1] * xa[:, 0], xb[:, 1] * xa[:, 1],
                  xb[:, 1], xa[:, 0], xa[:, 1], np.ones(5)], axis=0)  # fmt: skip  (9, 5) = M^T
    V = np.zeros((5, 9))
    for k in range(5):
        x = Q[k:, k]
        nx = sqrt(float(x @ x))
        if not nx > 0.0:
            return None
        v = x.copy()
        v[0] += nx if x[0] >= 0 else -nx
        vv = float(v @ v)
        V[k, k:] = v
        Q[k:, k:] -= np.outer(v, (2.0 / vv) * (v @ Q[k:, k:]))
    N = np.zeros((4, 9))
    for f in range(4):
        x = np.zeros(9)
        x[5 + f] = 1.0
        for k in range(4, -1, -1):
            v = V[k]
            x -= v * (2.0 * (v @ x) / (v @ v))
        N[f] = x
    return N


# ---- the degree-10 polynomial and its real roots (Sturm bisection, Newton polish) ------------------------------------
def _pmul(a, b):
    return np.convolve(a, b)  # ascending coefficients


def _psub_shift(a, b):
    """a(z) - z b(z), ascending coefficients."""
    o = np.zeros(max(len(a), len(b) + 1))
    o[: len(a)] += a
    o[1 : len(b) + 1] -= b
    return o


def _pad(a, n):
    o = np.zeros(n)
    o[: len(a)] = a
    return o


def _peval(p, x):
    """Horner, ascending coefficients."""
    v = 0.0
    for c in p[::-1]:
        v = v * x + c
    return v


def hidden_matrix(G):
    """B(z) (3, 3, 5 ascending coefficients) from the reduced constraint matrix G = [I | B] (10 x 20): the rows of
    x^2 z - z x^2, y^2 z - z y^2 and xyz - z xy, as polynomials in z times (x, y, 1)."""
    Bz = np.zeros((3, 3, 5))
    for r, (e, f) in enumerate(((4, 5), (6, 7), (8, 9))):
        a, b = G[e, 10:], G[f, 10:]
        # columns 10..19: xz^2 xz x | yz^2 yz y | z^3 z^2 z 1 -> ascending in z
        Bz[r, 0] = _pad(_psub_shift(a[[12 - 10, 11 - 10, 10 - 10]], b[[12 - 10, 11 - 10, 10 - 10]]), 5)
        Bz[r, 1] = _pad(_psub_shift(a[[15 - 10, 14 - 10, 13 - 10]], b[[15 - 10, 14 - 10, 13 - 10]]), 5)
        Bz[r, 2] = _pad(_psub_shift(a[[19 - 10, 18 - 10, 17 - 10, 16 - 10]], b[[19 - 10, 18 - 10, 17 - 10, 16 - 10]]), 5)
    return Bz


def det_poly(Bz):
    """det B(z), 11 ascending coefficients."""
    k, l, m = Bz
    p = (_pmul(k[0], _pmul(l[1], m[2]) - _pmul(l[2], m[1]))
         - _pmul(k[1], _pmul(l[0], m[2]) - _pmul(l[2], m[0]))
         + _pmul(k[2], _pmul(l[0], m[1]) - _pmul(l[1], m[0])))  # fmt: skip
    return _pad(p, 13)[:11]


def _prem(a, b):
    """Remainder of a / b (ascending, b's leading coefficient non-zero), degree < deg b."""
    a = a.copy()
    db = len(b) - 1
    for d in range(len(a) - 1, db - 1, -1):
        q = a[d] / b[db]
        a[d - db : d + 1] -= q * b
        a[d] = 0.0
    return a[:db]


def _trim(p):
    """Drop zero leading coefficients (keeps a constant)."""
    n = len(p)
    while n > 1 and p[n - 1] == 0.0:
        n -= 1
    return p[:n]


def sturm_chain(p):
    """Sturm sequence p, p', -rem(...), each scaled by a positive factor to max |coefficient| 1 (signs unchanged)."""
    p = _trim(np.asarray(p, np.float64))
    chain = [p / np.abs(p).max()]
    d = np.arange(1, len(p)) * p[1:]
    if len(d) == 0:
        return chain
    chain.append(d / np.abs(d).max())
    while len(chain[-1]) > 1:
        r = _trim(-_prem(chain[-2], chain[-1]))
        s = np.abs(r).max()
        if not s > 0.0:
            break
        chain.append(r / s)
    return chain


def _sign_changes(chain, x):
    n, last = 0, 0.0
    for p in chain:
        v = _peval(p, x)
        if v != 0.0:
            if last != 0.0 and (v < 0.0) != (last < 0.0):
                n += 1
            last = v
    return n


ROOT_STEPS = 200  # bisection steps at most per root


def real_roots(p):
    """Every distinct real root of p (ascending coefficients) in ascending order: Sturm counts bisect [-B, B] (B the
    Cauchy bound) until the r-th root is alone in (lo, hi] with p(lo), p(hi) of opposite signs, then bisection on the
    sign of p to the resolution of doubles (or ROOT_STEPS steps in all), then up to 3 Newton steps, each kept only when
    it does not raise |p|."""
    p = _trim(np.asarray(p, np.float64))
    if len(p) < 2 or not np.isfinite(p).all():
        return []
    bound = 1.0 + float(np.max(np.abs(p[:-1] / p[-1])))
    if not np.isfinite(bound):
        return []
    chain = sturm_chain(p)
    v0 = _sign_changes(chain, -bound)
    n = v0 - _sign_changes(chain, bound)
    dp = np.arange(1, len(p)) * p[1:]
    out = []
    for r in range(n):
        lo, hi, clo, chi = -bound, bound, 0, n  # clo / chi: roots <= lo / hi
        flo, fhi = _peval(p, lo), _peval(p, hi)
        steps = 0
        while steps < ROOT_STEPS and not (chi - clo == 1 and (flo < 0.0) != (fhi < 0.0) and flo != 0.0 and fhi != 0.0):
            mid = 0.5 * (lo + hi)
            cm = v0 - _sign_changes(chain, mid)
            if cm > r:
                hi, chi, fhi = mid, cm, _peval(p, mid)
            else:
                lo, clo, flo = mid, cm, _peval(p, mid)
            steps += 1
        while steps < ROOT_STEPS:
            mid = 0.5 * (lo + hi)
            if not (lo < mid < hi):
                break
            fm = _peval(p, mid)
            if fm == 0.0:
                lo = hi = mid
                break
            if (fm < 0.0) == (flo < 0.0):
                lo, flo = mid, fm
            else:
                hi, fhi = mid, fm
            steps += 1
        z = 0.5 * (lo + hi)
        fz = _peval(p, z)
        for _ in range(3):
            dz = _peval(dp, z)
            if not dz != 0.0:
                break
            zn = z - fz / dz
            fn = _peval(p, zn)
            if not abs(fn) <= abs(fz):
                break
            z, fz = zn, fn
        out.append(z)
    return out


POLISH_STEPS = 3


def cubic_residuals(E):
    """The ten cubic constraints of an essential matrix: det E, then 2 E E^T E - tr(E E^T) E row-major."""
    return np.r_[np.linalg.det(E), (2.0 * E @ E.T @ E - np.trace(E @ E.T) * E).ravel()]


def polish(N, x, y, z):
    """Up to POLISH_STEPS Gauss-Newton steps on (x, y, z) over the ten cubic constraints of E = x N0 + y N1 + z N2 + N3,
    each kept only when it lowers their sum of squares.  B(z)'s null vector loses accuracy where B(z) is nearly rank one;
    the constraints themselves stay well conditioned there."""
    p = np.array([x, y, z], np.float64)
    E = (p[0] * N[0] + p[1] * N[1] + p[2] * N[2] + N[3]).reshape(3, 3)
    f = cubic_residuals(E)
    for _ in range(POLISH_STEPS):
        EEt, EtE = E @ E.T, E.T @ E
        cof = np.stack([np.cross(E[1], E[2]), np.cross(E[2], E[0]), np.cross(E[0], E[1])])
        J = np.empty((10, 3))
        for k in range(3):
            D = N[k].reshape(3, 3)
            J[0, k] = (cof * D).sum()
            dF = 2.0 * (D @ EtE + E @ D.T @ E + EEt @ D) - 2.0 * (D * E).sum() * E - np.trace(EEt) * D
            J[1:, k] = dF.ravel()
        try:
            d = np.linalg.solve(J.T @ J, -(J.T @ f))
        except np.linalg.LinAlgError:
            break
        pn = p + d
        En = (pn[0] * N[0] + pn[1] * N[1] + pn[2] * N[2] + N[3]).reshape(3, 3)
        fn = cubic_residuals(En)
        if not fn @ fn < f @ f:
            break
        p, E, f = pn, En, fn
    return p[0], p[1], p[2]


def five_point(xa, xb):
    """Essential matrices (m, 3, 3) of five correspondences (normalised coordinates (5, 2) each), Nister's solver:
    null space, constraint matrix, Gauss-Jordan, the real roots of det B(z), (x, y) from B(z)'s null vector, then
    ``polish`` of (x, y, z) on the cubic constraints."""
    N = null_basis(np.asarray(xa, np.float64), np.asarray(xb, np.float64))
    if N is None:
        return np.zeros((0, 3, 3))
    G = constraint_matrix(N)
    if not _gauss_jordan(G, 10):
        return np.zeros((0, 3, 3))
    Bz = hidden_matrix(G)
    out = []
    for z in real_roots(det_poly(Bz)):
        B = np.array([[_peval(Bz[i, j], z) for j in range(3)] for i in range(3)])
        cands = [np.cross(B[0], B[1]), np.cross(B[0], B[2]), np.cross(B[1], B[2])]
        v = max(cands, key=lambda c: abs(c[2]))  # the first of equal |v_2|
        if not abs(v[2]) > 0.0:
            continue
        x, y, z = polish(N, v[0] / v[2], v[1] / v[2], z)
        E = (x * N[0] + y * N[1] + z * N[2] + N[3]).reshape(3, 3)
        if np.isfinite(E).all():
            out.append(E)
    return np.array(out).reshape(-1, 3, 3)


# ---- decomposition, depths, Sampson ------------------------------------------------------------------------------------
def skew(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def decompose(E):
    """The four poses of E in order (R1, t), (R1, -t), (R2, t), (R2, -t), |t| = 1, without an SVD: E scaled to
    |E|_F^2 = 2; t the largest cross product of two columns of E, normalised (t^T E = 0); R1,2 = cof(E) -+ [t]x E
    (for E = [t]x R with |t| = 1, cof(E) = t t^T R and [t]x E = (t t^T - I) R)."""
    E = np.asarray(E, np.float64) * (sqrt(2.0) / np.linalg.norm(E))
    c = [np.cross(E[:, 0], E[:, 1]), np.cross(E[:, 0], E[:, 2]), np.cross(E[:, 1], E[:, 2])]
    t = max(c, key=lambda v: float(v @ v))
    t = t / np.linalg.norm(t)
    cof = np.stack([np.cross(E[1], E[2]), np.cross(E[2], E[0]), np.cross(E[0], E[1])])
    tE = skew(t) @ E
    R1, R2 = cof - tE, cof + tE
    return [(R1, t), (R1, -t), (R2, t), (R2, -t)]


def depths(R, t, xa, xb):
    """(lambda_a, lambda_b) (n, 2): least squares of [R x_a, -x_b] (lambda_a, lambda_b)^T = -t, x = (x, y, 1)."""
    xa = np.asarray(xa, np.float64).reshape(-1, 2)
    xb = np.asarray(xb, np.float64).reshape(-1, 2)
    u = np.column_stack([xa, np.ones(len(xa))]) @ np.asarray(R).T
    v = np.column_stack([xb, np.ones(len(xb))])
    uu, vv, uv = (u * u).sum(1), (v * v).sum(1), (u * v).sum(1)
    ut, vt = u @ t, v @ t
    with np.errstate(divide="ignore", invalid="ignore"):
        det = uu * vv - uv * uv
        la = (uv * vt - ut * vv) / det
        lb = (uu * vt - uv * ut) / det
    return np.stack([la, lb], axis=1)


def sampson_parts(E, xa, xb, fa, fb):
    """(x_b^T E x_a, Sampson denominator in pixels^-2) of every correspondence; fa, fb = (fx, fy) of cameras a, b."""
    xa = np.asarray(xa).reshape(-1, 2)
    xb = np.asarray(xb).reshape(-1, 2)
    ha = np.concatenate([xa, np.ones((len(xa), 1), dtype=xa.dtype)], axis=1)
    hb = np.concatenate([xb, np.ones((len(xb), 1), dtype=xb.dtype)], axis=1)
    Ex = ha @ E.T
    Etx = hb @ E
    num = (hb * Ex).sum(1)
    den = Ex[:, 0] ** 2 / fb[0] ** 2 + Ex[:, 1] ** 2 / fb[1] ** 2 + Etx[:, 0] ** 2 / fa[0] ** 2 + Etx[:, 1] ** 2 / fa[1] ** 2
    return num, den


def sampson(E, xa, xb, fa, fb):
    """Squared Sampson distance in undistorted pixels."""
    num, den = sampson_parts(E, xa, xb, fa, fb)
    with np.errstate(divide="ignore", invalid="ignore"):
        return num * num / den


# ---- samples ---------------------------------------------------------------------------------------------------------
def candidate_samples(k: int, max_samples: int) -> list:
    """Positions of every candidate 5-sample of a pair of k correspondences, in order (None: the hashed draw gave up)."""
    T = k * (k - 1) * (k - 2) * (k - 3) * (k - 4) // 120
    if T <= max_samples:
        return list(combinations(range(k), 5))
    out = []
    for m in range(max_samples):
        got: list[int] = []
        for t in range(DRAWS):
            v = splitmix64((m << 32) + t) % k
            if v not in got:
                got.append(v)
                if len(got) == 5:
                    break
        out.append(tuple(sorted(got)) if len(got) == 5 else None)
    return out


def hypothesis(xa, xb):
    """Candidates c = 0..9 of one sample: (R, t) or None, in the solver's order."""
    out = []
    for E in five_point(xa, xb):
        pick = None
        for R, t in decompose(E):
            lam = depths(R, t, xa, xb)
            if (lam > 0).all():
                pick = (R, t)
                break
        out.append(pick)
    return out


# ---- refinement ------------------------------------------------------------------------------------------------------
def rodrigues(r):
    """Rotation matrix of a rotation vector; complex-safe (the complex step differentiates through it)."""
    r = np.asarray(r)
    th2 = r @ r
    K = np.array([[0.0, -r[2], r[1]], [r[2], 0.0, -r[0]], [-r[1], r[0], 0.0]], dtype=r.dtype)
    if abs(th2) < 1e-30:
        return np.eye(3) + K
    th = np.sqrt(th2)
    return np.eye(3) + np.sin(th) / th * K + (1.0 - np.cos(th)) / th2 * (K @ K)


def householder_basis(t0):
    """Columns 1 and 2 (u1, u2) of the reflector H = I - 2 v v^T / v^T v, v = t0 + sign(t0_z) |t0| e3 (sign(0) = +1),
    which takes t0 to -+|t0| e3."""
    t0 = np.asarray(t0, np.float64)
    s = 1.0 if t0[2] >= 0 else -1.0
    v = t0.copy()
    v[2] += s * np.linalg.norm(t0)
    H = np.eye(3) - 2.0 * np.outer(v, v) / (v @ v)
    return H[:, 0], H[:, 1]


def pose_of(q, t0, u1, u2):
    w = t0 + q[3] * u1 + q[4] * u2
    return rodrigues(q[:3]), w / np.sqrt(w @ w)


def residuals(q, t0, u1, u2, xa, xb, fa, fb):
    """Signed Sampson distances (pixels) at q = (r, alpha, beta)."""
    R, t = pose_of(q, t0, u1, u2)
    num, den = sampson_parts(skew_c(t) @ R, xa, xb, fa, fb)
    return num / np.sqrt(den)


def skew_c(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]], dtype=np.asarray(v).dtype)


def jacobian(q, t0, u1, u2, xa, xb, fa, fb):
    """(residuals, d r / d q) by complex step (exact to rounding)."""
    h = 1e-30
    r = residuals(q, t0, u1, u2, xa, xb, fa, fb)
    J = np.empty((len(r), 5))
    for i in range(5):
        qc = q.astype(complex)
        qc[i] += 1j * h
        J[:, i] = residuals(qc, t0, u1, u2, xa.astype(complex), xb.astype(complex), fa, fb).imag / h
    return r, J


def pd(H) -> bool:
    """Every Cholesky pivot of the Jacobi-scaled D^-1/2 H D^-1/2 above PD_RTOL (NaN fails)."""
    n = len(H)
    with np.errstate(divide="ignore", invalid="ignore"):
        s = 1.0 / np.sqrt(np.diag(H))
        A = H * s[:, None] * s[None, :]
        L = np.zeros((n, n))
        for j in range(n):
            d = A[j, j] - L[j, :j] @ L[j, :j]
            if not d > PD_RTOL:
                return False
            L[j, j] = sqrt(d)
            for i in range(j + 1, n):
                L[i, j] = (A[i, j] - L[i, :j] @ L[j, :j]) / L[j, j]
    return True


def _normal_eq(q, args):
    r, J = jacobian(q, *args)
    return float(r @ r), J.T @ J, J.T @ r


def refine(R0, t0, xa, xb, fa, fb, *, max_iter=20, xtol=1e-12):
    """Step 6 and the status of step 8 (2, 3, 4 or 0): (r, t, rmse, status); the hypothesis for status 2."""
    u1, u2 = householder_basis(t0)
    args = (t0, u1, u2, xa, xb, fa, fb)
    q0 = np.concatenate([rot_log(R0), [0.0, 0.0]])
    q = q0.copy()
    cost, H, g = _normal_eq(q, args)
    cost0, n = cost, len(xa)
    if not pd(H):
        return q0[:3], pose_of(q0, t0, u1, u2)[1], sqrt(cost0 / n), STATUS_NOT_PD
    status, lam, it = STATUS_OK, REFINE_LAMBDA0, 0
    while True:
        if it == max_iter:
            status = STATUS_MAX_ITER
            break
        d = np.linalg.solve(H + lam * np.diag(np.diag(H)), -g)
        ct, Ht, gt = _normal_eq(q + d, args)
        it += 1
        conv = np.linalg.norm(d) <= xtol * (np.linalg.norm(q) + xtol)
        if ct < cost:
            q, cost, H, g = q + d, ct, Ht, gt
            lam /= 10.0
        else:
            lam *= 10.0
        if conv:
            break
    if not pd(H):
        return q0[:3], pose_of(q0, t0, u1, u2)[1], sqrt(cost0 / n), STATUS_NOT_PD
    R, t = pose_of(q, t0, u1, u2)
    if status == STATUS_OK and not (depths(R, t, xa, xb) > 0).all():
        status = STATUS_BEHIND
    return q[:3], t, sqrt(cost / n), status


def covariance(r, t, xa, xb, fa, fb, pixel_sigma):
    """Step 7 at the pose (r, t): (6 x 6 covariance of (r, t), cov5 over (r, du))."""
    u1, u2 = householder_basis(t)
    q = np.concatenate([r, [0.0, 0.0]])
    _, J = jacobian(q, t, u1, u2, xa, xb, fa, fb)
    cov5 = pixel_sigma**2 * np.linalg.inv(J.T @ J)
    Jt = np.zeros((6, 5))
    Jt[:3, :3] = np.eye(3)
    Jt[3:, 3] = u1
    Jt[3:, 4] = u2
    cov = Jt @ cov5 @ Jt.T
    return 0.5 * (cov + cov.T), cov5


def parallax_deg(R, xa, xb):
    ba = np.column_stack([xa, np.ones(len(xa))]) @ np.asarray(R).T
    bb = np.column_stack([xb, np.ones(len(xb))])
    c = (ba * bb).sum(1) / (np.linalg.norm(ba, axis=1) * np.linalg.norm(bb, axis=1))
    return float(np.degrees(np.arccos(np.clip(c, -1.0, 1.0))).mean())


# ---- the whole rule --------------------------------------------------------------------------------------------------
def usable_coordinates(cam_flags, cam_const, cam_x, obs_cam, obs_px):
    """Float32-rounded normalised coordinates, NaN where a row is unusable (not finite, or a fisheye sentinel)."""
    norm = undistorted_coordinates(cam_flags, cam_const, cam_x, obs_cam, obs_px)
    fish = (np.asarray(cam_flags, np.int32)[np.asarray(obs_cam)] & 2) != 0
    bad = ~np.isfinite(norm).all(axis=1) | (fish & (norm[:, 0] == -1e6) & (norm[:, 1] == -1e6))
    norm[bad] = np.nan
    return norm


def correspondences(obs_cam, obs_key):
    """Step 0: {(a, b): (rows_a, rows_b)} in ascending (a, b)."""
    obs_cam = np.asarray(obs_cam, np.int64)
    order = np.argsort(np.asarray(obs_key, np.int64), kind="stable")
    keys = np.asarray(obs_key, np.int64)[order]
    bounds = np.flatnonzero(np.r_[True, keys[1:] != keys[:-1], True])
    pairs: dict = {}
    for g in range(len(bounds) - 1):
        rows = order[bounds[g] : bounds[g + 1]]
        for i in range(len(rows)):
            for j in range(i + 1, len(rows)):
                ra, rb = int(rows[i]), int(rows[j])
                ca, cb = int(obs_cam[ra]), int(obs_cam[rb])
                if ca == cb:
                    continue
                if ca > cb:
                    ca, cb, ra, rb = cb, ca, rb, ra
                pairs.setdefault((ca, cb), ([], []))
                pairs[(ca, cb)][0].append(ra)
                pairs[(ca, cb)][1].append(rb)
    return {p: (np.array(v[0]), np.array(v[1])) for p, v in sorted(pairs.items())}


def focal_lengths(cam_flags, cam_const, cam_x):
    """(n_cams, 2) fx, fy of every camera (s fx0, s fy0)."""
    flags = np.asarray(cam_flags, np.int32).ravel()
    const = np.asarray(cam_const, np.float64).reshape(-1, 9)
    cam_x = np.asarray(cam_x, np.float64)
    out, o = np.empty((len(flags), 2)), 0
    for c, f in enumerate(flags):
        s = cam_x[o + 6] if f & 1 else 1.0
        o += 9 if f & 1 else 6
        out[c] = s * const[c, 0], s * const[c, 1]
    return out


@dataclass
class RelPoseResult:
    cam_a: np.ndarray
    cam_b: np.ndarray
    pose: np.ndarray  # (P, 6)
    cov: np.ndarray  # (P, 6, 6)
    cov5: np.ndarray  # (P, 5, 5) in the chart at t*
    rmse_px: np.ndarray
    parallax_deg: np.ndarray
    count: np.ndarray
    n_inliers: np.ndarray
    status: np.ndarray
    inlier: list  # per pair, bool over its correspondences
    best: np.ndarray  # lowest score (+inf: no hypothesis)
    second: np.ndarray  # second-lowest score among the other slots (+inf: none)


def relative_poses_robust(cam_flags, cam_const, cam_x, obs_cam, obs_key, obs_px, *, threshold_px, min_inliers=15,
                          max_samples=64, pixel_sigma=1.0, max_iter=20, xtol=1e-12) -> RelPoseResult:  # fmt: skip
    """Steps 0-8 for every pair."""
    norm = usable_coordinates(cam_flags, cam_const, cam_x, obs_cam, obs_px)
    foc = focal_lengths(cam_flags, cam_const, cam_x)
    tau2 = threshold_px * threshold_px
    pairs = correspondences(obs_cam, obs_key)
    P = len(pairs)
    nan = np.nan
    res = RelPoseResult(cam_a=np.zeros(P, np.int32), cam_b=np.zeros(P, np.int32), pose=np.full((P, 6), nan),
                        cov=np.full((P, 6, 6), nan), cov5=np.full((P, 5, 5), nan), rmse_px=np.full(P, nan),
                        parallax_deg=np.full(P, nan), count=np.zeros(P, np.int32), n_inliers=np.zeros(P, np.int32),
                        status=np.zeros(P, np.int32), inlier=[], best=np.full(P, np.inf),
                        second=np.full(P, np.inf))  # fmt: skip
    for p, ((a, b), (ra, rb)) in enumerate(pairs.items()):
        res.cam_a[p], res.cam_b[p] = a, b
        k = len(ra)
        res.count[p] = k
        xa, xb = norm[ra], norm[rb]
        usable = np.isfinite(xa).all(1) & np.isfinite(xb).all(1)
        res.inlier.append(np.zeros(k, bool))
        if k < min_inliers:
            res.status[p] = STATUS_FEW
            continue
        slots, Rs, ts = [], [], []
        for m, smp in enumerate(candidate_samples(k, max_samples)):
            if smp is None or not usable[list(smp)].all():
                continue
            s = list(smp)
            for c, h in enumerate(hypothesis(xa[s], xb[s])):
                if h is not None:
                    slots.append(SLOTS_PER_SAMPLE * m + c)
                    Rs.append(h[0])
                    ts.append(h[1])
        if not slots:
            res.status[p] = STATUS_NO_CONSENSUS
            continue
        scores, inls = [], []
        for R, t in zip(Rs, ts):
            e2 = sampson(skew(t) @ R, xa, xb, foc[a], foc[b])
            with np.errstate(invalid="ignore"):
                ok = usable & (e2 <= tau2)
            scores.append(float(np.where(ok, e2, tau2).sum()))
            inls.append(ok)
        scores, slots = np.array(scores), np.array(slots)
        srt = np.lexsort((slots, scores))
        w = srt[0]
        res.best[p] = scores[w]
        if len(srt) > 1:
            res.second[p] = scores[srt[1]]
        with np.errstate(invalid="ignore"):
            cons = inls[w] & (depths(Rs[w], ts[w], xa, xb) > 0).all(1)
        if cons.sum() < min_inliers:
            res.status[p] = STATUS_NO_CONSENSUS
            continue
        res.inlier[p] = cons
        res.n_inliers[p] = int(cons.sum())
        ca, cb = xa[cons], xb[cons]
        r, t, rmse, st = refine(Rs[w], ts[w], ca, cb, foc[a], foc[b], max_iter=max_iter, xtol=xtol)
        res.pose[p] = np.concatenate([r, t])
        res.rmse_px[p], res.status[p] = rmse, st
        res.parallax_deg[p] = parallax_deg(rodrigues(res.pose[p, :3]), ca, cb)
        if st != STATUS_NOT_PD:
            res.cov[p], res.cov5[p] = covariance(res.pose[p, :3], t, ca, cb, foc[a], foc[b], pixel_sigma)
    return res
