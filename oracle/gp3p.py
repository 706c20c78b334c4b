"""CPU oracle of the generalized three-point pose (gP3P): the body poses that put three model points on three rays from
different cameras (``rig_gp3p`` in cb_rigid.cuh, DESIGN.md section 4.14).

TEST INFRASTRUCTURE ONLY — the product (caliscope_b200/) never imports this module.

Row i has the camera centre c_i, the unit ray d_i and the model point M_i, D_ij = |M_i - M_j|; the world points are
X_i = c_i + lambda_i d_i.
  0. None when the model triangle is degenerate (``rigid_pose_robust.horn``'s test) or the rays are parallel:
     det(A) <= GP3P_PARALLEL, A = sum (I - d_i d_i^T).
  1. Normalise: X^ = A^-1 b, b = sum (I - d_i d_i^T) c_i, the least-squares point of the three lines;
     lambda^_i = d_i . (X^ - c_i); c'_i = (c_i + lambda^_i d_i - X^) / s, s the longest model side; the unknowns
     u_i = (lambda_i - lambda^_i) / s and D_ij -> D_ij / s.
  2. Eliminate: for j = 2, 3, with w = c'_1 - c'_j, u_j = p_j +- sqrt(Delta_j), p_j = (d_1 . d_j) u_1 + d_j . w,
     Delta_j = p_j^2 - (u_1^2 + 2 u_1 d_1 . w + |w|^2 - D_1j^2).  The (2, 3) equation with w = c'_2 - c'_3 is
     P0 + P2 s_2 + P3 s_3 + P23 s_2 s_3 = 0, s_j = +-sqrt(Delta_j), a_23 = d_2 . d_3:
       P0 = p_2^2 + Delta_2 + p_3^2 + Delta_3 - 2 a_23 p_2 p_3 + 2 p_2 d_2 . w - 2 p_3 d_3 . w + |w|^2 - D_23^2,
       P2 = 2 p_2 - 2 a_23 p_3 + 2 d_2 . w,  P3 = 2 p_3 - 2 a_23 p_2 - 2 d_3 . w,  P23 = -2 a_23,
     and the product over the four signs is the octic F(u_1) = Q0^2 - Q1^2 Delta_2 Delta_3,
     Q0 = P0^2 + P23^2 Delta_2 Delta_3 - P2^2 Delta_2 - P3^2 Delta_3, Q1 = 2 (P0 P23 - P2 P3).
  3. The real roots of F with |u_1| <= GP3P_UMAX, ascending (here ``np.roots``, real when |Im| <= GP3P_IMAG
     max(1, |Re|)).  Per root: Delta_j < -GP3P_CLAMP (1 + p_j^2) for j = 2 or 3 skips it, else Delta_j is clamped at 0;
     of (p_2 + sqrt Delta_2, p_3 + sqrt Delta_3), (+, -), (-, +), (-, -) the one with the least |f_23|,
     f_ij = |c'_i + u_i d_i - c'_j - u_j d_j|^2 - D_ij^2 (the first on a tie); then at most GP3P_NEWTON Newton steps on
     (f_12, f_13, f_23) in (u_1, u_2, u_3), each kept only when it lowers their sum of squares (the first that does not
     ends the polish).  No hypothesis when some lambda_i = lambda^_i + s u_i <= 0 or a value is not finite.
  4. The pose of a root: ``horn`` on (M_i, X_i), X_i = X^ + s (c'_i + u_i d_i) (= c_i + lambda_i d_i); hypothesis c
     counts the roots that give one, in ascending root order.
"""
from __future__ import annotations

import numpy as np

from oracle.rigid_pose_robust import DEGENERATE, horn

GP3P_PARALLEL = 1e-12  # det(sum (I - d d^T)) at or below this: the rays are parallel
GP3P_CLAMP = 1e-8  # Delta_j >= -GP3P_CLAMP (1 + p_j^2) is clamped to 0, below it the root gives no hypothesis
GP3P_UMAX = 1e9  # roots beyond |u_1| = GP3P_UMAX (GP3P_UMAX model sizes from the lines' meeting point) are not sought
GP3P_NEWTON = 3  # Newton steps of the polish at most
GP3P_IMAG = 1e-6  # the oracle's real-root cut on np.roots: |Im| <= GP3P_IMAG max(1, |Re|)
GP3P_MAX = 8  # hypotheses of one sample at most (slot 1 + 8 m + c)

__all__ = ["GP3P_PARALLEL", "GP3P_CLAMP", "GP3P_UMAX", "GP3P_NEWTON", "GP3P_IMAG", "GP3P_MAX", "gp3p", "octic",
           "degenerate"]  # fmt: skip

P = np.polynomial.polynomial  # coefficients lowest degree first


def degenerate(M) -> bool:
    """``horn``'s test of the model triangle: |(M_1 - M_0) x (M_2 - M_0)| <= 1e-9 |M_1 - M_0| |M_2 - M_0|."""
    M = np.asarray(M, np.float64)
    u, v = M[1] - M[0], M[2] - M[0]
    with np.errstate(invalid="ignore", over="ignore"):
        c = np.cross(u, v)
        return not np.sqrt(c @ c) > DEGENERATE * np.sqrt(u @ u) * np.sqrt(v @ v)


def _normalise(c, d, M):
    """Step 1: (X^, lambda^, c', s, D / s) or None for parallel rays."""
    A = np.zeros((3, 3))
    b = np.zeros(3)
    for i in range(3):
        Pi = np.eye(3) - np.outer(d[i], d[i])
        A += Pi
        b += Pi @ c[i]
    if not np.linalg.det(A) > GP3P_PARALLEL:
        return None
    Xh = np.linalg.solve(A, b)
    lh = np.array([d[i] @ (Xh - c[i]) for i in range(3)])
    D = np.array([[np.linalg.norm(M[i] - M[j]) for j in range(3)] for i in range(3)])
    s = max(D[0, 1], D[0, 2], D[1, 2])
    cp = (c + lh[:, None] * d - Xh) / s
    return Xh, lh, cp, s, D / s


def _eliminate(cp, d, D):
    """Step 2: p_j, Delta_j (j = 2, 3) as polynomials in u_1 and the octic F, lowest degree first."""
    p, dl = [], []
    for j in (1, 2):
        w = cp[0] - cp[j]
        pj = np.array([d[j] @ w, d[0] @ d[j]])
        p.append(pj)
        dl.append(P.polysub(P.polymul(pj, pj), [w @ w - D[0, j] ** 2, 2.0 * (d[0] @ w), 1.0]))
    w = cp[1] - cp[2]
    a23 = d[1] @ d[2]
    p2, p3 = p
    P0 = P.polyadd(P.polyadd(P.polymul(p2, p2), dl[0]), P.polyadd(P.polymul(p3, p3), dl[1]))
    P0 = P.polysub(P0, 2.0 * a23 * P.polymul(p2, p3))
    P0 = P.polyadd(P0, P.polyadd(2.0 * (d[1] @ w) * p2, -2.0 * (d[2] @ w) * p3))
    P0 = P.polyadd(P0, [w @ w - D[1, 2] ** 2])
    P2 = P.polyadd(P.polysub(2.0 * p2, 2.0 * a23 * p3), [2.0 * (d[1] @ w)])
    P3 = P.polysub(P.polysub(2.0 * p3, 2.0 * a23 * p2), [2.0 * (d[2] @ w)])
    P23 = -2.0 * a23
    d23 = P.polymul(dl[0], dl[1])
    Q0 = P.polyadd(P.polymul(P0, P0), P23 * P23 * d23)
    Q0 = P.polysub(Q0, P.polyadd(P.polymul(P.polymul(P2, P2), dl[0]), P.polymul(P.polymul(P3, P3), dl[1])))
    Q1 = 2.0 * P.polysub(P23 * P0, P.polymul(P2, P3))
    F = P.polysub(P.polymul(Q0, Q0), P.polymul(P.polymul(Q1, Q1), d23))
    out = np.zeros(9)
    out[: len(F)] = F
    return p, dl, out


def octic(c, d, M) -> np.ndarray | None:
    """The coefficients of F (9, lowest degree first) of rows (c, d, M), None when step 0 gives no hypothesis."""
    c, d, M = (np.asarray(a, np.float64).reshape(3, 3) for a in (c, d, M))
    if degenerate(M):
        return None
    nz = _normalise(c, d, M)
    if nz is None:
        return None
    return _eliminate(nz[2], d, nz[4])[2]


def _residuals(cp, d, D, u):
    Y = cp + u[:, None] * d
    f = np.array([(Y[i] - Y[j]) @ (Y[i] - Y[j]) - D[i, j] ** 2 for i, j in ((0, 1), (0, 2), (1, 2))])
    return f, Y


def _polish(cp, d, D, u):
    f, Y = _residuals(cp, d, D, u)
    ss = f @ f
    for _ in range(GP3P_NEWTON):
        J = np.zeros((3, 3))
        for r, (i, j) in enumerate(((0, 1), (0, 2), (1, 2))):
            e = Y[i] - Y[j]
            J[r, i] = 2.0 * (e @ d[i])
            J[r, j] = -2.0 * (e @ d[j])
        with np.errstate(all="ignore"):
            try:
                un = u - np.linalg.solve(J, f)
            except np.linalg.LinAlgError:
                break
            fn, Yn = _residuals(cp, d, D, un)
            sn = fn @ fn
        if not sn < ss:
            break
        u, f, Y, ss = un, fn, Yn, sn
    return u


def gp3p(c, d, M) -> list:
    """Steps 0-4 on camera centres c (3, 3), unit rays d (3, 3) and model points M (3, 3): the hypotheses (R, t) with
    R M_i + t on ray i, in slot order (at most GP3P_MAX)."""
    c, d, M = (np.asarray(a, np.float64).reshape(3, 3) for a in (c, d, M))
    if degenerate(M):
        return []
    nz = _normalise(c, d, M)
    if nz is None:
        return []
    Xh, lh, cp, s, D = nz
    p, dl, F = _eliminate(cp, d, D)
    nzc = np.flatnonzero(F)
    if len(nzc) == 0 or nzc[-1] == 0:
        return []
    r = np.roots(F[: nzc[-1] + 1][::-1])
    r = np.sort(r[np.abs(r.imag) <= GP3P_IMAG * np.maximum(1.0, np.abs(r.real))].real)
    r = r[np.abs(r) <= GP3P_UMAX]
    out = []
    for u1 in r:
        pv = [P.polyval(u1, p[0]), P.polyval(u1, p[1])]
        dv = [P.polyval(u1, dl[0]), P.polyval(u1, dl[1])]
        if any(dv[j] < -GP3P_CLAMP * (1.0 + pv[j] * pv[j]) for j in range(2)):
            continue
        sq = [np.sqrt(max(v, 0.0)) for v in dv]
        best, bu = np.inf, None
        for s2, s3 in ((1, 1), (1, -1), (-1, 1), (-1, -1)):
            u = np.array([u1, pv[0] + s2 * sq[0], pv[1] + s3 * sq[1]])
            f = abs(_residuals(cp, d, D, u)[0][2])
            if f < best:
                best, bu = f, u
        if bu is None:
            continue
        u = _polish(cp, d, D, bu)
        lam = lh + s * u
        if not (np.isfinite(lam).all() and (lam > 0).all()):
            continue
        sol = horn(M, Xh + s * (cp + u[:, None] * d))
        if sol is not None:
            out.append(sol)
    return out[:GP3P_MAX]
