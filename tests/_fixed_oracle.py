"""NumPy statement of fixed camera parameters and fixed points (DESIGN.md section 4.12), the checker of
``cb_ba_problem_create_fixed`` (test infrastructure).  It builds on ``oracle/`` without changing it: a solve with fixed
parameters is the solve of the same problem over the free parameters alone, the fixed values constants taken from x0.

  solve_scipy_fixed   scipy's least_squares on the free subvector (the reference the engine is held to)
  lm_solve_dense      ``oracle.lm_schur.lm_solve_dense``'s iteration over the free subvector
  linearize           ``oracle.lm_schur.linearize`` with the fixed Jacobian columns zero
  schur_system        ``oracle.lm_schur.schur_system`` with the engine's masks
  dense_covariance    ``oracle.covariance.dense_covariance`` with fixed points as constants
"""
from __future__ import annotations

import numpy as np

from oracle import ba_oracle as O
from oracle import covariance as OC
from oracle import lm_schur as LS


def free_slots(free: np.ndarray, rig: O.Rig, P: int) -> tuple[np.ndarray, np.ndarray]:
    """A boolean mask over x -> (n_cams * P camera slots at stride P, padding slots False; n_pts points).  A point is free
    when its three coordinates are."""
    c, p = LS.split_x(np.asarray(free, np.float64), rig, P)
    return c.reshape(-1) > 0, p.min(axis=1) > 0


def solve_scipy_fixed(rig: O.Rig, x0: np.ndarray, free: np.ndarray, **kw):
    """``oracle.ba_oracle.solve_scipy`` over the free parameters alone: least_squares(method='trf', x_scale='jac') on
    x0[free], the fixed entries of x0 spliced back in for every residual and Jacobian evaluation; the Jacobian is
    ``ba_oracle.jacobian`` with the fixed columns deleted, the bounds those of the free entries.  ``free``: boolean over x.
    Returns scipy's result with ``x`` the whole parameter vector (fixed entries copied from x0)."""
    from scipy.optimize import least_squares

    x0 = np.asarray(x0, dtype=np.float64)
    cols = np.nonzero(np.asarray(free, bool))[0]

    def full(z):
        x = x0.copy()
        x[cols] = z
        return x

    lo, hi = rig.bounds()
    opts = dict(ftol=1e-8, xtol=1e-8, gtol=1e-8, max_nfev=None, loss="linear", f_scale=1.0, verbose=0)
    opts.update(kw)
    res = least_squares(lambda z: O.residuals(full(z), rig), x0[cols], jac=lambda z: O.jacobian(full(z), rig)[:, cols],
                        x_scale="jac", method="trf", bounds=(lo[cols], hi[cols]), **opts)  # fmt: skip
    res.x = full(res.x)
    return res


def lm_solve_dense(rig: O.Rig, x0: np.ndarray, free: np.ndarray, *, ftol: float = 1e-8, xtol: float = 1e-8,
                   gtol: float = 1e-8, max_nfev: int | None = None, loss: str = "linear", f_scale: float = 1.0,
                   lam0: float = 1e-4):  # fmt: skip
    """``oracle.lm_schur.lm_solve_dense``'s damped Gauss-Newton iteration on the full dense normal equations, over the
    free parameters alone: the step, the bounds, the gradient norm, |x| and the predicted reduction are those of the free
    subvector, and the fixed entries keep their values in x0.  With every parameter free it is that function, step for
    step."""
    x = np.asarray(x0, dtype=np.float64).copy()
    n = len(x)
    fi = np.nonzero(np.asarray(free, bool))[0]
    lo, hi = rig.bounds()
    if max_nfev is None:
        max_nfev = 100 * n

    def lin(xx):
        f = O.residuals(xx, rig)
        J = O.jacobian(xx, rig).toarray()
        cost = O.robust_cost(f, loss, f_scale)
        js, fs = O.robust_row_scales(f, loss, f_scale)
        Js = J * js[:, None]
        return cost, Js.T @ Js, Js.T @ fs

    cost, H, g = lin(x)
    nfev = njev = 1
    lam, nu = lam0, 2.0
    D = np.zeros(n)
    status, nit = 0, 0
    while True:
        D = np.maximum(D, np.diag(H))
        De = np.where(D > 0, D, 1.0)
        if np.abs(g[fi]).max() < gtol:
            status = 1
            break
        if nfev >= max_nfev:
            break
        nit += 1
        while True:
            d = np.zeros(n)
            d[fi] = np.linalg.solve((H + lam * np.diag(De))[np.ix_(fi, fi)], -g[fi])
            xn = x.copy()
            xn[fi] = np.clip(x[fi] + d[fi], lo[fi], hi[fi])
            de = xn - x
            pred = 0.5 * np.sum(de * (lam * De * de - g))
            fn = O.residuals(xn, rig)
            nfev += 1
            cn = O.robust_cost(fn, loss, f_scale) if np.all(np.isfinite(fn)) else np.inf
            actual = cost - cn
            ratio = actual / pred if pred > 0 else -1.0
            ft = actual < ftol * cost and ratio > 0.25
            xt = np.linalg.norm(de) < xtol * (xtol + np.linalg.norm(x[fi]))
            term = 4 if (ft and xt) else 2 if ft else 3 if xt else 0
            if actual > 0:
                lam = max(lam * max(1.0 / 3.0, 1 - (2 * ratio - 1) ** 3), 1e-15)
                nu = 2.0
                break
            lam = min(lam * nu, 1e12)
            nu *= 2
            if term or nfev >= max_nfev:
                break
        if actual > 0:
            x = xn
            if term:
                cost = cn
                status = term
                break
            cost, H, g = lin(x)
            njev += 1
        if term:
            status = term
            break
    return dict(x=x, cost=cost, status=status, nfev=nfev, njev=njev, nit=nit)


def linearize(x: np.ndarray, rig: O.Rig, free: np.ndarray, loss: str = "linear", f_scale: float = 1.0):
    """``oracle.lm_schur.linearize`` of the free parameters: the fixed Jacobian columns are zero (a fixed parameter is a
    constant of the problem), so U, g_c, V, g_p hold nothing of them."""
    P = LS.cam_stride(rig)
    lin = LS.linearize(x, rig, loss, f_scale)
    fc, fp = free_slots(free, rig, P)
    Jc = lin.Jc * fc.reshape(rig.n_cams, P)[rig.obs_cam][:, None, :]
    Jp = lin.Jp * fp[rig.obs_pt][:, None, None]
    rs = np.asarray(O.robust_row_scales(lin.f, loss, f_scale)[1]).reshape(-1, 2)
    U = np.zeros_like(lin.U)
    gc = np.zeros_like(lin.gc)
    V = np.zeros_like(lin.V)
    gp = np.zeros_like(lin.gp)
    np.add.at(U, rig.obs_cam, np.einsum("nki,nkj->nij", Jc, Jc))
    np.add.at(gc, rig.obs_cam, np.einsum("nki,nk->ni", Jc, rs))
    np.add.at(V, rig.obs_pt, np.einsum("nki,nkj->nij", Jp, Jp))
    np.add.at(gp, rig.obs_pt, np.einsum("nki,nk->ni", Jp, rs))
    return LS.Linearization(lin.cost, lin.f, U, gc, V, gp, Jc, Jp)


def schur_system(lin, rig: O.Rig, lam: float, Dc2: np.ndarray, Dp2: np.ndarray, fixed_slots: np.ndarray,
                 fixed_pts: np.ndarray):  # fmt: skip
    """The engine's masked reduced system: ``oracle.lm_schur.schur_system`` with Einv = 0 for the fixed points (no Schur
    term, no step), then unit rows and columns of S before the damping for the fixed camera slots (so 1 + lam Dc2 on the
    diagonal) and zero b.  ``fixed_slots``: boolean over the n_cams * P stride-P slots; ``fixed_pts``: boolean over
    points."""
    fp = np.asarray(fixed_pts, bool)
    # a fixed point's W = Jc^T Jp is left out (its Jp rows zero here; U, g_c keep its observations): no Schur term
    Jp = lin.Jp * (~fp)[rig.obs_pt][:, None, None]
    S, b, Einv, Wd = LS.schur_system(LS.Linearization(lin.cost, lin.f, lin.U, lin.gc, lin.V, lin.gp, lin.Jc, Jp), rig,
                                     lam, Dc2, Dp2)  # fmt: skip
    Einv[fp] = 0.0  # and no step
    f = np.nonzero(np.asarray(fixed_slots, bool))[0]
    S[f, :] = 0.0
    S[:, f] = 0.0
    S[f, f] = 1.0 + lam * np.asarray(Dc2).reshape(-1)[f]
    b[f] = 0.0
    return S, b, Einv, Wd


def dense_covariance(x, rig: O.Rig, fixed, fixed_points, loss: str = "linear", f_scale: float = 1.0,
                     variance_factor=None):  # fmt: skip
    """``oracle.covariance.dense_covariance`` with known points: the columns of ``fixed_points`` are deleted from J like
    those of the fixed camera parameters; their blocks are zero, their rank -2, and each counts 3 parameters fewer in the
    rank behind dof."""
    cost, H = OC._system(x, rig, loss, f_scale)
    ncp = rig.n_camera_params
    fix, masked = OC._masks(rig, fixed)
    fp = np.zeros(rig.n_pts, bool)
    fp[np.asarray(fixed_points, dtype=np.int64)] = True
    free = np.concatenate([~(fix | masked), np.repeat(~fp, 3)])
    comp = OC.constrained_points(rig)
    ranks = np.full(rig.n_pts, -1)
    ranks[fp] = -2
    defl = np.zeros_like(H)
    for j in np.nonzero(~comp & ~fp)[0]:
        sl = slice(ncp + 3 * j, ncp + 3 * j + 3)
        _, ranks[j], N = OC._point_pinv(H[sl, sl])
        defl[sl, sl] = N @ N.T
    idx = np.nonzero(free)[0]
    Hf = (H + defl)[np.ix_(idx, idx)]
    Sig = np.zeros_like(H)
    Sig[np.ix_(idx, idx)] = np.linalg.inv(Hf) - defl[np.ix_(idx, idx)]
    pts = np.stack([Sig[ncp + 3 * j : ncp + 3 * j + 3, ncp + 3 * j : ncp + 3 * j + 3] for j in range(rig.n_pts)])
    # laid out like oracle.covariance._finish, with the fixed points' 3 parameters each out of the rank
    m = 2 * rig.n_obs + rig.n_constraints
    null = int(sum(3 - r for r in ranks if r >= 0))
    dof = m - (rig.n_params - int(fix.sum()) - int(masked.sum()) - null - 3 * int(fp.sum()))
    s2 = variance_factor if variance_factor is not None and variance_factor > 0 else (2.0 * cost / dof if dof > 0 else np.nan)
    cam = s2 * Sig[:ncp, :ncp]
    cam[fix, :] = 0.0
    cam[:, fix] = 0.0
    cam[masked, :] = np.nan
    cam[:, masked] = np.nan
    pts = s2 * pts
    pts[ranks != 3] = np.nan
    pts[fp] = 0.0
    return dict(cameras=cam, points=pts, point_rank=ranks.astype(np.int32), variance_factor=s2, dof=dof)
