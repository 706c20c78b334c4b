"""NumPy statement of held parameters: fixed camera parameters and fixed points (DESIGN.md section 4.12) and Gaussian
priors on cameras and points (section 4.13), the checker of ``cb_ba_problem_create_priors`` (test infrastructure).  It
builds on ``oracle/`` without changing it.  A solve with fixed parameters is the solve of the same problem over the free
parameters alone, the fixed values constants taken from x0; a problem with priors is the least-squares problem whose
residual vector is extended by the rows W (x - mean) of every prior, W^T W = info, which the loss leaves linear.

  Priors              the priors in BAProblem's layout (camera means / information padded to 9)
  free_slots          a free mask over x as the engine's stride-P camera slots and points
  mixed_loss          scipy's callable loss: the named loss on the first rows, rho(z) = z on the prior rows
  solve_scipy         least_squares(method='trf', x_scale='jac') on the (augmented) residuals over the free subvector
  lm_solve_dense      ``oracle.lm_schur.lm_solve_dense``'s iteration over the free subvector
  linearize           ``oracle.lm_schur.linearize`` with the fixed Jacobian columns zero, plus the prior terms
  schur_system        ``oracle.lm_schur.schur_system`` with the engine's masks
  dense_covariance    ``oracle.covariance.dense_covariance`` of the augmented J, fixed points as constants
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np
from scipy import sparse

from oracle import ba_oracle as O
from oracle import covariance as OC
from oracle import lm_schur as LS

EIG_RTOL = 1e-12  # eigenvalues at or below this times the largest are zero (the engine's rank and PSD rule)


@dataclass
class Priors:
    cams: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int64))
    cam_mean: np.ndarray = field(default_factory=lambda: np.zeros((0, 9)))
    cam_info: np.ndarray = field(default_factory=lambda: np.zeros((0, 9, 9)))
    pts: np.ndarray = field(default_factory=lambda: np.zeros(0, np.int64))
    pt_mean: np.ndarray = field(default_factory=lambda: np.zeros((0, 3)))
    pt_info: np.ndarray = field(default_factory=lambda: np.zeros((0, 3, 3)))

    def kwargs(self) -> dict:
        """BAProblem's ``camera_priors`` / ``point_priors``."""
        out = {}
        if len(self.cams):
            out["camera_priors"] = (self.cams, self.cam_mean, self.cam_info)
        if len(self.pts):
            out["point_priors"] = (self.pts, self.pt_mean, self.pt_info)
        return out


def blocks(rig: O.Rig, pr: Priors | None):
    """[(x columns, mean, info)] of every prior, at the prior's own width."""
    if pr is None:
        return []
    out = []
    for k, c in enumerate(pr.cams):
        o, w = int(rig.cam_offsets[c]), int(rig.cam_offsets[c + 1] - rig.cam_offsets[c])
        out.append((np.arange(o, o + w), pr.cam_mean[k, :w], pr.cam_info[k, :w, :w]))
    ncp = rig.n_camera_params
    for k, j in enumerate(pr.pts):
        out.append((np.arange(ncp + 3 * j, ncp + 3 * j + 3), pr.pt_mean[k], pr.pt_info[k]))
    return out


def sqrt_info(L: np.ndarray) -> np.ndarray:
    """W with W^T W = L (L symmetric PSD, possibly singular): its eigen-rows scaled by sqrt(eigenvalue)."""
    w, Q = np.linalg.eigh(0.5 * (L + L.T))
    return np.sqrt(np.maximum(w, 0.0))[:, None] * Q.T


def rank(L: np.ndarray) -> int:
    w = np.linalg.eigvalsh(0.5 * (L + L.T))
    return int((w > EIG_RTOL * w.max()).sum()) if w.max() > 0 else 0


def prior_cost(x: np.ndarray, rig: O.Rig, pr: Priors | None) -> float:
    return sum(0.5 * float((x[c] - m) @ L @ (x[c] - m)) for c, m, L in blocks(rig, pr))


def prior_rank(rig: O.Rig, pr: Priors | None) -> int:
    return sum(rank(L) for _, _, L in blocks(rig, pr))


def info_matrix(rig: O.Rig, pr: Priors | None) -> np.ndarray:
    """The block-diagonal information over the whole x (dense)."""
    Lf = np.zeros((rig.n_params, rig.n_params))
    for c, _, L in blocks(rig, pr):
        Lf[np.ix_(c, c)] += L
    return Lf


def free_slots(free: np.ndarray, rig: O.Rig, P: int) -> tuple[np.ndarray, np.ndarray]:
    """A boolean mask over x -> (n_cams * P camera slots at stride P, padding slots False; n_pts points).  A point is free
    when its three coordinates are."""
    c, p = LS.split_x(np.asarray(free, np.float64), rig, P)
    return c.reshape(-1) > 0, p.min(axis=1) > 0


def mixed_loss(n_first: int, loss: str, f_scale: float):
    """scipy's callable loss over the augmented rows: ``loss`` on the first n_first (reprojection and constraint) rows,
    rho(z) = z on the rest.  scipy hands it z = (f / f_scale)^2 and multiplies rho by f_scale^2 (and rho'' by
    1 / f_scale^2), so a linear row contributes exactly f^2 / 2 to the cost and is left unscaled in J."""

    def rho(z):
        out = np.empty((3, len(z)))
        out[0, :n_first], out[1, :n_first], out[2, :n_first] = O.loss_rho(z[:n_first], loss)
        out[0, n_first:], out[1, n_first:], out[2, n_first:] = z[n_first:], 1.0, 0.0
        return out

    return rho


def solve_scipy(rig: O.Rig, x0: np.ndarray, free=None, priors: Priors | None = None, loss: str = "linear",
                f_scale: float = 1.0, **kw):  # fmt: skip
    """``oracle.ba_oracle.solve_scipy`` over the free entries of x (``free``: boolean over x, None: all), the fixed
    entries spliced back in from x0 for every residual and Jacobian evaluation: least_squares(method='trf',
    x_scale='jac') with the Jacobian's fixed columns deleted and the bounds of the free entries.  With priors the
    residuals are [joint_residuals(x); W (x - mean) ...] under ``mixed_loss``; without prior rows the named loss.
    Returns scipy's result with ``x`` the whole parameter vector."""
    from scipy.optimize import least_squares

    x0 = np.asarray(x0, dtype=np.float64)
    free = np.ones(len(x0), bool) if free is None else np.asarray(free, bool)
    cols = np.nonzero(free)[0]
    bl = [(c, m, sqrt_info(L)) for c, m, L in blocks(rig, priors)]

    def full(z):
        x = x0.copy()
        x[cols] = z
        return x

    if bl:
        rows = np.concatenate([np.repeat(np.arange(len(c)), len(c)) + off for (c, _, _), off in
                               zip(bl, np.cumsum([0] + [len(c) for c, _, _ in bl[:-1]]))])  # fmt: skip
        colsJ = np.concatenate([np.tile(c, len(c)) for c, _, _ in bl])
        vals = np.concatenate([W.ravel() for _, _, W in bl])
        Jpri = sparse.csr_matrix((vals, (rows, colsJ)), shape=(sum(len(c) for c, _, _ in bl), len(x0)))

        def res(z):
            x = full(z)
            return np.concatenate([O.residuals(x, rig)] + [W @ (x[c] - m) for c, m, W in bl])

        def jac(z):
            return sparse.vstack([O.jacobian(full(z), rig), Jpri]).tocsr()[:, cols]

        loss = mixed_loss(2 * rig.n_obs + rig.n_constraints, loss, f_scale)
    else:

        def res(z):
            return O.residuals(full(z), rig)

        def jac(z):
            return O.jacobian(full(z), rig)[:, cols]

    lo, hi = rig.bounds()
    opts = dict(ftol=1e-8, xtol=1e-8, gtol=1e-8, max_nfev=None, verbose=0)
    opts.update(kw)
    r = least_squares(res, x0[cols], jac=jac, x_scale="jac", method="trf", bounds=(lo[cols], hi[cols]), loss=loss,
                      f_scale=f_scale, **opts)  # fmt: skip
    r.x = full(r.x)
    return r


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


def linearize(x: np.ndarray, rig: O.Rig, free=None, priors: Priors | None = None, loss: str = "linear",
              f_scale: float = 1.0):  # fmt: skip
    """``oracle.lm_schur.linearize`` of the free parameters (``free``: boolean over x, None: all) with the priors.  The
    fixed Jacobian columns are zero (a fixed parameter is a constant of the problem), so U, g_c, V, g_p hold nothing of
    them.  The priors add info_c into U_c (at the camera's own slots of the stride-P block), info_c (x_c - mean_c) into
    g_c, info_j into V_j, info_j (X_j - mean_j) into g_j, and the prior cost into the cost.  The prior terms are whole: a
    fixed entry's information still couples to the free ones, as the engine's mask is applied to the reduced system
    afterwards."""
    lin = LS.linearize(x, rig, loss, f_scale)
    U, gc, V, gp, Jc, Jp = lin.U, lin.gc, lin.V, lin.gp, lin.Jc, lin.Jp
    if free is not None:
        fc, fp = free_slots(free, rig, LS.cam_stride(rig))
        Jc = Jc * fc.reshape(rig.n_cams, -1)[rig.obs_cam][:, None, :]
        Jp = Jp * fp[rig.obs_pt][:, None, None]
        rs = np.asarray(O.robust_row_scales(lin.f, loss, f_scale)[1]).reshape(-1, 2)
        U, gc, V, gp = np.zeros_like(U), np.zeros_like(gc), np.zeros_like(V), np.zeros_like(gp)
        np.add.at(U, rig.obs_cam, np.einsum("nki,nkj->nij", Jc, Jc))
        np.add.at(gc, rig.obs_cam, np.einsum("nki,nk->ni", Jc, rs))
        np.add.at(V, rig.obs_pt, np.einsum("nki,nkj->nij", Jp, Jp))
        np.add.at(gp, rig.obs_pt, np.einsum("nki,nk->ni", Jp, rs))
    if priors is None:
        return LS.Linearization(lin.cost, lin.f, U, gc, V, gp, Jc, Jp)
    U, gc, V, gp = U.copy(), gc.copy(), V.copy(), gp.copy()
    for k, c in enumerate(priors.cams):
        o, w = int(rig.cam_offsets[c]), int(rig.cam_offsets[c + 1] - rig.cam_offsets[c])
        L = priors.cam_info[k, :w, :w]
        U[c, :w, :w] += L
        gc[c, :w] += L @ (x[o : o + w] - priors.cam_mean[k, :w])
    ncp = rig.n_camera_params
    for k, j in enumerate(priors.pts):
        V[j] += priors.pt_info[k]
        gp[j] += priors.pt_info[k] @ (x[ncp + 3 * j : ncp + 3 * j + 3] - priors.pt_mean[k])
    return LS.Linearization(lin.cost + prior_cost(x, rig, priors), lin.f, U, gc, V, gp, Jc, Jp)


def scaling(x: np.ndarray, rig: O.Rig, priors: Priors | None = None, loss: str = "linear", f_scale: float = 1.0):
    """The engine's first Marquardt scaling (Dc2, Dp2): diag of the unmasked U_c, V_j with the priors' information, 1
    where that is 0."""
    lin = linearize(x, rig, None, priors, loss, f_scale)
    Dc2, Dp2 = np.einsum("cii->ci", lin.U), np.einsum("jii->ji", lin.V)
    return np.where(Dc2 > 0, Dc2, 1.0), np.where(Dp2 > 0, Dp2, 1.0)


def schur_system(lin, rig: O.Rig, lam: float, Dc2: np.ndarray, Dp2: np.ndarray, fixed_slots: np.ndarray,
                 fixed_pts: np.ndarray):  # fmt: skip
    """The engine's masked reduced system: ``oracle.lm_schur.schur_system`` with Einv = 0 for the fixed points (no Schur
    term, no step), then unit rows and columns of S before the damping for the fixed camera slots (so 1 + lam Dc2 on the
    diagonal) and zero b.  ``fixed_slots``: boolean over the n_cams * P stride-P slots; ``fixed_pts``: boolean over
    points.  Of a prior linearisation: the priors enter before the fixed-slot mask."""
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


def dense_covariance(x, rig: O.Rig, fixed=(), fixed_points=(), priors: Priors | None = None, loss: str = "linear",
                     f_scale: float = 1.0, variance_factor=None):  # fmt: skip
    """``oracle.covariance.dense_covariance`` of the augmented problem with known points: H = J^T J + info, the cost with
    the priors, and m counting sum rank(info) more rows.  The columns of ``fixed_points`` are deleted from J like those of
    the fixed camera parameters: their blocks are zero, their rank -2, and each counts 3 parameters fewer in the rank
    behind dof.  A point's rank is that of V_j + info_j."""
    cost, H = OC._system(x, rig, loss, f_scale)
    H = H + info_matrix(rig, priors)
    cost += prior_cost(x, rig, priors)
    ncp = rig.n_camera_params
    fix, masked = OC._masks(rig, list(fixed))
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
    m = 2 * rig.n_obs + rig.n_constraints + prior_rank(rig, priors)
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
    return dict(cameras=cam, points=pts, point_rank=ranks.astype(np.int32), variance_factor=s2, dof=dof, cost=cost)
