"""NumPy statement of Gaussian priors on cameras and points (DESIGN.md section 4.13), the checker of
``cb_ba_problem_create_priors`` (test infrastructure).  It builds on ``oracle/`` and ``tests/_fixed_oracle.py`` without
changing either: a problem with priors is the least-squares problem whose residual vector is extended by the rows
W (x - mean) of every prior, W^T W = info, which the loss leaves linear.

  Priors              the priors in BAProblem's layout (camera means / information padded to 9)
  mixed_loss          scipy's callable loss: the named loss on the first rows, rho(z) = z on the prior rows
  solve_scipy_prior   least_squares(method='trf', x_scale='jac') on the augmented residuals, over the free subvector
  linearize           ``_fixed_oracle.linearize`` plus the prior terms in U, g_c, V, g_p and the cost
  schur_system        ``_fixed_oracle.schur_system`` of that linearisation
  dense_covariance    ``_fixed_oracle.dense_covariance`` of the augmented J, m counting sum rank(info) more rows
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np
from scipy import sparse

from oracle import ba_oracle as O
from oracle import covariance as OC
from oracle import lm_schur as LS
from tests import _fixed_oracle as FO

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


def blocks(rig: O.Rig, pr: Priors):
    """[(x columns, mean, info)] of every prior, at the prior's own width."""
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


def prior_cost(x: np.ndarray, rig: O.Rig, pr: Priors) -> float:
    return sum(0.5 * float((x[c] - m) @ L @ (x[c] - m)) for c, m, L in blocks(rig, pr))


def prior_rank(rig: O.Rig, pr: Priors) -> int:
    return sum(rank(L) for _, _, L in blocks(rig, pr))


def info_matrix(rig: O.Rig, pr: Priors) -> np.ndarray:
    """The block-diagonal information over the whole x (dense)."""
    Lf = np.zeros((rig.n_params, rig.n_params))
    for c, _, L in blocks(rig, pr):
        Lf[np.ix_(c, c)] += L
    return Lf


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


def solve_scipy_prior(rig: O.Rig, x0: np.ndarray, pr: Priors, free=None, loss: str = "linear", f_scale: float = 1.0,
                      **kw):  # fmt: skip
    """least_squares(method='trf', x_scale='jac') on [joint_residuals(x); W (x - mean) ...] with ``mixed_loss``, over
    the free entries of x (``free``: boolean over x, None: all), the rest spliced in from x0.  Returns scipy's result with
    ``x`` the whole parameter vector."""
    from scipy.optimize import least_squares

    x0 = np.asarray(x0, dtype=np.float64)
    free = np.ones(len(x0), bool) if free is None else np.asarray(free, bool)
    cols = np.nonzero(free)[0]
    bl = [(c, m, sqrt_info(L)) for c, m, L in blocks(rig, pr)]
    n_first = 2 * rig.n_obs + rig.n_constraints
    if bl:
        rows = np.concatenate([np.repeat(np.arange(len(c)), len(c)) + off for (c, _, _), off in
                               zip(bl, np.cumsum([0] + [len(c) for c, _, _ in bl[:-1]]))])  # fmt: skip
        colsJ = np.concatenate([np.tile(c, len(c)) for c, _, _ in bl])
        vals = np.concatenate([W.ravel() for _, _, W in bl])
        Jpri = sparse.csr_matrix((vals, (rows, colsJ)), shape=(sum(len(c) for c, _, _ in bl), len(x0)))
    else:
        Jpri = sparse.csr_matrix((0, len(x0)))

    def full(z):
        x = x0.copy()
        x[cols] = z
        return x

    def res(z):
        x = full(z)
        r = [O.residuals(x, rig)] + [W @ (x[c] - m) for c, m, W in bl]
        return np.concatenate(r)

    def jac(z):
        return sparse.vstack([O.jacobian(full(z), rig), Jpri]).tocsr()[:, cols]

    lo, hi = rig.bounds()
    opts = dict(ftol=1e-8, xtol=1e-8, gtol=1e-8, max_nfev=None, verbose=0)
    opts.update(kw)
    r = least_squares(res, x0[cols], jac=jac, x_scale="jac", method="trf", bounds=(lo[cols], hi[cols]),
                      loss=mixed_loss(n_first, loss, f_scale), f_scale=f_scale, **opts)  # fmt: skip
    r.x = full(r.x)
    return r


def linearize(x: np.ndarray, rig: O.Rig, pr: Priors, free=None, loss: str = "linear", f_scale: float = 1.0):
    """``_fixed_oracle.linearize`` (``oracle.lm_schur.linearize`` when every parameter is free) with the priors: info_c
    into U_c (at the camera's own slots of the stride-P block), info_c (x_c - mean_c) into g_c, info_j into V_j,
    info_j (X_j - mean_j) into g_j, and the prior cost into the cost.  The prior terms are whole: a fixed entry's
    information still couples to the free ones, as the engine's mask is applied to the reduced system afterwards."""
    lin = LS.linearize(x, rig, loss, f_scale) if free is None else FO.linearize(x, rig, free, loss, f_scale)
    U, gc, V, gp = lin.U.copy(), lin.gc.copy(), lin.V.copy(), lin.gp.copy()
    for k, c in enumerate(pr.cams):
        o, w = int(rig.cam_offsets[c]), int(rig.cam_offsets[c + 1] - rig.cam_offsets[c])
        L = pr.cam_info[k, :w, :w]
        U[c, :w, :w] += L
        gc[c, :w] += L @ (x[o : o + w] - pr.cam_mean[k, :w])
    ncp = rig.n_camera_params
    for k, j in enumerate(pr.pts):
        V[j] += pr.pt_info[k]
        gp[j] += pr.pt_info[k] @ (x[ncp + 3 * j : ncp + 3 * j + 3] - pr.pt_mean[k])
    return LS.Linearization(lin.cost + prior_cost(x, rig, pr), lin.f, U, gc, V, gp, lin.Jc, lin.Jp)


def scaling(x: np.ndarray, rig: O.Rig, pr: Priors, loss: str = "linear", f_scale: float = 1.0):
    """The engine's first Marquardt scaling (Dc2, Dp2): diag of the unmasked U_c, V_j with the priors' information, 1
    where that is 0."""
    lin = linearize(x, rig, pr, None, loss, f_scale)
    Dc2, Dp2 = np.einsum("cii->ci", lin.U), np.einsum("jii->ji", lin.V)
    return np.where(Dc2 > 0, Dc2, 1.0), np.where(Dp2 > 0, Dp2, 1.0)


def schur_system(lin, rig: O.Rig, lam: float, Dc2, Dp2, fixed_slots, fixed_pts):
    """``_fixed_oracle.schur_system`` of a prior linearisation: the priors enter before the fixed-slot mask."""
    return FO.schur_system(lin, rig, lam, Dc2, Dp2, fixed_slots, fixed_pts)


def dense_covariance(x, rig: O.Rig, pr: Priors, fixed=(), fixed_points=(), loss: str = "linear", f_scale: float = 1.0,
                     variance_factor=None):  # fmt: skip
    """``_fixed_oracle.dense_covariance`` of the augmented problem: H = J^T J + info, the cost with the priors, and m
    counting sum rank(info) more rows.  A point's rank is that of V_j + info_j."""
    cost, H = OC._system(x, rig, loss, f_scale)
    H = H + info_matrix(rig, pr)
    cost += prior_cost(x, rig, pr)
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
    m = 2 * rig.n_obs + rig.n_constraints + prior_rank(rig, pr)
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
