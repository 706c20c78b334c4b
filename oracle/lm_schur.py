"""NumPy model of the Schur-complement Levenberg-Marquardt iteration that the CUDA
engine runs.  TEST INFRASTRUCTURE -- see ``oracle/__init__.py``.

This is NOT the reference's algorithm (the reference calls scipy's TRF+LSMR,
restated in ``ba_oracle.solve_scipy``); it is a CPU statement of the product's
own normal-equation pipeline so each CUDA stage (U/V/g accumulation, Schur
complement S, reduced rhs b, camera step, point back-substitution) can be
checked against dense linear algebra on small problems.  Parity claims are
made against ``ba_oracle`` / scipy, never against this file.
"""

from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from . import ba_oracle as O

EPS = np.finfo(float).eps


@dataclass
class Linearization:
    cost: float
    f: np.ndarray  # raw residuals (2 n_obs)
    U: np.ndarray  # (n_cams, P, P)
    gc: np.ndarray  # (n_cams, P)
    V: np.ndarray  # (n_pts, 3, 3)
    gp: np.ndarray  # (n_pts, 3)
    Jc: np.ndarray  # (n_obs, 2, P) robust-scaled
    Jp: np.ndarray  # (n_obs, 2, 3) robust-scaled


def cam_stride(rig: O.Rig) -> int:
    return 9 if (rig.cam_flags & O.FLAG_FREE_INTRINSICS).any() else 6


def split_x(x: np.ndarray, rig: O.Rig, P: int) -> tuple[np.ndarray, np.ndarray]:
    c = np.zeros((rig.n_cams, P))
    for i in range(rig.n_cams):
        w = rig.cam_offsets[i + 1] - rig.cam_offsets[i]
        c[i, :w] = x[rig.cam_offsets[i] : rig.cam_offsets[i + 1]]
    return c, x[rig.n_camera_params :].reshape(-1, 3).copy()


def join_x(c: np.ndarray, p: np.ndarray, rig: O.Rig) -> np.ndarray:
    parts = [c[i, : rig.cam_offsets[i + 1] - rig.cam_offsets[i]] for i in range(rig.n_cams)]
    return np.concatenate(parts + [p.ravel()])


def linearize(x: np.ndarray, rig: O.Rig, loss: str = "linear", f_scale: float = 1.0) -> Linearization:
    P = cam_stride(rig)
    f = O.residuals(x, rig)[: 2 * rig.n_obs]
    Jc9, Jp = O.jacobian_blocks(x, rig)
    Jc = Jc9[:, :, :P].copy()
    cost = O.robust_cost(f, loss, f_scale)
    js, fs = O.robust_row_scales(f, loss, f_scale)
    if loss != "linear":
        # J_s^T J_s = J^T w J,  J_s^T f_s = J^T rho' f
        Jc *= js.reshape(-1, 2)[:, :, None]
        Jp = Jp * js.reshape(-1, 2)[:, :, None]
    rs = fs.reshape(-1, 2)
    U = np.zeros((rig.n_cams, P, P))
    gc = np.zeros((rig.n_cams, P))
    V = np.zeros((rig.n_pts, 3, 3))
    gp = np.zeros((rig.n_pts, 3))
    np.add.at(U, rig.obs_cam, np.einsum("nki,nkj->nij", Jc, Jc))
    np.add.at(gc, rig.obs_cam, np.einsum("nki,nk->ni", Jc, rs))
    np.add.at(V, rig.obs_pt, np.einsum("nki,nkj->nij", Jp, Jp))
    np.add.at(gp, rig.obs_pt, np.einsum("nki,nk->ni", Jp, rs))
    return Linearization(cost, f, U, gc, V, gp, Jc, Jp)


def schur_system(lin: Linearization, rig: O.Rig, lam: float, Dc2: np.ndarray, Dp2: np.ndarray):
    """S (n_cams*P square), b (n_cams*P), Einv (n_pts,3,3), W (n_obs,P,3)."""
    n_cams, P = lin.gc.shape
    E = lin.V + lam * (Dp2[:, :, None] * np.eye(3)[None])
    # unobserved points: V == 0 and Dp2 == 1 -> E = lam I, gp = 0 -> no motion
    Einv = np.linalg.inv(E)
    W = np.einsum("nki,nkj->nij", lin.Jc, lin.Jp)  # (n_obs,P,3)
    # aggregate W per (cam, point) into a dense (n_pts, n_cams, P, 3) table
    Wd = np.zeros((rig.n_pts, n_cams, P, 3))
    np.add.at(Wd, (rig.obs_pt, rig.obs_cam), W)
    Y = np.einsum("jcpa,jab->jcpb", Wd, Einv)
    # sum over points j and point coordinates a as one (n_cams P) x (n_pts 3) matrix product
    Y2 = Y.transpose(1, 2, 0, 3).reshape(n_cams * P, -1)
    W2 = Wd.transpose(1, 2, 0, 3).reshape(n_cams * P, -1)
    S4 = -(Y2 @ W2.T).reshape(n_cams, P, n_cams, P)
    b = lin.gc - np.einsum("jcpa,ja->cp", Y, lin.gp)
    for c in range(n_cams):
        S4[c, :, c, :] += lin.U[c] + lam * np.diag(Dc2[c])
    return S4.reshape(n_cams * P, n_cams * P), b.reshape(-1), Einv, Wd


def block_jacobi_pcg(S: np.ndarray, rhs: np.ndarray, P: int, tol: float, maxit: int):
    """Preconditioned CG on the dense reduced camera system, P x P diagonal blocks as
    the preconditioner; stops on sqrt(r^T M^-1 r) <= tol * its initial value."""
    n = len(rhs)
    Minv = np.zeros_like(S)
    for i in range(n // P):
        sl = slice(i * P, (i + 1) * P)
        Minv[sl, sl] = np.linalg.inv(S[sl, sl])
    x = np.zeros(n)
    r = rhs.copy()
    z = Minv @ r
    p = z.copy()
    rz = r @ z
    if rz <= 0:
        return x, 0
    stop = tol * tol * rz
    for it in range(maxit):
        q = S @ p
        a = rz / (p @ q)
        x += a * p
        r -= a * q
        z = Minv @ r
        rz2 = r @ z
        if rz2 <= stop:
            return x, it + 1
        p = z + (rz2 / rz) * p
        rz = rz2
    return x, maxit


def lm_solve(
    rig: O.Rig,
    x0: np.ndarray,
    *,
    ftol: float = 1e-8,
    xtol: float = 1e-8,
    gtol: float = 1e-8,
    max_nfev: int | None = None,
    loss: str = "linear",
    f_scale: float = 1.0,
    lam0: float = 1e-4,
    verbose: int = 0,
    linear_solver: str = "direct",
    pcg_tol: float = 1e-10,
    lam_min: float = 0.0,
):
    P = cam_stride(rig)
    n_cams = rig.n_cams
    widths = rig.cam_offsets[1:] - rig.cam_offsets[:-1]
    active = np.arange(P)[None, :] < widths[:, None]  # (n_cams, P)
    lo, hi = rig.bounds()
    loc, _ = split_x(np.where(np.isfinite(lo), lo, -1e300), rig, P)
    hic, _ = split_x(np.where(np.isfinite(hi), hi, 1e300), rig, P)
    loc[~active] = -1e300
    hic[~active] = 1e300

    x = np.asarray(x0, dtype=np.float64).copy()
    if max_nfev is None:
        max_nfev = 100 * len(x)
    lin = linearize(x, rig, loss, f_scale)
    nfev = njev = 1
    lam, nu = lam0, 2.0
    Dc2 = np.zeros((n_cams, P))
    Dp2 = np.zeros((rig.n_pts, 3))
    status = 0
    nit = 0
    history = []
    while True:
        Dc2 = np.maximum(Dc2, np.einsum("cii->ci", lin.U))
        Dp2 = np.maximum(Dp2, np.einsum("jii->ji", lin.V))
        Dc2e = np.where(Dc2 > 0, Dc2, 1.0)
        Dp2e = np.where(Dp2 > 0, Dp2, 1.0)
        gnorm = max(np.abs(lin.gc[active]).max(), np.abs(lin.gp).max())
        if gnorm < gtol:
            status = 1
            break
        if nfev >= max_nfev:
            status = 0
            break
        nit += 1
        while True:
            S, b, Einv, Wd = schur_system(lin, rig, lam, Dc2e, Dp2e)
            # locked slots: unit diagonal, zero rhs
            ia = active.reshape(-1)
            S[~ia, :] = 0
            S[:, ~ia] = 0
            S[~ia, ~ia] = 1.0
            b = np.where(ia, b, 0.0)
            if linear_solver == "direct":
                dc = np.linalg.solve(S, -b).reshape(n_cams, P)
            else:
                dc, pcg_its = block_jacobi_pcg(S, -b, P, pcg_tol, 4 * len(b))
                dc = dc.reshape(n_cams, P)
            dp = -np.einsum("jab,jb->ja", Einv, lin.gp + np.einsum("jcpa,cp->ja", Wd, dc))
            c, p = split_x(x, rig, P)
            cn = np.clip(c + dc, loc, hic)
            dc_eff = cn - c
            x_new = join_x(cn, p + dp, rig)
            # model decrease 1/2 d^T (lam D^2 d - g)
            pred = 0.5 * (
                np.sum(dc_eff * (lam * Dc2e * dc_eff - lin.gc)) + np.sum(dp * (lam * Dp2e * dp - lin.gp))
            )
            f_new = O.residuals(x_new, rig)[: 2 * rig.n_obs]
            nfev += 1
            cost_new = O.robust_cost(f_new, loss, f_scale) if np.all(np.isfinite(f_new)) else np.inf
            actual = lin.cost - cost_new
            ratio = actual / pred if pred > 0 else -1.0
            step_norm = np.sqrt(np.sum(dc_eff**2) + np.sum(dp**2))
            x_norm = np.linalg.norm(x)
            ft = actual < ftol * lin.cost and ratio > 0.25
            xt = step_norm < xtol * (xtol + x_norm)
            history.append((nit, nfev, lin.cost, cost_new, ratio, lam, step_norm, gnorm))
            if verbose:
                print(
                    f"it {nit:3d} nfev {nfev:3d} cost {lin.cost:.15e} -> {cost_new:.15e} "
                    f"ratio {ratio:+.3f} lam {lam:.2e} |dx| {step_norm:.2e} |g| {gnorm:.2e}"
                )
            term = 4 if (ft and xt) else 2 if ft else 3 if xt else 0
            if actual > 0:
                lam = max(lam_min, lam * max(1.0 / 3.0, 1 - (2 * ratio - 1) ** 3))
                nu = 2.0
                break
            lam *= nu
            nu *= 2
            if term or nfev >= max_nfev:
                break
        if actual > 0:
            x = x_new
            lin = linearize(x, rig, loss, f_scale)
            njev += 1
        if term:
            status = term
            break
    return dict(x=x, cost=lin.cost, status=status, nfev=nfev, njev=njev, nit=nit, history=history)


def lm_solve_dense(
    rig: O.Rig,
    x0: np.ndarray,
    *,
    ftol: float = 1e-8,
    xtol: float = 1e-8,
    gtol: float = 1e-8,
    max_nfev: int | None = None,
    loss: str = "linear",
    f_scale: float = 1.0,
    lam0: float = 1e-4,
    verbose: int = 0,
):
    """The same damped Gauss-Newton iteration on the FULL dense normal equations, constraint rows included
    (any point-point coupling is handled by brute force).  Small problems only; used to check the
    component-wise elimination of the CUDA engine when rigid-distance rows are present."""
    x = np.asarray(x0, dtype=np.float64).copy()
    n = len(x)
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
        gnorm = np.abs(g).max()
        if gnorm < gtol:
            status = 1
            break
        if nfev >= max_nfev:
            break
        nit += 1
        while True:
            d = np.linalg.solve(H + lam * np.diag(De), -g)
            xn = np.clip(x + d, lo, hi)
            de = xn - x
            pred = 0.5 * np.sum(de * (lam * De * de - g))
            fn = O.residuals(xn, rig)
            nfev += 1
            cn = O.robust_cost(fn, loss, f_scale) if np.all(np.isfinite(fn)) else np.inf
            actual = cost - cn
            ratio = actual / pred if pred > 0 else -1.0
            sn = np.linalg.norm(de)
            ft = actual < ftol * cost and ratio > 0.25
            xt = sn < xtol * (xtol + np.linalg.norm(x))
            term = 4 if (ft and xt) else 2 if ft else 3 if xt else 0
            if verbose:
                print(f"it {nit:3d} nfev {nfev:3d} cost {cost:.15e} -> {cn:.15e} ratio {ratio:+.3f} lam {lam:.2e} |dx| {sn:.2e}")
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
