"""NumPy statement of the parameter covariance at a bundle-adjustment solution (DESIGN.md section 4.6), the checker of
``cb_ba_covariance``.  TEST INFRASTRUCTURE -- see ``oracle/__init__.py``.

J is ``ba_oracle.jacobian`` (pixels / fx_initial, then the constraint rows) after the robust row rescaling at x, exactly
as ``lm_schur.linearize`` / ``lm_solve_dense`` use it.  Sigma = s2 (J_F^T J_F)^-1 over the free parameters F (neither
fixed by the gauge nor masked: cameras without observations).  The null directions of rank-deficient point blocks V_j
(points seen by one camera, unobserved points) are exact null vectors of J^T J; they are not parameters of F.

Two forms that must agree:
  dense_covariance  the full J_F^T J_F with those null directions deflated, inverted densely;
  schur_covariance  the reduced camera system S = U - sum_j W_j V_j^+ W_j^T (- the constrained points' block, eliminated
                    densely), inverted on F, and the per-point marginals V_j^+ + V_j^+ W_j^T S_F^-1 W_j V_j^+.
"""

from __future__ import annotations

import numpy as np
from scipy.sparse import diags

from . import ba_oracle as O

EIG_RTOL = 1e-12  # eigenvalues of V_j at or below this times the largest are zero (cb_covariance.cuh COV_EIG_RTOL)


def _system(x, rig: O.Rig, loss: str, f_scale: float):
    f = O.residuals(x, rig)
    js, _ = O.robust_row_scales(f, loss, f_scale)
    Js = diags(js) @ O.jacobian(x, rig)
    return O.robust_cost(f, loss, f_scale), (Js.T @ Js).toarray()


def constrained_points(rig: O.Rig) -> np.ndarray:
    m = np.zeros(rig.n_pts, bool)
    if rig.n_constraints:
        m[np.asarray(rig.groups_a).ravel()] = True
        m[np.asarray(rig.groups_b).ravel()] = True
    return m


def observed_cameras(rig: O.Rig) -> np.ndarray:
    return np.bincount(rig.obs_cam, minlength=rig.n_cams) > 0


def _masks(rig: O.Rig, fixed):
    ncp = rig.n_camera_params
    masked = np.zeros(ncp, bool)
    for c in np.nonzero(~observed_cameras(rig))[0]:
        masked[rig.cam_offsets[c] : rig.cam_offsets[c + 1]] = True
    fix = np.zeros(ncp, bool)
    fix[np.asarray(fixed, dtype=np.int64)] = True
    fix &= ~masked
    return fix, masked


def _point_pinv(Vj):
    w, Q = np.linalg.eigh(Vj)
    wmax = max(w.max(), 0.0)
    nz = (w > EIG_RTOL * wmax) if wmax > 0 else np.zeros(3, bool)
    Vp = (Q[:, nz] / w[nz]) @ Q[:, nz].T
    return Vp, int(nz.sum()), Q[:, ~nz]


def _finish(rig, fix, masked, cost, ranks, s2_given, cam_hat, pts_hat):
    """Scale by s2 and lay out like the engine: NaN for masked rows / columns, 0 for fixed ones, NaN point blocks for
    rank-deficient and constrained points."""
    ncp = rig.n_camera_params
    m = 2 * rig.n_obs + rig.n_constraints
    null = int(sum(3 - r for r in ranks if r >= 0))
    dof = m - (rig.n_params - int(fix.sum()) - int(masked.sum()) - null)
    s2 = s2_given if s2_given is not None and s2_given > 0 else (2.0 * cost / dof if dof > 0 else np.nan)
    cam = s2 * cam_hat
    cam[fix, :] = 0.0
    cam[:, fix] = 0.0
    cam[masked, :] = np.nan
    cam[:, masked] = np.nan
    pts = s2 * pts_hat
    pts[np.asarray(ranks) != 3] = np.nan
    return dict(cameras=cam.reshape(ncp, ncp), points=pts, point_rank=np.asarray(ranks, np.int32), variance_factor=s2,
                dof=dof)


def dense_covariance(x, rig: O.Rig, fixed, loss: str = "linear", f_scale: float = 1.0, variance_factor=None):
    cost, H = _system(x, rig, loss, f_scale)
    ncp = rig.n_camera_params
    fix, masked = _masks(rig, fixed)
    free = np.concatenate([~(fix | masked), np.ones(3 * rig.n_pts, bool)])
    comp = constrained_points(rig)
    ranks = np.full(rig.n_pts, -1)
    defl = np.zeros_like(H)
    for j in np.nonzero(~comp)[0]:
        sl = slice(ncp + 3 * j, ncp + 3 * j + 3)
        _, ranks[j], N = _point_pinv(H[sl, sl])
        defl[sl, sl] = N @ N.T
    idx = np.nonzero(free)[0]
    Hf = (H + defl)[np.ix_(idx, idx)]
    Sig = np.zeros_like(H)
    Sig[np.ix_(idx, idx)] = np.linalg.inv(Hf) - defl[np.ix_(idx, idx)]
    pts = np.stack([Sig[ncp + 3 * j : ncp + 3 * j + 3, ncp + 3 * j : ncp + 3 * j + 3] for j in range(rig.n_pts)])
    return _finish(rig, fix, masked, cost, ranks, variance_factor, Sig[:ncp, :ncp], pts)


def schur_covariance(x, rig: O.Rig, fixed, loss: str = "linear", f_scale: float = 1.0, variance_factor=None):
    cost, H = _system(x, rig, loss, f_scale)
    ncp = rig.n_camera_params
    fix, masked = _masks(rig, fixed)
    comp = constrained_points(rig)
    U = H[:ncp, :ncp]
    W = H[:ncp, ncp:].reshape(ncp, rig.n_pts, 3)  # camera x point blocks
    Vp = np.zeros((rig.n_pts, 3, 3))
    ranks = np.full(rig.n_pts, -1)
    for j in np.nonzero(~comp)[0]:
        Vp[j], ranks[j], _ = _point_pinv(H[ncp + 3 * j : ncp + 3 * j + 3, ncp + 3 * j : ncp + 3 * j + 3])
    Z = np.einsum("cja,jab->jcb", W, Vp)  # (n_pts, ncp, 3): W_j V_j^+
    S = U - np.tensordot(Z, W, axes=([0, 2], [1, 2]))
    if comp.any():  # constraint components: their point block (incl. the constraint rows) eliminated as one
        cols = (ncp + 3 * np.nonzero(comp)[0][:, None] + np.arange(3)[None]).ravel()
        Wc = H[:ncp, cols]
        S -= Wc @ np.linalg.solve(H[np.ix_(cols, cols)], Wc.T)
    f = ~(fix | masked)
    Shat = np.zeros((ncp, ncp))
    Shat[np.ix_(f, f)] = np.linalg.inv(S[np.ix_(f, f)])
    pts = Vp + np.einsum("jca,jcb->jab", Z, np.einsum("cd,jdb->jcb", Shat, Z, optimize=True))
    return _finish(rig, fix, masked, cost, ranks, variance_factor, Shat, pts)


def reduced_pivots(x, rig: O.Rig, fixed, loss: str = "linear", f_scale: float = 1.0) -> np.ndarray:
    """Cholesky pivots of S_F over its diagonal, in F's order, for a problem without constraint rows (the engine's
    singularity test compares them with CB_COV_PIVOT_RTOL)."""
    _, H = _system(x, rig, loss, f_scale)
    ncp = rig.n_camera_params
    fix, masked = _masks(rig, fixed)
    S = H[:ncp, :ncp].copy()
    for j in np.nonzero(~constrained_points(rig))[0]:
        sl = slice(ncp + 3 * j, ncp + 3 * j + 3)
        Vp, _, _ = _point_pinv(H[sl, sl])
        S -= H[:ncp, sl] @ Vp @ H[sl, :ncp]
    f = ~(fix | masked)
    A = S[np.ix_(f, f)].copy()
    d0 = np.diag(A).copy()
    piv = np.empty(len(A))
    for k in range(len(A)):
        piv[k] = A[k, k] / d0[k]
        A[k + 1 :, k + 1 :] -= np.outer(A[k + 1 :, k], A[k, k + 1 :]) / A[k, k]
    return piv
