"""Closed-form first derivatives of exact moment matching ('EM') w.r.t. the test input mean z and the
input covariance Sigma  --  TEST INFRASTRUCTURE ONLY (the checker of gpmpc_predict_em_grad).

With ``gp_method='EM'`` CasADi differentiates ``gp_exact_moment`` (``gp_functions.py:344-418``) inside
``nlpsol`` (``mpc_class.py:390-412``, ``:496-513``).  The reference has no closed forms; these follow
from ``gp_oracle.gp_exact_moment`` and are checked by ``em_grad_fd``.  Per output a, pair (a, b):

    v_i = x_i - z,  Lambda_a = diag(ell_a^2),  iR_a = (Sigma + Lambda_a)^-1,  q_ai = c_a exp(-1/2 v_i^T iR_a v_i)
    d mean_a / dz     = iR_a s_a,                          s_a = sum_i beta_ai q_ai v_i
    d mean_a / dSigma = 1/2 iR_a S_a iR_a - 1/2 mean_a iR_a,  S_a = sum_i beta_ai q_ai v_i v_i^T
    P = Lambda_a^-1 + Lambda_b^-1,  C = (I + P Sigma)^-1,  g_ij = C (Lambda_a^-1 v_i + Lambda_b^-1 v_j)
    d log(t Q_ij) / dz = g_ij,   d log(t Q_ij) / dSigma = 1/2 g_ij g_ij^T - 1/2 C P
    T_a = t tr(K^-1 Q_aa):  dT/dz = 2 C Lambda^-1 sum_i v_i r_i,  r = diag(K^-1 tQ)
                            dT/dSigma = C Lambda^-1 [sum_i r_i v_i v_i^T + V^T (K^-1 o tQ) V] Lambda^-1 C^T - 1/2 C P T

The cross term is differentiated as written (t beta^T Q beta minus the product of the means, each summed
in numpy longdouble), not in the regrouped form the engine uses, so the two are independent.  Every K^-1
term goes through the Cholesky factor: the rank-one backbone e e^T of Q_aa through triangular solves, the
O(Sigma) remainder through K^-1 = cho_solve(L, I).  d/dSigma[d][e] holds every other entry fixed.
"""
from __future__ import annotations

import numpy as np
from scipy.linalg import cho_solve, solve_triangular

from oracle import gp_oracle as orc

LD = np.longdouble


def _sigmas(Sigma, H, Nx):
    Sigma = np.asarray(Sigma, dtype=np.float64)
    return np.broadcast_to(Sigma, (H, Nx, Nx)) if Sigma.ndim == 2 else Sigma


def _point(X, hyper, alpha, chol, kinv, z, S):
    N, Nx = X.shape
    Ny = hyper.shape[0]
    eye = np.eye(Nx)
    v = (X - z[None, :]).astype(LD)
    al = [alpha[a].astype(LD) for a in range(Ny)]
    lam = [hyper[a, :Nx] ** 2 for a in range(Ny)]
    sf2 = [hyper[a, Nx] ** 2 for a in range(Ny)]
    iR, mean, J, dmS, logk = [], np.zeros(Ny), np.zeros((Ny, Nx)), np.zeros((Ny, Nx, Nx)), []
    for a in range(Ny):
        R = S + np.diag(lam[a])
        iRa = np.linalg.inv(R)
        c = sf2[a] * np.prod(hyper[a, :Nx]) / np.sqrt(np.linalg.det(R))
        q = LD(c) * np.exp(-0.5 * np.sum((v @ iRa.astype(LD)) * v, 1))
        u = al[a] * q
        m = np.sum(u)
        s = (v.T @ u).astype(np.float64)
        Sa = (v.T @ (u[:, None] * v)).astype(np.float64)
        iR.append(iRa); mean[a] = float(m)
        J[a] = iRa @ s
        dmS[a] = 0.5 * iRa @ Sa @ iRa - 0.5 * float(m) * iRa
        logk.append(LD(2 * np.log(hyper[a, Nx])) - 0.5 * np.sum((v / hyper[a, :Nx].astype(LD)) ** 2, 1))
    cov = np.zeros((Ny, Ny)); dcz = np.zeros((Ny, Ny, Nx)); dcS = np.zeros((Ny, Ny, Nx, Nx))
    for a in range(Ny):
        for b in range(a + 1):
            P = np.diag(1.0 / lam[a] + 1.0 / lam[b])
            C = np.linalg.inv(eye + P @ S)
            Fa = C / lam[a][None, :]; Fb = C / lam[b][None, :]
            Rm = S @ P + eye
            t = 1.0 / np.sqrt(np.linalg.det(Rm))
            Qm = np.linalg.solve(Rm, 0.5 * S).astype(LD)
            ii = v / lam[a].astype(LD); ij = v / lam[b].astype(LD)
            ea = logk[a] + np.sum((ii @ Qm) * ii, 1)
            eb = logk[b] + np.sum((ij @ Qm) * ij, 1)
            cr = 2 * (ii @ Qm) @ ij.T
            tQ = LD(t) * np.exp(ea[:, None] + eb[None, :] + cr)
            W = np.outer(al[a], al[b]) * tQ
            r, cs, tot = W.sum(1), W.sum(0), W.sum()
            Gi = (v.T @ (r[:, None] * v)).astype(np.float64)
            Gj = (v.T @ (cs[:, None] * v)).astype(np.float64)
            B = (v.T @ W @ v).astype(np.float64)
            Wg = Fa @ (v.T @ r).astype(np.float64) + Fb @ (v.T @ cs).astype(np.float64)
            Wgg = Fa @ Gi @ Fa.T + Fa @ B @ Fb.T + Fb @ B.T @ Fa.T + Fb @ Gj @ Fb.T
            cz = Wg - (J[a] * mean[b] + mean[a] * J[b])
            cS = 0.5 * Wgg - 0.5 * float(tot) * (C @ P) - (dmS[a] * mean[b] + mean[a] * dmS[b])
            c_ab = float(tot - LD(mean[a]) * LD(mean[b]))
            if a == b:
                e = np.exp(ea).astype(np.float64)
                ke = cho_solve((chol[a], True), e)
                Y = solve_triangular(chol[a], e[:, None] * v.astype(np.float64), lower=True)
                rr = LD(t) * e.astype(LD) * ke.astype(LD)
                Bl = t * (Y.T @ Y)
                Qr = LD(t) * np.exp(ea[:, None] + eb[None, :]) * np.expm1(cr)
                Km = kinv[a].astype(LD) * Qr
                rr = rr + Km.sum(1)
                Bl = Bl + (v.T @ Km @ v).astype(np.float64)
                T = float(np.sum(rr))
                cz = cz - 2 * Fa @ (v.T @ rr).astype(np.float64)
                cS = cS - (Fa @ ((v.T @ (rr[:, None] * v)).astype(np.float64) + Bl) @ Fa.T - 0.5 * T * (C @ P))
                c_ab += sf2[a] - T
            cov[a, b] = cov[b, a] = c_ab
            dcz[a, b] = dcz[b, a] = cz
            dcS[a, b] = cS
            dcS[b, a] = cS.T
    return mean, cov, J, dmS, dcz, dcS


def em_grad_closed(X, hyper, alpha, chol, Z, Sigma):
    """Closed-form 'EM' first derivatives (what gpmpc_predict_em_grad computes).  ``alpha`` (Ny,N) and
    ``chol`` (Ny,N,N) may be the engine's own (``gpmpc_get``).  Sigma: (Nx,Nx) shared or (H,Nx,Nx).
    Returns dict(mean (H,Ny), cov (H,Ny,Ny), dmean_dz (H,Ny,Nx), dmean_dSigma (H,Ny,Nx,Nx),
    dcov_dz (H,Ny,Ny,Nx), dcov_dSigma (H,Ny,Ny,Nx,Nx))."""
    X = np.asarray(X, dtype=np.float64)
    Z = np.atleast_2d(np.asarray(Z, dtype=np.float64))
    hyper = np.atleast_2d(np.asarray(hyper, dtype=np.float64))
    alpha = np.atleast_2d(np.asarray(alpha, dtype=np.float64))
    H, Nx = Z.shape
    Ny = hyper.shape[0]
    N = X.shape[0]
    kinv = []
    for a in range(Ny):
        Ki = cho_solve((chol[a], True), np.eye(N))
        kinv.append(0.5 * (Ki + Ki.T))
    Sg = _sigmas(Sigma, H, Nx)
    keys = ('mean', 'cov', 'dmean_dz', 'dmean_dSigma', 'dcov_dz', 'dcov_dSigma')
    res = [_point(X, hyper, alpha, chol, kinv, Z[h], Sg[h]) for h in range(H)]
    return {k: np.stack([r[i] for r in res]) for i, k in enumerate(keys)}


def sym_pair(dS):
    """The derivative along the symmetric perturbation Sigma[d][e] = Sigma[e][d] += eps: dS[d][e] + dS[e][d]
    off the diagonal, dS[d][d] on it (the quantity ``em_grad_fd`` differences)."""
    out = dS + np.swapaxes(dS, -1, -2)
    Nx = dS.shape[-1]
    out[..., np.arange(Nx), np.arange(Nx)] *= 0.5
    return out


def em_grad_fd(invK, X, Y, hyper, Z, Sigma, hz=3e-2, hs=3e-4):
    """Fourth-order central differences of ``gp_oracle.gp_exact_moment(extended=True)``: every entry of z,
    and Sigma along each symmetric pair (d, e) (compare with ``sym_pair`` of the closed form).  Returns
    dict(dmean_dz, dmean_dSigma, dcov_dz, dcov_dSigma) shaped as ``em_grad_closed``'s."""
    Z = np.atleast_2d(np.asarray(Z, dtype=np.float64))
    hyper = np.atleast_2d(np.asarray(hyper, dtype=np.float64))
    H, Nx = Z.shape
    Ny = hyper.shape[0]
    Sg = _sigmas(Sigma, H, Nx)
    out = dict(dmean_dz=np.zeros((H, Ny, Nx)), dmean_dSigma=np.zeros((H, Ny, Nx, Nx)),
               dcov_dz=np.zeros((H, Ny, Ny, Nx)), dcov_dSigma=np.zeros((H, Ny, Ny, Nx, Nx)))

    def f(z, S):
        return orc.gp_exact_moment(invK, X, Y, hyper, z, S, extended=True)

    def d4(fun, st):
        r = {k: fun(k * st) for k in (-2, -1, 1, 2)}
        return tuple((r[-2][i] - 8 * r[-1][i] + 8 * r[1][i] - r[2][i]) / (12 * st) for i in range(2))

    for h in range(H):
        for d in range(Nx):
            st = hz * max(1.0, abs(Z[h, d]))
            ez = np.zeros(Nx); ez[d] = 1.0
            dm, dc = d4(lambda s: f(Z[h] + s * ez, Sg[h]), st)
            out['dmean_dz'][h, :, d] = dm; out['dcov_dz'][h, :, :, d] = dc
        for d in range(Nx):
            for e in range(d + 1):
                E = np.zeros((Nx, Nx)); E[d, e] = E[e, d] = 1.0
                dm, dc = d4(lambda s: f(Z[h], Sg[h] + s * E), hs)
                out['dmean_dSigma'][h, :, d, e] = out['dmean_dSigma'][h, :, e, d] = dm
                out['dcov_dSigma'][h, :, :, d, e] = out['dcov_dSigma'][h, :, :, e, d] = dc
    return out
