"""Closed-form second derivatives of exact moment matching ('EM') w.r.t. the test input mean z and the input
covariance Sigma  --  TEST INFRASTRUCTURE ONLY (the checker of gpmpc_predict_em_hess).

Every term of the 'EM' moments is a Gaussian expectation over x ~ N(z, Sigma) of a product of squared-exponential
kernels, so it is Gaussian in z and its z-derivatives are multivariate Hermite polynomials:  for a term
c exp(-1/2 (m - z)^T S (m - z)),  d^k / dz^k = term He_k(y; S),  y = S (m - z), with
    He_1 = y,  He_2 = y y^T - S,  He_3 = y y y - (3 placements of S y),  He_4 = y^4 - (6 placements of S y y) + (3 of S S).
    mean_a:       y = iR_a v_i,           S = iR_a = (Sigma + Lambda_a)^-1
    t Q_ij:       y = g_ij = Fa v_i + Fb v_j,  S = C P   (em_grad_oracle's notation, Fa = C Lambda_a^-1)
And d/dSigma = 1/2 d^2/dz^2 for any Gaussian expectation (the heat equation), which gives every Sigma block from the
z-derivatives of mean up to order 4 and of cov up to order 4 (the product mean_a mean_b adds product-rule terms).

Per output and pair everything is summed in numpy longdouble on the engine's own alpha and factor.  The cross term is
differentiated as written -- d^k (t beta_a^T Q beta_b) minus d^k (mean_a mean_b) by the product rule -- not in the
engine's regrouped form.  The trace term t tr(K^-1 Q_aa) goes through the Cholesky factor: the rank-one backbone e e^T
of Q_aa through triangular solves, the O(Sigma) remainder through K^-1 = cho_solve(L, I).
"""
from __future__ import annotations

import itertools

import numpy as np
from scipy.linalg import cho_solve, solve_triangular

from oracle import em_grad_oracle as emg

LD = np.longdouble
KEYS = ('d2mean_dz2', 'd2mean_dSigma_dz', 'd2mean_dSigma2', 'd2cov_dz2', 'd2cov_dSigma_dz', 'd2cov_dSigma2')


def _outer_rows(Y, k):
    """rows y_i^(x)k flattened: (N, Nx^k)"""
    N, Nx = Y.shape
    out = np.ones((N, 1), dtype=Y.dtype)
    for _ in range(k):
        out = (out[:, :, None] * Y[:, None, :]).reshape(N, -1)
    return out


def _place(S, T, k):
    """sum over the placements of S on two of the k axes, T (order k - 2) on the rest"""
    Nx = S.shape[0]
    out = np.zeros((Nx,) * k, dtype=T.dtype)
    for i, j in itertools.combinations(range(k), 2):
        rest = [q for q in range(k) if q not in (i, j)]
        letters = 'defg'[:k]
        expr = letters[i] + letters[j] + ',' + ''.join(letters[q] for q in rest) + '->' + letters
        out = out + np.einsum(expr, S, T)
    return out


def hermite(G, S):
    """[sum W He_k(y; S)]_k from G_k = sum W y^(x)k (k = 0..4, G_0 scalar)"""
    S = S.astype(G[1].dtype)
    H2 = G[2] - S * G[0]
    H3 = G[3] - _place(S, G[1], 3)
    pp = np.einsum('de,fg->defg', S, S) + np.einsum('df,eg->defg', S, S) + np.einsum('dg,ef->defg', S, S)
    H4 = G[4] - _place(S, G[2], 4) + pp * G[0]
    return [G[0], G[1], H2, H3, H4]


def _subsets(k, Xpq):
    """sum over the subsets S of the k axes of Xpq[|S|][k-|S|] with its first |S| axes placed on S"""
    out = 0
    for r in range(k + 1):
        for S in itertools.combinations(range(k), r):
            Sc = [q for q in range(k) if q not in S]
            perm = list(S) + Sc                      # axis s of X goes to position perm[s]
            out = out + np.transpose(Xpq[r][k - r], np.argsort(perm))
    return out


def leibniz(A, B, k):
    """d^k (f g) from A_p = d^p f, B_q = d^q g"""
    return _subsets(k, [[np.multiply.outer(A[p], B[q]) if p + q == k else None for q in range(5)] for p in range(5)])


def _bilinear(Pi, W, Pj, Nx):
    """X[p][q] = sum_ij W_ij (row i of Pi[p]) (x) (row j of Pj[q]), reshaped to (Nx,)*(p+q)"""
    X = [[None] * 5 for _ in range(5)]
    WPj = {q: W @ Pj[q] for q in range(3)}
    PiW = {p: Pi[p].T @ W for p in range(2)}
    for p in range(5):
        for q in range(5 - p):
            M = Pi[p].T @ WPj[q] if q <= 2 else PiW[p] @ Pj[q]
            X[p][q] = np.asarray(M).reshape((Nx,) * (p + q))
    return X


def _point(X, hyper, alpha, chol, kinv, z, S):
    N, Nx = X.shape
    Ny = hyper.shape[0]
    eye = np.eye(Nx)
    v = (X - z[None, :]).astype(LD)
    al = [alpha[a].astype(LD) for a in range(Ny)]
    lam = [hyper[a, :Nx] ** 2 for a in range(Ny)]
    D, logk = [], []
    for a in range(Ny):
        iRa = np.linalg.inv(S + np.diag(lam[a]))
        c = hyper[a, Nx] ** 2 * np.prod(hyper[a, :Nx]) / np.sqrt(np.linalg.det(S + np.diag(lam[a])))
        q = LD(c) * np.exp(-0.5 * np.sum((v @ iRa.astype(LD)) * v, 1))
        u = al[a] * q
        y = v @ iRa.astype(LD)
        G = [np.sum(u)] + [(u @ _outer_rows(y, k)).reshape((Nx,) * k) for k in range(1, 5)]
        D.append(hermite(G, iRa))
        logk.append(LD(2 * np.log(hyper[a, Nx])) - 0.5 * np.sum((v / hyper[a, :Nx].astype(LD)) ** 2, 1))
    Ck = {}
    for a in range(Ny):
        for b in range(a + 1):
            P = np.diag(1.0 / lam[a] + 1.0 / lam[b])
            C = np.linalg.inv(eye + P @ S)
            Fa = C / lam[a][None, :]; Fb = C / lam[b][None, :]
            CP = C @ P; CP = 0.5 * (CP + CP.T)
            Rm = S @ P + eye
            t = 1.0 / np.sqrt(np.linalg.det(Rm))
            Qm = np.linalg.solve(Rm, 0.5 * S).astype(LD)
            ii = v / lam[a].astype(LD); ij = v / lam[b].astype(LD)
            ea = logk[a] + np.sum((ii @ Qm) * ii, 1)
            eb = logk[b] + np.sum((ij @ Qm) * ij, 1)
            cr = 2 * (ii @ Qm) @ ij.T
            tQ = LD(t) * np.exp(ea[:, None] + eb[None, :] + cr)
            Ga = v @ Fa.T.astype(LD); Gb = v @ Fb.T.astype(LD)
            Pa = [_outer_rows(Ga, k) for k in range(5)]
            Pb = [_outer_rows(Gb, k) for k in range(5)]
            Xc = _bilinear(Pa, np.outer(al[a], al[b]) * tQ, Pb, Nx)
            G = [_subsets(k, Xc) for k in range(5)]
            cross = hermite(G, CP)
            out = [cross[k] - leibniz(D[a], D[b], k) for k in range(5)]
            if a == b:
                # backbone e e^T (e = exp(ea)) through L: rows e o g^(x)p, Gram of L^-1 rows for p, q <= 2
                e = np.exp(ea).astype(np.float64)
                Pe = [(e[:, None] * Pa[k].astype(np.float64)) for k in range(5)]
                Y = [solve_triangular(chol[a], Pe[k], lower=True) for k in range(3)]
                Ke = [cho_solve((chol[a], True), Pe[k]) for k in range(2)]
                Xb = [[None] * 5 for _ in range(5)]
                for p in range(5):
                    for q in range(5 - p):
                        if p <= 2 and q <= 2:
                            M = Y[p].T @ Y[q]
                        elif q <= 1:
                            M = Pe[p].T @ Ke[q]
                        else:
                            M = (Pe[q].T @ Ke[p]).T
                        Xb[p][q] = M.astype(LD).reshape((Nx,) * (p + q))
                Qr = np.exp(ea[:, None] + eb[None, :]) * np.expm1(cr)
                Xr = _bilinear(Pa, kinv[a].astype(LD) * Qr, Pa, Nx)
                Gt = [LD(t) * (_subsets(k, Xb) + _subsets(k, Xr)) for k in range(5)]
                tr = hermite(Gt, CP)
                out = [out[k] - tr[k] for k in range(5)]
            Ck[a, b] = Ck[b, a] = out
    f64 = lambda x: np.asarray(x, dtype=np.float64)
    res = {k: [] for k in KEYS}
    for a in range(Ny):
        res['d2mean_dz2'].append(f64(D[a][2]))
        res['d2mean_dSigma_dz'].append(f64(0.5 * D[a][3]))
        res['d2mean_dSigma2'].append(f64(0.25 * D[a][4]))
    c2 = np.zeros((Ny, Ny) + (Nx,) * 2); c3 = np.zeros((Ny, Ny) + (Nx,) * 3); c4 = np.zeros((Ny, Ny) + (Nx,) * 4)
    for a in range(Ny):
        for b in range(Ny):
            J = [f64(D[a][1]), f64(D[b][1])]; Hh = [f64(D[a][2]), f64(D[b][2])]; M3 = [f64(D[a][3]), f64(D[b][3])]
            C2, C3, C4 = f64(Ck[a, b][2]), f64(Ck[a, b][3]), f64(Ck[a, b][4])
            c2[a, b] = C2
            # d/dz_f of dcov/dSigma[d][e] = 1/2 C2 + 1/2 (J_a J_b^T + J_b J_a^T)
            c3[a, b] = 0.5 * C3
            for x, y in ((0, 1), (1, 0)):
                c3[a, b] += 0.5 * (np.einsum('df,e->def', Hh[x], J[y]) + np.einsum('d,ef->def', J[x], Hh[y]))
            # d/dSigma[f][g] of the same: 1/4 C4 + 1/4 d_d d_e (J_a,f J_b,g + J_b,f J_a,g) + 1/4 (dJ/dSigma terms)
            t4 = 0.25 * C4
            for x, y in ((0, 1), (1, 0)):
                t4 = t4 + 0.25 * (np.einsum('fde,g->defg', M3[x], J[y]) + np.einsum('fd,ge->defg', Hh[x], Hh[y])
                                  + np.einsum('fe,gd->defg', Hh[x], Hh[y]) + np.einsum('f,gde->defg', J[x], M3[y]))
                t4 = t4 + 0.25 * (np.einsum('dfg,e->defg', M3[x], J[y]) + np.einsum('d,efg->defg', J[x], M3[y]))
            c4[a, b] = t4
    res = {k: np.stack(vv) for k, vv in res.items() if vv}
    res.update(d2cov_dz2=c2, d2cov_dSigma_dz=c3, d2cov_dSigma2=c4)
    return res, D


def em_hess_closed(X, hyper, alpha, chol, Z, Sigma):
    """Closed-form 'EM' second derivatives (what gpmpc_predict_em_hess adds to gpmpc_predict_em_grad), shaped as its
    outputs with H first.  ``alpha`` (Ny,N) and ``chol`` (Ny,N,N) may be the engine's own.  Also returns d3mean_dz3
    (H,Ny,Nx,Nx,Nx) and d4mean_dz4 for the identities the tests check."""
    X = np.asarray(X, dtype=np.float64)
    Z = np.atleast_2d(np.asarray(Z, dtype=np.float64))
    hyper = np.atleast_2d(np.asarray(hyper, dtype=np.float64))
    alpha = np.atleast_2d(np.asarray(alpha, dtype=np.float64))
    H, Nx = Z.shape
    N = X.shape[0]
    kinv = []
    for c in chol:
        Ki = cho_solve((c, True), np.eye(N))
        kinv.append(0.5 * (Ki + Ki.T))
    Sg = emg._sigmas(Sigma, H, Nx)
    out = {k: [] for k in KEYS + ('d3mean_dz3', 'd4mean_dz4')}
    for h in range(H):
        r, D = _point(X, hyper, alpha, chol, kinv, Z[h], Sg[h])
        for k in KEYS:
            out[k].append(r[k])
        out['d3mean_dz3'].append(np.stack([np.asarray(d[3], dtype=np.float64) for d in D]))
        out['d4mean_dz4'].append(np.stack([np.asarray(d[4], dtype=np.float64) for d in D]))
    return {k: np.stack(v) for k, v in out.items()}


def em_hess_terms(X, hyper, alpha, chol, Z, Sigma):
    """Sums of |terms| that bound the entries of the order-k z-derivatives, in float64, per point: mean (H,Ny,5) with
    sum_i |beta_ai q_ai| (|y_i|_inf + max|S|^1/2)^k, and cov (H,Ny,Ny,5) with the same over the cross term's |beta beta tQ|,
    the product rule's sum_p C(k,p) mean_p(a) mean_(k-p)(b) and, for a = b, |K^-1 o tQ| of the trace term.  Errors of a
    block are normalised by the scale of its output (pair) and its highest z-order (2, 3, 4)."""
    from math import comb
    X = np.asarray(X, dtype=np.float64)
    Z = np.atleast_2d(np.asarray(Z, dtype=np.float64))
    hyper = np.atleast_2d(np.asarray(hyper, dtype=np.float64))
    H, Nx = Z.shape
    Ny, N = hyper.shape[0], X.shape[0]
    Sg = emg._sigmas(Sigma, H, Nx)
    kinv = [cho_solve((c, True), np.eye(N)) for c in chol]
    ks = np.arange(5)
    mean = np.zeros((H, Ny, 5)); cov = np.zeros((H, Ny, Ny, 5))
    for h in range(H):
        S = Sg[h]; v = X - Z[h][None, :]
        lam = [hyper[a, :Nx] ** 2 for a in range(Ny)]
        for a in range(Ny):
            iR = np.linalg.inv(S + np.diag(lam[a]))
            c = hyper[a, Nx] ** 2 * np.prod(hyper[a, :Nx]) / np.sqrt(np.linalg.det(S + np.diag(lam[a])))
            u = np.abs(alpha[a] * c * np.exp(-0.5 * np.sum((v @ iR) * v, 1)))
            r = np.abs(v @ iR).max(1) + np.sqrt(np.abs(iR).max())
            mean[h, a] = (u[:, None] * r[:, None] ** ks).sum(0)
        for a in range(Ny):
            for b in range(a + 1):
                P = np.diag(1.0 / lam[a] + 1.0 / lam[b])
                C = np.linalg.inv(np.eye(Nx) + P @ S)
                CP = C @ P
                t = 1.0 / np.sqrt(np.linalg.det(S @ P + np.eye(Nx)))
                Qm = np.linalg.solve(S @ P + np.eye(Nx), 0.5 * S)
                ii = v / lam[a]; ij = v / lam[b]
                la_ = 2 * np.log(hyper[a, Nx]) - 0.5 * np.sum(v * v / lam[a], 1)
                lb_ = 2 * np.log(hyper[b, Nx]) - 0.5 * np.sum(v * v / lam[b], 1)
                E = la_ + np.sum((ii @ Qm) * ii, 1); F = lb_ + np.sum((ij @ Qm) * ij, 1)
                tQ = t * np.exp(E[:, None] + F[None, :] + 2 * (ii @ Qm) @ ij.T)
                Ga = v @ (C / lam[a][None, :]).T; Gb = v @ (C / lam[b][None, :]).T
                g = np.abs(Ga[:, None, :] + Gb[None, :, :]).max(2) + np.sqrt(np.abs(CP).max())
                W = np.abs(np.outer(alpha[a], alpha[b]) * tQ)
                if a == b:
                    W = W + np.abs(kinv[a] * tQ)
                sc = np.array([(W * g ** k).sum() for k in ks])
                sc += np.array([sum(comb(k, p) * mean[h, a, p] * mean[h, b, k - p] for p in range(k + 1)) for k in ks])
                cov[h, a, b] = cov[h, b, a] = sc
    return dict(mean=mean, cov=cov)


def normalised_errors(o, ref, terms):
    """max |o - ref| of each block of the six outputs over the scale (em_hess_terms) of its output or pair and order"""
    out = {}
    for key, k in (('d2mean_dz2', 2), ('d2mean_dSigma_dz', 3), ('d2mean_dSigma2', 4)):
        err = np.abs(np.asarray(o[key]) - ref[key]).reshape(ref[key].shape[:2] + (-1,)).max(2)
        out[key] = float((err / terms['mean'][..., k]).max())
    for key, k in (('d2cov_dz2', 2), ('d2cov_dSigma_dz', 3), ('d2cov_dSigma2', 4)):
        err = np.abs(np.asarray(o[key]) - ref[key]).reshape(ref[key].shape[:3] + (-1,)).max(3)
        out[key] = float((err / terms['cov'][..., k]).max())
    return out
