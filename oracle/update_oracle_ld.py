"""The factor updates of gpmpc_append, gpmpc_append_greedy and gpmpc_remove in np.longdouble, applied to the engine's
own pre-update factor (GET_CHOL, GET_LINV: exact bits), with the sum of |terms| of every entry they form.

A ``Factor`` carries L and L^-1 of one output (N x N, lower) and SL, SLi: for each entry the sum of |terms| of the
sums that formed it, carried through every update (a fresh factor from the engine starts at |L|, |L^-1|).  Each
update evaluates its formulas on (L, Li) and the same formulas on (SL, SLi) with every subtraction turned into an
addition, so a kernel's rounding in any entry is measured against the scale of what that entry was summed from,
whatever cond(K) is.  The formulas and their order follow the kernels:

* append (append_row_kernel): l = L^-1 k, lambda^2 = kss - l^T l, row N of L^-1 = -(l^T L^-1) / lambda, 1 / lambda;
* remove (remove_* kernels, kernels.cuh; oracle/remove_oracle.py): p, d, g, the suffix sums along the rows of L and
  the prefix sums down the columns of the L^-1 rows, several indices one at a time in descending order;
* greedy (greedy_* kernels): the pool's V = L^-1 k and variances sf2 - |v|^2, the pick of the largest summed score
  (ties to the lowest index), the append from the gathered V row and the downdate of the rest of the pool.
"""
from collections import namedtuple

import numpy as np

LD = np.longdouble

Factor = namedtuple('Factor', 'L Li SL SLi')


def factor(L, Li):
    """A Factor from an engine's L and L^-1 (N x N): its entries are exact, their scales themselves."""
    L = np.asarray(L, dtype=LD)
    Li = np.asarray(Li, dtype=LD)
    return Factor(L, Li, np.abs(L), np.abs(Li))


def kvec(X, Z, hyper_a, scale=False):
    """k(X, Z) (N, H) of one output by direct differences, in long double; scale=True: (k, k (1 + q)), q the exponent's
    sum of squares, whose rounding the exponential carries into k."""
    X = np.asarray(X, dtype=LD)
    Z = np.atleast_2d(np.asarray(Z, dtype=LD))
    hyper_a = np.asarray(hyper_a, dtype=LD)
    Nx = X.shape[1]
    diff = (X[:, None, :] - Z[None, :, :]) / hyper_a[:Nx]
    q = np.sum(diff * diff, axis=2)
    k = hyper_a[Nx] ** 2 * np.exp(-q / 2)
    return (k, k * (1 + q)) if scale else k


def kss(hyper_a, jitter=0.0):
    """k(x, x) + sn2 + the jitter the output's factorisation used."""
    Nx = len(hyper_a) - 2
    return LD(hyper_a[Nx]) ** 2 + LD(hyper_a[Nx + 1]) ** 2 + LD(jitter)


def append_row(F, l, sl, kdiag):
    """(Factor with row N appended, lambda, its scale) from l = L^-1 k and its scale sl."""
    N = F.L.shape[0]
    lam2 = kdiag - l @ l
    slam2 = kdiag + 2 * np.abs(l) @ sl               # kdiag and the first-order error of l^T l
    lam = np.sqrt(lam2)
    slam = lam + slam2 / (2 * lam)                   # the rounding of the sqrt and the first-order error of lam2
    r = F.Li.T @ l
    sr = F.SLi.T @ sl
    L2, Li2, SL2, SLi2 = (np.zeros((N + 1, N + 1), dtype=LD) for _ in range(4))
    for dst, src in ((L2, F.L), (Li2, F.Li), (SL2, F.SL), (SLi2, F.SLi)):
        dst[:N, :N] = src
    L2[N, :N], L2[N, N] = l, lam
    SL2[N, :N], SL2[N, N] = sl, slam
    Li2[N, :N], Li2[N, N] = -r / lam, 1 / lam
    SLi2[N, :N], SLi2[N, N] = sr / lam + np.abs(r) * slam / lam ** 2, slam / lam ** 2
    return Factor(L2, Li2, SL2, SLi2), lam, slam


def append_point(F, X, x, hyper_a, jitter=0.0):
    """gpmpc_append of x to the training inputs X for one output: (Factor of N + 1 points, lambda, its scale)."""
    k, sk = kvec(X, x, hyper_a, scale=True)
    return append_row(F, F.Li @ k[:, 0], F.SLi @ sk[:, 0], kss(hyper_a, jitter))


def remove_point(F, i):
    """The Factor of the N - 1 points left after removing point i (every row below i rewritten)."""
    L, Li, SL, SLi = F
    N = L.shape[0]
    keep = np.r_[0:i, i + 1:N]
    out = [M[np.ix_(keep, keep)].copy() for M in F]
    if i == N - 1:
        return Factor(*out)
    L2, Li2, SL2, SLi2 = out
    p = -L[i, i] * Li[i + 1:, i]
    sp = SL[i, i] * SLi[i + 1:, i]
    t = 1 + np.cumsum(p * p)
    st = 1 + np.cumsum(sp * sp)
    tp = np.concatenate([[LD(1)], t[:-1]])
    stp = np.concatenate([[LD(1)], st[:-1]])
    rel = 1 + st / t + stp / tp                      # relative scale of d and of 1 / sqrt(t tp)
    d = np.sqrt(t / tp)
    g = p / np.sqrt(t * tp)
    sd = d * rel
    sg = sp / np.sqrt(t * tp) + np.abs(g) * rel
    # rows of L: d_j A_rj + g_j sum_{k > j} p_k A_rk (A = L33, lower)
    A, SA = L[i + 1:, i + 1:], SL[i + 1:, i + 1:]

    def suffix_excl(M):
        s = np.cumsum(M[:, ::-1], axis=1)[:, ::-1]
        return np.concatenate([s[:, 1:], np.zeros((M.shape[0], 1), dtype=LD)], axis=1)

    L2[i:, i:] = d * A + g * suffix_excl(p * A)
    SL2[i:, i:] = sd * SA + sg * suffix_excl(sp * SA)
    # rows of L^-1: R_r / d_r - g_r sum_{s < r} p_s R_s,  R_r = Li[i+1+r] + p_r Li[i] (column i dropped)
    R = Li[i + 1:][:, keep] + p[:, None] * Li[i, keep][None, :]
    SR = SLi[i + 1:][:, keep] + sp[:, None] * SLi[i, keep][None, :]

    def prefix_excl(M):
        s = np.cumsum(M, axis=0)
        return np.concatenate([np.zeros((1, M.shape[1]), dtype=LD), s[:-1]], axis=0)

    Li2[i:, :] = R / d[:, None] - g[:, None] * prefix_excl(p[:, None] * R)
    SLi2[i:, :] = SR * (sd / d ** 2)[:, None] + sg[:, None] * prefix_excl(sp[:, None] * SR)
    return Factor(L2, Li2, SL2, SLi2)


def remove(F, idx):
    """remove_point for every index of idx (indices before the call), in descending order, as gpmpc_remove does."""
    for i in sorted((int(k) for k in idx), reverse=True):
        F = remove_point(F, i)
    return F


def greedy(Fs, X, hyper, Xc, n_new, jitter=None):
    """gpmpc_append_greedy of n_new points of the pool Xc (n, Nx) for every output (Fs: one Factor per output, hyper
    their rows).  Returns dict(Fs (the updated Factors), picked (n_new,), score, sscore (the pick's summed variance and
    its scale), gap (n_new,): the smallest |score - score_c| / sscore over the active candidates c whose inputs differ
    from the pick's -- how far the pick is from a tie the device could break the other way)."""
    Xc = np.asarray(Xc, dtype=np.float64)
    n, Nx = Xc.shape
    Ny = len(Fs)
    jitter = np.zeros(Ny) if jitter is None else jitter
    K = [kvec(X, Xc, hyper[a], scale=True) for a in range(Ny)]      # (N, n) each
    V = [Fs[a].Li @ K[a][0] for a in range(Ny)]
    SV = [Fs[a].SLi @ K[a][1] for a in range(Ny)]
    sf2 = [LD(hyper[a, Nx]) ** 2 for a in range(Ny)]
    var = [sf2[a] - np.sum(V[a] * V[a], axis=0) for a in range(Ny)]
    svar = [sf2[a] + 2 * np.sum(np.abs(V[a]) * SV[a], axis=0) for a in range(Ny)]
    active = np.ones(n, dtype=bool)
    Fs = list(Fs)
    picked, score, sscore, gap = [], [], [], []
    for _ in range(int(n_new)):
        s = var[0].copy()
        ss = svar[0].copy()
        for a in range(1, Ny):
            s += var[a]
            ss += svar[a]
        s[~active] = -np.inf
        c = int(np.argmax(s))                                        # the first of equal maxima: the lowest index
        other = active & np.any(Xc != Xc[c], axis=1)
        gap.append(float(np.min(np.abs(s[c] - s[other]) / ss[c])) if other.any() else np.inf)
        picked.append(c)
        score.append(s[c])
        sscore.append(ss[c])
        active[c] = False
        for a in range(Ny):
            l, sl = V[a][:, c].copy(), SV[a][:, c].copy()
            Fs[a], lam, slam = append_row(Fs[a], l, sl, kss(hyper[a], jitter[a]))
            kc, skc = (x[0] for x in kvec(Xc[c:c + 1], Xc, hyper[a], scale=True))   # k(x*, c) for every candidate
            w = (kc - l @ V[a]) / lam
            sw = (skc + np.abs(l) @ SV[a] + sl @ np.abs(V[a])) / lam + np.abs(w) * slam / lam
            w[~active] = 0
            sw[~active] = 0
            V[a] = np.vstack([V[a], w])
            SV[a] = np.vstack([SV[a], sw])
            var[a] = var[a] - w * w
            svar[a] = svar[a] + 2 * np.abs(w) * sw
    return dict(Fs=Fs, picked=np.array(picked, dtype=np.int64), score=np.array(score), sscore=np.array(sscore),
                gap=np.array(gap))


def alpha(F, y):
    """(alpha = L^-T (L^-1 y), its scale) on the factor F."""
    y = np.asarray(y, dtype=LD)
    u = F.Li @ y
    su = F.SLi @ np.abs(y)
    return F.Li.T @ u, F.SLi.T @ su


def logdet(F):
    """(log det K = 2 sum log L_ii, its scale) on the factor F."""
    dg, sdg = np.diag(F.L), np.diag(F.SL)
    return 2 * np.sum(np.log(dg)), 2 * np.sum(np.abs(np.log(dg)) + sdg / dg)
