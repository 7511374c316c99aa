"""Removal of training points from a factorised GP, restated in numpy: the O(N^2) update gpmpc_remove performs.

Removing point i from K = L L^T leaves K' whose trailing block is L33 L33^T + l32 l32^T = L33 (I + p p^T) L33^T with
p = L33^-1 l32 = -L[i][i] Li[i+1:, i].  With t_-1 = 1, t_r = t_{r-1} + p_r^2, d_r = sqrt(t_r / t_{r-1}) and
g_r = p_r / sqrt(t_r t_{r-1}):

    chol(I + p p^T) = diag(d) + strict_lower(p g^T),   its inverse  diag(1/d) - strict_lower(g p^T)

so the new trailing rows of L are L33 (diag(d) + strict_lower(p g^T)), a suffix sum along each row, and the new rows of
L^-1 are (diag(1/d) - strict_lower(g p^T)) R with R = Li[i+1:, cols != i] + p Li[i, cols != i], a prefix sum down each
column.  Rows above i are unchanged.  Every t_r >= 1: the update cannot lose positive definiteness.

The functions work on unpadded N x N factors.  The reference refits instead (replace_data_all, gp_class.py:553-626).
"""
import numpy as np


def coefficients(L, Li, i):
    """(p, d, g) of the removal of point i, each of length N - i - 1."""
    p = -L[i, i] * Li[i + 1:, i]
    t = 1.0 + np.cumsum(p * p)
    tp = np.concatenate([[1.0], t[:-1]])
    return p, np.sqrt(t / tp), p / np.sqrt(t * tp)


def remove_point(L, Li, i):
    """(L', Li') of the N-1 points left after removing point i (suffix / prefix sums, O(N^2))."""
    N = L.shape[0]
    keep = np.r_[0:i, i + 1:N]
    p, d, g = coefficients(L, Li, i)
    L2 = L[np.ix_(keep, keep)].copy()
    Li2 = Li[np.ix_(keep, keep)].copy()
    if i < N - 1:
        A = L[i + 1:, i + 1:]                                   # L33, lower triangular
        S = p[None, :] * A
        suffix = np.cumsum(S[:, ::-1], axis=1)[:, ::-1]          # sum over k >= j
        excl = np.concatenate([suffix[:, 1:], np.zeros((A.shape[0], 1))], axis=1)
        L2[i:, i:] = d[None, :] * A + g[None, :] * excl
        R = Li[i + 1:, keep] + p[:, None] * Li[i, keep][None, :]
        pre = np.cumsum(p[:, None] * R, axis=0)
        pre = np.concatenate([np.zeros((1, R.shape[1])), pre[:-1]], axis=0)   # sum over s < r
        Li2[i:, :] = R / d[:, None] - g[:, None] * pre
    return L2, Li2


def remove(L, Li, idx):
    """remove_point for every index in idx (indices before the call), in descending order, as gpmpc_remove does."""
    for i in sorted((int(k) for k in idx), reverse=True):
        L, Li = remove_point(L, Li, i)
    return L, Li


def append_point(L, Li, k, kss):
    """The rank-1 append of gpmpc_append: k = k(X, x_new), kss = k(x_new, x_new) + sn2."""
    l = Li @ k
    lam = np.sqrt(kss - l @ l)
    N = L.shape[0]
    L2 = np.zeros((N + 1, N + 1)); Li2 = np.zeros((N + 1, N + 1))
    L2[:N, :N] = L; Li2[:N, :N] = Li
    L2[N, :N] = l; L2[N, N] = lam
    Li2[N, :N] = -(l @ Li) / lam; Li2[N, N] = 1.0 / lam
    return L2, Li2


def alpha(Li, y):
    """K^-1 y = Li^T (Li y)."""
    return Li.T @ (Li @ y)
