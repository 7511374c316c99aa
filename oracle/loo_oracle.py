"""Leave-one-out cross-validation of a GP, restated in numpy (Rasmussen & Williams section 5.4.2, eqs. 5.10-5.14): what
gpmpc_loo and gpmpc_loo_nlpp compute.

With K = k(X, X) + sn2 I (+ the jitter if the factorisation needed it), C = K^-1 = Li^T Li, alpha = C y and
c_i = C_ii = sum_k Li[k][i]^2:

    LOO mean  mu_i = y_i - alpha_i / c_i,   LOO variance  s2_i = 1 / c_i   (of the noisy y_i),
    NLPP = sum_i [ 1/2 log 2pi - 1/2 log c_i + alpha_i^2 / (2 c_i) ]

and the gradient of the NLPP in theta = [ell_1..ell_Nx, sf, sn] (standard deviations), R&W eq. 5.13 with Z_j = C dK_j:

    dNLPP/dtheta_j = -sum_i [ alpha_i (Z_j alpha)_i - 1/2 (1 + alpha_i^2 / c_i) (Z_j C)_ii ] / c_i

which is the trace tr(W dK_j) with W = C diag(w) C - sym(b alpha^T), w_i = (1 + alpha_i^2 / c_i) / (2 c_i),
b = C (alpha / c).  The reference has no LOO; its validation needs a test set (gp_class.py:145-190).
"""
import numpy as np
from scipy.linalg import solve_triangular

from oracle import gp_oracle as orc

HALF_LOG_2PI = 0.5 * np.log(2 * np.pi)


def _factor(X, hyper_a):
    """(K with the jitter the factorisation used, L^-1)."""
    K = orc.assemble_K(X, hyper_a)
    L, jit = orc.chol_with_jitter(K)
    if jit:
        K = K + 1e-8 * np.eye(K.shape[0])
    return K, solve_triangular(L, np.eye(K.shape[0]), lower=True)


def closed_form(X, y, hyper_a):
    """dict(mean, var, nlpp, alpha, c, C) of the LOO predictions of every training point, from one factorisation."""
    y = np.asarray(y, dtype=np.float64).reshape(-1)
    _, Li = _factor(X, np.asarray(hyper_a, dtype=np.float64))
    C = Li.T @ Li
    alpha = Li.T @ (Li @ y)
    c = np.sum(Li * Li, axis=0)
    r = alpha / c
    nlpp = np.sum(HALF_LOG_2PI - 0.5 * np.log(c) + 0.5 * alpha * r)
    return dict(mean=y - r, var=1.0 / c, nlpp=nlpp, alpha=alpha, c=c, C=C)


def brute_force(X, y, hyper_a):
    """(mean, var, nlpp) by N drop-one refits: point i predicted by the GP on the other N-1 points (var includes sn2)."""
    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64).reshape(-1)
    K = orc.assemble_K(X, np.asarray(hyper_a, dtype=np.float64))
    N = X.shape[0]
    mean, var = np.empty(N), np.empty(N)
    for i in range(N):
        keep = np.r_[0:i, i + 1:N]
        L = np.linalg.cholesky(K[np.ix_(keep, keep)])
        v = solve_triangular(L, K[keep, i], lower=True)
        mean[i] = v @ solve_triangular(L, y[keep], lower=True)
        var[i] = K[i, i] - v @ v
    nlpp = np.sum(0.5 * np.log(2 * np.pi * var) + (y - mean) ** 2 / (2 * var))
    return mean, var, nlpp


def dK(X, hyper_a):
    """[dK/dell_1 .. dK/dell_Nx, dK/dsf, dK/dsn] as (Nx+2, N, N)."""
    X = np.asarray(X, dtype=np.float64)
    N, D = X.shape
    ell, sf, sn = hyper_a[:D], hyper_a[D], hyper_a[D + 1]
    Kf = orc.covSEard(X, X, ell, sf ** 2)
    out = np.empty((D + 2, N, N))
    for d in range(D):
        out[d] = Kf * (X[:, d][:, None] - X[:, d][None, :]) ** 2 / ell[d] ** 3
    out[D] = 2.0 * Kf / sf
    out[D + 1] = 2.0 * sn * np.eye(N)
    return out


def grad_eq513(X, y, hyper_a):
    """dNLPP/dtheta by R&W eq. 5.13 (one Z_j = C dK_j per hyper-parameter, O(N^3) each)."""
    cf = closed_form(X, y, hyper_a)
    C, alpha, c = cf['C'], cf['alpha'], cf['c']
    g = []
    for Dj in dK(X, np.asarray(hyper_a, dtype=np.float64)):
        Z = C @ Dj
        s = np.einsum('ik,ki->i', Z, C)
        g.append(-np.sum((alpha * (Z @ alpha) - 0.5 * (1.0 + alpha ** 2 / c) * s) / c))
    return np.array(g)


def w_matrix(X, y, hyper_a):
    """W = C diag(w) C - sym(b alpha^T): dNLPP/dtheta_j = tr(W dK_j)."""
    cf = closed_form(X, y, hyper_a)
    C, alpha, c = cf['C'], cf['alpha'], cf['c']
    w = (1.0 + alpha ** 2 / c) / (2.0 * c)
    b = C @ (alpha / c)
    return (C * w[None, :]) @ C - 0.5 * (np.outer(b, alpha) + np.outer(alpha, b))


def grad_trace(X, y, hyper_a):
    """dNLPP/dtheta as the traces tr(W dK_j): the form gpmpc_loo_nlpp evaluates."""
    W = w_matrix(X, y, hyper_a)
    return np.array([np.sum(W * Dj) for Dj in dK(X, np.asarray(hyper_a, dtype=np.float64))])


def grad_fd(X, y, hyper_a, rel=1e-3, f=None):
    """Five-point central differences of the NLPP (of f(theta) when given, e.g. an engine's value) with the step
    rel * |theta_j|: sn is about 1e-3 on the fixtures, so an absolute step would cross zero, and the NLPP of an
    ill-conditioned K carries cond(K) eps of noise that a short step amplifies."""
    f = f or (lambda t: closed_form(X, y, t)['nlpp'])
    hyper_a = np.asarray(hyper_a, dtype=np.float64)
    g = np.zeros_like(hyper_a)
    for j in range(hyper_a.size):
        h = rel * (abs(hyper_a[j]) or 1.0)
        e = np.zeros_like(hyper_a)
        e[j] = h
        g[j] = (8.0 * (f(hyper_a + e) - f(hyper_a - e)) - (f(hyper_a + 2 * e) - f(hyper_a - 2 * e))) / (12.0 * h)
    return g
