"""CPU oracle of the unscented transform ('UT', include/gpmpc.h GPMPC_METHOD_UT)  --  TEST INFRASTRUCTURE ONLY.

The rule, as the engine defines it, for n = Nx and parameters (alpha, beta, kappa):
  lambda = alpha^2 (n + kappa) - n,  c = sqrt(n + lambda)
  sigma points z_0 = z, z_{2j-1} = z + c S_j, z_{2j} = z - c S_j (j = 1..n), S the lower Cholesky factor of Sigma with a
  column set to zero where its pivot is <= 1e-14 max(diag Sigma) or <= 0
  W0m = lambda / (n + lambda), W0c = W0m + 1 - alpha^2 + beta, Wi = 1 / (2 (n + lambda))
  mean = sum_i Wim m_i,  cov = sum_i Wic (m_i - mean)(m_i - mean)^T + diag(sum_i Wim v_i)
The square root and the sums run in the engine's order with separate multiplies and adds (a Python loop over the index
that the sum runs over, vectorised over points), so the oracle's sigma points are what a correctly rounded evaluation of
the rule gives.  ``ut`` takes any callable of per-point means and variances; ``ut_me`` is the float64 'UT' of
``gp_oracle``'s 'ME' prediction.
"""
from __future__ import annotations

import numpy as np

from oracle import gp_oracle as orc

DEFAULT_PARAMS = (1.0, 0.0, 0.0)


def sqrt_psd(Sigma, rel_tol=1e-14):
    """Lower Cholesky factor S of Sigma (..., n, n), S S^T = Sigma, from its lower triangle, left-looking column by column;
    a pivot <= rel_tol max(diag Sigma) (or <= 0) makes its column exactly zero."""
    A = np.array(Sigma, dtype=np.float64)
    n = A.shape[-1]
    L = np.tril(A)
    tol = rel_tol * np.maximum(np.max(np.diagonal(A, axis1=-2, axis2=-1), axis=-1), 0.0)
    for j in range(n):
        d = L[..., j, j].copy()
        for k in range(j):
            d = d - L[..., j, k] * L[..., j, k]
        keep = d > tol
        piv = np.where(keep, np.sqrt(np.where(keep, d, 1.0)), 0.0)
        s = L[..., j + 1:, j].copy()
        for k in range(j):
            s = s - L[..., j + 1:, k] * L[..., j, k][..., None]
        L[..., j + 1:, j] = np.where(keep[..., None], s / np.where(keep, piv, 1.0)[..., None], 0.0)
        L[..., j, j] = piv
    return L


def weights(n, params=DEFAULT_PARAMS):
    """(c, Wm (2n+1,), Wc (2n+1,)) of the rule; the scalars are formed in the engine's operation order."""
    alpha, beta, kappa = (float(v) for v in params)
    a2 = alpha * alpha
    lam = a2 * (n + kappa) - n
    c = np.sqrt(n + lam)
    wi = 1.0 / (2.0 * (n + lam))
    wm = np.full(2 * n + 1, wi); wc = np.full(2 * n + 1, wi)
    wm[0] = lam / (n + lam)
    wc[0] = lam / (n + lam) + 1.0 - a2 + beta
    return float(c), wm, wc


def sigma_points(Z, Sigma, params=DEFAULT_PARAMS):
    """Z (H, n), Sigma (n, n) or (H, n, n) -> the sigma points (H, 2n+1, n) in the engine's order."""
    Z = np.atleast_2d(np.asarray(Z, dtype=np.float64))
    H, n = Z.shape
    S = sqrt_psd(np.broadcast_to(np.asarray(Sigma, dtype=np.float64), (H, n, n)))
    c = weights(n, params)[0]
    P = np.empty((H, 2 * n + 1, n))
    P[:, 0] = Z
    for j in range(n):
        s = c * S[:, :, j]
        P[:, 2 * j + 1] = Z + s
        P[:, 2 * j + 2] = Z - s
    return P


def combine(m, v, n, params=DEFAULT_PARAMS):
    """m, v (H, 2n+1, Ny): the means and variances at the sigma points -> mean (H, Ny), var (H, Ny), cov (H, Ny, Ny),
    every sum from point 0 in point order."""
    _, wm, wc = weights(n, params)
    H, P, Ny = m.shape
    mean = np.zeros((H, Ny)); sv = np.zeros((H, Ny))
    for k in range(P):
        mean = mean + wm[k] * m[:, k]
        sv = sv + wm[k] * v[:, k]
    cov = np.zeros((H, Ny, Ny))
    for k in range(P):
        d = m[:, k] - mean
        cov = cov + wc[k] * (d[:, :, None] * d[:, None, :])
    idx = np.arange(Ny)
    cov[:, idx, idx] = cov[:, idx, idx] + sv
    return mean, cov[:, idx, idx].copy(), cov


def ut(fun, Z, Sigma, params=DEFAULT_PARAMS):
    """The rule over any fun(points (M, n)) -> (means (M, Ny), variances (M, Ny)): mean, var, cov as ``combine``."""
    P = sigma_points(Z, Sigma, params)
    H, Np, n = P.shape
    m, v = fun(P.reshape(H * Np, n))
    m = np.asarray(m, dtype=np.float64).reshape(H, Np, -1)
    v = np.asarray(v, dtype=np.float64).reshape(H, Np, -1)
    return combine(m, v, n, params)


def ut_me(X, hyper, alpha, chol, Z, Sigma, params=DEFAULT_PARAMS):
    """float64 'UT' of gp_oracle's 'ME' (a fitted model's X, hyper, alpha, chol) -> mean, var, cov, jac, with jac the 'ME'
    Jacobian at Z."""
    mean, var, cov = ut(lambda P: orc.gp_mean_var(X, hyper, alpha, chol, P), Z, Sigma, params)
    return mean, var, cov, orc.gp_mean_jac(X, hyper, alpha, Z)
