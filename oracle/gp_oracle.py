"""CPU oracle for the GP hot path of helgeanl/GP-MPC  --  TEST INFRASTRUCTURE ONLY.

This file is a numpy/LAPACK restatement of the reference's dense GP regression
path.  It is the checker, never the product: only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl
reference`` legs may import it.  Nothing under ``gp-mpc_b200/`` imports it.

Pinning status ("how do we know the oracle is right"):
  * The reference has NO tests; its only result-pinning artifacts are the two
    saved models ``examples/models/gp_{tank,car}_example.json``.  This oracle
    reproduces their stored ``chol`` / ``alpha`` / ``invK`` from the stored
    ``(X, Y, hyper)`` (``tests/test_oracle_golden.py``).
  * The reference's numpy-only functions (``optimize.calc_cov_matrix``,
    ``optimize.calc_NLL_numpy``, ``GP.covSEard``, ``GP.covar``) were imported
    VERBATIM in the build container (casadi/pyDOE/matplotlib stubbed, see
    ``oracle/ref_loader.py``) and their outputs on the fixtures are committed
    under ``tests/golden/`` by ``oracle/make_golden.py``; this oracle is checked
    against them.
  * The CasADi-only graph builders (``build_gp``, ``build_TA_cov``,
    ``gp_exact_moment``) cannot run here (CasADi, unpinned "tested with 3.4",
    README.md:21, is absent).  They are restated below following the cited
    lines; that part is "parity unpinned by reference execution" and is
    cross-checked by finite differences and limiting cases instead.

All citations are ``file:line`` relative to the reference checkout.
Arithmetic is fp64 throughout.
"""
from __future__ import annotations

import numpy as np

try:  # scipy is only needed for the triangular solves / SLSQP driver
    from scipy.linalg import solve_triangular as _solve_tri
except Exception:  # pragma: no cover
    _solve_tri = None


# ----------------------------------------------------------------------------
# a1  ARD squared-exponential kernel
# ----------------------------------------------------------------------------
def covSEard(X, Z, ell, sf2):
    """k(x,z) = sf2 * exp(-1/2 sum_d (x_d - z_d)^2 / ell_d^2), direct differences.

    Follows the CasADi kernel ``gp_functions.py:17-22`` (``(x - z)**2 / ell**2``
    summed, then one exp).  X:(n1,D)  Z:(n2,D)  ->  (n1,n2).
    """
    X = np.atleast_2d(np.asarray(X, dtype=np.float64))
    Z = np.atleast_2d(np.asarray(Z, dtype=np.float64))
    ell = np.asarray(ell, dtype=np.float64).reshape(-1)
    if X.shape[1] != Z.shape[1]:
        # same error behaviour as GP.covSEard, gp_class.py:342-344
        raise ValueError('Input dimensions are not the same! D_x=' + str(X.shape[1])
                         + ', D_z=' + str(Z.shape[1]))
    dist = np.zeros((X.shape[0], Z.shape[0]))
    for d in range(X.shape[1]):
        diff = X[:, d][:, None] - Z[:, d][None, :]
        dist += diff * diff / ell[d] ** 2
    return sf2 * np.exp(-0.5 * dist)


def covSEard_expanded(X, Z, ell, sf2):
    """Same kernel through the a^2 + b^2 - 2ab expansion per dimension.

    Follows the numeric twins ``optimize.py:303-319`` (``calc_cov_matrix``) and
    ``gp_class.py:345-350`` (``GP.covSEard``): per dimension
    ``(sum(x1**2) + sum(x2**2) - 2 x1 x2^T) / ell_i**2`` accumulated, one exp.
    """
    X = np.atleast_2d(np.asarray(X, dtype=np.float64))
    Z = np.atleast_2d(np.asarray(Z, dtype=np.float64))
    dist = 0
    n1, n2 = X.shape[0], Z.shape[0]
    for i in range(X.shape[1]):
        x1 = X[:, i].reshape(n1, 1)
        x2 = Z[:, i].reshape(n2, 1)
        dist = (np.sum(x1 ** 2, 1).reshape(-1, 1) + np.sum(x2 ** 2, 1)
                - 2 * np.dot(x1, x2.T)) / ell[i] ** 2 + dist
    return sf2 * np.exp(-.5 * dist)


def covSEard_blas(X, Z, ell, sf2):
    """The expansion form of ``optimize.py:303-319`` with the D per-dimension rank-1
    updates folded into one BLAS product on the pre-scaled inputs (same arithmetic up to
    summation order; used where N is too large for D full-size temporaries)."""
    X = np.atleast_2d(np.asarray(X, dtype=np.float64)) / np.asarray(ell, dtype=np.float64)
    Z = np.atleast_2d(np.asarray(Z, dtype=np.float64)) / np.asarray(ell, dtype=np.float64)
    d = -2.0 * (X @ Z.T)
    d += np.sum(X * X, 1)[:, None]
    d += np.sum(Z * Z, 1)[None, :]
    np.maximum(d, 0.0, out=d)
    d *= -0.5
    np.exp(d, out=d)
    d *= sf2
    return d


def calc_cov_matrix(X, ell, sf2):
    """``optimize.py:303-319``: K(X,X) without noise (expansion form)."""
    return covSEard_expanded(X, X, ell, sf2)


def mean_function(hyper_a, X, func='zero'):
    """``get_mean_function`` ``gp_functions.py:25-69`` evaluated numerically: parameters are the tail
    of the hyper row -- const: m = hyp[-1] (:46-50); linear: a = hyp[-Nx-1:-1], b = hyp[-1],
    m = a^T x + b (:51-56); polynomial: a = hyp[-2Nx-1:-Nx-1], b = hyp[-Nx-1:-1], c = hyp[-1],
    m = a^T x^2 + b^T x + c (:57-63).  X:(n,Nx) -> (n,)."""
    X = np.atleast_2d(np.asarray(X, dtype=np.float64))
    hyp = np.asarray(hyper_a, dtype=np.float64).reshape(-1)
    n, Nx = X.shape
    m = np.zeros(n)
    for i in range(n):                                   # the reference's per-point loop
        if func == 'zero':
            m[i] = 0.0
        elif func == 'const':
            m[i] = hyp[-1]
        elif func == 'linear':
            m[i] = np.dot(hyp[-Nx - 1:-1], X[i]) + hyp[-1]
        elif func == 'polynomial':
            m[i] = np.dot(hyp[-2 * Nx - 1:-Nx - 1], X[i] ** 2) + np.dot(hyp[-Nx - 1:-1], X[i]) + hyp[-1]
        else:
            raise NameError('No mean function called: ' + func)
    return m


# ----------------------------------------------------------------------------
# a2/a3  K assembly + Cholesky with the single 1e-8 jitter retry
# ----------------------------------------------------------------------------
def assemble_K(X, hyper_a):
    """``optimize.py:338-344`` / ``:476-482``: K = k(X,X) + sn2 I, symmetrised."""
    X = np.asarray(X, dtype=np.float64)
    n, D = X.shape
    ell = hyper_a[:D]
    sf2 = hyper_a[D] ** 2
    sn2 = hyper_a[D + 1] ** 2
    K = calc_cov_matrix(X, ell, sf2)
    K = K + sn2 * np.eye(n)
    K = (K + K.T) * 0.5
    return K


def chol_with_jitter(K, jitter=1e-8):
    """``optimize.py:345-350`` (= ``:483-488``, ``gp_class.py:524-529``).

    Returns (L, jitter_used).  A second failure propagates LinAlgError like the
    reference does.
    """
    try:
        return np.linalg.cholesky(K), False
    except np.linalg.LinAlgError:
        K = K + np.eye(K.shape[0]) * jitter
        return np.linalg.cholesky(K), True


# ----------------------------------------------------------------------------
# a4-a6  NLML (no N/2 log 2pi term, zero mean only)
# ----------------------------------------------------------------------------
def calc_NLL(hyper_a, X, y, lapack_general_solve=True):
    """``optimize.py:322-356`` (``calc_NLL_numpy``).

    ``lapack_general_solve=True`` reproduces the reference's use of
    ``np.linalg.solve`` (general LU) on the triangular factor (``:353-354``);
    False uses true triangular solves (results agree to rounding).
    """
    y = np.asarray(y, dtype=np.float64).reshape(-1)
    K = assemble_K(X, np.asarray(hyper_a, dtype=np.float64))
    L, _ = chol_with_jitter(K)
    logK = 2 * np.sum(np.log(np.abs(np.diag(L))))            # :352
    if lapack_general_solve or _solve_tri is None:
        invLy = np.linalg.solve(L, y)                        # :353
        alpha = np.linalg.solve(L.T, invLy)                  # :354
    else:
        invLy = _solve_tri(L, y, lower=True)
        alpha = _solve_tri(L.T, invLy, lower=False)
    return 0.5 * np.dot(y.T, alpha) + 0.5 * logK             # :355


def calc_NLL_grad_fd(hyper_a, X, y, rel=1e-6):
    """Central differences of ``calc_NLL`` -- the oracle for the analytic
    gradient the GPU engine adds (the reference has none: SLSQP uses forward
    differences, ``optimize.py:466-467``)."""
    hyper_a = np.asarray(hyper_a, dtype=np.float64)
    g = np.zeros_like(hyper_a)
    for j in range(hyper_a.size):
        h = rel * max(1.0, abs(hyper_a[j]))
        hp = hyper_a.copy(); hp[j] += h
        hm = hyper_a.copy(); hm[j] -= h
        g[j] = (calc_NLL(hp, X, y, False) - calc_NLL(hm, X, y, False)) / (2 * h)
    return g


def calc_NLL_grad_analytic(hyper_a, X, y):
    """Closed-form gradient (Rasmussen & Williams eq. 5.9) in the reference's
    parametrisation hyper=[ell.., sf, sn] (standard deviations, not logs,
    ``gp_class.py:139-142``).  d/dtheta = 1/2 tr((K^-1 - alpha alpha^T) dK/dtheta).
    CPU cross-check of the GPU gradient kernel; validated against
    ``calc_NLL_grad_fd`` in tests."""
    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64).reshape(-1)
    hyper_a = np.asarray(hyper_a, dtype=np.float64)
    n, D = X.shape
    ell = hyper_a[:D]; sf = hyper_a[D]; sn = hyper_a[D + 1]
    Kf = covSEard(X, X, ell, sf ** 2)
    K = Kf + sn ** 2 * np.eye(n)
    L = np.linalg.cholesky(K)
    Linv = _solve_tri(L, np.eye(n), lower=True)
    Kinv = Linv.T @ Linv
    alpha = Kinv @ y
    W = Kinv - np.outer(alpha, alpha)
    g = np.zeros(D + 2)
    for d in range(D):
        diff2 = (X[:, d][:, None] - X[:, d][None, :]) ** 2
        g[d] = 0.5 * np.sum(W * Kf * diff2) / ell[d] ** 3
    g[D] = 0.5 * np.sum(W * Kf) * 2.0 / sf
    g[D + 1] = 0.5 * np.trace(W) * 2.0 * sn
    return g


# ----------------------------------------------------------------------------
# a5  post-fit block: chol, invK, alpha per output
# ----------------------------------------------------------------------------
def postfit(X, Y, hyper, lapack_general_solve=True, mean_func='zero'):
    """``optimize.py:472-494`` (twins ``:267-285``, ``gp_class.py:516-537``).

    hyper:(Ny, Nx+2[+mean params]); zero prior mean ('zero' mean function, the
    only one the numpy path supports, ``optimize.py:377-379``).
    Returns dict(chol:(Ny,N,N) lower with zeros above, alpha:(Ny,N),
    invK:(Ny,N,N), jitter:(Ny,) bool).
    """
    X = np.asarray(X, dtype=np.float64)
    Y = np.asarray(Y, dtype=np.float64)
    hyper = np.atleast_2d(np.asarray(hyper, dtype=np.float64))
    N = X.shape[0]
    Ny = hyper.shape[0]
    chol = np.zeros((Ny, N, N)); invK = np.zeros((Ny, N, N)); alpha = np.zeros((Ny, N))
    jit = np.zeros(Ny, dtype=bool)
    for a in range(Ny):
        K = assemble_K(X, hyper[a])
        L, jit[a] = chol_with_jitter(K)
        if lapack_general_solve or _solve_tri is None:
            invL = np.linalg.solve(L, np.eye(N))                         # :489
            invK[a] = np.linalg.solve(L.T, invL)                         # :490
            alpha[a] = np.linalg.solve(L.T, np.linalg.solve(L, Y[:, a] - mean_function(hyper[a], X, mean_func)))  # :492-494
        else:
            invL = _solve_tri(L, np.eye(N), lower=True)
            invK[a] = _solve_tri(L.T, invL, lower=False)
            alpha[a] = _solve_tri(L.T, _solve_tri(L, Y[:, a] - mean_function(hyper[a], X, mean_func), lower=True), lower=False)
        chol[a] = L                                                      # :491
    return dict(chol=chol, alpha=alpha, invK=invK, jitter=jit)


def factor_large(X, y, hyper_a):
    """Post-fit block ``optimize.py:476-494`` for ONE output at the BASELINE sizes
    (N = 4096 ... 16384), where ``postfit`` (Nx full-size temporaries per K, dense invK) is
    too slow for a test: K through ``covSEard_blas`` (the reference's expansion with the
    per-dimension rank-1 updates folded into one BLAS product), ``np.linalg.cholesky`` with
    the single 1e-8 jitter retry (:483-488), alpha by true triangular solves (q11) and the
    NLL of ``optimize.py:352-355``.  invK is not formed.
    Returns dict(chol, alpha, nll, jitter)."""
    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64).reshape(-1)
    hyper_a = np.asarray(hyper_a, dtype=np.float64)
    n, D = X.shape
    K = covSEard_blas(X, X, hyper_a[:D], hyper_a[D] ** 2)
    K[np.diag_indices(n)] += hyper_a[D + 1] ** 2
    K = (K + K.T) * 0.5                                        # :482
    L, jit = chol_with_jitter(K)
    del K
    invLy = _solve_tri(L, y, lower=True, check_finite=False)
    alpha = _solve_tri(L, invLy, lower=True, trans='T', check_finite=False)
    nll = 0.5 * float(np.dot(y, alpha)) + float(np.sum(np.log(np.abs(np.diag(L)))))
    return dict(chol=L, alpha=alpha, nll=nll, jitter=jit)


def predict_large(X, hyper_a, alpha_a, L_a, Z):
    """Numeric predict of ONE output for a batch (``gp_functions.py:111-147``; the numeric twin
    ``GP.covar`` ``gp_class.py:353-381``) with BLAS-folded ks and Jacobian sums, for the
    BASELINE sizes: mean (H,), var (H,), J (H,Nx)."""
    X = np.asarray(X, dtype=np.float64)
    Z = np.atleast_2d(np.asarray(Z, dtype=np.float64))
    Nx = X.shape[1]
    ell = np.asarray(hyper_a[:Nx], dtype=np.float64); sf2 = float(hyper_a[Nx]) ** 2
    ks = covSEard(X, Z, ell, sf2) if X.shape[0] * Z.shape[0] <= (1 << 22) else covSEard_blas(X, Z, ell, sf2)
    mean = ks.T @ alpha_a
    v = _solve_tri(L_a, ks, lower=True, check_finite=False)
    var = sf2 - np.sum(v * v, axis=0)
    w = ks * alpha_a[:, None]                                  # (N,H)
    # J[h,d] = sum_i w_ih (X_id - z_hd)/ell_d^2 = ((X^T w)_dh - z_hd sum_i w_ih)/ell_d^2
    J = ((X.T @ w).T - Z * np.sum(w, axis=0)[:, None]) / ell[None, :] ** 2
    return mean, var, J


# ----------------------------------------------------------------------------
# a8/a9/a10  posterior mean / variance / Jacobian / Taylor covariance
# ----------------------------------------------------------------------------
def gp_mean_var(X, hyper, alpha, chol, Z, lapack_general_solve=False):
    """Restatement of ``build_gp`` ``gp_functions.py:111-136`` for a batch.

    per output a:  ks_i = covSE(X_i, z, ell_a, sf2_a)        (:114-117,132)
                   mean_a = ks^T alpha_a + 0                 (:119-120,135; the
                       prior mean is always 'zero' because GP.__init__ never
                       forwards meanFunc, gp_class.py:69-71)
                   v = L_a \\ ks ;  var_a = sf2_a - v^T v      (:122-126,133,136)
    Z:(H,Nx) in the GP's (standardised) input space.  Returns mean:(H,Ny),
    var:(H,Ny).  Noise is NOT added (q3).
    """
    X = np.asarray(X, dtype=np.float64)
    Z = np.atleast_2d(np.asarray(Z, dtype=np.float64))
    hyper = np.atleast_2d(np.asarray(hyper, dtype=np.float64))
    Ny = hyper.shape[0]
    Nx = X.shape[1]
    H = Z.shape[0]
    mean = np.zeros((H, Ny)); var = np.zeros((H, Ny))
    for a in range(Ny):
        ell = hyper[a, :Nx]; sf2 = hyper[a, Nx] ** 2
        ks = covSEard(X, Z, ell, sf2)                       # (N,H)
        mean[:, a] = ks.T @ alpha[a]
        if lapack_general_solve or _solve_tri is None:
            v = np.linalg.solve(chol[a], ks)                # GP.covar style, gp_class.py:379
        else:
            v = _solve_tri(chol[a], ks, lower=True)         # ca.solve on lower-sparsity L
        var[:, a] = sf2 - np.sum(v * v, axis=0)
    return mean, var


def gp_mean_jac(X, hyper, alpha, Z):
    """Closed form of ``ca.jacobian(mean_func(z), z)`` ``gp_functions.py:146-147``:
    J[a,d] = sum_i alpha_{a,i} ks_i (X_{i,d} - z_d) / ell_{a,d}^2.
    Returns (H,Ny,Nx).  Cross-checked by central differences in tests."""
    X = np.asarray(X, dtype=np.float64)
    Z = np.atleast_2d(np.asarray(Z, dtype=np.float64))
    hyper = np.atleast_2d(np.asarray(hyper, dtype=np.float64))
    Ny = hyper.shape[0]; Nx = X.shape[1]; H = Z.shape[0]
    J = np.zeros((H, Ny, Nx))
    for a in range(Ny):
        ell = hyper[a, :Nx]; sf2 = hyper[a, Nx] ** 2
        ks = covSEard(X, Z, ell, sf2)                       # (N,H)
        w = ks * alpha[a][:, None]                          # (N,H)
        for d in range(Nx):
            diff = X[:, d][:, None] - Z[:, d][None, :]      # (N,H)
            J[:, a, d] = np.sum(w * diff, axis=0) / ell[d] ** 2
    return J


def ta_cov(var, J, Sigma):
    """``build_TA_cov`` ``gp_functions.py:167-171``: diag(var) + J Sigma J^T.
    var:(H,Ny) J:(H,Ny,Nx) Sigma:(Nx,Nx) or (H,Nx,Nx) -> (H,Ny,Ny)."""
    var = np.asarray(var); J = np.asarray(J)
    H, Ny = var.shape
    Sigma = np.asarray(Sigma, dtype=np.float64)
    if Sigma.ndim == 2:
        Sigma = np.broadcast_to(Sigma, (H,) + Sigma.shape)
    cov = np.zeros((H, Ny, Ny))
    for h in range(H):
        cov[h] = np.diag(var[h]) + J[h] @ Sigma[h] @ J[h].T
    return cov


def me_cov(var):
    """'ME' covariance ``gp_functions.py:142`` / ``gp_class.py:213-215``: diag(var)."""
    var = np.asarray(var)
    H, Ny = var.shape
    cov = np.zeros((H, Ny, Ny))
    for h in range(H):
        cov[h] = np.diag(var[h])
    return cov


# ----------------------------------------------------------------------------
# 'EM' exact moment matching  (next-row f2; restated for parity tests)
# ----------------------------------------------------------------------------
def _maha(a1, b1, Q1):
    """``maha`` ``gp_functions.py:421-430``."""
    aQ = a1 @ Q1
    bQ = b1 @ Q1
    return (np.sum(aQ * a1, 1)[:, None] + np.sum(bQ * b1, 1)[None, :]
            - 2 * aQ @ b1.T)


def gp_exact_moment(invK, X, Y, hyper, inputmean, inputcov, extended=False, beta=None):
    """``gp_exact_moment`` ``gp_functions.py:344-418``, one test point.

    ``extended=True`` evaluates the N x N sums (which cancel ~6-7 digits: beta beta^T vs
    invK) in numpy longdouble -- a higher-precision yardstick for judging fp64 noise.
    ``beta`` (Ny, N), e.g. an engine's own alpha, replaces the reference's ``invK @ Y`` (the
    default), so a comparison can separate the evaluation's error from alpha's conditioning.

    Quirks kept: hyper=log(hyper) then exponentiated (:367); det through the
    product of the QR diagonal (:378-380) -- restated with slogdet's value
    (identical when the QR diagonal is positive, NaN otherwise in the
    reference); ``A -= invK[a]`` on the diagonal blocks (:410-411); ``+sf2``
    (:415); ``- mean mean^T`` (:416).  Returns mean:(Ny,), cov:(Ny,Ny)
    (standardised space; zero prior mean).
    """
    X = np.asarray(X, dtype=np.float64); Y = np.asarray(Y, dtype=np.float64)
    hyper = np.atleast_2d(np.asarray(hyper, dtype=np.float64))
    inputmean = np.asarray(inputmean, dtype=np.float64).reshape(1, -1)
    inputcov = np.asarray(inputcov, dtype=np.float64)
    beta_in = None if beta is None else np.asarray(beta, dtype=np.float64)
    lh = np.log(hyper)
    Ny = len(invK)
    N, Nx = X.shape
    mean = np.zeros(Ny); beta = np.zeros((N, Ny)); log_k = np.zeros((N, Ny))
    v = X - np.repeat(inputmean, N, 0)
    covariance = np.zeros((Ny, Ny))
    det = np.linalg.det
    eye = np.eye(Nx)
    for a in range(Ny):
        beta[:, a] = invK[a] @ Y[:, a] if beta_in is None else beta_in[a]
        iLambda = np.diag(np.exp(-2 * lh[a, :Nx]))
        R = inputcov + np.diag(np.exp(2 * lh[a, :Nx]))
        iR = iLambda @ (eye - np.linalg.solve(eye + inputcov @ iLambda, inputcov @ iLambda))
        T = v @ iR
        c = np.exp(2 * lh[a, Nx]) / np.sqrt(det(R)) * np.exp(np.sum(lh[a, :Nx]))
        q2 = c * np.exp(-np.sum(T * v, 1) * 0.5)
        qb = q2 * beta[:, a]
        mean[a] = np.sum(qb)
        t = np.repeat(np.exp(lh[a, :Nx]).reshape(1, -1), N, 0)
        v1 = v / t
        log_k[:, a] = 2 * lh[a, Nx] - np.sum(v1 * v1, 1) * 0.5
    for a in range(Ny):
        ii = v / np.exp(2 * lh[a, :Nx])[None, :]
        for b in range(a + 1):
            R = inputcov @ np.diag(np.exp(-2 * lh[a, :Nx]) + np.exp(-2 * lh[b, :Nx])) + eye
            t = 1.0 / np.sqrt(det(R))
            ij = v / np.exp(2 * lh[b, :Nx])[None, :]
            Qm = np.linalg.solve(R, inputcov * 0.5)
            if extended:
                ld = np.longdouble
                Q = np.exp(log_k[:, a].astype(ld)[:, None] + log_k[:, b].astype(ld)[None, :]
                           + _maha(ii.astype(ld), -ij.astype(ld), Qm.astype(ld)))
                A = np.outer(beta[:, a].astype(ld), beta[:, b].astype(ld))
                if b == a:
                    A = A - np.asarray(invK[a]).astype(ld)
                covariance[a, b] = float(t * np.sum(A * Q))
                covariance[b, a] = covariance[a, b]
                continue
            Q = np.exp(log_k[:, a][:, None] + log_k[:, b][None, :] + _maha(ii, -ij, Qm))
            A = np.outer(beta[:, a], beta[:, b])
            if b == a:
                A = A - invK[a]
            A = A * Q
            covariance[a, b] = t * np.sum(A)
            covariance[b, a] = covariance[a, b]
        covariance[a, a] = covariance[a, a] + np.exp(2 * lh[a, Nx])
    covariance = covariance - np.outer(mean, mean)
    return mean, covariance


def gp_exact_moment_mp(X, Y, hyper, inputmean, inputcov, dps=40):
    """The formula of ``gp_exact_moment`` (``gp_functions.py:344-418``) evaluated in ``dps``-digit
    arithmetic (mpmath) FROM (X, Y, hyper): K, K^-1, beta = K^-1 y and every N x N sum are exact to
    ~dps digits, so this is what the reference's expression means mathematically -- the yardstick
    for any fp64 evaluation (the fp64 restatement above loses 4-8 digits to the beta beta^T - invK
    cancellation; the GPU engine evaluates an algebraically identical, better conditioned form).
    Slow (pure Python): used offline by ``oracle/make_golden_em.py``.  Returns mean:(Ny,), cov:(Ny,Ny)."""
    import mpmath as mp
    mp.mp.dps = dps
    X = np.asarray(X, dtype=np.float64); Y = np.asarray(Y, dtype=np.float64)
    hyper = np.atleast_2d(np.asarray(hyper, dtype=np.float64))
    mu = [mp.mpf(float(t)) for t in np.asarray(inputmean, dtype=np.float64).reshape(-1)]
    N, Nx = X.shape
    Ny = hyper.shape[0]
    S = mp.matrix([[mp.mpf(float(inputcov[i, j])) for j in range(Nx)] for i in range(Nx)])
    Xm = [[mp.mpf(float(X[i, d])) for d in range(Nx)] for i in range(N)]
    v = [[Xm[i][d] - mu[d] for d in range(Nx)] for i in range(N)]
    eye = mp.eye(Nx)
    ell2 = [[mp.mpf(float(hyper[a, d])) ** 2 for d in range(Nx)] for a in range(Ny)]
    sf2 = [mp.mpf(float(hyper[a, Nx])) ** 2 for a in range(Ny)]
    sn2 = [mp.mpf(float(hyper[a, Nx + 1])) ** 2 for a in range(Ny)]
    invK = []; beta = []; q = []; logk = []
    for a in range(Ny):
        K = mp.matrix(N, N)
        for i in range(N):
            for j in range(i + 1):
                d2 = sum((Xm[i][d] - Xm[j][d]) ** 2 / ell2[a][d] for d in range(Nx))
                K[i, j] = K[j, i] = sf2[a] * mp.exp(-d2 / 2)
            K[i, i] += sn2[a]
        Ki = K ** -1
        invK.append(Ki)
        beta.append(Ki * mp.matrix([mp.mpf(float(Y[i, a])) for i in range(N)]))
        R = S + mp.diag(ell2[a])                                         # :383
        iR = R ** -1
        c = sf2[a] / mp.sqrt(mp.det(R)) * mp.sqrt(mp.fprod(ell2[a]))   # :386-387 (prod ell = sqrt(prod ell^2))
        qa = []
        for i in range(N):
            vi = mp.matrix(v[i])
            qa.append(c * mp.exp(-(vi.T * iR * vi)[0] / 2))              # :385,388
        q.append(qa)
        logk.append([mp.log(sf2[a]) - sum(v[i][d] ** 2 / ell2[a][d] for d in range(Nx)) / 2 for i in range(N)])  # :389-391
    mean = [sum(q[a][i] * beta[a][i] for i in range(N)) for a in range(Ny)]
    cov = np.zeros((Ny, Ny))
    for a in range(Ny):
        ii = [mp.matrix([v[i][d] / ell2[a][d] for d in range(Nx)]) for i in range(N)]
        for b in range(a + 1):
            ij = [mp.matrix([v[i][d] / ell2[b][d] for d in range(Nx)]) for i in range(N)]
            R = S * mp.diag([1 / ell2[a][d] + 1 / ell2[b][d] for d in range(Nx)]) + eye     # :396-397
            t = 1 / mp.sqrt(mp.det(R))
            Qm = (R ** -1) * S / 2                                      # :402
            Qi = [Qm.T * ii[i] for i in range(N)]                       # maha(ii, -ij, Qm) = (ii+ij)^T Qm (ii+ij)
            Qj = [Qm * ij[j] for j in range(N)]
            dii = [(ii[i].T * Qm * ii[i])[0] for i in range(N)]
            djj = [(ij[j].T * Qm * ij[j])[0] for j in range(N)]
            acc = mp.mpf(0)
            for i in range(N):
                for j in range(N):
                    mh = dii[i] + djj[j] + (ii[i].T * Qj[j])[0] + (Qi[i].T * ij[j])[0]
                    Aij = beta[a][i] * beta[b][j] - (invK[a][i, j] if a == b else 0)      # :409-411
                    acc += Aij * mp.exp(logk[a][i] + logk[b][j] + mh)
            cab = t * acc
            if a == b:
                cab += sf2[a]                                           # :415
            cab -= mean[a] * mean[b]                                    # :416
            cov[a, b] = cov[b, a] = float(cab)
    return np.array([float(m) for m in mean]), cov


# ----------------------------------------------------------------------------
# a11/a12/a13  predict wrapper, linearisation, scalers
# ----------------------------------------------------------------------------
def standardize(v, mean, std):
    """``gp_class.py:629-630`` / ``optimize.py:580-582``."""
    return (v - mean) / std


def inverse_mean(x, mean, std):
    """``gp_class.py:635-638``."""
    return (x * std) + mean


def data_stats(X, Y, Ny):
    """``GP.optimize`` ``gp_class.py:92-99`` (population std, ddof=0)."""
    X = np.asarray(X, dtype=np.float64); Y = np.asarray(Y, dtype=np.float64)
    return dict(meanY=np.mean(Y, 0), stdY=np.std(Y, 0),
                meanZ=np.mean(X, 0), stdZ=np.std(X, 0),
                meanX=np.mean(X[:, :Ny], 0), stdX=np.std(X[:, :Ny], 0),
                meanU=np.mean(X[:, Ny:], 0), stdU=np.std(X[:, Ny:], 0))


def predict(model, x, u, cov, method='TA'):
    """``GP.predict`` ``gp_class.py:245-263`` + ``set_method`` ``:212-224``.

    ``model`` = dict(X, Y, hyper, alpha, chol, invK, normalize, meta).
    Standardises x,u when normalize (:253-255); the input covariance is used
    as-is and the output covariance is NOT rescaled (:259-262, q4); the mean is
    de-standardised (:260).  Returns mean:(Ny,1), cov:(Ny,Ny) like the DMs the
    reference returns.
    """
    X = model['X']; hyper = model['hyper']
    Ny = np.atleast_2d(hyper).shape[0]
    x = np.asarray(x, dtype=np.float64).reshape(-1)
    u = np.asarray(u, dtype=np.float64).reshape(-1)
    if model.get('normalize', False):
        m = model['meta']
        x_s = standardize(x, np.asarray(m['meanX']), np.asarray(m['stdX']))
        u_s = standardize(u, np.asarray(m['meanU']), np.asarray(m['stdU']))
    else:
        x_s, u_s = x, u
    z = np.concatenate([x_s, u_s]).reshape(1, -1)
    if method == 'ME':
        mean, var = gp_mean_var(X, hyper, model['alpha'], model['chol'], z)
        c = me_cov(var)[0]; mu = mean[0]
    elif method == 'TA':
        mean, var = gp_mean_var(X, hyper, model['alpha'], model['chol'], z)
        J = gp_mean_jac(X, hyper, model['alpha'], z)
        c = ta_cov(var, J, np.asarray(cov, dtype=np.float64))[0]; mu = mean[0]
    elif method == 'EM':
        mu, c = gp_exact_moment(model['invK'], X, model['Y'], hyper, z, cov)
    else:
        raise NameError('No GP method called: ' + method)      # gp_class.py:237
    if model.get('normalize', False):
        mu = inverse_mean(mu, np.asarray(model['meta']['meanY']), np.asarray(model['meta']['stdY']))
    return mu.reshape(Ny, 1), c


def discrete_linearize(model, x0, u0, cov0=None):
    """``GP.discrete_linearize`` ``gp_class.py:647-661`` for methods ME/TA:
    A = d mean / d x, B = d mean / d u of the (standardised-space) predictor
    (``:239-242``); inputs standardised when normalize (:656-658), outputs not
    rescaled."""
    hyper = model['hyper']
    Ny = np.atleast_2d(hyper).shape[0]
    x0 = np.asarray(x0, dtype=np.float64).reshape(-1)
    u0 = np.asarray(u0, dtype=np.float64).reshape(-1)
    if model.get('normalize', False):
        m = model['meta']
        x0 = standardize(x0, np.asarray(m['meanX']), np.asarray(m['stdX']))
        u0 = standardize(u0, np.asarray(m['meanU']), np.asarray(m['stdU']))
    z = np.concatenate([x0, u0]).reshape(1, -1)
    J = gp_mean_jac(model['X'], hyper, model['alpha'], z)[0]
    return J[:, :Ny].copy(), J[:, Ny:].copy()


def covar(model, X_new):
    """``GP.covar`` ``gp_class.py:353-381``: per output full posterior
    covariance ``kss - v^T v`` between the rows of X_new, in the oddly shaped
    (D,n,n) buffer of which only the first Ny slabs are filled (q12)."""
    X_new = np.atleast_2d(np.asarray(X_new, dtype=np.float64))
    n, D = X_new.shape
    hyper = np.atleast_2d(model['hyper'])
    Ny = hyper.shape[0]; Nx = model['X'].shape[1]
    out = np.zeros((D, n, n))
    for a in range(Ny):
        ell = hyper[a, :Nx]; sf2 = hyper[a, Nx] ** 2
        ks = covSEard_expanded(model['X'], X_new, ell, sf2)
        v = np.linalg.solve(model['chol'][a], ks)
        out[a] = sf2 - v.T @ v
    return out


def validate(model, X_test, Y_test):
    """``GP.validate`` ``gp_class.py:145-190``: SMSE = MSE/std(Y_test) (q15),
    MNLP with var + sn2 (:161).  Returns (SMSE, MNLP), each (Ny,)."""
    X_test = np.asarray(X_test, dtype=np.float64).copy()
    Y_test = np.asarray(Y_test, dtype=np.float64).copy()
    hyper = np.atleast_2d(model['hyper'])
    Nx = model['X'].shape[1]
    if model.get('normalize', False):
        m = model['meta']
        Y_test = standardize(Y_test, np.asarray(m['meanY']), np.asarray(m['stdY']))
        X_test = standardize(X_test, np.asarray(m['meanZ']), np.asarray(m['stdZ']))
    N = Y_test.shape[0]
    mean, var = gp_mean_var(model['X'], hyper, model['alpha'], model['chol'], X_test)
    var = var + (hyper[:, Nx + 1] ** 2)[None, :]
    loss = np.sum((Y_test - mean) ** 2, 0) / N
    NLP = np.sum(0.5 * np.log(2 * np.pi * var) + (Y_test - mean) ** 2 / (2 * var), 0)
    SMSE = loss / np.std(Y_test, 0)
    MNLP = NLP / N
    return SMSE.flatten(), MNLP.flatten()


# ----------------------------------------------------------------------------
# a7  hyper-parameter fit driver (SLSQP, finite differences)
# ----------------------------------------------------------------------------
def train_bounds_init(X, y):
    """Bounds and initial point of ``train_gp_numpy`` ``optimize.py:433-451``
    (zero mean).  NB ``lb[:Nx] = 1-2`` = -1 is the reference's typo (q7)."""
    X = np.asarray(X, dtype=np.float64)
    N, Nx = X.shape
    num_hyp = Nx + 2
    lb = -np.inf * np.ones(num_hyp); ub = np.inf * np.ones(num_hyp)
    lb[:Nx] = 1 - 2
    ub[:Nx] = 2e2
    lb[Nx] = 1e-8
    ub[Nx] = 1e2
    lb[Nx + 1] = 10 ** -10
    ub[Nx + 1] = 10 ** -2
    bounds = np.hstack((lb.reshape(num_hyp, 1), ub.reshape(num_hyp, 1)))
    hyp_init = np.zeros(num_hyp)
    hyp_init[:Nx] = np.std(X, 0)
    hyp_init[Nx] = np.std(y)
    hyp_init[Nx + 1] = 1e-5
    return bounds, hyp_init


def train_gp(X, Y, options=None):
    """``train_gp_numpy`` ``optimize.py:359-503`` restated for meanFunc='zero':
    per output SLSQP (tol 1e-12, maxiter 1e4, finite-difference gradients,
    ``:466-467``) from the reference's init, then the post-fit block."""
    from scipy.optimize import minimize
    X = np.asarray(X, dtype=np.float64); Y = np.asarray(Y, dtype=np.float64)
    N, Nx = X.shape; Ny = Y.shape[1]
    opts = {'disp': False, 'maxiter': 10000}
    if options:
        opts.update(options)
    hyp_opt = np.zeros((Ny, Nx + 2))
    for a in range(Ny):
        bounds, init = train_bounds_init(X, Y[:, a])
        res = minimize(calc_NLL, init, args=(X, Y[:, a]), method='SLSQP',
                       options=opts, bounds=bounds, tol=1e-12)
        hyp_opt[a] = res.x
    out = postfit(X, Y, hyp_opt)
    out['hyper'] = hyp_opt
    return out


# ----------------------------------------------------------------------------
# first derivatives w.r.t. the test input: checker for gpmpc_predict_grad
# ----------------------------------------------------------------------------
def predict_grad_fd(X, hyper, alpha, chol, Z, Sigma, method='TA', rel=1e-4):
    """Central differences of the restated prediction (``gp_mean_var`` / ``gp_mean_jac`` /
    ``ta_cov``, i.e. ``gp_functions.py:111-173``) w.r.t. every test-input coordinate: what
    CasADi's AD computes for the MPC's NLP (``mpc_class.py:390-412``, ``:496-513``).  Oracle for
    the analytic derivative kernels of the GPU engine (the reference has no closed forms).
    Z:(H,Nx), Sigma:(Nx,Nx)|(H,Nx,Nx).  Returns dict(dmean (H,Ny,Nx), dvar (H,Ny,Nx),
    dcov (H,Ny,Ny,Nx), hess (H,Ny,Nx,Nx))."""
    X = np.asarray(X, dtype=np.float64)
    Z = np.atleast_2d(np.asarray(Z, dtype=np.float64))
    hyper = np.atleast_2d(np.asarray(hyper, dtype=np.float64))
    H, Nx = Z.shape
    Ny = hyper.shape[0]

    def f(Zp):
        m, v = gp_mean_var(X, hyper, alpha, chol, Zp)
        J = gp_mean_jac(X, hyper, alpha, Zp)
        c = ta_cov(v, J, Sigma) if method == 'TA' else me_cov(v)
        return m, v, c, J

    out = dict(dmean=np.zeros((H, Ny, Nx)), dvar=np.zeros((H, Ny, Nx)), dcov=np.zeros((H, Ny, Ny, Nx)),
               hess=np.zeros((H, Ny, Nx, Nx)))
    for e in range(Nx):
        h = rel * np.maximum(1.0, np.abs(Z[:, e]))
        Zp = Z.copy(); Zp[:, e] += h
        Zm = Z.copy(); Zm[:, e] -= h
        mp, vp, cp, Jp = f(Zp)
        mm, vm, cm, Jm = f(Zm)
        out['dmean'][:, :, e] = (mp - mm) / (2 * h[:, None])
        out['dvar'][:, :, e] = (vp - vm) / (2 * h[:, None])
        out['dcov'][:, :, :, e] = (cp - cm) / (2 * h[:, None, None])
        out['hess'][:, :, :, e] = (Jp - Jm) / (2 * h[:, None, None])
    return out


# ----------------------------------------------------------------------------
# fixtures / synthetic workloads shared by tests and bench
# ----------------------------------------------------------------------------
def synthetic_problem(N, Nx, Ny, config_id=0, H=30):
    """Seeded synthetic workload of SURVEY.md section 8(d)."""
    rng = np.random.default_rng(1234 + config_id)
    X = rng.standard_normal((N, Nx))
    W = rng.standard_normal((Nx, Ny)) / np.sqrt(Nx)
    F = np.sin(X @ W) + 0.1 * (X @ W) ** 2
    Y = F + 1e-2 * rng.standard_normal((N, Ny))
    Y = (Y - Y.mean(0)) / Y.std(0)
    hyper = np.zeros((Ny, Nx + 2))
    hyper[:, :Nx] = rng.uniform(2.0, 6.0, size=(Ny, Nx))
    hyper[:, Nx] = 1.0
    hyper[:, Nx + 1] = 1e-2
    rt = np.random.default_rng(7)
    Z = 0.5 * rt.standard_normal((H, Nx))
    A = rt.standard_normal((Nx, Nx))
    Sigma = 1e-4 * np.eye(Nx) + 1e-5 * A @ A.T
    return dict(X=X, Y=Y, hyper=hyper, Z=Z, Sigma=Sigma)
