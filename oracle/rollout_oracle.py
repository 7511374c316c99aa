"""The numeric loop of ``GP.predict_compare`` (reference gp_class.py:746-804), open loop and with LQR
feedback, minus the plotting and the plant simulation  --  TEST INFRASTRUCTURE ONLY (the checker of
``GP.rollout`` and ``gpmpc_rollout_batch``).

Per method: start from x0 with the input covariance diag(sn2) (+1e-6 on the inputs; the covariance is
shared across methods), and per step predict with ``gp_oracle.predict``.  With feedback the GP is
linearised at (x0, u[0]) through the oracle's posterior-mean Jacobian, the gain comes from the discrete
algebraic Riccati equation (mpc_class.py:956-976), and every step applies u_t = K (mean_t - x_ref) with
the input blocks Sigma_uu = K cov K^T and Sigma_xu = cov K^T (gp_class.py:770-804).
"""
from __future__ import annotations

import numpy as np
import scipy.linalg

from oracle import gp_oracle as orc


def _mm(A, B):
    """A @ B summed in index order with separate multiplies and adds: the order the engine uses for the feedback
    products.  The closed loop amplifies a single rounding difference (to 1e-10 on the car model), so a BLAS product,
    whose order varies between builds, could not be compared at 1e-12."""
    out = np.zeros((A.shape[0], B.shape[1]))
    for k in range(A.shape[1]):
        out = out + A[:, k:k + 1] * B[k:k + 1, :]
    return out


def lqr_gain(A, B, Q, R):
    """u = K x with K = -(R + B^T P B)^-1 B^T P A, P from the DARE."""
    P = scipy.linalg.solve_discrete_are(A, B, Q, R)
    return -np.linalg.solve(R + B.T @ P @ B, B.T @ P @ A), P


def predict_compare_loop(model, x0, u, methods, feedback=False, x_ref=None, Q=None, R=None):
    """``model`` as for ``gp_oracle.predict``; x0:(Ny,), u:(Nt,Nu).  Returns mean, var of shape
    (len(methods), Nt+1, Ny), var rescaled by stdY^2 when the model normalises (gp_class.py:795-796)."""
    hyper = np.atleast_2d(model['hyper'])
    Ny, Nx = hyper.shape[0], model['X'].shape[1]
    Nu = Nx - Ny
    x0 = np.asarray(x0, dtype=np.float64).reshape(Ny)
    u = np.asarray(u, dtype=np.float64).reshape(-1, Nu)
    Nt = u.shape[0]
    init_var = hyper[:, Nx + 1] ** 2
    mean = np.zeros((len(methods), Nt + 1, Ny))
    var = np.zeros((len(methods), Nt + 1, Ny))
    covar = np.eye(Nx) * 1e-6
    Q = np.eye(Ny) if Q is None else np.asarray(Q, dtype=np.float64)
    R = np.eye(Nu) if R is None else np.asarray(R, dtype=np.float64)
    if feedback and x_ref is None:
        x_ref = np.zeros(Ny)
    for i, meth in enumerate(methods):
        mean_t = x0
        covar[:Ny, :Ny] = np.diag(init_var)
        mean[i, 0] = x0
        if feedback:
            A, Bm = orc.discrete_linearize(model, x0, u[0])
            K = lqr_gain(A, Bm, Q, R)[0]
        for t in range(1, Nt + 1):
            u_t = _mm(K, (mean_t - x_ref)[:, None])[:, 0] if feedback else u[t - 1]
            m, covar_x = orc.predict(model, mean_t, u_t, covar, meth)
            mean_t = m.reshape(Ny)
            mean[i, t] = mean_t
            var[i, t] = np.diag(covar_x)
            if model.get('normalize', False):
                var[i, t] = var[i, t] * np.asarray(model['meta']['stdY']) ** 2
            if feedback:
                cov_xu = _mm(covar_x, K.T)
                covar[Ny:, Ny:] = _mm(_mm(K, covar_x), K.T)
                covar[Ny:, :Ny] = cov_xu.T
                covar[:Ny, Ny:] = cov_xu
            covar[:Ny, :Ny] = covar_x
    return mean, var
