"""Sampled roll-outs (DESIGN 4.12, ``gpmpc_rollout_sample``) in numpy  --  TEST INFRASTRUCTURE ONLY.

``conditional_draw`` runs the sequential conditioning of one (trajectory, output) from the posterior moments of its
visited points, with the engine's delta rule; ``joint_draw`` forms m + R eps with R = chol of the joint posterior
covariance of the kept points, the identity the sequential draw must satisfy.  ``path_moments`` gives those moments from
a given factor (L^-1, alpha), and ``rollout_sample`` restates the whole entry (dynamics included) for the oracle-backed
engine of the CPU tests.
"""
from __future__ import annotations

import numpy as np

from oracle import gp_oracle as orc

DELTA = 1e-12       # a conditional variance <= DELTA sf2 is rounding: the point is not added (gpmpc.cu, SAMPLE_DELTA)


def path_moments(X, hyper_a, alpha_a, Linv_a, Z):
    """Posterior mean m (T,) and joint covariance C (T, T) of one output at the points Z (T, Nx): ks^T alpha and
    k(Z, Z) - V^T V with V = L^-1 k(X, Z)."""
    Nx = X.shape[1]
    ell, sf2 = hyper_a[:Nx], hyper_a[Nx] ** 2
    ks = orc.covSEard(X, Z, ell, sf2)
    V = Linv_a @ ks
    return ks.T @ alpha_a, orc.covSEard(Z, Z, ell, sf2) - V.T @ V


def conditional_draw(m, C, eps, sf2, delta=DELTA):
    """Step by step: w = R^-1 C[t, S], d = C[t, t] - |w|^2, f_t = m_t + w . eps_S (+ sqrt(d) eps_t and t joins S when
    d > delta sf2).  Returns f (T,) and kept (T,) bool."""
    T = len(m)
    R = np.zeros((T, T))
    S, f, kept = [], np.empty(T), np.zeros(T, dtype=bool)
    for t in range(T):
        k = len(S)
        w = np.zeros(0)
        if k:
            c = C[t, S]
            w = np.empty(k)
            for j in range(k):
                w[j] = (c[j] - R[j, :j] @ w[:j]) / R[j, j]
        d = C[t, t] - w @ w
        f[t] = m[t] + (w @ eps[S] if k else 0.0)
        if d > delta * sf2:
            f[t] += np.sqrt(d) * eps[t]
            R[k, :k] = w
            R[k, k] = np.sqrt(d)
            S.append(t)
            kept[t] = True
    return f, kept


def joint_draw(m, C, eps, kept):
    """m + R eps over the kept points, R = cholesky(C[kept, kept]) (LAPACK)."""
    idx = np.flatnonzero(kept)
    R = np.linalg.cholesky(C[np.ix_(idx, idx)])
    return m[idx] + R @ eps[idx]


def rollout_sample(model, Linv, z0, U, eps, xi=None, scale=None, K=None, x_ref=None, uscale=None):
    """The whole of gpmpc_rollout_sample for one factor: model dict(X, hyper, alpha), Linv (Ny, N, N); arguments and
    returns as Engine.rollout_sample (samples, z_out, kept), trajectory by trajectory."""
    X, hyper, alpha = model['X'], np.atleast_2d(model['hyper']), model['alpha']
    Ny, Nx = hyper.shape[0], X.shape[1]
    Nu = Nx - Ny
    z0 = np.asarray(z0, dtype=np.float64).reshape(-1, Nx)
    B, Nt = z0.shape[0], eps.shape[1]
    samples, z_out, kept = np.empty((B, Nt, Ny)), np.empty((B, Nt, Nx)), np.zeros((B, Nt, Ny), dtype=np.int32)
    for b in range(B):
        z = z0[b].copy()
        R = np.zeros((Ny, Nt, Nt))
        S = [[] for _ in range(Ny)]
        for t in range(Nt):
            z_out[b, t] = z
            Zp = z_out[b, :t + 1]
            for a in range(Ny):
                m, C = path_moments(X, hyper[a], alpha[a], Linv[a], Zp)
                k = len(S[a])
                w = np.empty(k)
                for j in range(k):
                    w[j] = (C[t, S[a][j]] - R[a, j, :j] @ w[:j]) / R[a, j, j]
                d = C[t, t] - w @ w
                f = m[t] + (w @ eps[b, S[a], a] if k else 0.0)
                if d > DELTA * hyper[a, Nx] ** 2:
                    f += np.sqrt(d) * eps[b, t, a]
                    R[a, k, :k] = w
                    R[a, k, k] = np.sqrt(d)
                    S[a].append(t)
                    kept[b, t, a] = 1
                samples[b, t, a] = f + (hyper[a, Nx + 1] * xi[b, t, a] if xi is not None else 0.0)
            if t + 1 == Nt:
                break
            x = samples[b, t]
            zx = x
            if scale is not None:
                x = x * scale[0] + scale[1]
                zx = (x - scale[2]) / scale[3]
            if K is None:
                un = U[b, t + 1] if Nu > 0 else np.zeros(0)
            else:
                un = np.asarray(K) @ (x - (0.0 if x_ref is None else x_ref))
                if uscale is not None:
                    un = (un - uscale[0]) / uscale[1]
            z = np.concatenate([zx, un])
    return samples, z_out, kept
