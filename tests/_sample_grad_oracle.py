"""Pathwise derivatives of sampled roll-outs (DESIGN 4.16, ``gpmpc_rollout_sample_grad``) in numpy  --  TEST
INFRASTRUCTURE ONLY (the checker of ``GP.sample_rollout_grad`` and the device entry).

The same forward-mode recursion as the device, over ``oracle/sample_oracle.py``'s sequential conditioning, with J and
dvar_dz from ``hess_oracle.predict_grad_closed``.  Per output a and step t, with beta_s = K^-1 ks_s:

    dm = J dz_t,  dc_tt = dvar_dz . dz_t,  dc_s = g(t,s) . dz_t + g(s,t) . dz_s   (s in the conditioning set S),
    g(t,s)_e = -(z_t,e - z_s,e) / ell_e^2 k(z_t, z_s) + sum_i (z_t,e - x_i,e) / ell_e^2 ks_t[i] beta_s[i],
    dw = R^-1 (dc - dR w),  dd = dc_tt - 2 w . dw,  df = dm + dw . eps_S (+ dd / (2 sqrt d) eps_t when kept),

and a kept point appends [dw, dd / (2 sqrt d)] to dR.  The next tangent is that of sample_oracle's input update.
"""
from __future__ import annotations

import numpy as np

from oracle import gp_oracle as orc
from oracle import hess_oracle
from oracle import sample_oracle as so


class Conditioner:
    """The sequential conditioning of one (trajectory, output) and its tangents over P parameter columns."""

    def __init__(self, X, hyper_a, alpha_a, chol_a, Linv_a, Nt, P):
        self.X, self.hyp, self.alpha, self.chol, self.Linv = X, hyper_a, alpha_a, chol_a, Linv_a
        self.S, self.R, self.dR = [], np.zeros((Nt, Nt)), np.zeros((Nt, Nt, P))

    def step(self, Z, dZ, eps, keep=None):
        """Step t = len(Z) - 1 along the points Z (t+1, Nx) with tangents dZ (t+1, Nx, P) and normals eps (t+1,):
        returns f, df (P,), d and whether the point was kept (``keep`` forces the branch; None: the delta rule)."""
        X, hyp, Nx = self.X, self.hyp, self.X.shape[1]
        t, S, k = Z.shape[0] - 1, self.S, len(self.S)
        ell2, sf2 = hyp[:Nx] ** 2, hyp[Nx] ** 2
        m, C = so.path_moments(X, hyp, self.alpha, self.Linv, Z)
        w = np.empty(k)
        for j in range(k):
            w[j] = (C[t, S[j]] - self.R[j, :j] @ w[:j]) / self.R[j, j]
        d = C[t, t] - w @ w
        if keep is None:
            keep = d > so.DELTA * sf2
        g = hess_oracle.predict_grad_closed(X, hyp[None], self.alpha[None], self.chol[None], Z[t][None], None, 'ME')
        df = g['dmean'][0, 0] @ dZ[t]
        dct = g['dvar'][0, 0] @ dZ[t]
        f = m[t] + (w @ eps[S] if k else 0.0)
        dw = np.zeros((0, dZ.shape[2]))
        if k:
            ks = orc.covSEard(X, Z, hyp[:Nx], sf2)                       # (N, t+1)
            beta = self.Linv.T @ (self.Linv @ ks)
            dc = np.empty((k, dZ.shape[2]))
            for j, s in enumerate(S):
                kts = sf2 * np.exp(-0.5 * np.sum((Z[t] - Z[s]) ** 2 / ell2))
                gts = (-(Z[t] - Z[s]) * kts + ((Z[t] - X) * (ks[:, t] * beta[:, s])[:, None]).sum(0)) / ell2
                gst = (-(Z[s] - Z[t]) * kts + ((Z[s] - X) * (ks[:, s] * beta[:, t])[:, None]).sum(0)) / ell2
                dc[j] = gts @ dZ[t] + gst @ dZ[s]
            rhs = dc - np.einsum('jip,i->jp', self.dR[:k, :k], w)
            dw = np.empty_like(rhs)
            for j in range(k):
                dw[j] = (rhs[j] - self.R[j, :j] @ dw[:j]) / self.R[j, j]
            df = df + dw.T @ eps[S]
        if keep:
            sd = np.sqrt(d)
            q = (dct - 2 * w @ dw) / (2 * sd)
            f += sd * eps[t]
            df = df + q * eps[t]
            self.R[k, :k], self.R[k, k] = w, sd
            self.dR[k, :k], self.dR[k, k] = dw, q
            S.append(t)
        return f, df, d, bool(keep)


def rollout_sample_grad(model, Linv, z0, U, eps, xi=None, scale=None, K=None, x_ref=None, uscale=None):
    """gpmpc_rollout_sample_grad for one factor: model dict(X, hyper, alpha, chol), Linv (Ny, N, N); arguments as
    Engine.rollout_sample_grad.  Returns dict(samples, z_out, kept, dsamples (B, Nt, Ny, P) with the entry's columns,
    d (B, Nt, Ny) the conditional variance of every step, for margin checks against the delta rule)."""
    X, hyper, alpha, chol = model['X'], np.atleast_2d(model['hyper']), model['alpha'], model['chol']
    Ny, Nx = hyper.shape[0], X.shape[1]
    Nu = Nx - Ny
    z0 = np.asarray(z0, dtype=np.float64).reshape(-1, Nx)
    eps = np.asarray(eps, dtype=np.float64)
    B, Nt = z0.shape[0], eps.shape[1]
    P = Nx + (Nu * Ny if K is not None else (Nt - 1) * Nu)
    samples, z_out = np.empty((B, Nt, Ny)), np.empty((B, Nt, Nx))
    kept, D, dvals = np.zeros((B, Nt, Ny), dtype=np.int32), np.empty((B, Nt, Ny, P)), np.empty((B, Nt, Ny))
    if scale is not None:
        sY, mY, mX, sX = (np.asarray(v, dtype=np.float64) for v in scale)
    for b in range(B):
        z, dz = z0[b].copy(), np.eye(Nx, P)
        Z, dZ = np.empty((Nt, Nx)), np.empty((Nt, Nx, P))
        conds = [Conditioner(X, hyper[a], alpha[a], chol[a], Linv[a], Nt, P) for a in range(Ny)]
        for t in range(Nt):
            Z[t], dZ[t] = z, dz
            for a in range(Ny):
                f, df, dvals[b, t, a], kp = conds[a].step(Z[:t + 1], dZ[:t + 1], eps[b, :t + 1, a])
                kept[b, t, a] = kp
                samples[b, t, a] = f + (hyper[a, Nx + 1] * xi[b, t, a] if xi is not None else 0.0)
                D[b, t, a] = df
            if t + 1 == Nt:
                break
            x, dx = samples[b, t], D[b, t]
            zx, dzx = x, dx
            if scale is not None:
                x, dx = x * sY + mY, dx * sY[:, None]
                zx, dzx = (x - mX) / sX, dx / sX[:, None]
            if K is None:
                un = U[b, t + 1] if Nu > 0 else np.zeros(0)
                du = np.zeros((Nu, P))
                du[:, Nx + t * Nu:Nx + (t + 1) * Nu] = np.eye(Nu)
            else:
                K = np.asarray(K, dtype=np.float64)
                xt = x - (0.0 if x_ref is None else x_ref)
                un, du = K @ xt, K @ dx
                for i in range(Nu):
                    du[i, Nx + i * Ny:Nx + (i + 1) * Ny] += xt
                if uscale is not None:
                    un, du = (un - uscale[0]) / uscale[1], du / np.asarray(uscale[1])[:, None]
            z, dz = np.concatenate([zx, un]), np.concatenate([dzx, du])
        z_out[b] = Z
    return dict(samples=samples, z_out=z_out, kept=kept, dsamples=D, d=dvals)


MARGIN = 1e3                # every d is at least MARGIN delta sf2 away from the delta rule's threshold


def assert_margin(d, hyper):
    Nx = hyper.shape[1] - 2
    thr = so.DELTA * hyper[:, Nx] ** 2
    assert (np.abs(d - thr) >= MARGIN * thr).all(), 'a step sits within the margin of the delta rule'
