"""Forward-mode derivatives of ``rollout_oracle.predict_compare_loop``'s 'EM' arithmetic  --  TEST INFRASTRUCTURE ONLY
(the checker of ``GP.rollout_grad(method='EM')`` and ``gpmpc_rollout_batch_em_grad``).  The 'EM' counterpart of
``oracle/rollout_grad_oracle.py`` (which covers 'ME' and 'TA'), with the same parameters, units and feedback recurrences.

Per step, in the GP's input units z = [(x - meanX)/stdX, (u - meanU)/stdU] with input covariance S, the primal is
``gp_oracle.gp_exact_moment`` (the arithmetic ``predict_compare_loop`` runs for 'EM'; ``model`` needs Y and invK) and the
derivatives are ``em_grad_oracle.em_grad_closed``'s at (z, S) with the model's alpha and chol.  The mean depends on S, so

    d mean_std = dmean_dz dz + sum_{d,e} dmean_dSigma[., d, e] dS[d, e],
    d C = dcov_dz dz + sum_{d,e} dcov_dSigma[., ., d, e] dS[d, e],

over every entry of the symmetric dS (the blocks hold every other entry fixed), and

    x_{t+1} = mean_std stdY + meanY,   u_{t+1} = K (x_{t+1} - x_ref)  or  u[t],
    S_{t+1} = [C, C K^T; K C, K C K^T] with feedback, S's x block = C open loop.

The variance is C's diagonal times stdY^2, as ``predict_compare_loop`` records it.
"""
from __future__ import annotations

import numpy as np

from oracle import em_grad_oracle
from oracle import gp_oracle as orc
from oracle import rollout_oracle


def rollout_em_grad(model, x0, u, feedback=False, x_ref=None, Q=None, R=None, K=None):
    """``model`` as for ``gp_oracle.predict`` (X, Y, hyper, alpha, chol, invK, normalize, meta); x0:(Ny,), u:(Nt,Nu).  With
    feedback, K (Nu,Ny) defaults to ``predict_compare_loop``'s gain of the linearisation at (x0, u[0]).  Returns
    ``GP.rollout_grad``'s dict for one trajectory: mean, var (Nt+1,Ny), dmean_dx0, dvar_dx0 (Nt+1,Ny,Ny), and
    dmean_du, dvar_du (Nt+1,Ny,Nt,Nu) open loop or dmean_dK, dvar_dK (Nt+1,Ny,Nu,Ny) with feedback."""
    hyper = np.atleast_2d(model['hyper'])
    Ny, Nx = hyper.shape[0], model['X'].shape[1]
    Nu = Nx - Ny
    x0 = np.asarray(x0, dtype=np.float64).reshape(Ny)
    u = np.asarray(u, dtype=np.float64)
    u = u.reshape(-1, Nu) if Nu > 0 else u.reshape(u.shape[0], 0)
    Nt = u.shape[0]
    if model.get('normalize', False):
        st = model['meta']
        mX, sX, mU, sU = (np.asarray(st[k], dtype=np.float64) for k in ('meanX', 'stdX', 'meanU', 'stdU'))
        mY, sY = np.asarray(st['meanY'], dtype=np.float64), np.asarray(st['stdY'], dtype=np.float64)
    else:
        mX, sX, mU, sU, mY, sY = np.zeros(Ny), np.ones(Ny), np.zeros(Nu), np.ones(Nu), np.zeros(Ny), np.ones(Ny)
    if feedback:
        x_ref = np.zeros(Ny) if x_ref is None else np.asarray(x_ref, dtype=np.float64).reshape(Ny)
        if K is None:
            Q = np.eye(Ny) if Q is None else np.asarray(Q, dtype=np.float64)
            R = np.eye(Nu) if R is None else np.asarray(R, dtype=np.float64)
            A, Bm = orc.discrete_linearize(model, x0, u[0])
            K = rollout_oracle.lqr_gain(A, Bm, Q, R)[0]
        K = np.asarray(K, dtype=np.float64).reshape(Nu, Ny)
    # parameters: x0 (Ny) then u row-major (Nt Nu) or K row-major (Nu Ny)
    nrest = Nu * Ny if feedback else Nt * Nu
    P = Ny + nrest
    mean = np.zeros((Nt + 1, Ny)); var = np.zeros((Nt + 1, Ny))
    Dm = np.zeros((Nt + 1, Ny, P)); Dv = np.zeros((Nt + 1, Ny, P))
    mean[0] = x0
    Dm[0, :, :Ny] = np.eye(Ny)
    S = np.eye(Nx) * 1e-6
    S[:Ny, :Ny] = np.diag(hyper[:, Nx + 1] ** 2)
    dS = np.zeros((Nx, Nx, P))
    x, dx = x0, np.concatenate([np.eye(Ny), np.zeros((Ny, nrest))], 1)
    for t in range(Nt):
        if feedback:
            xt = x - x_ref
            ut = rollout_oracle._mm(K, xt[:, None])[:, 0]
            dut = K @ dx
            for i in range(Nu):
                dut[i, Ny + i * Ny:Ny + (i + 1) * Ny] += xt
        else:
            ut = u[t]
            dut = np.zeros((Nu, P))
            dut[:, Ny + t * Nu:Ny + (t + 1) * Nu] = np.eye(Nu)
        z = np.concatenate([(x - mX) / sX, (ut - mU) / sU])
        dz = np.concatenate([dx / sX[:, None], dut / sU[:, None]])
        m_std, C = orc.gp_exact_moment(model['invK'], model['X'], model['Y'], hyper, z, S)
        g = em_grad_oracle.em_grad_closed(model['X'], hyper, model['alpha'], model['chol'], z[None], S)
        dm = g['dmean_dz'][0] @ dz + np.einsum('ade,dep->ap', g['dmean_dSigma'][0], dS)
        dC = np.einsum('ace,ep->acp', g['dcov_dz'][0], dz) + np.einsum('acde,dep->acp', g['dcov_dSigma'][0], dS)
        x = m_std * sY + mY
        dx = dm * sY[:, None]
        mean[t + 1] = x
        Dm[t + 1] = dx
        var[t + 1] = np.diag(C) * sY ** 2
        Dv[t + 1] = np.einsum('aap->ap', dC) * (sY ** 2)[:, None]
        dSn = dS.copy()
        dSn[:Ny, :Ny] = dC
        if feedback:
            KC = K @ C
            dxu = np.einsum('rkp,ik->rip', dC, K)                        # dC K^T
            dKC = np.einsum('ik,kcp->icp', K, dC)                        # K dC
            duu = np.einsum('ikp,jk->ijp', dKC, K)                       # K dC K^T
            for i in range(Nu):
                for k in range(Ny):
                    p = Ny + i * Ny + k                                  # dK = E_ik
                    dxu[:, i, p] += C[:, k]                              # C dK^T
                    duu[i, :, p] += (C @ K.T)[k, :]                      # dK C K^T
                    duu[:, i, p] += KC[:, k]                             # K C dK^T
            dSn[:Ny, Ny:] = dxu
            dSn[Ny:, :Ny] = np.transpose(dxu, (1, 0, 2))
            dSn[Ny:, Ny:] = duu
            cov_xu = rollout_oracle._mm(C, K.T)
            S[Ny:, Ny:] = rollout_oracle._mm(rollout_oracle._mm(K, C), K.T)
            S[Ny:, :Ny] = cov_xu.T
            S[:Ny, Ny:] = cov_xu
        dS = dSn
        S[:Ny, :Ny] = C
    out = dict(mean=mean, var=var, dmean_dx0=Dm[..., :Ny], dvar_dx0=Dv[..., :Ny])
    if feedback:
        out.update(dmean_dK=Dm[..., Ny:].reshape(Nt + 1, Ny, Nu, Ny), dvar_dK=Dv[..., Ny:].reshape(Nt + 1, Ny, Nu, Ny))
    else:
        out.update(dmean_du=Dm[..., Ny:].reshape(Nt + 1, Ny, Nt, Nu), dvar_du=Dv[..., Ny:].reshape(Nt + 1, Ny, Nt, Nu))
    return out
