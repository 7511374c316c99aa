"""The device roll-outs (gpmpc_rollout_batch, gpmpc_rollout_batch_grad, gpmpc_rollout_sample) in np.longdouble, on the
engine's own alpha and L^-1 (GET_ALPHA, GET_LINV), with the sum of |terms| of every value they return.

Everything is in the engine's units: inputs z = [x, u] and Sigma as the GP sees them, means and variances in its output
units.  One step is ``hess_oracle.derivs_core_ld`` (first-order outputs only) and ``hess_oracle.cov_derivs``; the
recursion follows rollout_feedback_kernel and rollout_tangent_kernel (gpmpc.cu, the comments above them):

    open loop:  z_{t+1} = [zx(mean_t), U[t+1]],                Sigma x block = cov_t, u blocks kept
    feedback:   x = mean_t sY + mY (or mean_t), u = K (x - x_ref) [then (u - mU) / sU],
                Sigma = [cov_t, cov_t K^T; K cov_t, (K cov_t) K^T]
    zx(m) = (m sY + mY - mX) / sX with scale = [sY | mY | mX | sX], else m.

Tangents are forward mode over P parameters, [z0 (Nx) | U rows 1 .. Nt-1] open loop or [z0 | K row-major] with K:
dm = J dz, dC = dcov_dz . dz + J dS J^T ('TA') or diag(dvar_dz . dz) ('ME'), and the derivatives of the next input.

Each value v comes with s_v, its sum of |terms| carried through the steps as ``update_oracle_ld`` does, so that a
kernel's error in v is a few units of rounding times s_v whatever the cancellation.  Inside a step the sums are those of
``derivs_core_ld(absolute=True)``; an operand formed in an earlier step (z, Sigma, the tangents dz, dS) enters a product
with its carried sum times the |value| of the other factor, e(A B) = e(A) |B| + |A| e(B), and enters a step's outputs
through their true derivatives in z: |J| (mean), |dvar_dz| (var) and |hess| (J).  The z-dependence of dvar_dz, hess
and dcov_dz is left out: it is second order in the derivative chain.  Inputs the caller supplies (z0, Sigma0, U) carry
their |values|: the differences x_i - z of ks round on that scale.

``sample_ld`` restates sample_cond_kernel (kernels.cuh) on given inputs: the engine's z_out, so no error propagates
from step to step, with the conditioning sets of the engine's kept flags when they are given.  Its sums follow the same
first-order rule through V = L^-1 k, the covariances c, the forward substitution w = R^-1 c and d = c_tt - |w|^2, so
that a small pivot of R amplifies them as it amplifies the kernel's rounding.
"""
import numpy as np

from oracle import hess_oracle
from oracle.update_oracle_ld import LD, kvec

DELTA = 1e-12       # gpmpc.cu, SAMPLE_DELTA: a conditional variance <= DELTA sf2 is rounding and the point is not kept
# a keep decision whose margin |d - DELTA sf2| / s_d is below this could go either way on the device: the kernel's error
# in d is a few units of rounding (~1e-16) times s_d, 1e4-fold below it
MARGIN = 1e-12

# blocks of Sigma (its value, written by rollout_feedback_kernel) and of dS (its tangent) that ``rollout_ld(drop=...)``
# can leave out: a lost Sigma write keeps the previous step's block, a dropped dS term is zero
SIGMA_BLOCKS = ('Sxu', 'Sux', 'Suu')
DS_BLOCKS = ('xx', 'xu', 'ux', 'uu')


def _blocks(M, Ny, name):
    """The (rows, cols) slices of block name ('xx', 'xu', 'ux', 'uu' or 'S' + one of them) of an Nx x Nx matrix."""
    x, u = slice(0, Ny), slice(Ny, None)
    r, c = name[-2:]
    return (slice(None),) + ((x if r == 'x' else u), (x if c == 'x' else u))


def _k_units(Nu, Ny, P, Nx):
    """E (Nu, Ny, P): E[i, k, p] = 1 where parameter p is the entry (i, k) of K."""
    E = np.zeros((Nu, Ny, P), dtype=LD)
    for i in range(Nu):
        for k in range(Ny):
            E[i, k, Nx + i * Ny + k] = 1
    return E


def feedback_inputs64(means, scale=None, K=None, x_ref=None, uscale=None, U_next=None):
    """The next inputs (B, Nx) that rollout_feedback_kernel forms from float64 means (B, Ny), with its operation order
    and no fused multiply-add, so that fed the engine's means they are the engine's inputs bit for bit.  U_next (B, Nu):
    the open-loop inputs."""
    means = np.asarray(means, dtype=np.float64)
    B, Ny = means.shape
    x = z = means
    if scale is not None:
        sc = np.asarray(scale, dtype=np.float64)
        x = means * sc[0] + sc[1]
        z = (x - sc[2]) / sc[3]
    if K is None:
        return np.concatenate([z, np.asarray(U_next, dtype=np.float64).reshape(B, -1)], 1)
    K = np.asarray(K, dtype=np.float64)
    xt = x - np.asarray(x_ref, dtype=np.float64) if x_ref is not None else x
    u = np.zeros((B, K.shape[0]))
    for k in range(Ny):
        u = u + K[:, k][None, :] * xt[:, k][:, None]
    if uscale is not None:
        us = np.asarray(uscale, dtype=np.float64)
        u = (u - us[0]) / us[1]
    return np.concatenate([z, u], 1)


def rollout_ld(X, hyper, alpha, linv, z0, U, Sigma0, method, scale=None, K=None, x_ref=None, uscale=None,
               tangents=False, means_in=None, drop=()):
    """gpmpc_rollout_batch(_grad) for B trajectories: z0 (B, Nx), U (B, Nt, Nu) (with K only its shape is used), Sigma0
    (B, Nx, Nx), method 'TA' or 'ME', scale (4, Ny), K (Nu, Ny), x_ref (Ny,), uscale (2, Nu) as Engine.rollout_batch;
    linv (Ny, N, N), best already np.longdouble.  ``means_in`` (B, Nt, Ny): form every next input from these means (the
    engine's) with ``feedback_inputs64`` instead of from the reference's own; ``drop``: names of SIGMA_BLOCKS / DS_BLOCKS
    to leave out (the guards).  Returns dict(mean, var (B, Nt, Ny), cov_last (B, Ny, Ny)[, dmean, dvar (B, Nt, Ny, P)])
    and for each key k its sum of |terms| 's_' + k."""
    hyper = np.atleast_2d(np.asarray(hyper, dtype=np.float64))
    Ny, Nx = hyper.shape[0], X.shape[1]
    Nu = Nx - Ny
    Li = np.asarray(linv, dtype=LD)
    z = np.asarray(z0, dtype=LD).reshape(-1, Nx)
    B = z.shape[0]
    Nt = int(np.shape(U)[1])
    U = np.asarray(U, dtype=LD).reshape(B, Nt, Nu)
    S = np.array(np.broadcast_to(np.asarray(Sigma0, dtype=LD), (B, Nx, Nx)))
    ez, eS = np.abs(z), np.abs(S)
    fb = K is not None
    if scale is not None:
        sY, mY, mX, sX = np.asarray(scale, dtype=LD)
    if fb:
        Kl = np.asarray(K, dtype=LD)
        aK = np.abs(Kl)
        xr = np.zeros(Ny, dtype=LD) if x_ref is None else np.asarray(x_ref, dtype=LD)
        if uscale is not None:
            mU, sU = np.asarray(uscale, dtype=LD)
    P = Nx + (Nu * Ny if fb else (Nt - 1) * Nu)
    out = {k: np.zeros((B, Nt, Ny), dtype=LD) for k in ('mean', 'var', 's_mean', 's_var')}
    if tangents:
        out.update({k: np.zeros((B, Nt, Ny, P), dtype=LD) for k in ('dmean', 'dvar', 's_dmean', 's_dvar')})
        dz = np.zeros((B, Nx, P), dtype=LD)
        dz[:, np.arange(Nx), np.arange(Nx)] = 1
        edz = np.abs(dz)
        dS = np.zeros((B, Nx, Nx, P), dtype=LD)
        edS = np.zeros_like(dS)
        EK = _k_units(Nu, Ny, P, Nx) if fb else None
    for t in range(Nt):
        c = hess_oracle.derivs_core_ld(X, hyper, alpha, Li, z, second=False)
        a = hess_oracle.derivs_core_ld(X, hyper, alpha, Li, z, absolute=True, second=False)
        J, H, dv = c['J'], c['hess'], c['dvar_dz']
        aJ, aH, adv = np.abs(J), np.abs(H), np.abs(dv)
        eJ = a['J'] + np.einsum('bade,be->bad', aH, ez)                 # J's own terms and the error z carries into it
        eH, edv = a['hess'], a['dvar_dz']
        aS = np.abs(S)
        cv = hess_oracle.cov_derivs(c, S, method)
        C = cv['cov']
        evar = a['var'] + np.einsum('bad,bd->ba', adv, ez)
        eC = np.zeros_like(C)
        eC[:, np.arange(Ny), np.arange(Ny)] = evar
        if method == 'TA':
            eC += (np.einsum('bad,bde,bce->bac', eJ, aS, aJ) + np.einsum('bad,bde,bce->bac', aJ, aS, eJ)
                   + np.einsum('bad,bde,bce->bac', aJ, eS, aJ))
        out['mean'][:, t] = c['mean']
        out['s_mean'][:, t] = a['mean'] + np.einsum('bad,bd->ba', aJ, ez)
        out['var'][:, t] = np.diagonal(C, axis1=1, axis2=2)
        out['s_var'][:, t] = np.diagonal(eC, axis1=1, axis2=2)
        if t + 1 == Nt:
            out['cov_last'], out['s_cov_last'] = C, eC
        if tangents:
            adz, adS = np.abs(dz), np.abs(dS)
            dm = np.einsum('bae,bep->bap', J, dz)
            edm = np.einsum('bae,bep->bap', eJ, adz) + np.einsum('bae,bep->bap', aJ, edz)
            if method == 'TA':
                dcv = cv['dcov_dz']
                edcv = np.zeros_like(dcv)
                edcv[:, np.arange(Ny), np.arange(Ny)] = edv
                for X1, S1, X2 in ((eH, aS, aJ), (aH, aS, eJ), (aH, eS, aJ)):
                    edcv += np.einsum('badf,bde,bce->bacf', X1, S1, X2) + np.einsum('bce,bde,badf->bcaf', X2, S1, X1)
                dC = np.einsum('bace,bep->bacp', dcv, dz) + np.einsum('bae,befp,bcf->bacp', J, dS, J, optimize=True)
                edC = (np.einsum('bace,bep->bacp', edcv, adz) + np.einsum('bace,bep->bacp', np.abs(dcv), edz)
                       + np.einsum('bae,befp,bcf->bacp', eJ, adS, aJ, optimize=True)
                       + np.einsum('bae,befp,bcf->bacp', aJ, adS, eJ, optimize=True)
                       + np.einsum('bae,befp,bcf->bacp', aJ, edS, aJ, optimize=True))
            else:
                dC = np.zeros((B, Ny, Ny, P), dtype=LD)
                edC = np.zeros_like(dC)
                dC[:, np.arange(Ny), np.arange(Ny)] = np.einsum('bae,bep->bap', dv, dz)
                edC[:, np.arange(Ny), np.arange(Ny)] = (np.einsum('bae,bep->bap', edv, adz)
                                                        + np.einsum('bae,bep->bap', adv, edz))
            out['dmean'][:, t], out['s_dmean'][:, t] = dm, edm
            out['dvar'][:, t] = np.diagonal(dC, axis1=1, axis2=2).transpose(0, 2, 1)
            out['s_dvar'][:, t] = np.diagonal(edC, axis1=1, axis2=2).transpose(0, 2, 1)
        if t + 1 == Nt:
            break
        # the next input and Sigma (rollout_feedback_kernel)
        if means_in is not None:
            m = np.asarray(means_in, dtype=np.float64)[:, t]
            znew = np.asarray(feedback_inputs64(m, scale, K, x_ref, uscale, None if fb else U[:, t + 1]), dtype=LD)
            m, em = m.astype(LD), np.abs(m).astype(LD)
        else:
            m, em = out['mean'][:, t], out['s_mean'][:, t]
        x, ex = m, em
        zx, ezx = m, em
        if scale is not None:
            x, ex = m * sY + mY, em * np.abs(sY) + np.abs(mY)
            zx, ezx = (x - mX) / sX, (ex + np.abs(mX)) / np.abs(sX)
        S2, eS2 = S.copy(), eS.copy()
        S2[:, :Ny, :Ny], eS2[:, :Ny, :Ny] = C, eC
        if fb:
            xt, ext = x - xr, ex + np.abs(xr)
            u, eu = xt @ Kl.T, ext @ aK.T
            if uscale is not None:
                u, eu = (u - mU) / sU, (eu + np.abs(mU)) / np.abs(sU)
            CKt, eCKt = C @ Kl.T, eC @ aK.T
            S2[:, :Ny, Ny:], eS2[:, :Ny, Ny:] = CKt, eCKt
            S2[:, Ny:, :Ny], eS2[:, Ny:, :Ny] = CKt.transpose(0, 2, 1), eCKt.transpose(0, 2, 1)
            S2[:, Ny:, Ny:], eS2[:, Ny:, Ny:] = Kl @ C @ Kl.T, aK @ eC @ aK.T
            for name in drop:
                if name in SIGMA_BLOCKS:
                    blk = _blocks(S, Ny, name)
                    S2[blk], eS2[blk] = S[blk], eS[blk]
        else:
            u, eu = U[:, t + 1], np.abs(U[:, t + 1])
        z, ez = np.concatenate([zx, u], 1), np.concatenate([ezx, eu], 1)
        if means_in is not None:
            z = znew
        if tangents:
            dx, edx = dm, edm
            if scale is not None:
                dx, edx = dm * sY[None, :, None], edm * np.abs(sY)[None, :, None]
            dzx, edzx = dm, edm
            if scale is not None:
                dzx, edzx = dx / sX[None, :, None], edx / np.abs(sX)[None, :, None]
            dS2, edS2 = np.zeros_like(dS), np.zeros_like(edS)
            dS2[:, :Ny, :Ny], edS2[:, :Ny, :Ny] = dC, edC
            if fb:
                du = np.einsum('ik,bkp->bip', Kl, dx) + np.einsum('ikp,bk->bip', EK, xt)
                edu = np.einsum('ik,bkp->bip', aK, edx) + np.einsum('ikp,bk->bip', EK, ext)
                if uscale is not None:
                    du, edu = du / sU[None, :, None], edu / np.abs(sU)[None, :, None]
                dxu = np.einsum('bxkp,ik->bxip', dC, Kl) + np.einsum('bxk,ikp->bxip', C, EK)
                edxu = np.einsum('bxkp,ik->bxip', edC, aK) + np.einsum('bxk,ikp->bxip', eC, EK)
                duu = (np.einsum('ikp,bkl,jl->bijp', EK, C, Kl, optimize=True)
                       + np.einsum('ik,bklp,jl->bijp', Kl, dC, Kl, optimize=True)
                       + np.einsum('ik,bkl,jlp->bijp', Kl, C, EK, optimize=True))
                eduu = (np.einsum('ikp,bkl,jl->bijp', EK, eC, aK, optimize=True)
                        + np.einsum('ik,bklp,jl->bijp', aK, edC, aK, optimize=True)
                        + np.einsum('ik,bkl,jlp->bijp', aK, eC, EK, optimize=True))
                dS2[:, :Ny, Ny:], edS2[:, :Ny, Ny:] = dxu, edxu
                dS2[:, Ny:, :Ny], edS2[:, Ny:, :Ny] = dxu.transpose(0, 2, 1, 3), edxu.transpose(0, 2, 1, 3)
                dS2[:, Ny:, Ny:], edS2[:, Ny:, Ny:] = duu, eduu
            else:
                du = np.zeros((B, Nu, P), dtype=LD)
                for i in range(Nu):
                    du[:, i, Nx + t * Nu + i] = 1
                edu = np.abs(du)
            for name in drop:
                if name in DS_BLOCKS:
                    blk = _blocks(dS2, Ny, name)
                    dS2[blk] = 0
            dz, edz = np.concatenate([dzx, du], 1), np.concatenate([edzx, edu], 1)
            dS, edS = dS2, edS2
        S, eS = S2, eS2
    return out


def sample_ld(X, hyper, alpha, linv, z_out, eps, xi=None, kept=None, delta=DELTA):
    """gpmpc_rollout_sample's draws along given inputs z_out (B, Nt, Nx) with normals eps (and xi) (B, Nt, Ny).  ``kept``
    (B, Nt, Ny), the engine's flags: draw every step on the conditioning set they define (else on the reference's own
    decisions).  Returns dict(samples (B, Nt, Ny), s_samples (their sums of |terms|), kept (the reference's own
    decisions, bool), d (the conditional variances), margin = |d - delta sf2| / s_d)."""
    hyper = np.atleast_2d(np.asarray(hyper, dtype=np.float64))
    Ny, Nx = hyper.shape[0], X.shape[1]
    z_out = np.asarray(z_out, dtype=np.float64)
    B, Nt = z_out.shape[:2]
    eps = np.asarray(eps, dtype=LD)
    out = dict(samples=np.zeros((B, Nt, Ny), dtype=LD), s_samples=np.zeros((B, Nt, Ny), dtype=LD),
               kept=np.zeros((B, Nt, Ny), dtype=bool), d=np.zeros((B, Nt, Ny), dtype=LD),
               margin=np.zeros((B, Nt, Ny)))
    Zall = z_out.reshape(B * Nt, Nx)
    for a in range(Ny):
        Li = np.asarray(linv[a], dtype=LD)
        al = np.asarray(alpha[a], dtype=LD)
        k, sk = kvec(X, Zall, hyper[a], scale=True)                 # (N, B Nt)
        V, sV = Li @ k, np.abs(Li) @ sk
        m, sm = k.T @ al, sk.T @ np.abs(al)
        sf2 = LD(hyper[a, Nx]) ** 2
        sn = LD(hyper[a, Nx + 1])
        for b in range(B):
            rows = np.arange(b * Nt, (b + 1) * Nt)
            Vb, sVb = V[:, rows], sV[:, rows]
            kz, skz = kvec(z_out[b], z_out[b], hyper[a], scale=True)  # k(z_s, z_t) of the path
            R = np.zeros((Nt, Nt), dtype=LD)
            sR = np.zeros((Nt, Nt), dtype=LD)
            S = []
            for t in range(Nt):
                n = len(S)
                c = kz[S, t] - Vb[:, S].T @ Vb[:, t]
                sc = skz[S, t] + sVb[:, S].T @ np.abs(Vb[:, t]) + np.abs(Vb[:, S]).T @ sVb[:, t]
                w, sw = np.zeros(n, dtype=LD), np.zeros(n, dtype=LD)
                for j in range(n):                                     # forward substitution, as the kernel
                    w[j] = (c[j] - R[j, :j] @ w[:j]) / R[j, j]
                    sw[j] = ((sc[j] + sR[j, :j] @ np.abs(w[:j]) + np.abs(R[j, :j]) @ sw[:j]) / R[j, j]
                             + abs(w[j]) * sR[j, j] / R[j, j])
                d = sf2 - Vb[:, t] @ Vb[:, t] - w @ w
                sd = sf2 + 2 * np.abs(Vb[:, t]) @ sVb[:, t] + 2 * np.abs(w) @ sw
                e = eps[b, S, a]
                f, sf = m[rows[t]] + w @ e, sm[rows[t]] + (np.abs(w) + sw) @ np.abs(e)
                own = bool(d > delta * sf2)
                keep = own if kept is None else bool(kept[b, t, a])
                if keep:
                    # a step kept with d <= 0 would leave a zero pivot in R and NaN in every later step
                    assert d > 0, ('kept with a conditional variance <= 0 in long double', b, t, a, float(d))
                    sq = np.sqrt(d)
                    ssq = sq + sd / (2 * sq)
                    f, sf = f + sq * eps[b, t, a], sf + ssq * abs(eps[b, t, a])
                    R[n, :n], sR[n, :n] = w, sw
                    R[n, n], sR[n, n] = sq, ssq
                    S.append(t)
                if xi is not None:
                    f, sf = f + sn * LD(xi[b, t, a]), sf + abs(sn * LD(xi[b, t, a]))
                out['samples'][b, t, a], out['s_samples'][b, t, a] = f, sf
                out['kept'][b, t, a], out['d'][b, t, a] = own, d
                out['margin'][b, t, a] = float(abs(d - delta * sf2) / sd)
    return out
