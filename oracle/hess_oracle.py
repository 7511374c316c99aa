"""Closed-form first and second derivatives of the restated prediction w.r.t. the test input  --
TEST INFRASTRUCTURE ONLY (the checker of gpmpc_predict_grad / gpmpc_predict_hess).

With IPOPT's default exact Hessian (``hessian_approximation``), CasADi differentiates the symbolic
``build_gp`` / ``build_TA_cov`` graphs (``gp_functions.py:111-173``) twice inside ``nlpsol``
(``mpc_class.py:390-412``, ``:496-513``).  The reference has no closed forms; these are derived
from ``gp_oracle.gp_mean_var`` / ``gp_mean_jac`` / ``ta_cov`` and checked by central differences
(``predict_hess_fd``).  Per output a, test point z, standardised input space, with
``k_i = ks_i``, ``s_id = (x_id - z_d)/ell_d^2``, ``beta = K^-1 k``, J / H the mean Jacobian / Hessian:

    d3 mean / dz_d dz_e dz_f = M3_def - d_de J_f/ell_d^2 - d_df J_e/ell_d^2 - d_ef J_d/ell_e^2,
                               M3_def = sum_i alpha_i k_i s_id s_ie s_if
    d2 var / dz_d dz_e       = -2 [G_de + B2_de - d_de (k^T K^-1 k)/ell_d^2],
                               B2_de = sum_i beta_i k_i s_id s_ie,  G_de = (L^-1 d_d k)^T (L^-1 d_e k)
    'ME': d2 cov_ab = delta_ab d2 var_a
    'TA': d2 cov_ab / dz_f dz_g = delta_ab d2 var_a + sum_de [T_a,dfg S_de J_b,e + H_a,df S_de H_b,eg
                                  + H_a,dg S_de H_b,ef + J_a,d S_de T_b,efg]        (S = Sigma, not symmetrised)

Every solve goes through the Cholesky factor: the explicit K^-1 loses ~1e-4 relative on the car fixture.
"""
from __future__ import annotations

import numpy as np
from scipy.linalg import solve_triangular

from oracle import gp_oracle as orc


def _parts(X, hyper_a, alpha_a, L_a, Z):
    """Per-output building blocks for a batch: ks (N,H), s (H,N,Nx), beta (N,H), v (N,H)."""
    Nx = X.shape[1]
    ell = hyper_a[:Nx]; sf2 = hyper_a[Nx] ** 2
    ks = orc.covSEard(X, Z, ell, sf2)
    v = solve_triangular(L_a, ks, lower=True, check_finite=False)
    beta = solve_triangular(L_a, v, lower=True, trans='T', check_finite=False)
    s = (X[None, :, :] - Z[:, None, :]) / ell ** 2
    return ell, ks, s, v, beta


def _sigmas(Sigma, H, Nx):
    Sigma = np.asarray(Sigma, dtype=np.float64)
    return np.broadcast_to(Sigma, (H, Nx, Nx)) if Sigma.ndim == 2 else Sigma


def predict_grad_closed(X, hyper, alpha, chol, Z, Sigma, method='TA'):
    """Closed-form first derivatives (what gpmpc_predict_grad computes).  Same arguments as
    ``gp_oracle.predict_grad_fd``; returns dict(dmean (H,Ny,Nx), dvar (H,Ny,Nx), dcov (H,Ny,Ny,Nx),
    hess (H,Ny,Nx,Nx)) plus mean, var (H,Ny)."""
    X = np.asarray(X, dtype=np.float64)
    Z = np.atleast_2d(np.asarray(Z, dtype=np.float64))
    hyper = np.atleast_2d(np.asarray(hyper, dtype=np.float64))
    H, Nx = Z.shape
    Ny = hyper.shape[0]
    mean = np.zeros((H, Ny)); var = np.zeros((H, Ny))
    J = np.zeros((H, Ny, Nx)); dvar = np.zeros((H, Ny, Nx)); Hm = np.zeros((H, Ny, Nx, Nx))
    for a in range(Ny):
        ell, ks, s, v, beta = _parts(X, hyper[a], alpha[a], chol[a], Z)
        mean[:, a] = ks.T @ alpha[a]
        var[:, a] = hyper[a, Nx] ** 2 - np.sum(v * v, axis=0)
        for h in range(H):
            wa = alpha[a] * ks[:, h]
            J[h, a] = wa @ s[h]
            dvar[h, a] = -2 * (beta[:, h] * ks[:, h]) @ s[h]
            Hm[h, a] = (s[h] * wa[:, None]).T @ s[h] - np.diag(mean[h, a] / ell ** 2)
    dcov = np.zeros((H, Ny, Ny, Nx))
    if method == 'TA':
        S = _sigmas(Sigma, H, Nx)
        dcov += np.einsum('hade,hbd->habe', Hm, np.einsum('hde,hbe->hbd', S, J))
        dcov += np.einsum('had,hbde->habe', np.einsum('had,hde->hae', J, S), Hm)
    for a in range(Ny):
        dcov[:, a, a, :] += dvar[:, a, :]
    return dict(mean=mean, var=var, dmean=J, dvar=dvar, dcov=dcov, hess=Hm)


def predict_hess(X, hyper, alpha, chol, Z, Sigma, method='TA'):
    """Closed-form second derivatives (what gpmpc_predict_hess adds to gpmpc_predict_grad).  Same
    arguments as ``gp_oracle.predict_grad_fd`` (chol may hold ``factor_large`` factors).  Returns
    ``predict_grad_closed``'s dict plus d2var (H,Ny,Nx,Nx), d3mean (H,Ny,Nx,Nx,Nx),
    d2cov (H,Ny,Ny,Nx,Nx)."""
    X = np.asarray(X, dtype=np.float64)
    Z = np.atleast_2d(np.asarray(Z, dtype=np.float64))
    hyper = np.atleast_2d(np.asarray(hyper, dtype=np.float64))
    H, Nx = Z.shape
    Ny = hyper.shape[0]
    out = predict_grad_closed(X, hyper, alpha, chol, Z, Sigma, method)
    J, Hm = out['dmean'], out['hess']
    d2var = np.zeros((H, Ny, Nx, Nx)); d3 = np.zeros((H, Ny, Nx, Nx, Nx))
    eye = np.eye(Nx)
    for a in range(Ny):
        ell, ks, s, v, beta = _parts(X, hyper[a], alpha[a], chol[a], Z)
        il2 = 1.0 / ell ** 2
        for h in range(H):
            dk = ks[:, h][:, None] * s[h]                                  # (N,Nx): d_d k
            Vd = solve_triangular(chol[a], dk, lower=True, check_finite=False)
            G = Vd.T @ Vd
            B2 = (s[h] * (beta[:, h] * ks[:, h])[:, None]).T @ s[h]
            q = float(np.sum(v[:, h] ** 2))                               # k^T K^-1 k
            d2var[h, a] = -2 * (G + B2 - np.diag(il2) * q)
            M3 = np.einsum('i,id,ie,if->def', alpha[a] * ks[:, h], s[h], s[h], s[h], optimize=True)
            Lj = (eye * il2[:, None])                                      # Lambda^-1
            d3[h, a] = (M3 - np.einsum('de,f->def', Lj, J[h, a]) - np.einsum('df,e->def', Lj, J[h, a])
                        - np.einsum('ef,d->def', Lj, J[h, a]))
    d2cov = np.zeros((H, Ny, Ny, Nx, Nx))
    if method == 'TA':
        S = _sigmas(Sigma, H, Nx)
        d2cov += np.einsum('hadfg,hde,hbe->habfg', d3, S, J, optimize=True)
        d2cov += np.einsum('hadf,hde,hbeg->habfg', Hm, S, Hm, optimize=True)
        d2cov += np.einsum('hadg,hde,hbef->habfg', Hm, S, Hm, optimize=True)
        d2cov += np.einsum('had,hde,hbefg->habfg', J, S, d3, optimize=True)
    for a in range(Ny):
        d2cov[:, a, a] += d2var[:, a]
    out.update(d2var=d2var, d3mean=d3, d2cov=d2cov)
    return out


def derivs_core_ld(X, hyper, alpha, linv, Z, absolute=False, second=True):
    """The Sigma-free part of ``predict_derivs_ld``: dict(mean, var (H,Ny), J (H,Ny,Nx), dvar_dz (H,Ny,Nx),
    hess (H,Ny,Nx,Nx), d2var_dz2 (H,Ny,Nx,Nx), d3mean_dz3 (H,Ny,Nx,Nx,Nx)) in np.longdouble, on the path of the
    kernels: ks by direct differences, v = L^-1 ks, beta = L^-T v and V_d = L^-1 d_d ks as products with ``linv``
    (Ny,N,N, lower, as GET_LINV returns it), k^T K^-1 k = |v|^2.  ``absolute``: the sums of |terms| of every output
    (see ``predict_derivs_ld``).  ``second=False`` leaves out d2var_dz2 and d3mean_dz3 (what gpmpc_predict_grad and
    the roll-outs need; V_d and the third moments dominate the cost at large Nx)."""
    ld = np.longdouble
    X = np.asarray(X, dtype=ld)
    Z = np.atleast_2d(np.asarray(Z, dtype=ld))
    hyper = np.atleast_2d(np.asarray(hyper, dtype=ld))
    H, Nx = Z.shape
    Ny = hyper.shape[0]
    sg = 1 if absolute else -1                                    # the sign of every subtraction
    shapes = (('mean', (H, Ny)), ('var', (H, Ny)), ('J', (H, Ny, Nx)), ('dvar_dz', (H, Ny, Nx)), ('hess', (H, Ny, Nx, Nx)))
    if second:
        shapes += (('d2var_dz2', (H, Ny, Nx, Nx)), ('d3mean_dz3', (H, Ny, Nx, Nx, Nx)))
    out = {k: np.zeros(s, dtype=ld) for k, s in shapes}
    eye = np.eye(Nx, dtype=ld)
    for a in range(Ny):
        ell = hyper[a, :Nx]
        sf2 = hyper[a, Nx] ** 2
        il2 = 1 / ell ** 2
        Li = np.asarray(linv[a], dtype=ld)
        al = np.asarray(alpha[a], dtype=ld)
        if absolute:
            Li, al = np.abs(Li), np.abs(al)
        diff = (X[None, :, :] - Z[:, None, :]) / ell                 # (H,N,Nx)
        ks = sf2 * np.exp(-np.sum(diff * diff, axis=2) / 2)          # (H,N)
        s = (X[None, :, :] - Z[:, None, :]) * il2                    # (H,N,Nx)
        if absolute:
            s = np.abs(s)
        v = Li @ ks.T                                                # (N,H)
        beta = Li.T @ v
        q = np.sum(v * v, axis=0)                                    # k^T K^-1 k
        wa = al[None, :] * ks                                        # (H,N)
        wb = beta.T * ks
        mean = wa.sum(1)
        J = np.einsum('hi,hid->hd', wa, s)
        out['mean'][:, a] = mean
        out['var'][:, a] = sf2 + sg * q
        out['J'][:, a] = J
        out['dvar_dz'][:, a] = 2 * sg * np.einsum('hi,hid->hd', wb, s)
        out['hess'][:, a] = np.einsum('hi,hid,hie->hde', wa, s, s) + sg * mean[:, None, None] * np.diag(il2)
        if not second:
            continue
        dk = ks[:, :, None] * s                                      # (H,N,Nx): d_d ks
        Vd = (Li @ np.transpose(dk, (1, 0, 2)).reshape(-1, H * Nx)).reshape(-1, H, Nx)
        G = np.einsum('ihd,ihe->hde', Vd, Vd)
        B2 = np.einsum('hi,hid,hie->hde', wb, s, s)
        # the kernels take k^T K^-1 k as sf2 - var, whose sum of |terms| is sf2 + |var|
        qn = sf2 + out['var'][:, a] if absolute else q
        out['d2var_dz2'][:, a] = 2 * sg * (G + B2 + sg * qn[:, None, None] * np.diag(il2))
        M3 = np.einsum('hi,hid,hie,hif->hdef', wa, s, s, s, optimize=True)
        Lj = eye * il2[:, None]
        out['d3mean_dz3'][:, a] = M3 + sg * (np.einsum('de,hf->hdef', Lj, J) + np.einsum('df,he->hdef', Lj, J)
                                             + np.einsum('ef,hd->hdef', Lj, J))
    return out


def cov_derivs(core, Sigma, method):
    """cov (H,Ny,Ny), dcov_dz (H,Ny,Ny,Nx) and d2cov_dz2 (H,Ny,Ny,Nx,Nx) from ``derivs_core_ld``'s outputs and Sigma
    ((Nx,Nx) shared or (H,Nx,Nx), not symmetrised): diag(var) + J Sigma J^T and its derivatives for 'TA', diag(var) and
    its derivatives for 'ME'.  Fed a core with absolute=True and |Sigma|, the sums of |terms|.  A core made with
    second=False gives no d2cov_dz2."""
    second = 'd3mean_dz3' in core
    var, J, Hm = (core[k] for k in ('var', 'J', 'hess'))
    H, Ny, Nx = J.shape
    cov = np.zeros((H, Ny, Ny), dtype=var.dtype)
    dcov = np.zeros((H, Ny, Ny, Nx), dtype=var.dtype)
    d2cov = np.zeros((H, Ny, Ny, Nx, Nx) if second else (0,), dtype=var.dtype)
    if method == 'TA':
        S = np.asarray(Sigma, dtype=var.dtype)
        S = np.broadcast_to(S, (H, Nx, Nx)) if S.ndim == 2 else S
        cov += np.einsum('had,hde,hbe->hab', J, S, J)
        dcov += np.einsum('hadf,hde,hbe->habf', Hm, S, J) + np.einsum('had,hde,hbef->habf', J, S, Hm)
    if method == 'TA' and second:
        T3 = core['d3mean_dz3']
        d2cov += (np.einsum('hadfg,hde,hbe->habfg', T3, S, J, optimize=True)
                  + np.einsum('hadf,hde,hbeg->habfg', Hm, S, Hm, optimize=True)
                  + np.einsum('hadg,hde,hbef->habfg', Hm, S, Hm, optimize=True)
                  + np.einsum('had,hde,hbefg->habfg', J, S, T3, optimize=True))
    for a in range(Ny):
        cov[:, a, a] += var[:, a]
        dcov[:, a, a] += core['dvar_dz'][:, a]
        if second:
            d2cov[:, a, a] += core['d2var_dz2'][:, a]
    out = dict(cov=cov, dcov_dz=dcov)
    if second:
        out['d2cov_dz2'] = d2cov
    return out


def predict_derivs_ld(X, hyper, alpha, linv, Z, Sigma, method, absolute=False):
    """Every output of gpmpc_predict_hess in np.longdouble, on the engine's own alpha (Ny,N) and L^-1 (Ny,N,N) (GET_ALPHA,
    GET_LINV) so that cond(K) enters neither side of a comparison: dict(mean, var, J, dvar_dz, hess, d2var_dz2,
    d3mean_dz3, cov, dcov_dz, d2cov_dz2) shaped as gpmpc_predict_hess's outputs, with the module docstring's formulas.

    ``absolute=True`` evaluates the same expressions on |L^-1|, |alpha|, |s|, |Sigma| with every subtraction turned into
    an addition (var -> sf2 + |v|^2, the -delta/ell^2 terms added): the sum of |terms| of each output, including the
    cancellation inside L^-1 ks itself.  It is the scale against which a kernel's rounding is measured."""
    core = derivs_core_ld(X, hyper, alpha, linv, Z, absolute)
    if absolute and Sigma is not None:
        Sigma = np.abs(np.asarray(Sigma, dtype=np.float64))
    core.update(cov_derivs(core, Sigma, method))
    return core


def predict_hess_fd(X, hyper, alpha, chol, Z, Sigma, method='TA', rel=1e-4):
    """Central differences of ``predict_grad_closed`` w.r.t. every test-input coordinate: the
    checker of ``predict_hess``.  Returns dict(d2var, d3mean, d2cov) shaped as there."""
    Z = np.atleast_2d(np.asarray(Z, dtype=np.float64))
    hyper = np.atleast_2d(np.asarray(hyper, dtype=np.float64))
    H, Nx = Z.shape
    Ny = hyper.shape[0]
    out = dict(d2var=np.zeros((H, Ny, Nx, Nx)), d3mean=np.zeros((H, Ny, Nx, Nx, Nx)),
               d2cov=np.zeros((H, Ny, Ny, Nx, Nx)))
    for g in range(Nx):
        step = rel * np.maximum(1.0, np.abs(Z[:, g]))
        Zp = Z.copy(); Zp[:, g] += step
        Zm = Z.copy(); Zm[:, g] -= step
        p = predict_grad_closed(X, hyper, alpha, chol, Zp, Sigma, method)
        m = predict_grad_closed(X, hyper, alpha, chol, Zm, Sigma, method)
        out['d2var'][..., g] = (p['dvar'] - m['dvar']) / (2 * step[:, None, None])
        out['d3mean'][..., g] = (p['hess'] - m['hess']) / (2 * step[:, None, None, None])
        out['d2cov'][..., g] = (p['dcov'] - m['dcov']) / (2 * step[:, None, None, None])
    return out
