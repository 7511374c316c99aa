"""gpmpc_predict_hess, the jac_jac_gp_b200 CasADi external and GP.predict_batch_hess on the GPU: second
derivatives of the prediction against the closed-form oracle (triangular solves with the factor) and
central differences, bit-identity of the first-order outputs with gpmpc_predict_grad, exact symmetry,
reproducibility and the argument checks."""
import ctypes as C
import itertools

import numpy as np
import pytest

from gp_mpc_b200 import _lib as L
from oracle import gp_oracle as orc
from oracle import hess_oracle as hor
from tests._engines import ccs, fit, gp_from_fixture
from tests._util import load_fixture, load_golden, relinf

pytestmark = pytest.mark.gpu

FIRST = ('mean', 'var', 'cov', 'jac', 'dvar_dz', 'dcov_dz', 'hess')


def _case(case):
    """X, Y, hyper, Z, Sigma and the CPU factor (alpha, chol per output)."""
    if case in ('tank', 'car'):
        m = load_fixture(case); X, Y, hyper = m['X'], m['Y'], m['hyper']
        rng = np.random.default_rng(5)
        Z = X[rng.choice(X.shape[0], 6, replace=False)] + 0.05 * rng.standard_normal((6, X.shape[1]))
        A = rng.standard_normal((X.shape[1],) * 2); Sigma = 1e-3 * np.eye(X.shape[1]) + 1e-4 * A @ A.T
        post = orc.postfit(X, Y, hyper, lapack_general_solve=False)
        return X, Y, hyper, Z, Sigma, post['alpha'], post['chol']
    N, Nx, Ny, H = {'syn700': (700, 7, 3, 9), 'syn1500': (1500, 17, 3, 66), 'syn4200': (4200, 12, 2, 70)}[case]
    p = orc.synthetic_problem(N, Nx, Ny, config_id=N, H=H)
    X, Y, hyper, Z, Sigma = p['X'], p['Y'], p['hyper'], p['Z'], p['Sigma']
    facs = [orc.factor_large(X, Y[:, a], hyper[a]) for a in range(Ny)]
    return X, Y, hyper, Z, Sigma, np.stack([f['alpha'] for f in facs]), np.stack([f['chol'] for f in facs])


def _all_perms_equal(T):
    return all(np.array_equal(T, np.transpose(T, (0, 1) + tuple(2 + p for p in perm)))
               for perm in itertools.permutations(range(3)))


@pytest.mark.parametrize('case', ['tank', 'car', 'syn700', 'syn1500', 'syn4200'])
def test_predict_hess_vs_oracle(case):
    """syn4200 (Nx = 12): 5 points per derivative pass, 14 passes per 64-point chunk, two chunks, N > 4096."""
    X, Y, hyper, Z, Sigma, alpha, chol = _case(case)
    eng = fit(X, Y, hyper)
    Sg = np.stack([Sigma * (1 + 0.05 * h) for h in range(Z.shape[0])])
    tol = 3e-5 if case == 'car' else 1e-6
    for method, name, S in ((L.METHOD_TA, 'TA', Sg), (L.METHOD_ME, 'ME', None)):
        o = eng.predict_hess(Z, S, method)
        g = eng.predict_grad(Z, S, method, want_hess=True)
        for k in FIRST:
            assert np.array_equal(o[k], g[k]), k
        ref = hor.predict_hess(X, hyper, alpha, chol, Z, Sg if name == 'TA' else None, name)
        errs = dict(d2var=relinf(o['d2var_dz2'], ref['d2var']), d3mean=relinf(o['d3mean_dz3'], ref['d3mean']),
                    d2cov=relinf(o['d2cov_dz2'], ref['d2cov']))
        assert max(errs.values()) < tol, (name, errs)
        assert np.array_equal(o['d2var_dz2'], np.swapaxes(o['d2var_dz2'], 2, 3))
        assert np.array_equal(o['d2cov_dz2'], np.swapaxes(o['d2cov_dz2'], 3, 4))
        assert _all_perms_equal(o['d3mean_dz3'])
        o2 = eng.predict_hess(Z, S, method)
        for k in o:
            assert np.array_equal(o[k], o2[k]), k
    eng.close()


def test_predict_hess_argument_checks():
    lib = L.load()
    m = load_fixture('tank'); X, Y, hyper = m['X'], m['Y'], m['hyper']
    Ny, Nx = Y.shape[1], X.shape[1]
    eng = fit(X, Y, hyper)
    Z = X[:3] + 0.01
    S = 1e-3 * np.eye(Nx)
    with pytest.raises(L.GpmpcError) as e:
        eng.predict_hess(Z, S, L.METHOD_EM)
    assert e.value.code == L.ERR_ARG
    # every output is optional: only d2cov requested
    full = eng.predict_hess(Z, S, L.METHOD_TA)
    d2cov = np.empty((3, Ny, Ny, Nx, Nx))
    dp = C.POINTER(C.c_double)
    Zc = np.ascontiguousarray(Z)
    rc = lib.gpmpc_predict_hess(eng.h, L.METHOD_TA, 3, Zc.ctypes.data_as(dp), S.ctypes.data_as(dp), 0,
                                *([None] * 9), d2cov.ctypes.data_as(dp))
    assert rc == L.OK and np.array_equal(d2cov, full['d2cov_dz2'])
    eng.close()
    # a handle that owns only some of the outputs
    part = fit(X, Y, hyper, out_begin=0, out_count=Ny - 1)
    with pytest.raises(L.GpmpcError) as e:
        part.predict_hess(Z, S, L.METHOD_TA)
    assert e.value.code == L.ERR_STATE
    part.close()


def _dense(pat, vals):
    nrow, ncol, colind, rows = pat
    D = np.zeros((nrow, ncol))
    for c in range(ncol):
        for k in range(colind[c], colind[c + 1]):
            D[rows[k], c] = vals[k]
    return D


@pytest.mark.parametrize('method', ['TA', 'ME'])
def test_jac_jac_external_entry_points(method):
    """jac_jac_gp_b200 through ctypes the way CasADi drives it: the 16 patterns, their values against
    gpmpc_predict_hess and against central differences of jac_gp_b200's own outputs."""
    m = load_fixture('tank'); X, Y, hyper = m['X'], m['Y'], m['hyper']
    Ny, Nx, Nt = 4, 6, 5
    eng = fit(X, Y, hyper)
    lib = L.load()
    meth = L.METHOD_TA if method == 'TA' else L.METHOD_ME
    rng = np.random.default_rng(8)
    Z = X[:Nt] + 0.1 * rng.standard_normal((Nt, Nx))
    Sg = np.stack([1e-3 * np.eye(Nx) + 1e-4 * (lambda A: A @ A.T)(rng.standard_normal((Nx, Nx))) for _ in range(Nt)])
    assert lib.gp_b200_bind(eng.h, meth, Nt) == 0
    dp = C.POINTER(C.c_double)

    def call(fn, ins, outs):
        arg = (dp * len(ins))(*[a.ctypes.data_as(dp) for a in ins])
        res = (dp * len(outs))(*[a.ctypes.data_as(dp) for a in outs])
        assert fn(arg, res, None, None, 0) == 0

    z_cm = np.ascontiguousarray(Z)                                        # Nx x Nt column-major
    s_cm = np.ascontiguousarray(np.transpose(Sg, (0, 2, 1)))               # Nx x Nx*Nt column-major
    mean_cm = np.empty((Nt, Ny)); cov_cm = np.empty((Nt, Ny, Ny))
    call(lib.gp_b200, [z_cm, s_cm], [mean_cm, cov_cm])
    jpats = [ccs(lib.jac_gp_b200_sparsity_out(k)) for k in range(4)]

    def jac_dense(z, s):
        outs = [np.zeros(max(1, p[2][-1])) for p in jpats]
        call(lib.jac_gp_b200, [z, s, mean_cm, cov_cm], outs)
        return [_dense(p, v) for p, v in zip(jpats, outs)]

    for k in range(4):                                                    # inputs 4..7 carry jac_gp_b200's patterns
        assert ccs(lib.jac_jac_gp_b200_sparsity_in(4 + k)) == jpats[k]
    n_in = [Nx * Nt, Nx * Nx * Nt, Ny * Nt, Ny * Ny * Nt]
    n_o = [p[0] * p[1] for p in jpats]
    pats = [ccs(lib.jac_jac_gp_b200_sparsity_out(k)) for k in range(16)]
    ta = method == 'TA'
    nnz = {0: Nt * Ny * Nx * Nx, 8: Nt * Ny * Ny * Nx * Nx, 9: Nt * Ny * Ny * Nx ** 3 if ta else 0,
           12: Nt * Ny * Ny * Nx ** 3 if ta else 0}
    for k, p in enumerate(pats):
        assert (p[0], p[1], p[2][-1]) == (n_o[k // 4], n_in[k % 4], nnz.get(k, 0)), k
    outs = [np.zeros(max(1, p[2][-1])) for p in pats]
    call(lib.jac_jac_gp_b200, [z_cm, s_cm, mean_cm, cov_cm] + [np.zeros(max(1, p[2][-1])) for p in jpats], outs)
    D = [_dense(p, v) for p, v in zip(pats, outs)]
    # values against gpmpc_predict_hess: mean_z_z and cov_z_z per node
    o = eng.predict_hess(Z, Sg if ta else None, meth)
    for t in range(Nt):
        for a in range(Ny):
            for d in range(Nx):
                r = (a + Ny * t) + Ny * Nt * (d + Nx * t)
                assert np.array_equal(D[0][r, Nx * t:Nx * (t + 1)], o['hess'][t, a, d])
        for a in range(Ny):
            for b in range(Ny):
                for e in range(Nx):
                    r = (a + Ny * b + Ny * Ny * t) + Ny * Ny * Nt * (e + Nx * t)
                    assert np.array_equal(D[8][r, Nx * t:Nx * (t + 1)], o['d2cov_dz2'][t, a, b, e])
    # central differences of jac_gp_b200 w.r.t. z and (TA) sigma, column-major vec of each Jacobian
    for i_in, base in ((0, z_cm), (1, s_cm)):
        flat = base.reshape(-1)
        for c in range(flat.size):
            st = 1e-4 * max(1.0, abs(flat[c])) if i_in == 0 else 1e-3
            zp, zm = base.copy(), base.copy()
            zp.reshape(-1)[c] += st; zm.reshape(-1)[c] -= st
            jp = jac_dense(zp if i_in == 0 else z_cm, zp if i_in == 1 else s_cm)
            jm = jac_dense(zm if i_in == 0 else z_cm, zm if i_in == 1 else s_cm)
            for oi in range(4):
                fd = (jp[oi].reshape(-1, order='F') - jm[oi].reshape(-1, order='F')) / (2 * st)
                got = D[oi * 4 + i_in][:, c]
                den = max(np.abs(D[oi * 4 + i_in]).max(), 1e-300)
                assert np.abs(got - fd).max() / den < 1e-5, (oi, i_in, c)
    lib.gp_b200_unbind()
    assert not lib.jac_jac_gp_b200_sparsity_out(0)
    eng.close()


def test_gp_predict_batch_hess_vs_central_differences():
    gp, m = gp_from_fixture('tank')
    assert m['normalize']
    d = load_golden('derived', 'tank')
    xs = np.tile(d['x0'], (3, 1)) * (1 + 0.02 * np.arange(3)[:, None]); us = np.tile(d['u0'], (3, 1))
    Sigma = d['Sigma']
    gh = gp.predict_batch_hess(xs, us, Sigma)
    gg = gp.predict_batch_grad(xs, us, Sigma)
    for k in gg:
        assert np.array_equal(gh[k], gg[k]), k
    zs = np.hstack([xs, us])
    for e in range(zs.shape[1]):
        # fourth-order central differences: the covariance derivatives are ~1e-8, so a second-order stencil small
        # enough for its truncation error drowns in the rounding of the first derivatives
        h = 1e-3 * max(1.0, abs(zs[0, e]))
        g = {}
        for k in (-2, -1, 1, 2):
            zk = zs.copy(); zk[:, e] += k * h
            g[k] = gp.predict_batch_grad(zk[:, :4], zk[:, 4:], Sigma)
        fd = lambda n: (g[-2][n] - 8 * g[-1][n] + 8 * g[1][n] - g[2][n]) / (12 * h)
        assert relinf(gh['d2mean_dz2'][..., e], fd('dmean_dz')) < 1e-5
        assert relinf(gh['d2cov_dz2'][..., e], fd('dcov_dz')) < 1e-5
        assert relinf(gh['dcov_dSigma_hess'][..., e], fd('dcov_dSigma_factor')) < 1e-5
    with pytest.raises(NotImplementedError):
        gp.predict_batch_hess(xs, us, Sigma, method='EM')
    gp.close()
