"""gpmpc_predict_em_hess and GP.predict_batch_em_hess on the GPU: 'EM' second derivatives against the long-double closed
form on the engine's own alpha and factor, against fourth-order differences of the engine's gpmpc_predict_em_grad, the
heat-equation identities at an arbitrary Sigma, the Sigma = 0 limit against the ME / TA Hessian entries, bit-identity of
the first outputs with gpmpc_predict_em_grad, exact symmetry, reproducibility and batch independence, the argument checks,
the CasADi external bound with gp_b200_bind_em_hess, and the GP's chain rule through the scalers."""
import ctypes as C

import numpy as np
import pytest

from gp_mpc_b200 import _lib as L
from oracle import em_grad_oracle as emg
from oracle import em_hess_oracle as emh
from oracle import gp_oracle as orc
from tests._em_cases import em_problem, engine_alpha_chol, grad_case, sigmas
from tests._engines import ccs, fit, gp_from_fixture
from tests._util import d4, load_fixture, load_golden, relinf

pytestmark = pytest.mark.gpu

FIRST = ('mean', 'var', 'cov', 'dmean_dz', 'dmean_dSigma', 'dcov_dz', 'dcov_dSigma')
MEAN_KEYS = ('d2mean_dz2', 'd2mean_dSigma_dz', 'd2mean_dSigma2')
COV_KEYS = ('d2cov_dz2', 'd2cov_dSigma_dz', 'd2cov_dSigma2')


def _hess_case(case):
    """test_em_grad_gpu's cases, plus '<shape>_s1e-5', 'car' (cond(K) ~ 1e10) and 'nx16' (N = 300, Nx = 16: every feature
    slot of the 16 bucket); the synthetic cases, car and the shapes at one point (the long-double oracle takes 10-20 s per
    point at N ~ 1000 or Nx >= 12)."""
    if case == 'car':
        m = load_fixture('car'); X, Y, hyper = m['X'], m['Y'], m['hyper']
        rng = np.random.default_rng(5)
        Nx = X.shape[1]
        Z = X[:1] + 0.05 * rng.standard_normal((1, Nx))
        A = rng.standard_normal((Nx, Nx))
        return X, Y, hyper, Z, 1e-3 * np.eye(Nx) + 1e-4 * A @ A.T, None
    if case == 'nx16':
        p = orc.synthetic_problem(300, 16, 2, config_id=316, H=1)
        hyper = p['hyper'].copy(); hyper[:, 17] = 0.3
        return p['X'], p['Y'], hyper, p['Z'][:1], sigmas(hyper, 16)['0.1'], None
    X, Y, hyper, Z, Sigma, cap = grad_case(case)
    if '_s' in case or case.startswith('syn'):
        Z = Z[:1]
    return X, Y, hyper, Z, Sigma, cap


def _symmetric(o):
    """every returned tensor is exactly symmetric under its index symmetries"""
    m3, m4 = o['d2mean_dSigma_dz'], o['d2mean_dSigma2']
    c3, c4 = o['d2cov_dSigma_dz'], o['d2cov_dSigma2']
    assert np.array_equal(o['d2mean_dz2'], np.swapaxes(o['d2mean_dz2'], 2, 3))
    for perm in ((0, 1, 3, 2, 4), (0, 1, 2, 4, 3), (0, 1, 4, 3, 2)):
        assert np.array_equal(m3, np.transpose(m3, perm))
    for perm in ((0, 1, 3, 2, 4, 5), (0, 1, 2, 4, 3, 5), (0, 1, 2, 3, 5, 4), (0, 1, 4, 5, 2, 3)):
        assert np.array_equal(m4, np.transpose(m4, perm))
    assert np.array_equal(o['d2cov_dz2'], np.swapaxes(o['d2cov_dz2'], 3, 4))
    assert np.array_equal(o['d2cov_dz2'], np.swapaxes(o['d2cov_dz2'], 1, 2))
    assert np.array_equal(c3, np.swapaxes(c3, 3, 4)) and np.array_equal(c3, np.swapaxes(c3, 1, 2))
    for perm in ((0, 2, 1, 3, 4, 5, 6), (0, 1, 2, 4, 3, 5, 6), (0, 1, 2, 3, 4, 6, 5), (0, 1, 2, 5, 6, 3, 4)):
        assert np.array_equal(c4, np.transpose(c4, perm))


def em_hess_errors(case):
    """The engine's predict_em_hess on a case against em_hess_closed on the engine's own alpha and factor, after the
    bit-level checks: errors of every output / pair block normalised by its sum of |terms| (em_hess_terms)."""
    X, Y, hyper, Z, Sigma, cap = _hess_case(case)
    Ny = Y.shape[1]
    eng = fit(X, Y, hyper, capacity=cap)
    o = eng.predict_em_hess(Z, Sigma)
    g = eng.predict_em_grad(Z, Sigma)
    for k in FIRST:
        assert np.array_equal(o[k], g[k]), k
    for k in MEAN_KEYS + COV_KEYS:
        assert np.all(np.isfinite(o[k])), k
    _symmetric(o)
    o2 = eng.predict_em_hess(Z, Sigma)
    for k in o:
        assert np.array_equal(o[k], o2[k]), k
    alpha, chol = engine_alpha_chol(eng, Ny)
    eng.close()
    ref = emh.em_hess_closed(X, hyper, alpha, chol, Z, Sigma)
    return emh.normalised_errors(o, ref, emh.em_hess_terms(X, hyper, alpha, chol, Z, Sigma))


SHAPES = [n + s for n in ('nx1', 'ny9', 'reserved', 'nx8') for s in ('_s1e-5', '_s0.1', '_s1')]
# (mean blocks, cov blocks) bars on the errors normalised by the sums of |terms|, measured on an H100 SXM at 700 W over every
# case: mean <= 5.6e-17 (tank_large), cov <= 5.4e-19 (ny9 at Sigma = Lambda)
HESS_TOL = (3e-16, 3e-18)


@pytest.mark.parametrize('case', ['tank', 'tank_pp', 'tank_large', 'car', 'syn1000', 'syn12', 'nx16'] + SHAPES)
def test_em_hess_vs_closed_oracle(case):
    """syn1000: Nx = 8, N ~ 1000; syn12: Nx = 12 and nx16: Nx = 16, the 16 bucket; tank_pp: one Sigma per point; the shapes of
    test_em_shapes_gpu at Sigma = 1e-5 Lambda, 0.1 Lambda (correlated) and Lambda: nx1 (one live dimension), ny9 (45
    pairs), reserved (an identity tail of L^-1) and nx8 (N = 1030, a partial last tile)."""
    errs = em_hess_errors(case)
    tm, tc = HESS_TOL
    assert all(errs[k] < tm for k in MEAN_KEYS), errs
    assert all(errs[k] < tc for k in COV_KEYS), errs


def test_em_hess_points_are_independent_of_their_batch():
    X, Y, hyper, Z, Sigma, _ = grad_case('tank_pp')
    eng = fit(X, Y, hyper)
    full = eng.predict_em_hess(Z, Sigma)
    for p in (0, Z.shape[0] - 1):
        one = eng.predict_em_hess(Z[p:p + 1], Sigma[p:p + 1])
        for k in one:
            assert np.array_equal(one[k][0], full[k][p]), (p, k)
    eng.close()


@pytest.mark.parametrize('case,tol', [('tank', 1e-5), ('car', 1e-3)])
def test_em_hess_vs_differences_of_the_engine(case, tol):
    """Fourth-order differences of the engine's own gpmpc_predict_em_grad in each z_f and along each symmetric Sigma
    pair (f, g)."""
    m = load_fixture(case); X, Y, hyper = m['X'], m['Y'], m['hyper']
    Nx = X.shape[1]
    rng = np.random.default_rng(11)
    Z = X[:2] + 0.05 * rng.standard_normal((2, Nx))
    A = rng.standard_normal((Nx, Nx)); S = 1e-3 * np.eye(Nx) + 1e-4 * A @ A.T
    eng = fit(X, Y, hyper)
    o = eng.predict_em_hess(Z, S)
    pairs = (('dmean_dz', 'd2mean_dz2'), ('dmean_dSigma', 'd2mean_dSigma_dz'), ('dcov_dz', 'd2cov_dz2'),
             ('dcov_dSigma', 'd2cov_dSigma_dz'))
    fz = {k: np.zeros_like(o[k2]) for k, k2 in pairs}
    for f in range(Nx):
        e = np.zeros(Nx); e[f] = 1.0
        d = d4(lambda s: eng.predict_em_grad(Z + s * e, S), 3e-2)
        for k in fz:
            fz[k][..., f] = d[k]
    for k, k2 in pairs:
        assert relinf(o[k2], fz[k]) < tol, k2
    for f in range(Nx):
        for g in range(f + 1):
            E = np.zeros((Nx, Nx)); E[f, g] = E[g, f] = 1.0
            d = d4(lambda s: eng.predict_em_grad(Z, S + s * E), 3e-4)
            sc = 1.0 if f == g else 2.0
            assert relinf(sc * o['d2mean_dSigma2'][..., f, g], d['dmean_dSigma']) < tol, (f, g)
            assert relinf(sc * o['d2cov_dSigma2'][..., f, g], d['dcov_dSigma']) < tol, (f, g)
    eng.close()


def test_em_hess_heat_equation_identities():
    """At an arbitrary Sigma: dmean_dSigma = 1/2 d2mean_dz2, dcov_dSigma = 1/2 d2cov_dz2 + sym(J_a J_b^T), and
    d2mean_dSigma2 is fully symmetric in its four Sigma / z indices (it is 1/4 d^4 mean / dz^4)."""
    X, Y, hyper, Z, Sigma, _ = grad_case('syn12')
    eng = fit(X, Y, hyper)
    o = eng.predict_em_hess(Z, Sigma)
    eng.close()
    assert relinf(o['dmean_dSigma'], 0.5 * o['d2mean_dz2']) < 1e-12
    J = o['dmean_dz']
    JJ = np.einsum('had,hbe->habde', J, J)
    assert relinf(o['dcov_dSigma'], 0.5 * o['d2cov_dz2'] + 0.5 * (JJ + np.swapaxes(JJ, 1, 2))) < 1e-11
    m4 = o['d2mean_dSigma2']
    assert np.array_equal(m4, np.transpose(m4, (0, 1, 2, 4, 3, 5)))      # e <-> f: across the Sigma / Sigma pair


def test_em_hess_at_zero_sigma_against_me_ta():
    """Sigma = 0 against gpmpc_predict_hess: d2mean_dz2 = the ME Hessian, d2mean_dSigma_dz = 1/2 d3mean_dz3, the diagonal
    of d2cov_dz2 = d2var_dz2 and its off-diagonal ~ 0, and d2cov_dSigma_dz for a != b = the symmetrised TA mixed term."""
    m = load_fixture('tank'); X, Y, hyper = m['X'], m['Y'], m['hyper']
    Nx, Ny = X.shape[1], Y.shape[1]
    rng = np.random.default_rng(4)
    Z = X[:3] + 0.05 * rng.standard_normal((3, Nx))
    eng = fit(X, Y, hyper)
    o = eng.predict_em_hess(Z, np.zeros((Nx, Nx)))
    me = eng.predict_hess(Z, None, L.METHOD_ME)
    eng.close()
    assert relinf(o['d2mean_dz2'], me['hess']) < 1e-9
    assert relinf(o['d2mean_dSigma_dz'], 0.5 * me['d3mean_dz3']) < 1e-9
    d2var = me['d2var_dz2']
    J, Hm = me['jac'], me['hess']
    for a in range(Ny):
        assert relinf(o['d2cov_dz2'][:, a, a], d2var[:, a]) < 1e-7
        for b in range(Ny):
            if a == b:
                continue
            assert np.abs(o['d2cov_dz2'][:, a, b]).max() < 1e-7 * np.abs(d2var).max()
            mix = np.einsum('hdf,he->hdef', Hm[:, a], J[:, b]) + np.einsum('hd,hef->hdef', J[:, a], Hm[:, b])
            assert relinf(o['d2cov_dSigma_dz'][:, a, b], 0.5 * (mix + np.swapaxes(mix, 1, 2))) < 1e-7


def test_em_hess_argument_checks():
    """Nx = 17, a null Sigma, a handle that owns only some outputs and an unfactorised handle return their codes; the
    model still predicts the same afterwards."""
    import gp_mpc_b200
    lib = L.load()
    dp = C.POINTER(C.c_double)
    m = load_fixture('tank'); X, Y, hyper = m['X'], m['Y'], m['hyper']
    Ny, Nx = Y.shape[1], X.shape[1]
    Z = np.ascontiguousarray(X[:2] + 0.01)
    S = 1e-3 * np.eye(Nx)
    eng = fit(X, Y, hyper)
    before = eng.predict_em_hess(Z, S)
    assert lib.gpmpc_predict_em_hess(eng.h, 2, Z.ctypes.data_as(dp), None, 0, *([None] * 13)) == L.ERR_ARG
    assert lib.gpmpc_predict_em_hess(eng.h, 0, Z.ctypes.data_as(dp), S.ctypes.data_as(dp), 0, *([None] * 13)) == L.ERR_ARG
    after = eng.predict_em_hess(Z, S)
    for k in before:
        assert np.array_equal(before[k], after[k]), k
    eng.close()
    part = fit(X, Y, hyper, out_begin=0, out_count=Ny - 1)
    with pytest.raises(L.GpmpcError) as e:
        part.predict_em_hess(Z, S)
    assert e.value.code == L.ERR_STATE
    part.close()
    raw = gp_mpc_b200.Engine(X.shape[0], Nx, Ny, device=0)
    raw.set_data(X, Y); raw.set_hyper(hyper)
    with pytest.raises(L.GpmpcError) as e:
        raw.predict_em_hess(Z, S)
    assert e.value.code == L.ERR_STATE
    raw.close()
    X17, Y17, h17, Z17 = em_problem('nx17')
    e17 = fit(X17, Y17, h17)
    with pytest.raises(L.GpmpcError) as e:
        e17.predict_em_hess(Z17[:1], sigmas(h17, 17)['0.1'])
    assert e.value.code == L.ERR_ARG
    assert lib.gp_b200_bind_em_hess(e17.h, 2) == L.ERR_ARG
    e17.close()


def test_casadi_external_with_em_hess():
    """gp_b200_bind_em_hess driven through ctypes as CasADi drives it: gp_b200 and jac_gp_b200 equal the
    gp_b200_bind(EM) results bit for bit, and jac_jac_gp_b200's eight non-zero blocks equal gpmpc_predict_em_hess in
    pattern order while the other eight are empty."""
    m = load_fixture('tank'); X, Y, hyper = m['X'], m['Y'], m['hyper']
    Ny, Nx, Nt = Y.shape[1], X.shape[1], 3
    eng = fit(X, Y, hyper)
    lib = L.load()
    rng = np.random.default_rng(8)
    Z = X[:Nt] + 0.1 * rng.standard_normal((Nt, Nx))
    Sg = np.stack([1e-3 * np.eye(Nx) + 1e-4 * (lambda A: A @ A.T)(rng.standard_normal((Nx, Nx))) for _ in range(Nt)])
    dp = C.POINTER(C.c_double)

    def call(fn, ins, outs):
        arg = (dp * len(ins))(*[a.ctypes.data_as(dp) for a in ins])
        res = (dp * len(outs))(*[a.ctypes.data_as(dp) for a in outs])
        return fn(arg, res, None, None, 0)

    z_cm = np.ascontiguousarray(Z)
    s_cm = np.ascontiguousarray(np.transpose(Sg, (0, 2, 1)))

    def run():
        mean_cm = np.empty((Nt, Ny)); cov_cm = np.empty((Nt, Ny, Ny))
        assert call(lib.gp_b200, [z_cm, s_cm], [mean_cm, cov_cm]) == 0
        pats = [ccs(lib.jac_gp_b200_sparsity_out(k)) for k in range(4)]
        outs = [np.zeros(p[2][-1]) for p in pats]
        assert call(lib.jac_gp_b200, [z_cm, s_cm, mean_cm, cov_cm], outs) == 0
        return mean_cm, cov_cm, pats, outs

    assert lib.gp_b200_bind(eng.h, L.METHOD_EM, Nt) == 0
    ref = run()
    assert lib.gp_b200_bind_em_hess(eng.h, Nt) == 0
    got = run()
    assert np.array_equal(ref[0], got[0]) and np.array_equal(ref[1], got[1])
    assert ref[2] == got[2]
    for a, b in zip(ref[3], got[3]):
        assert np.array_equal(a, b)
    mean_cm, cov_cm, pats, outs = got
    jj = [ccs(lib.jac_jac_gp_b200_sparsity_out(k)) for k in range(16)]
    res = [np.zeros(max(1, p[2][-1])) for p in jj]
    assert call(lib.jac_jac_gp_b200, [z_cm, s_cm, mean_cm, cov_cm] + outs, res) == 0
    o = eng.predict_em_hess(Z, Sg)
    # nonzeros in pattern order: node t, column (f, or f + Nx g for Sigma[f][g]), rows ascending
    exp = {0: np.transpose(o['d2mean_dz2'], (0, 3, 2, 1))}             # [t, a, d, e] -> t, e, d, a
    exp[1] = np.transpose(o['d2mean_dSigma_dz'], (0, 3, 2, 4, 1))     # [t, a, f, g, d] -> t, g, f, d, a
    exp[4] = np.transpose(o['d2mean_dSigma_dz'], (0, 4, 3, 2, 1))     # [t, a, d, e, f] -> t, f, e, d, a
    exp[5] = np.transpose(o['d2mean_dSigma2'], (0, 5, 4, 3, 2, 1))    # [t, a, d, e, f, g] -> t, g, f, e, d, a
    exp[8] = np.transpose(o['d2cov_dz2'], (0, 4, 3, 2, 1))            # [t, a, b, e, f] -> t, f, e, b, a
    exp[9] = np.transpose(o['d2cov_dSigma_dz'], (0, 4, 3, 5, 2, 1))   # [t, a, b, f, g, e] -> t, g, f, e, b, a
    exp[12] = np.transpose(o['d2cov_dSigma_dz'], (0, 5, 4, 3, 2, 1))  # [t, a, b, d, e, f] -> t, f, e, d, b, a
    exp[13] = np.transpose(o['d2cov_dSigma2'], (0, 6, 5, 4, 3, 2, 1))  # [t, a, b, d, e, f, g] -> t, g, f, e, d, b, a
    for k in range(16):
        if k in exp:
            assert jj[k][2][-1] == exp[k].size, k
            assert np.array_equal(res[k], exp[k].reshape(-1)), k
        else:
            assert jj[k][2][-1] == 0, k
    lib.gp_b200_unbind()
    eng.close()


def test_gp_predict_batch_em_hess_vs_differences():
    """GP.predict_batch_em_hess (normalize=True) against fourth-order differences of GP.predict_batch_grad('EM') in the
    caller's units, and its first-order entries bit-identical to predict_batch_grad's."""
    gp, m = gp_from_fixture('tank')
    assert m['normalize']
    d = load_golden('derived', 'tank')
    xs = np.tile(d['x0'], (2, 1)) * (1 + 0.02 * np.arange(2)[:, None]); us = np.tile(d['u0'], (2, 1))
    Sigma = d['Sigma']
    h = gp.predict_batch_em_hess(xs, us, Sigma)
    g = gp.predict_batch_grad(xs, us, Sigma, method='EM')
    for k in g:
        assert np.array_equal(h[k], g[k]), k
    zs = np.hstack([xs, us])
    Ny, Nx = xs.shape[1], zs.shape[1]
    for f in range(Nx):
        st = 1e-2 * max(1.0, abs(zs[0, f]))
        e = np.zeros(Nx); e[f] = 1.0
        dd = d4(lambda s: gp.predict_batch_grad((zs + s * e)[:, :Ny], (zs + s * e)[:, Ny:], Sigma, method='EM'), st)
        assert relinf(h['d2mean_dz2'][..., f], dd['dmean_dz']) < 1e-4
        assert relinf(h['d2mean_dSigma_dz'][..., f], dd['dmean_dSigma']) < 1e-4
        assert relinf(h['d2cov_dz2'][..., f], dd['dcov_dz']) < 1e-3
        assert relinf(h['d2cov_dSigma_dz'][..., f], dd['dcov_dSigma']) < 1e-3
    E = np.zeros((Nx, Nx)); E[0, 1] = E[1, 0] = 1.0
    dd = d4(lambda s: gp.predict_batch_grad(xs, us, Sigma + s * E, method='EM'), 3e-4)
    assert relinf(2 * h['d2mean_dSigma2'][..., 0, 1], dd['dmean_dSigma']) < 1e-4
    assert relinf(2 * h['d2cov_dSigma2'][..., 0, 1], dd['dcov_dSigma']) < 1e-3
    gp.close()
