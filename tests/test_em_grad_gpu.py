"""gpmpc_predict_em_grad and GP.predict_batch_grad('EM') on the GPU: 'EM' first derivatives and the forward mean and cov
against the closed-form oracle fed with the engine's own alpha and factor, against fourth-order differences of the engine's
own EM prediction, bit-identity of the forward outputs with gpmpc_predict(EM), exact symmetry, reproducibility, the K^-1
cache after append and the argument checks."""
import ctypes as C

import numpy as np
import pytest
from scipy.linalg import cho_solve

from gp_mpc_b200 import _lib as L
from oracle import em_grad_oracle as emo
from oracle import gp_oracle as orc
from tests._em_cases import check_case, em_errors, em_terms, engine_alpha_chol, grad_case, tma_on_device
from tests._engines import ccs, fit, gp_from_fixture, require
from tests._util import load_fixture, load_golden, relinf

pytestmark = pytest.mark.gpu

DERIV = ('dmean_dz', 'dmean_dSigma', 'dcov_dz', 'dcov_dSigma')


def forward_errors(o, ref, X, hyper, alpha, chol, Z, Sigma):
    """Largest errors of the engine's EM mean and cov against the closed form's over the points, normalised by the sums of
    |terms| (test_em_shapes_gpu.em_terms) with K^-1 from the engine's factor."""
    N = X.shape[0]
    kinv = np.stack([cho_solve((c, True), np.eye(N), check_finite=False) for c in chol])
    kinv = 0.5 * (kinv + np.swapaxes(kinv, 1, 2))
    Sg = emo._sigmas(Sigma, Z.shape[0], X.shape[1])
    e = dict(mean=0.0, cov=0.0)
    for h in range(Z.shape[0]):
        eh = em_errors(o['mean'][h], o['cov'][h], (ref['mean'][h], ref['cov'][h]), em_terms(X, hyper, alpha, kinv, Z[h], Sg[h]))
        e = {k: max(e[k], eh[k]) for k in e}
    return e


NEW_SHAPES = [n + s for n in ('nx1', 'nx32', 'tma', 'ny9', 'reserved') for s in ('_s0.1', '_s1')]
# (dmean, dcov) bars against the closed form: the fixtures and the sn = 1e-2 synthetic cases carry cond(K) eps; the
# well-conditioned cases (sn = 0.3) were measured on an H100 SXM at 700 W: syn12 dmean 5.7e-15, dcov 2.8e-13; the
# shapes of test_em_shapes_gpu dmean <= 1.5e-14 (nx32), dcov <= 1.6e-13 (ny9 at Sigma = Lambda)
GRAD_TOL = dict({'syn12': (1e-13, 3e-12)}, **{c: (1e-13, 3e-12) for c in NEW_SHAPES})
# (mean, cov) bar against the closed form's, normalised by the sums of |terms|; measured on an H100 SXM at 700 W over every
# case: mean <= 1.7e-16 (nx32), cov <= 4.5e-18
FWD_TOL = (1e-15, 1e-15)


def em_grad_errors(case):
    """The engine's predict_em_grad on a case against em_grad_closed on the engine's own alpha and factor: relative errors
    of the four derivatives and normalised errors of mean and cov, after the bit-level checks."""
    X, Y, hyper, Z, Sigma, cap = grad_case(case)
    Ny = Y.shape[1]
    eng = fit(X, Y, hyper, capacity=cap)
    o = eng.predict_em_grad(Z, Sigma)
    mean, var, cov, _ = eng.predict(Z, Sigma, L.METHOD_EM, want_jac=False)
    assert np.array_equal(o['mean'], mean) and np.array_equal(o['var'], var) and np.array_equal(o['cov'], cov)
    for k in DERIV:
        assert np.all(np.isfinite(o[k])), k
    assert np.array_equal(o['dmean_dSigma'], np.swapaxes(o['dmean_dSigma'], 2, 3))
    assert np.array_equal(o['dcov_dSigma'], np.swapaxes(o['dcov_dSigma'], 3, 4))
    assert np.array_equal(o['dcov_dSigma'], np.swapaxes(o['dcov_dSigma'], 1, 2))
    assert np.array_equal(o['dcov_dz'], np.swapaxes(o['dcov_dz'], 1, 2))
    o2 = eng.predict_em_grad(Z, Sigma)
    for k in o:
        assert np.array_equal(o[k], o2[k]), k
    alpha, chol = engine_alpha_chol(eng, Ny)
    eng.close()
    ref = emo.em_grad_closed(X, hyper, alpha, chol, Z, Sigma)
    errs = {k: relinf(o[k], ref[k]) for k in DERIV}
    errs.update(forward_errors(o, ref, X, hyper, alpha, chol, Z, Sigma))
    return errs


@pytest.mark.parametrize('case', ['tank', 'tank_pp', 'tank_large', 'syn1000', 'syn300', 'syn12'] + NEW_SHAPES)
def test_em_grad_vs_closed_oracle(case):
    """syn1000: Nx = 8, N ~ 1000 (16 tiles); syn300: Nx = 17, the 32 bucket; syn12: Nx = 12, the 16 bucket of em_prep,
    em_owner_rec and em_pair_rec; tank_pp: one Sigma per point.  The shapes of test_em_shapes_gpu at Sigma = 0.1 Lambda
    and Lambda: nx1, nx32 (em_pair_rec_kernel<32, 2>'s opt-in shared memory at its largest), tma (em_owner_rec,
    em_backbone_rows and trmv_lower_T on the 3072 pad), ny9 (nine outputs' records) and reserved (an identity tail of
    L^-1)."""
    if case.startswith('tma'):
        require(tma_on_device(), 'the TMA feed')
    errs = em_grad_errors(case)
    tm, tc = GRAD_TOL.get(case, (1e-6, 1e-5))
    assert errs['dmean_dz'] < tm and errs['dmean_dSigma'] < tm, errs
    assert errs['dcov_dz'] < tc and errs['dcov_dSigma'] < tc, errs
    fm, fc = FWD_TOL
    assert errs['mean'] < fm and errs['cov'] < fc, errs


def test_em_forward_nxp16_vs_exact_moment():
    """The forward 'EM' moments at Nx = 12 (em_prep / em_owner_rec<16, 2>) on the well-conditioned syn12 model against the
    fp64 restatement gp_exact_moment with postfit's K^-1.  Measured on an H100 SXM at 700 W: mean 1.2e-13, cov
    3.9e-11 (the restatement's own cancellation between beta beta^T and K^-1).  Then the nx12 case of test_em_shapes_gpu
    (N = 600, Ny = 3) against the long-double formula on the engine's alpha and factor at Sigma = 1e-5 Lambda, 0.1 Lambda
    and Lambda, under that file's bars (measured: mean 2.7e-17, cov 1.2e-18 of the sums of |terms|)."""
    X, Y, hyper, Z, Sigma, _ = grad_case('syn12')
    eng = fit(X, Y, hyper)
    mean, _, cov, _ = eng.predict(Z, Sigma, L.METHOD_EM, want_jac=False)
    eng.close()
    post = orc.postfit(X, Y, hyper, lapack_general_solve=False)
    for h in range(Z.shape[0]):
        mo, co = orc.gp_exact_moment(post['invK'], X, Y, hyper, Z[h], Sigma)
        assert relinf(mean[h], mo) < 1e-12 and relinf(cov[h], co) < 1e-9, h
    check_case('nx12')


@pytest.mark.parametrize('case,tol', [('tank', 1e-5), ('car', 1e-3)])
def test_em_grad_vs_differences_of_the_engine(case, tol):
    """Fourth-order differences of the engine's own gpmpc_predict(EM).  The car fixture (cond K ~ 1e10) gets 1e-3:
    its EM covariance carries the alpha floor of DESIGN 4.8, which the differences amplify."""
    m = load_fixture(case); X, Y, hyper = m['X'], m['Y'], m['hyper']
    Nx, Ny = X.shape[1], Y.shape[1]
    rng = np.random.default_rng(11)
    Z = X[:2] + 0.05 * rng.standard_normal((2, Nx))
    A = rng.standard_normal((Nx, Nx)); S = 1e-3 * np.eye(Nx) + 1e-4 * A @ A.T
    eng = fit(X, Y, hyper)
    o = eng.predict_em_grad(Z, S)
    for k in DERIV:
        assert np.all(np.isfinite(o[k])), k

    def f(Zp, Sp):
        mean, _, cov, _ = eng.predict(Zp, Sp, L.METHOD_EM, want_jac=False)
        return mean, cov

    def d4(fun, h):
        r = {k: fun(k * h) for k in (-2, -1, 1, 2)}
        return [(r[-2][i] - 8 * r[-1][i] + 8 * r[1][i] - r[2][i]) / (12 * h) for i in range(2)]

    dmz = np.zeros_like(o['dmean_dz']); dcz = np.zeros_like(o['dcov_dz'])
    for d in range(Nx):
        e = np.zeros(Nx); e[d] = 1.0
        dmz[:, :, d], dcz[:, :, :, d] = d4(lambda s: f(Z + s * e, S), 3e-2)
    dmS = np.zeros_like(o['dmean_dSigma']); dcS = np.zeros_like(o['dcov_dSigma'])
    for d in range(Nx):
        for e in range(d + 1):
            E = np.zeros((Nx, Nx)); E[d, e] = E[e, d] = 1.0
            dm, dc = d4(lambda s: f(Z, S + s * E), 3e-4)
            dmS[:, :, d, e] = dmS[:, :, e, d] = dm
            dcS[:, :, :, d, e] = dcS[:, :, :, e, d] = dc
    assert relinf(o['dmean_dz'], dmz) < tol and relinf(o['dcov_dz'], dcz) < tol
    assert relinf(emo.sym_pair(o['dmean_dSigma']), dmS) < tol
    assert relinf(emo.sym_pair(o['dcov_dSigma']), dcS) < tol
    eng.close()


def test_em_grad_argument_checks():
    lib = L.load()
    m = load_fixture('tank'); X, Y, hyper = m['X'], m['Y'], m['hyper']
    Ny, Nx = Y.shape[1], X.shape[1]
    eng = fit(X, Y, hyper)
    Z = np.ascontiguousarray(X[:3] + 0.01)
    S = 1e-3 * np.eye(Nx)
    dp = C.POINTER(C.c_double)
    rc = lib.gpmpc_predict_em_grad(eng.h, 3, Z.ctypes.data_as(dp), None, 0, *([None] * 7))
    assert rc == L.ERR_ARG
    with pytest.raises(L.GpmpcError) as e:
        eng.predict_grad(Z, S, L.METHOD_EM)
    assert e.value.code == L.ERR_ARG
    full = eng.predict_em_grad(Z, S)
    names = ('mean', 'var', 'cov') + DERIV
    for k, name in enumerate(names):            # every output is optional: one at a time
        out = np.empty_like(full[name])
        ptrs = [None] * 7
        ptrs[k] = out.ctypes.data_as(dp)
        assert lib.gpmpc_predict_em_grad(eng.h, 3, Z.ctypes.data_as(dp), S.ctypes.data_as(dp), 0, *ptrs) == L.OK
        assert np.array_equal(out, full[name]), name
    eng.close()
    part = fit(X, Y, hyper, out_begin=0, out_count=Ny - 1)
    with pytest.raises(L.GpmpcError) as e:
        part.predict_em_grad(Z, S)
    assert e.value.code == L.ERR_STATE
    part.close()


def test_em_grad_after_append_matches_a_refit():
    """The cached K^-1 must follow gpmpc_append."""
    m = load_fixture('tank'); X, Y, hyper = m['X'], m['Y'], m['hyper']
    Nx = X.shape[1]
    rng = np.random.default_rng(3)
    Z = X[:3] + 0.05 * rng.standard_normal((3, Nx))
    S = 1e-3 * np.eye(Nx)
    eng = fit(X[:-2], Y[:-2], hyper)
    eng.predict_em_grad(Z, S)                   # builds the cache for the smaller model
    assert eng.append(X[-2], Y[-2]) and eng.append(X[-1], Y[-1])
    got = eng.predict_em_grad(Z, S)
    eng.close()
    ref_eng = fit(X, Y, hyper)
    ref = ref_eng.predict_em_grad(Z, S)
    ref_eng.close()
    for k in DERIV:
        assert relinf(got[k], ref[k]) < 1e-8, k


def test_gp_predict_batch_grad_em_vs_central_differences():
    gp, m = gp_from_fixture('tank')
    assert m['normalize']
    d = load_golden('derived', 'tank')
    xs = np.tile(d['x0'], (3, 1)) * (1 + 0.02 * np.arange(3)[:, None]); us = np.tile(d['u0'], (3, 1))
    Sigma = d['Sigma']
    g = gp.predict_batch_grad(xs, us, Sigma, method='EM')
    mb, cb = gp.predict_batch(xs, us, Sigma, method='EM')
    assert np.array_equal(g['mean'], mb) and np.array_equal(g['cov'], cb)
    zs = np.hstack([xs, us])
    Nx = zs.shape[1]
    for e in range(Nx):
        h = 1e-2 * max(1.0, abs(zs[0, e]))
        r = {}
        for k in (-2, -1, 1, 2):
            zk = zs.copy(); zk[:, e] += k * h
            r[k] = gp.predict_batch(zk[:, :4], zk[:, 4:], Sigma, method='EM')
        fd = [(r[-2][i] - 8 * r[-1][i] + 8 * r[1][i] - r[2][i]) / (12 * h) for i in range(2)]
        assert relinf(g['dmean_dz'][..., e], fd[0]) < 1e-5
        assert relinf(g['dcov_dz'][..., e], fd[1]) < 1e-4
    E = np.zeros((Nx, Nx)); E[0, 1] = E[1, 0] = 1.0
    hs = 3e-4
    r = {k: gp.predict_batch(xs, us, Sigma + k * hs * E, method='EM') for k in (-2, -1, 1, 2)}
    fd = [(r[-2][i] - 8 * r[-1][i] + 8 * r[1][i] - r[2][i]) / (12 * hs) for i in range(2)]
    assert relinf(g['dmean_dSigma'][..., 0, 1] + g['dmean_dSigma'][..., 1, 0], fd[0]) < 1e-4
    assert relinf(g['dcov_dSigma'][..., 0, 1] + g['dcov_dSigma'][..., 1, 0], fd[1]) < 1e-4
    gp.close()


def test_casadi_external_entry_points_with_em():
    """gp_b200_bind(EM) driven through ctypes the way CasADi drives it: gp_b200 equals gpmpc_predict(EM), the CCS
    nonzeros of jac_gp_b200 equal gpmpc_predict_em_grad (jac_mean_sigma and jac_cov_sigma block-diagonal, column
    d + Nx*e <-> Sigma[d][e]), and jac_jac_gp_b200 reports failure."""
    m = load_fixture('tank'); X, Y, hyper = m['X'], m['Y'], m['hyper']
    Ny, Nx, Nt = Y.shape[1], X.shape[1], 4
    eng = fit(X, Y, hyper)
    lib = L.load()
    rng = np.random.default_rng(8)
    Z = X[:Nt] + 0.1 * rng.standard_normal((Nt, Nx))
    Sg = np.stack([1e-3 * np.eye(Nx) + 1e-4 * (lambda A: A @ A.T)(rng.standard_normal((Nx, Nx))) for _ in range(Nt)])
    assert lib.gp_b200_bind(eng.h, L.METHOD_EM, Nt) == 0
    dp = C.POINTER(C.c_double)

    def call(fn, ins, outs):
        arg = (dp * len(ins))(*[a.ctypes.data_as(dp) for a in ins])
        res = (dp * len(outs))(*[a.ctypes.data_as(dp) for a in outs])
        return fn(arg, res, None, None, 0)

    z_cm = np.ascontiguousarray(Z)                                        # Nx x Nt column-major
    s_cm = np.ascontiguousarray(np.transpose(Sg, (0, 2, 1)))               # Nx x Nx*Nt column-major
    mean_cm = np.empty((Nt, Ny)); cov_cm = np.empty((Nt, Ny, Ny))
    assert call(lib.gp_b200, [z_cm, s_cm], [mean_cm, cov_cm]) == 0
    o = eng.predict_em_grad(Z, Sg)
    assert np.array_equal(mean_cm, o['mean'])
    assert np.array_equal(cov_cm, np.transpose(o['cov'], (0, 2, 1)))
    pats = [ccs(lib.jac_gp_b200_sparsity_out(k)) for k in range(4)]
    assert [(p[0], p[1], p[2][-1]) for p in pats] == [
        (Ny * Nt, Nx * Nt, Ny * Nx * Nt), (Ny * Nt, Nx * Nx * Nt, Ny * Nx * Nx * Nt),
        (Ny * Ny * Nt, Nx * Nt, Ny * Ny * Nx * Nt), (Ny * Ny * Nt, Nx * Nx * Nt, Ny * Ny * Nx * Nx * Nt)]
    outs = [np.zeros(p[2][-1]) for p in pats]
    assert call(lib.jac_gp_b200, [z_cm, s_cm, mean_cm, cov_cm], outs) == 0
    # nonzeros in pattern order: node t, column (d + Nx*e for Sigma), rows ascending (a, or a + Ny*b)
    exp_mz = np.transpose(o['dmean_dz'], (0, 2, 1)).reshape(-1)                        # t, d, a
    exp_ms = np.transpose(o['dmean_dSigma'], (0, 3, 2, 1)).reshape(-1)                 # t, e, d, a
    exp_cz = np.transpose(o['dcov_dz'], (0, 3, 2, 1)).reshape(-1)                      # t, e, b, a
    exp_cs = np.transpose(o['dcov_dSigma'], (0, 4, 3, 2, 1)).reshape(-1)               # t, e, d, b, a
    for got, exp in zip(outs, (exp_mz, exp_ms, exp_cz, exp_cs)):
        assert np.array_equal(got, exp)
    jj = [ccs(lib.jac_jac_gp_b200_sparsity_out(k)) for k in range(16)]
    jins = [z_cm, s_cm, mean_cm, cov_cm] + [np.zeros(max(1, p[2][-1])) for p in pats]
    assert call(lib.jac_jac_gp_b200, jins, [np.zeros(max(1, p[2][-1])) for p in jj]) != 0
    lib.gp_b200_unbind()
    assert not lib.jac_gp_b200_sparsity_out(0)
    eng.close()
