"""Parity of the CUDA path (through the C ABI) against the CPU oracle and the committed
golden fixtures.  Tolerances: mean / covariance 1e-6 batch-inf-norm relative (BASELINE.json
north_star); chol 2e-9; NLL 1e-9; index work exact."""
import json
import os

import numpy as np
import pytest

from gp_mpc_b200 import _lib as L
from oracle import gp_oracle as orc
from tests._engines import fit, gp_from_fixture
from tests._util import load_fixture, load_golden, relinf

pytestmark = pytest.mark.gpu

TOL = 1e-6


def _engine(N, Nx, Ny, **kw):
    import gp_mpc_b200
    return gp_mpc_b200.Engine(N, Nx, Ny, device=0, **kw)


# ------------------------------------------------------------------ a1/a2 K build
@pytest.mark.parametrize('case', ['tank', 'car', 'syn300', 'syn1000'])
def test_kbuild_matches_oracle(case):
    if case in ('tank', 'car'):
        m = load_fixture(case); X, Y, hyper = m['X'], m['Y'], m['hyper']
    else:
        n = int(case[3:]); p = orc.synthetic_problem(n, 7, 2, config_id=n); X, Y, hyper = p['X'], p['Y'], p['hyper']
    N, Nx = X.shape
    eng = _engine(N, Nx, Y.shape[1]); eng.set_data(X, Y); eng.set_hyper(hyper)
    for a in range(Y.shape[1]):
        K = eng.build_K(a)
        Ko = orc.covSEard(X, X, hyper[a, :Nx], hyper[a, Nx] ** 2) + hyper[a, Nx + 1] ** 2 * np.eye(N)
        assert relinf(K, Ko) < 1e-13
        assert np.array_equal(K, K.T)                     # exactly symmetric (q10)
        assert relinf(K, orc.assemble_K(X, hyper[a])) < 1e-11   # the reference's expansion form
    eng.close()


# ------------------------------------------------------------------ a3-a5 factorisation
@pytest.mark.parametrize('name', ['tank', 'car'])
def test_factorize_reproduces_stored_model(name):
    m = load_fixture(name)
    eng, info = fit(m['X'], m['Y'], m['hyper'], with_info=True)
    assert not info.any()
    N = m['X'].shape[0]
    for a in range(m['hyper'].shape[0]):
        chol = eng.get(L.GET_CHOL, a)
        assert np.all(np.triu(chol, 1) == 0.0)            # GET_CHOL's stored-model layout (extract_kernel writes these zeros)
        assert relinf(chol, m['chol'][a]) < (1e-10 if name == 'tank' else 2e-9)
        linv = eng.get(L.GET_LINV, a)
        assert relinf(linv @ chol, np.eye(N)) < 1e-9
        alpha = eng.get(L.GET_ALPHA, a)
        # alpha itself is cond(K)*eps limited (1e-9 tank / 1e-5 car, as for the oracle's own rerun)
        assert relinf(alpha, m['alpha'][a]) < (1e-7 if name == 'tank' else 1e-4)
        invK = eng.get(L.GET_INVK, a)
        assert np.array_equal(invK, invK.T)
        assert relinf(invK, m['invK'][a]) < (1e-7 if name == 'tank' else 1e-4)
        K = eng.get(L.GET_K, a)
        assert relinf(chol @ chol.T, K) < 1e-13
        logdet = eng.get(L.GET_LOGDET, a)[0]
        assert logdet == pytest.approx(2 * np.sum(np.log(np.diag(m['chol'][a]))), rel=1e-8)
    eng.close()


@pytest.mark.parametrize('N', [129, 384, 1000])
def test_factorize_synthetic_vs_oracle(N):
    p = orc.synthetic_problem(N, 8, 3, config_id=N)
    post = orc.postfit(p['X'], p['Y'], p['hyper'], lapack_general_solve=False)
    eng, info = fit(p['X'], p['Y'], p['hyper'], with_info=True)
    for a in range(3):
        assert relinf(eng.get(L.GET_CHOL, a), post['chol'][a]) < 1e-10
        assert relinf(eng.get(L.GET_ALPHA, a), post['alpha'][a]) < 1e-7
    eng.close()


def test_jitter_retry_and_not_pd():
    """optimize.py:483-488: one 1e-8 jitter retry, then LinAlgError."""
    rng = np.random.default_rng(0)
    X = rng.standard_normal((40, 3)); X[20:] = X[:20]      # exact duplicates -> singular Kf
    Y = rng.standard_normal((40, 1))
    hyper = np.array([[1.0, 1.0, 1.0, 1.0, 1e-10]])        # sn2 = 1e-20: K numerically singular
    eng = _engine(40, 3, 1); eng.set_data(X, Y); eng.set_hyper(hyper)
    info = eng.factorize(1e-8)
    assert info[0] == 1                                     # succeeded after jitter
    Ko = orc.covSEard(X, X, hyper[0, :3], 1.0) + (1e-20 + 1e-8) * np.eye(40)
    assert relinf(eng.get(L.GET_CHOL, 0), np.linalg.cholesky(Ko)) < 1e-6
    with pytest.raises(np.linalg.LinAlgError):
        eng.factorize(0.0)                                  # retry with zero jitter must fail again
    eng.close()


# ------------------------------------------------------------------ a8-a11 prediction
@pytest.mark.parametrize('name', ['tank', 'car'])
def test_predict_fixture_batch(name):
    m = load_fixture(name); d = load_golden('derived', name)
    eng, _ = fit(m['X'], m['Y'], m['hyper'], with_info=True)
    mean, var, cov, jac = eng.predict(d['Zs'], d['Sigma'], L.METHOD_TA)
    assert relinf(mean, d['mean_b']) < TOL
    assert relinf(var, d['var_b']) < TOL
    assert relinf(jac, d['J_b']) < TOL
    assert relinf(cov, d['cov_b']) < TOL
    mean2, var2, cov2, _ = eng.predict(d['Zs'], None, L.METHOD_ME, want_jac=False)
    assert np.array_equal(mean2, mean) and np.array_equal(var2, var)
    assert relinf(cov2, orc.me_cov(d['var_b'])) < TOL
    # refinement step must agree as well
    eng.set_option('refine', 1)
    mean3, var3, _, _ = eng.predict(d['Zs'], d['Sigma'], L.METHOD_TA)
    assert relinf(var3, d['var_b']) < TOL and relinf(mean3, d['mean_b']) < TOL
    eng.close()


@pytest.mark.parametrize('N,Nx,Ny,H', [(1000, 8, 6, 30), (300, 5, 2, 70), (130, 10, 3, 1), (2048, 17, 1, 50)])
def test_predict_synthetic_vs_oracle(N, Nx, Ny, H):
    p = orc.synthetic_problem(N, Nx, Ny, config_id=N + H, H=H)
    post = orc.postfit(p['X'], p['Y'], p['hyper'], lapack_general_solve=False)
    mo, vo = orc.gp_mean_var(p['X'], p['hyper'], post['alpha'], post['chol'], p['Z'])
    Jo = orc.gp_mean_jac(p['X'], p['hyper'], post['alpha'], p['Z'])
    co = orc.ta_cov(vo, Jo, p['Sigma'])
    eng, _ = fit(p['X'], p['Y'], p['hyper'], with_info=True)
    mean, var, cov, jac = eng.predict(p['Z'], p['Sigma'], L.METHOD_TA)
    assert relinf(mean, mo) < TOL and relinf(var, vo) < TOL and relinf(jac, Jo) < TOL and relinf(cov, co) < TOL
    assert (var > 0).all()
    # per-point input covariances (one Sigma per shooting node, mpc_class.py:265-275)
    Sg = np.stack([p['Sigma'] * (1 + 0.1 * h) for h in range(H)])
    _, _, cov_pp, _ = eng.predict(p['Z'], Sg, L.METHOD_TA)
    assert relinf(cov_pp, orc.ta_cov(vo, Jo, Sg)) < TOL
    # the stream-K partition (persistent grid size) must not change the result beyond rounding,
    # and a fixed partition is bit-reproducible (parked partials are added in contributor order)
    mean_b, var_b, cov_b, jac_b = eng.predict(p['Z'], p['Sigma'], L.METHOD_TA)
    assert np.array_equal(var_b, var) and np.array_equal(mean_b, mean) and np.array_equal(cov_b, cov)
    for ctas in (1, 7, 1000):
        eng.set_option('predict_ctas', ctas)
        mean_s, var_s, cov_s, jac_s = eng.predict(p['Z'], p['Sigma'], L.METHOD_TA)
        assert relinf(var_s, var) < 1e-9 and np.array_equal(mean_s, mean) and np.array_equal(jac_s, jac)
        assert relinf(cov_s, cov) < 1e-9
    eng.close()


def test_profiling_entry_points_leave_the_engine_intact():
    """gpmpc_profile (ks / product / product + tail selectors), gpmpc_profile_balance and gpmpc_profile_tail run the
    production kernels on the engine's own buffers: times are positive and the next predict call is bit-identical."""
    p = orc.synthetic_problem(700, 6, 3, config_id=77, H=40)
    eng, _ = fit(p['X'], p['Y'], p['hyper'], with_info=True)
    ref = eng.predict(p['Z'], p['Sigma'], L.METHOD_TA)
    for what in (L.PROF_KS, L.PROF_TRIGEMM, L.PROF_PREDICT_TAIL):
        ms = eng.profile(what, n=40, reps=3)
        assert np.isfinite(ms) and ms > 0.0
    bal = eng.profile_balance(40)
    assert 0.0 <= bal['min_us'] <= bal['max_us'] <= bal['span_us'] and bal['span_us'] > 0.0
    tail = eng.profile_tail(40)
    assert tail['output_done'] <= tail['records'] <= tail['step_counter'] <= tail['staged'] <= tail['jsigma'] <= tail['written']
    assert tail['written'] < 1e3 and tail['kernel_span'] > 0.0
    again = eng.predict(p['Z'], p['Sigma'], L.METHOD_TA)
    for a, b in zip(ref, again):
        assert np.array_equal(a, b)
    eng.close()


def test_full_size_properties_n4096():
    """C3-size (N=4096) checks that do not need the O(N^3) CPU oracle: L Linv = I on probe
    columns, the interpolation identity Kf alpha = y - sn2 alpha at training points, var > 0."""
    N, Nx, Ny = 4096, 8, 2
    p = orc.synthetic_problem(N, Nx, Ny, config_id=3, H=30)
    eng, _ = fit(p['X'], p['Y'], p['hyper'], with_info=True)
    idx = np.arange(0, N, 137)[:30]
    mean, var, _, _ = eng.predict(p['X'][idx], None, L.METHOD_ME, want_jac=False)
    for a in range(Ny):
        alpha = eng.get(L.GET_ALPHA, a)
        sn2 = p['hyper'][a, Nx + 1] ** 2
        assert relinf(mean[:, a], p['Y'][idx, a] - sn2 * alpha[idx]) < 1e-7
    assert (var > 0).all() and (var < 1.0).all()
    chol = eng.get(L.GET_CHOL, 0); linv = eng.get(L.GET_LINV, 0)
    probe = np.zeros((N, 4)); probe[[0, 777, 2048, 4095], range(4)] = 1.0
    assert relinf(chol @ (linv @ probe), probe) < 1e-9
    K = orc.covSEard(p['X'][:512], p['X'][:512], p['hyper'][0, :Nx], 1.0) + 1e-4 * np.eye(512)
    assert relinf((chol @ chol.T)[:512, :512], K) < 1e-12
    eng.close()


def test_full_size_properties_n16384():
    """BASELINE.json's full size (C5: N=16384, Nx=10, H=50), one output: oracle-free
    properties.  (1) interpolation identity  Kf alpha = y - sn2 alpha  read off the predicted
    mean at training points; (2) var in (0, sf2); (3) L L^-1 = I on probe columns;
    (4) L L^T reproduces K on a 512 block; (5) TA covariance is symmetric PSD-plus-diagonal and
    reduces to ME when Sigma = 0; (6) refinement and split-K variants agree."""
    N, Nx, H = 16384, 10, 50
    p = orc.synthetic_problem(N, Nx, 1, config_id=5, H=H)
    eng, info = fit(p['X'], p['Y'], p['hyper'], with_info=True)
    assert not info.any()
    idx = np.arange(0, N, 331)[:H]
    mean, var, _, _ = eng.predict(p['X'][idx], None, L.METHOD_ME, want_jac=False)
    alpha = eng.get(L.GET_ALPHA, 0)
    sn2 = p['hyper'][0, Nx + 1] ** 2
    assert relinf(mean[:, 0], p['Y'][idx, 0] - sn2 * alpha[idx]) < 1e-6
    assert (var > 0).all() and (var < 1.0).all()
    chol = eng.get(L.GET_CHOL, 0)
    assert np.all(chol[0, 1:] == 0.0) and np.all(np.diag(chol) > 0)
    Kb = orc.covSEard(p['X'][:512], p['X'][:512], p['hyper'][0, :Nx], 1.0) + sn2 * np.eye(512)
    assert relinf(chol[:512, :512] @ chol[:512, :512].T, Kb) < 1e-12
    linv = eng.get(L.GET_LINV, 0)
    probe = np.zeros((N, 3)); probe[[5, 8191, 16383], range(3)] = 1.0
    assert relinf(chol @ (linv @ probe), probe) < 1e-8
    del chol, linv
    mean_t, var_t, cov_t, jac_t = eng.predict(p['Z'], p['Sigma'], L.METHOD_TA)
    _, _, cov_0, _ = eng.predict(p['Z'], np.zeros((Nx, Nx)), L.METHOD_TA)
    assert np.array_equal(cov_0[:, 0, 0], var_t[:, 0])
    assert relinf(cov_t[:, 0, 0], var_t[:, 0] + np.einsum('hd,de,he->h', jac_t[:, 0], p['Sigma'], jac_t[:, 0])) < 1e-12
    eng.set_option('refine', 1)
    _, var_r, _, _ = eng.predict(p['Z'], p['Sigma'], L.METHOD_TA)
    assert relinf(var_r, var_t) < 1e-6
    eng.set_option('refine', 0); eng.set_option('predict_ctas', 100)
    _, var_k, _, _ = eng.predict(p['Z'], p['Sigma'], L.METHOD_TA)
    assert relinf(var_k, var_t) < 1e-8
    eng.close()


# ------------------------------------------------------------------ BASELINE sizes against an independent CPU factor
def test_c3_full_size_vs_oracle():
    """BASELINE config C3 (N=4096, Nx=8, Ny=6, H=30, TA) at its stated size: every output against
    an independent CPU Cholesky (np.linalg.cholesky + triangular solves, oracle factor_large /
    predict_large): chol <= 1e-9, mean / var / J / cov <= 1e-6 (batch-inf-norm relative)."""
    N, Nx, Ny, H = 4096, 8, 6, 30
    p = orc.synthetic_problem(N, Nx, Ny, config_id=3, H=H)
    eng, info = fit(p['X'], p['Y'], p['hyper'], with_info=True)
    assert not info.any()
    mean, var, cov, jac = eng.predict(p['Z'], p['Sigma'], L.METHOD_TA)
    mo = np.zeros((H, Ny)); vo = np.zeros((H, Ny)); Jo = np.zeros((H, Ny, Nx))
    for a in range(Ny):
        f = orc.factor_large(p['X'], p['Y'][:, a], p['hyper'][a])
        assert not f['jitter']
        assert relinf(eng.get(L.GET_CHOL, a), f['chol']) < 1e-9
        assert relinf(eng.get(L.GET_ALPHA, a), f['alpha']) < 1e-6
        assert eng.get(L.GET_LOGDET, a)[0] == pytest.approx(2 * np.sum(np.log(np.diag(f['chol']))), rel=1e-10)
        mo[:, a], vo[:, a], Jo[:, a] = orc.predict_large(p['X'], p['hyper'][a], f['alpha'], f['chol'], p['Z'])
    co = orc.ta_cov(vo, Jo, p['Sigma'])
    assert relinf(mean, mo) < TOL and relinf(var, vo) < TOL and relinf(jac, Jo) < TOL and relinf(cov, co) < TOL
    # cancellation-aware view (SURVEY 8d): |dvar| / sf2
    assert np.abs(var - vo).max() < 1e-9
    eng.close()


def test_c4_nlml_and_gradient_at_n8192():
    """BASELINE config C4 (N=8192, Nx=8, one output): NLL <= 1e-9 relative vs the CPU restatement
    of calc_NLL_numpy (optimize.py:322-356) and the analytic gradient vs central differences of
    that NLL on three components (one length scale, sf, sn) <= 1e-5."""
    N, Nx = 8192, 8
    p = orc.synthetic_problem(N, Nx, 1, config_id=4)
    eng = _engine(N, Nx, 1); eng.set_data(p['X'], p['Y'])
    th = p['hyper'][0].copy(); th[:Nx] *= 0.8; th[Nx] = 0.9; th[Nx + 1] = 8e-3
    nll, g = eng.nlml(0, th, grad=True)
    y = p['Y'][:, 0]
    ref = orc.factor_large(p['X'], y, th)['nll']
    assert nll == pytest.approx(ref, rel=1e-9)
    for j in (2, Nx, Nx + 1):
        h = 1e-5 * max(1.0, abs(th[j])) if j <= Nx else 1e-5 * th[j]
        tp = th.copy(); tp[j] += h
        tm = th.copy(); tm[j] -= h
        fd = (orc.factor_large(p['X'], y, tp)['nll'] - orc.factor_large(p['X'], y, tm)['nll']) / (2 * h)
        assert abs(g[j] - fd) <= 1e-5 * max(abs(fd), np.abs(g).max() * 1e-2), (j, g[j], fd)
    # the GPU's own NLL differences agree with its gradient too (same stencil, GPU evaluations)
    j = 0
    h = 1e-5 * th[j]
    tp = th.copy(); tp[j] += h
    tm = th.copy(); tm[j] -= h
    fd_gpu = (eng.nlml(0, tp, grad=False) - eng.nlml(0, tm, grad=False)) / (2 * h)
    assert abs(g[j] - fd_gpu) <= 1e-5 * max(abs(fd_gpu), np.abs(g).max() * 1e-2)
    eng.close()


def test_c5_full_size_vs_independent_cholesky():
    """BASELINE config C5's per-GPU problem (N=16384, Nx=10, H=50, one output, TA) against an
    INDEPENDENT CPU factor (np.linalg.cholesky of the reference's expansion-form K + triangular
    solves): chol <= 1e-9, mean / var / J / cov <= 1e-6."""
    N, Nx, H = 16384, 10, 50
    p = orc.synthetic_problem(N, Nx, 1, config_id=5, H=H)
    eng, info = fit(p['X'], p['Y'], p['hyper'], with_info=True)
    assert not info.any()
    mean, var, cov, jac = eng.predict(p['Z'], p['Sigma'], L.METHOD_TA)
    f = orc.factor_large(p['X'], p['Y'][:, 0], p['hyper'][0])
    assert not f['jitter']
    mo, vo, Jo = orc.predict_large(p['X'], p['hyper'][0], f['alpha'], f['chol'], p['Z'])
    chol = eng.get(L.GET_CHOL, 0)
    assert relinf(chol, f['chol']) < 1e-9
    del chol
    assert relinf(eng.get(L.GET_ALPHA, 0), f['alpha']) < 1e-5          # alpha is cond(K)*eps limited
    assert eng.get(L.GET_LOGDET, 0)[0] == pytest.approx(2 * np.sum(np.log(np.diag(f['chol']))), rel=1e-10)
    co = orc.ta_cov(vo[:, None], Jo[:, None, :], p['Sigma'])
    assert relinf(mean[:, 0], mo) < TOL and relinf(var[:, 0], vo) < TOL
    assert relinf(jac[:, 0], Jo) < TOL and relinf(cov, co) < TOL
    assert np.abs(var[:, 0] - vo).max() < 1e-9
    eng.close()


# ------------------------------------------------------------------ derivatives for the CasADi adapter (8f row 1)
@pytest.mark.parametrize('case', ['tank', 'car', 'syn700', 'syn1500'])
def test_predict_grad_vs_central_differences(case):
    """gpmpc_predict_grad: d var / d z, d cov / d z (ME and TA) and the mean Hessian against central
    differences of the oracle prediction (<= 1e-5, the FD truncation/rounding level); the values
    themselves must equal gpmpc_predict's bit for bit."""
    if case in ('tank', 'car'):
        m = load_fixture(case); X, Y, hyper = m['X'], m['Y'], m['hyper']
        rng = np.random.default_rng(5)
        Z = X[rng.choice(X.shape[0], 6, replace=False)] + 0.05 * rng.standard_normal((6, X.shape[1]))
        A = rng.standard_normal((X.shape[1],) * 2); Sigma = 1e-3 * np.eye(X.shape[1]) + 1e-4 * A @ A.T
    else:
        n = int(case[3:]); p = orc.synthetic_problem(n, 7 if n == 700 else 17, 3, config_id=n, H=9 if n == 700 else 66)
        X, Y, hyper, Z, Sigma = p['X'], p['Y'], p['hyper'], p['Z'], p['Sigma']
    Ny, Nx = Y.shape[1], X.shape[1]
    eng, _ = fit(X, Y, hyper, with_info=True)
    post = orc.postfit(X, Y, hyper, lapack_general_solve=False)
    Sg = np.stack([Sigma * (1 + 0.05 * h) for h in range(Z.shape[0])])
    for method, name, S in ((L.METHOD_TA, 'TA', Sg), (L.METHOD_ME, 'ME', None)):
        g = eng.predict_grad(Z, S, method, want_hess=True)
        mean, var, cov, jac = eng.predict(Z, S, method)
        assert np.array_equal(g['mean'], mean) and np.array_equal(g['var'], var)
        assert np.array_equal(g['cov'], cov) and np.array_equal(g['jac'], jac)
        fd = orc.predict_grad_fd(X, hyper, post['alpha'], post['chol'], Z, S, name)
        tol = 1e-5 if case != 'car' else 3e-5        # car: cond(K) ~ 1e10 makes the FD of var itself noisy
        assert relinf(g['jac'], fd['dmean']) < tol
        assert relinf(g['hess'], fd['hess']) < tol
        assert relinf(g['dvar_dz'], fd['dvar']) < tol
        assert relinf(g['dcov_dz'], fd['dcov']) < tol
        assert np.array_equal(g['hess'], np.swapaxes(g['hess'], 2, 3))
    eng.close()


def test_casadi_external_entry_points():
    """The `casadi.external`-shaped C entry points (include/gpmpc_casadi.h) driven through ctypes the
    way CasADi's importer drives them: sizes / sparsity patterns, gp_b200 == gpmpc_predict over all
    shooting nodes, jac_gp_b200's block-diagonal CCS nonzeros == gpmpc_predict_grad."""
    import ctypes as C
    m = load_fixture('tank'); X, Y, hyper = m['X'], m['Y'], m['hyper']
    Ny, Nx, Nt = 4, 6, 5
    eng, _ = fit(X, Y, hyper, with_info=True)
    lib = L.load()
    rng = np.random.default_rng(8)
    Z = X[:Nt] + 0.1 * rng.standard_normal((Nt, Nx))
    Sg = np.stack([1e-3 * np.eye(Nx) + 1e-4 * (lambda A: A @ A.T)(rng.standard_normal((Nx, Nx))) for _ in range(Nt)])
    assert lib.gp_b200_bind(eng.h, L.METHOD_TA, Nt) == 0
    assert lib.gp_b200_n_in() == 2 and lib.gp_b200_n_out() == 2
    assert lib.jac_gp_b200_n_in() == 4 and lib.jac_gp_b200_n_out() == 4
    assert lib.gp_b200_name_in(0) == b'z' and lib.gp_b200_name_out(1) == b'cov'
    assert [lib.gp_b200_sparsity_in(0)[k] for k in range(3)] == [Nx, Nt, 1]
    assert [lib.gp_b200_sparsity_in(1)[k] for k in range(3)] == [Nx, Nx * Nt, 1]
    assert [lib.gp_b200_sparsity_out(0)[k] for k in range(3)] == [Ny, Nt, 1]
    assert [lib.gp_b200_sparsity_out(1)[k] for k in range(3)] == [Ny, Ny * Nt, 1]
    dp = C.POINTER(C.c_double)

    def call(fn, ins, outs):
        arg = (dp * len(ins))(*[a.ctypes.data_as(dp) for a in ins])
        res = (dp * len(outs))(*[a.ctypes.data_as(dp) for a in outs])
        assert fn(arg, res, None, None, 0) == 0

    # column-major dense: z (Nx x Nt) is (Nt,Nx) row-major; sigma (Nx x Nx*Nt): block t column-major
    z_cm = np.ascontiguousarray(Z)
    s_cm = np.ascontiguousarray(np.transpose(Sg, (0, 2, 1)))
    mean_cm = np.empty((Nt, Ny)); cov_cm = np.empty((Nt, Ny, Ny))
    call(lib.gp_b200, [z_cm, s_cm], [mean_cm, cov_cm])
    mean, var, cov, jac = eng.predict(Z, Sg, L.METHOD_TA)
    assert np.array_equal(mean_cm, mean) and np.array_equal(cov_cm, np.transpose(cov, (0, 2, 1)))   # column-major blocks
    g = eng.predict_grad(Z, Sg, L.METHOD_TA)

    def ccs(ptr):
        nrow, ncol = ptr[0], ptr[1]
        colind = [ptr[2 + k] for k in range(ncol + 1)]
        rows = [ptr[2 + ncol + 1 + k] for k in range(colind[-1])]
        return nrow, ncol, colind, rows

    pats = [ccs(lib.jac_gp_b200_sparsity_out(k)) for k in range(4)]
    assert (pats[0][0], pats[0][1], pats[0][2][-1]) == (Ny * Nt, Nx * Nt, Nt * Ny * Nx)
    assert (pats[1][0], pats[1][1], pats[1][2][-1]) == (Ny * Nt, Nx * Nx * Nt, 0)
    assert (pats[2][0], pats[2][1], pats[2][2][-1]) == (Ny * Ny * Nt, Nx * Nt, Nt * Ny * Ny * Nx)
    assert (pats[3][0], pats[3][1], pats[3][2][-1]) == (Ny * Ny * Nt, Nx * Nx * Nt, Nt * Ny * Ny * Nx * Nx)
    outs = [np.zeros(max(1, pt[2][-1])) for pt in pats]
    call(lib.jac_gp_b200, [z_cm, s_cm, mean_cm, cov_cm], outs)

    def dense(pat, vals):
        nrow, ncol, colind, rows = pat
        D = np.zeros((nrow, ncol))
        for c in range(ncol):
            for k in range(colind[c], colind[c + 1]):
                D[rows[k], c] = vals[k]
        return D

    Jm = dense(pats[0], outs[0]); Jc = dense(pats[2], outs[2]); Js = dense(pats[3], outs[3])
    for t in range(Nt):
        assert np.array_equal(Jm[t * Ny:(t + 1) * Ny, t * Nx:(t + 1) * Nx], g['jac'][t])
        blk = Jc[t * Ny * Ny:(t + 1) * Ny * Ny, t * Nx:(t + 1) * Nx]         # rows a + Ny*b
        assert np.array_equal(blk.reshape(Ny, Ny, Nx).transpose(1, 0, 2), g['dcov_dz'][t])
        sb = Js[t * Ny * Ny:(t + 1) * Ny * Ny, t * Nx * Nx:(t + 1) * Nx * Nx]  # cols d + Nx*e
        want = np.einsum('ad,be->baed', g['jac'][t], g['jac'][t]).reshape(Ny * Ny, Nx * Nx)
        assert np.array_equal(sb, want)
    Jm[:, :] = np.where(np.kron(np.eye(Nt), np.ones((Ny, Nx))) > 0, 0.0, Jm)
    assert not Jm.any()                                                       # nothing off the block diagonal
    # d cov / d Sigma against a finite difference of the restated TA covariance (linear in Sigma)
    post = orc.postfit(X, Y, hyper, lapack_general_solve=False)
    mo, vo = orc.gp_mean_var(X, hyper, post['alpha'], post['chol'], Z[:1])
    Jo = orc.gp_mean_jac(X, hyper, post['alpha'], Z[:1])
    E = np.zeros((Nx, Nx)); E[1, 3] = 1.0
    dS = (orc.ta_cov(vo, Jo, Sg[0] + E) - orc.ta_cov(vo, Jo, Sg[0]))[0]
    assert relinf(Js[:Ny * Ny, 1 + Nx * 3].reshape(Ny, Ny).T, dS) < 1e-6
    lib.gp_b200_unbind()
    assert not lib.gp_b200_sparsity_in(0)
    eng.close()
    # the GP-class view: derivatives in the caller's units (chain rule through the scalers) vs central
    # differences of GP.predict_batch itself
    gp, m = gp_from_fixture('tank')
    d = load_golden('derived', 'tank')
    xs = np.tile(d['x0'], (3, 1)) * (1 + 0.02 * np.arange(3)[:, None]); us = np.tile(d['u0'], (3, 1))
    gg = gp.predict_batch_grad(xs, us, d['Sigma'])
    mb, cb = gp.predict_batch(xs, us, d['Sigma'])
    assert np.array_equal(gg['mean'], mb) and np.array_equal(gg['cov'], cb)
    zs = np.hstack([xs, us])
    for e in range(6):
        h = 1e-4 * max(1.0, abs(zs[0, e]))
        zp = zs.copy(); zp[:, e] += h
        zm = zs.copy(); zm[:, e] -= h
        mp_, cp_ = gp.predict_batch(zp[:, :4], zp[:, 4:], d['Sigma'])
        mm_, cm_ = gp.predict_batch(zm[:, :4], zm[:, 4:], d['Sigma'])
        assert relinf(gg['dmean_dz'][:, :, e], (mp_ - mm_) / (2 * h)) < 1e-5
        assert relinf(gg['dcov_dz'][:, :, :, e], (cp_ - cm_) / (2 * h)) < 2e-4    # FD of a 1e-5-sized covariance at h ~ 1e-3
    gp.close()


# ------------------------------------------------------------------ 'EM' exact moment matching (8f row 2)
def test_exact_moment_matching_vs_extended_precision():
    """gp_exact_moment (gp_functions.py:344-418) on the GPU against the SAME formula evaluated in
    40-digit arithmetic from (X, Y, hyper) (oracle gp_exact_moment_mp, committed as
    tests/golden/em_mp_*.npz by oracle/make_golden_em.py).  The engine evaluates an algebraically
    identical, better conditioned form (Cholesky-based trace for the invK term, expm1 for
    t Q - q q^T), so unlike the reference's fp64 expression it stays meaningful on the car fixture
    (cond(K) ~ 1e10, where the reference formula in fp64 returns negative variances, SURVEY q18)."""
    # accuracy floor: alpha = K^-1 y itself carries eps*cond(K) relative error (5e-9 tank, 7e-6 car), amplified by the
    # beta^T (t Q - q q^T) beta contraction -- a property of the formula in fp64, shared by every evaluation order
    for name, tol_cov in (('tank', 1e-4), ('car', 0.25)):
        m = load_fixture(name); g = load_golden('em_mp', name)
        eng, _ = fit(m['X'], m['Y'], m['hyper'], with_info=True)
        mean, var, cov, _ = eng.predict(g['Z'], g['Sigma'], L.METHOD_EM, want_jac=False)
        assert relinf(mean, g['mean']) < (TOL if name == 'tank' else 1e-3), relinf(mean, g['mean'])
        assert relinf(cov, g['cov']) < tol_cov, relinf(cov, g['cov'])
        assert (var > 0).all() and np.array_equal(var, np.einsum('haa->ha', cov))
        assert relinf(cov, np.transpose(cov, (0, 2, 1))) == 0.0
        # the plain fp64 restatement of the reference expression (its own invK) for comparison
        post = orc.postfit(m['X'], m['Y'], m['hyper'], lapack_general_solve=False)
        mo, co = orc.gp_exact_moment(post['invK'], m['X'], m['Y'], m['hyper'], g['Z'][0], g['Sigma'][0])
        assert relinf(cov[0], g['cov'][0]) <= max(relinf(co, g['cov'][0]), 1e-9)      # never worse than the reference form
        # EM -> ME as the input covariance vanishes
        Nx = m['X'].shape[1]
        mean0, _, cov0, _ = eng.predict(g['Z'], 1e-14 * np.eye(Nx), L.METHOD_EM, want_jac=False)
        mean_me, var_me, _, _ = eng.predict(g['Z'], None, L.METHOD_ME, want_jac=False)
        assert relinf(mean0, mean_me) < 1e-7
        assert relinf(np.einsum('haa->ha', cov0), var_me) < (1e-6 if name == 'tank' else 1e-3)
        # ... and EM ~ TA for a small input covariance (first-order agreement)
        S = 1e-6 * np.diag(m['X'].var(0))
        _, _, cov_em, _ = eng.predict(g['Z'], S, L.METHOD_EM, want_jac=False)
        _, _, cov_ta, _ = eng.predict(g['Z'], S, L.METHOD_TA, want_jac=False)
        assert relinf(cov_em, cov_ta) < 1e-2
        eng.close()
    # through the GP class at the example's operating point, against the stored-model answer
    d = load_golden('derived', 'tank')
    gp, m = gp_from_fixture('tank')
    gp.set_method('EM')
    mean, cov = gp.predict(d['x0'], d['u0'], d['Sigma'])
    assert relinf(mean, d['mean_em']) < TOL
    assert relinf(np.diag(cov), np.diag(d['cov_em'])) < 2e-2
    gp.close()


# ------------------------------------------------------------------ a6/a7 NLML + gradient
@pytest.mark.parametrize('name', ['tank', 'car'])
def test_nlml_matches_reference_values(name):
    m = load_fixture(name); g = load_golden('ref_verbatim', name)
    eng = _engine(m['X'].shape[0], m['X'].shape[1], m['Y'].shape[1]); eng.set_data(m['X'], m['Y'])
    for a in range(m['hyper'].shape[0]):
        nll = eng.nlml(a, m['hyper'][a], grad=False)
        # car: cond(K) ~ 1e10-7e10, the log-determinant itself is only defined to ~1e-8
        # (numpy triangular-vs-LU reruns of the reference formula differ by 1e-9 already)
        assert nll == pytest.approx(g['nll'][a], rel=1e-9 if name == 'tank' else 5e-8)
    eng.close()


def test_nlml_gradient_vs_oracle():
    p = orc.synthetic_problem(200, 4, 2, config_id=11)
    eng = _engine(200, 4, 2); eng.set_data(p['X'], p['Y'])
    for a in range(2):
        th = p['hyper'][a].copy(); th[:4] *= 0.5; th[5] = 5e-3
        nll, g = eng.nlml(a, th, grad=True)
        assert nll == pytest.approx(orc.calc_NLL(th, p['X'], p['Y'][:, a]), rel=1e-10)
        assert relinf(g, orc.calc_NLL_grad_analytic(th, p['X'], p['Y'][:, a])) < 1e-8
        assert relinf(g, orc.calc_NLL_grad_fd(th, p['X'], p['Y'][:, a])) < 1e-5
    eng.close()


def test_prior_mean_functions_on_the_gpu():
    """get_mean_function (gp_functions.py:25-69) through the engine: alpha on the residual y - m(X)
    (optimize.py:492-494) for given mean parameters; the q2 flag; and the joint fit of kernel + mean
    parameters ('fit_mean', objective of the CasADi twin optimize.py:22-97) lowers the NLL of the
    residual below the zero-mean fit on data with a linear trend."""
    import gp_mpc_b200
    from gp_mpc_b200 import mean_functions as mf
    rng = np.random.default_rng(6)
    p = orc.synthetic_problem(150, 3, 2, config_id=41, H=7)
    X = p['X']; Y = p['Y'] + X @ np.array([[0.8, -0.3], [0.1, 0.5], [-0.4, 0.2]]) + np.array([0.7, -1.1])
    hyper = np.hstack([p['hyper'], 0.2 * rng.standard_normal((2, 4))])
    post = orc.postfit(X, Y, hyper, lapack_general_solve=False, mean_func='linear')
    gp = gp_mpc_b200.GP(X, Y, hyper=dict(hyper=hyper), normalize=False, mean_func='linear')
    assert relinf(gp.get_alpha(), post['alpha']) < 1e-7 and relinf(gp.get_chol(), post['chol']) < 1e-10
    mo, vo = orc.gp_mean_var(X, hyper, post['alpha'], post['chol'], p['Z'])
    mean, cov = gp.predict_batch(p['Z'][:, :2], p['Z'][:, 2:], p['Sigma'])
    assert relinf(mean, mo) < TOL                                   # q2: m(z) is not added back
    gp_f = gp_mpc_b200.GP(X, Y, hyper=dict(hyper=hyper), normalize=False, mean_func='linear', prior_mean_in_predict=True)
    mean_f, _ = gp_f.predict_batch(p['Z'][:, :2], p['Z'][:, 2:], p['Sigma'])
    M = np.column_stack([orc.mean_function(hyper[a], p['Z'], 'linear') for a in range(2)])
    assert relinf(mean_f, mo + M) < TOL
    gp.close(); gp_f.close()
    # joint fit: gradient block of the mean parameters vs central differences of the restated NLL
    eng = _engine(150, 3, 2); eng.set_data(X, Y)
    Phi = mf.mean_design(X, 'linear')
    th = hyper[0].copy()
    eng.set_y(0, Y[:, 0] - Phi @ th[5:])
    nll, g = eng.nlml(0, th[:5], grad=True)
    gm = -Phi.T @ eng.get(L.GET_ALPHA_NLML, 0)
    ref = lambda t: orc.calc_NLL(t[:5], X, Y[:, 0] - Phi @ t[5:], False)
    assert nll == pytest.approx(ref(th), rel=1e-10)
    for j in range(4):
        e = np.zeros(9); e[5 + j] = 1e-6
        assert gm[j] == pytest.approx((ref(th + e) - ref(th - e)) / 2e-6, rel=1e-5, abs=1e-6)
    eng.close()
    opts = {'maxiter': 200, 'fixed_bounds': True}
    gp0 = gp_mpc_b200.GP(X, Y, normalize=False, mean_func='linear', optimizer_opts=dict(opts))
    h0 = np.column_stack([gp0.get_hyper_parameters()['length_scale'], np.sqrt(gp0.get_hyper_parameters()['signal_var']),
                          gp0.get_hyper_parameters()['mean']])
    assert h0.shape == (2, 9) and np.all(h0[:, 5:] == 0.0)          # reference numeric path: mean parameters stay 0
    gp1 = gp_mpc_b200.GP(X, Y, normalize=False, mean_func='linear', optimizer_opts=dict(opts, fit_mean=True))
    h1 = np.column_stack([gp1.get_hyper_parameters()['length_scale'], np.sqrt(gp1.get_hyper_parameters()['signal_var']),
                          gp1.get_hyper_parameters()['mean']])
    assert np.abs(h1[:, 5:8]).max() <= 1e-2 + 1e-12                  # slope bounds of optimize.py:458-459
    from gp_mpc_b200.optimize import bounds_and_init
    for a in range(2):
        # SLSQP made progress on the joint objective from the reference's start (kernel init of
        # optimize.py:445-449, mean parameters 0 clipped into their bounds) and respected the bounds
        bk, init = bounds_and_init(X, Y[:, a], True)
        mb = mf.mean_bounds(Y[:, a], 3, 'linear')
        m0 = np.clip(np.zeros(4), mb[:, 0], mb[:, 1])
        n_init = orc.calc_NLL(init, X, Y[:, a] - Phi @ m0, False)
        n1 = orc.calc_NLL(h1[a, :5], X, Y[:, a] - Phi @ h1[a, 5:], False)
        assert n1 < n_init
        assert np.all(h1[a, 5:] >= mb[:, 0] - 1e-12) and np.all(h1[a, 5:] <= mb[:, 1] + 1e-12)
        assert h1[a, 8] != 0.0                                       # the offset moved into its (data-mean) interval
    gp0.close(); gp1.close()


# ------------------------------------------------------------------ the GP class (drop-in boundary)


@pytest.mark.parametrize('name', ['tank', 'car'])
def test_gp_class_known_answers(name):
    gp, m = gp_from_fixture(name)
    d = load_golden('derived', name)
    N, Ny, Nu = gp.get_size()
    assert (N, Ny, Nu) == (m['X'].shape[0], m['Y'].shape[1], m['X'].shape[1] - m['Y'].shape[1])
    gp.set_method('TA')
    mean, cov = gp.predict(d['x0'], d['u0'], d['Sigma'])
    assert mean.shape == (Ny, 1) and cov.shape == (Ny, Ny)
    assert relinf(mean, d['mean_ta']) < TOL and relinf(cov, d['cov_ta']) < TOL
    gp.set_method('ME')
    mean, cov = gp.predict(d['x0'], d['u0'], d['Sigma'])
    assert relinf(mean, d['mean_me']) < TOL and relinf(cov, d['cov_me']) < TOL
    A, B = gp.discrete_linearize(d['x0'], d['u0'], d['Sigma'])
    assert relinf(A, d['A']) < TOL and relinf(B, d['B']) < TOL
    with pytest.raises(NameError):
        gp.set_method('nope')
    gp.close()


def test_gp_class_validate_and_io(tmp_path):
    gp, m = gp_from_fixture('tank')
    rng = np.random.default_rng(1)
    Xt = m['meta']['meanZ'] + m['meta']['stdZ'] * rng.standard_normal((25, 6)) * 0.5
    Yt = m['meta']['meanY'] + m['meta']['stdY'] * rng.standard_normal((25, 4)) * 0.5
    smse, mnlp = gp.validate(Xt, Yt)
    so, mo = orc.validate(m, Xt, Yt)
    assert relinf(smse, so) < TOL and relinf(mnlp, mo) < TOL
    path = str(tmp_path / 'model')
    gp.save_model(path)
    with open(path + '.json') as f:
        dd = json.load(f)
    assert set(dd) == {'X', 'Y', 'hyper', 'mean_func', 'normalize', 'xlb', 'xub', 'ulb', 'uub', 'meta'}
    assert set(dd['hyper']) == {'hyper', 'invK', 'alpha', 'chol', 'length_scale', 'signal_var', 'noise_var', 'mean'}
    assert relinf(np.array(dd['hyper']['chol']), m['chol']) < 1e-10
    import gp_mpc_b200
    gp2 = gp_mpc_b200.GP.load_model(path)
    d = load_golden('derived', 'tank')
    m1, c1 = gp.predict(d['x0'], d['u0'], d['Sigma'])
    m2, c2 = gp2.predict(d['x0'], d['u0'], d['Sigma'])
    assert np.array_equal(m1, m2) and np.array_equal(c1, c2)
    gp.save_model_npz(path)
    gp3 = gp_mpc_b200.GP.load_model_npz(path)
    m3, c3 = gp3.predict(d['x0'], d['u0'], d['Sigma'])
    assert np.array_equal(m1, m3) and np.array_equal(c1, c3)
    gp3.close()
    # batched horizon call == per-point calls
    xs = np.tile(d['x0'], (5, 1)) * (1 + 0.01 * np.arange(5)[:, None]); us = np.tile(d['u0'], (5, 1))
    mb, cb = gp.predict_batch(xs, us, d['Sigma'])
    for h in range(5):
        mh, ch = gp.predict(xs[h], us[h], d['Sigma'])
        assert relinf(mb[h], mh.ravel()) < 1e-12 and relinf(cb[h], ch) < 1e-12
    # sequential roll-out (numeric part of predict_compare, gp_class.py:777-804) vs the oracle loop
    useq = np.tile(d['u0'], (6, 1)) * (1 + 0.02 * np.arange(6)[:, None])
    rm, rv = gp.rollout(d['x0'], useq, methods=['TA', 'ME'], device_rollout=False)      # one host call per step
    for i, meth in enumerate(['TA', 'ME']):
        cv = np.eye(6) * 1e-6; cv[:4, :4] = np.diag(m['hyper'][:, 7] ** 2); xt = d['x0'].copy()
        for t in range(6):
            mo_, co_ = orc.predict(m, xt, useq[t], cv, meth)
            xt = mo_.ravel(); cv[:4, :4] = co_
            assert relinf(rm[i, t + 1], xt) < TOL
            assert relinf(rv[i, t + 1], np.diag(co_) * m['meta']['stdY'] ** 2) < 1e-5
    # kernel helper keeps the reference's error behaviour
    with pytest.raises(ValueError):
        gp.covSEard(np.zeros((3, 6)), np.zeros((2, 5)), np.ones(6), 1.0)
    # GP.covar: full posterior covariance between test points, odd (D,n,n) shape kept (q12)
    g = load_golden('ref_verbatim', 'tank')
    cv = gp.covar(g['Zt'])
    assert cv.shape == g['covar'].shape and np.all(cv[4:] == 0.0)
    for a in range(4):
        assert relinf(cv[a], g['covar'][a]) < TOL            # vs the reference's own GP.covar output
    k = gp.covSEard(m['X'][:5], m['X'][5:9], m['hyper'][0, :6], 2.0)
    assert relinf(k, orc.covSEard(m['X'][:5], m['X'][5:9], m['hyper'][0, :6], 2.0)) < 1e-13
    gp.close(); gp2.close()


def test_gp_class_trains_like_the_reference_driver():
    """train_gp_numpy semantics (optimize.py:359-503): same init / bounds / SLSQP; the GPU fit
    (analytic gradient) must reach an NLL at least as low as the FD-gradient CPU restatement."""
    import gp_mpc_b200
    p = orc.synthetic_problem(60, 3, 2, config_id=77)
    Xr = 3.0 + 2.0 * p['X']; Yr = 1.0 + 0.5 * p['Y']
    gp = gp_mpc_b200.GP(Xr, Yr, normalize=True, xlb=[0] * 2, xub=[1] * 2, ulb=[0], uub=[1],
                        optimizer_opts={'maxiter': 300})
    hy = np.column_stack([gp.get_hyper_parameters()['length_scale'],
                          np.sqrt(gp.get_hyper_parameters()['signal_var']),
                          np.sqrt(gp.get_hyper_parameters()['noise_var'])])
    st = orc.data_stats(Xr, Yr, 2)
    Xs = (Xr - st['meanZ']) / st['stdZ']; Ys = (Yr - st['meanY']) / st['stdY']
    ref = orc.train_gp(Xs, Ys, options={'maxiter': 300})
    for a in range(2):
        nll_gpu = orc.calc_NLL(hy[a], Xs, Ys[:, a])
        nll_ref = orc.calc_NLL(ref['hyper'][a], Xs, Ys[:, a])
        assert nll_gpu <= nll_ref + 1e-3 * abs(nll_ref)
    # jac='fd' follows the reference's finite-difference trajectory
    gp_fd = gp_mpc_b200.GP(Xr, Yr, normalize=True, xlb=[0] * 2, xub=[1] * 2, ulb=[0], uub=[1],
                           optimizer_opts={'maxiter': 300, 'jac': 'fd'})
    hy_fd = np.column_stack([gp_fd.get_hyper_parameters()['length_scale'],
                             np.sqrt(gp_fd.get_hyper_parameters()['signal_var']),
                             np.sqrt(gp_fd.get_hyper_parameters()['noise_var'])])
    for a in range(2):
        assert orc.calc_NLL(hy_fd[a], Xs, Ys[:, a]) == pytest.approx(
            orc.calc_NLL(ref['hyper'][a], Xs, Ys[:, a]), rel=1e-4, abs=1e-3)
    gp.close(); gp_fd.close()


def test_parallel_per_output_fits_equal_the_sequential_loop():
    """train_gp_b200 runs the independent per-output SLSQP fits concurrently (one scratch engine and host
    thread per output); every output's iterates only depend on its own data, so the fitted rows are
    identical to the sequential loop's."""
    import gp_mpc_b200
    p = orc.synthetic_problem(300, 4, 3, config_id=55)
    kw = dict(normalize=False)
    gp_s = gp_mpc_b200.GP(p['X'], p['Y'], optimizer_opts={'maxiter': 40, 'parallel_fits': False}, **kw)
    gp_p = gp_mpc_b200.GP(p['X'], p['Y'], optimizer_opts={'maxiter': 40}, **kw)
    hs, hp_ = gp_s.get_hyper_parameters(), gp_p.get_hyper_parameters()
    for k in ('length_scale', 'signal_var', 'noise_var'):
        assert np.array_equal(hs[k], hp_[k])
    gp_s.close(); gp_p.close()


# ------------------------------------------------------------------ edge cases / error behaviour
@pytest.mark.parametrize('N,Nx,Ny,H', [(1, 1, 1, 1), (2, 3, 2, 5), (127, 4, 1, 64), (128, 4, 1, 65), (129, 2, 2, 129),
                                       (257, 32, 1, 3), (200, 3, 11, 9), (300, 10, 12, 64)])
def test_edge_sizes(N, Nx, Ny, H):
    """smallest / ragged / maximum-Nx shapes: padding to 128, H chunking at 64, Nx = NX_MAX; more than 8 outputs (second
    column block of the row-wise assembly), and a batch whose records do not fit the fused tail's shared memory (flat
    assembly from L2)."""
    rng = np.random.default_rng(N * 7 + H)
    X = rng.standard_normal((N, Nx)); Y = rng.standard_normal((N, Ny))
    hyper = np.column_stack([rng.uniform(1.0, 3.0, (Ny, Nx)), np.full(Ny, 1.3), np.full(Ny, 0.05)])
    Z = rng.standard_normal((H, Nx)); A = rng.standard_normal((Nx, Nx)); Sig = 1e-3 * (np.eye(Nx) + 0.1 * A @ A.T)
    post = orc.postfit(X, Y, hyper, lapack_general_solve=False)
    mo, vo = orc.gp_mean_var(X, hyper, post['alpha'], post['chol'], Z)
    Jo = orc.gp_mean_jac(X, hyper, post['alpha'], Z); co = orc.ta_cov(vo, Jo, Sig)
    eng, info = fit(X, Y, hyper, with_info=True)
    mean, var, cov, jac = eng.predict(Z, Sig, L.METHOD_TA)
    assert relinf(mean, mo) < TOL and relinf(var, vo) < TOL and relinf(cov, co) < TOL and relinf(jac, Jo) < TOL
    assert relinf(eng.get(L.GET_CHOL, Ny - 1), post['chol'][Ny - 1]) < 1e-10
    pc = eng.posterior_cov(Z[:min(H, 7)])
    ks = orc.covSEard(X, Z[:min(H, 7)], hyper[0, :Nx], hyper[0, Nx] ** 2)
    v = np.linalg.solve(post['chol'][0], ks)
    assert relinf(pc[0], hyper[0, Nx] ** 2 - v.T @ v) < TOL
    eng.close()


def test_argument_errors_fail_loudly():
    import gp_mpc_b200
    with pytest.raises(L.GpmpcError):
        gp_mpc_b200.Engine(10, 33, 1, device=0)                  # Nx above NX_MAX
    with pytest.raises(L.GpmpcError):
        gp_mpc_b200.Engine(10, 2, 2, out_begin=1, out_count=2, device=0)
    eng = gp_mpc_b200.Engine(10, 2, 1, device=0)
    with pytest.raises(L.GpmpcError):
        eng.factorize()                                          # no data / hyper yet
    rng = np.random.default_rng(0)
    eng.set_data(rng.standard_normal((10, 2)), rng.standard_normal((10, 1)))
    with pytest.raises(L.GpmpcError):
        eng.set_hyper(np.array([[0.0, 1.0, 1.0, 0.1]]))          # zero length scale
    eng.set_hyper(np.array([[1.0, 1.0, 1.0, 0.1]]))
    with pytest.raises(L.GpmpcError):
        eng.predict(np.zeros((1, 2)))                            # not factorised
    eng.factorize()
    with pytest.raises(L.GpmpcError):
        eng.get(L.GET_CHOL, 3)                                   # output not owned
    for name in ('no_such_option', 'gemm_variant', 'leaf_variant', 'overlap', 'lookahead', 'lookahead_min', 'zero_copy'):
        with pytest.raises(L.GpmpcError):
            eng.set_option(name, 1)
    with pytest.raises(L.GpmpcError):
        eng.predict(np.zeros((2, 2)), None, L.METHOD_EM, want_jac=False)     # EM needs Sigma
    eng.close()
    gp = gp_mpc_b200.GP(rng.standard_normal((12, 3)), rng.standard_normal((12, 2)), normalize=False,
                        hyper=dict(hyper=np.array([[1., 1., 1., 1., .1], [1., 2., 1., 1., .1]])))
    with pytest.raises(NotImplementedError):
        gp.set_method('old_TA')
    with pytest.raises(NotImplementedError):
        gp.update_data(np.zeros((1, 3)), np.zeros((1, 2)))
    gp.update_data_all(rng.standard_normal((4, 3)), rng.standard_normal((4, 2)))
    assert gp.get_size() == (16, 2, 1)
    gp.replace_data_all(rng.standard_normal((5, 3)), rng.standard_normal((5, 2)))
    assert gp.get_size() == (5, 2, 1)
    gp.close()


def test_autonomous_system_nu_zero_rollout():
    """van_der_pol.py:20-47 pattern: no control inputs (Nu = 0), a long sequential numeric
    gp.predict roll-out with 'ME' -- each call is one H=1 pass through the engine."""
    import gp_mpc_b200
    rng = np.random.default_rng(12)
    X = rng.uniform(-2, 2, (40, 2))
    Y = np.column_stack([X[:, 0] + 0.1 * X[:, 1], X[:, 1] + 0.1 * (-X[:, 0] + (1 - X[:, 0] ** 2) * X[:, 1])])
    Y = Y + 2e-2 * rng.standard_normal(Y.shape)          # measurement noise, as the example adds (van_der_pol.py:66-71)
    gp = gp_mpc_b200.GP(X, Y, normalize=True, xlb=[-2, -2], xub=[2, 2], ulb=[], uub=[], gp_method='ME',
                        optimizer_opts={'maxiter': 100})
    assert gp.get_size() == (40, 2, 0)
    hy = np.column_stack([gp.get_hyper_parameters()['length_scale'], np.sqrt(gp.get_hyper_parameters()['signal_var']),
                          np.sqrt(gp.get_hyper_parameters()['noise_var'])])
    st = orc.data_stats(X, Y, 2)
    model = dict(X=(X - st['meanZ']) / st['stdZ'], Y=(Y - st['meanY']) / st['stdY'], hyper=hy, normalize=True, meta=st)
    model.update(orc.postfit(model['X'], model['Y'], hy, lapack_general_solve=False))
    x = np.array([1.0, 0.5]); xo = x.copy()
    for t in range(25):
        mean, cov = gp.predict(x, [], np.zeros((2, 2)))
        mo, co = orc.predict(model, xo, np.zeros(0), np.zeros((2, 2)), 'ME')
        assert relinf(mean, mo) < TOL and relinf(np.diag(cov), np.diag(co)) < TOL
        x = np.array(mean).flatten(); xo = mo.flatten()
    gp.close()


@pytest.mark.parametrize('name', ['tank', 'car'])
def test_device_rollout_equals_the_host_loop(name):
    """gpmpc_rollout (all steps enqueued on the device, state fed back by a kernel) against GP.rollout's host loop
    (one predict call per step, gp_class.py:777-804): same operation order, so the trajectories agree to rounding."""
    gp, m = gp_from_fixture(name)
    d = load_golden('derived', name)
    useq = np.tile(d['u0'], (12, 1)) * (1 + 0.02 * np.arange(12)[:, None])
    rm, rv = gp.rollout(d['x0'], useq, methods=['TA', 'ME'])
    rm_h, rv_h = gp.rollout(d['x0'], useq, methods=['TA', 'ME'], device_rollout=False)
    assert rm.shape == rm_h.shape and relinf(rm, rm_h) < 1e-12 and relinf(rv, rv_h) < 1e-12
    assert (rv[:, 1:] > 0).all()
    gp.close()


def test_device_rollout_autonomous_system():
    """Nu = 0 (van_der_pol.py): 25 'ME' steps on the device equal 25 sequential GP.predict calls."""
    import gp_mpc_b200
    rng = np.random.default_rng(12)
    X = rng.uniform(-2, 2, (40, 2))
    Y = np.column_stack([X[:, 0] + 0.1 * X[:, 1], X[:, 1] + 0.1 * (-X[:, 0] + (1 - X[:, 0] ** 2) * X[:, 1])])
    Y = Y + 2e-2 * rng.standard_normal(Y.shape)
    hyper = np.column_stack([np.full((2, 2), 1.5), np.full(2, 1.2), np.full(2, 0.05)])
    gp = gp_mpc_b200.GP(X, Y, normalize=False, gp_method='ME', hyper=dict(hyper=hyper))
    x = np.array([1.0, 0.5]); traj = []
    for t in range(25):
        mean, cov = gp.predict(x, [], np.zeros((2, 2)))
        x = np.array(mean).flatten(); traj.append(x.copy())
    rm, rv = gp.rollout(np.array([1.0, 0.5]), np.zeros((25, 0)), methods=['ME'])
    assert rm.shape == (1, 26, 2) and relinf(rm[0, 1:], np.array(traj)) < 1e-12 and (rv[0, 1:] > 0).all()
    gp.close()


def test_rank1_append_matches_a_full_refit():
    """SURVEY 8f row 3: O(N^2) append of training points == refactorising from scratch (oracle
    postfit on the concatenated data); crossing the padded capacity falls back to a refit."""
    import gp_mpc_b200
    p = orc.synthetic_problem(134, 5, 2, config_id=31, H=12)
    X, Y, hyper = p['X'], p['Y'], p['hyper']
    gp = gp_mpc_b200.GP(X[:123], Y[:123], normalize=False, hyper=dict(hyper=hyper))
    gp.append_data(X[123:128], Y[123:128])                  # fills the 128-row capacity by rank-1 updates
    assert gp.get_size()[0] == 128 and gp.engine.N == 128
    post = orc.postfit(X[:128], Y[:128], hyper, lapack_general_solve=False)
    assert relinf(gp.get_chol(), post['chol']) < 1e-10
    assert relinf(gp.get_alpha(), post['alpha']) < 1e-7
    mo, vo = orc.gp_mean_var(X[:128], hyper, post['alpha'], post['chol'], p['Z'])
    mean, var, _, _ = gp.engine.predict(p['Z'], None, L.METHOD_ME, want_jac=False)
    assert relinf(mean, mo) < TOL and relinf(var, vo) < TOL
    gp.append_data(X[128:], Y[128:])                        # capacity exceeded -> refit path
    assert gp.get_size()[0] == 134
    post = orc.postfit(X, Y, hyper, lapack_general_solve=False)
    assert relinf(gp.get_chol(), post['chol']) < 1e-10
    gp.append_data(X[:1] + 0.37, Y[:1])                     # rank-1 again on the new 256-row handle
    assert gp.get_size()[0] == 135
    Xa = np.vstack([X, X[:1] + 0.37]); Ya = np.vstack([Y, Y[:1]])
    post = orc.postfit(Xa, Ya, hyper, lapack_general_solve=False)
    assert relinf(gp.get_chol(), post['chol']) < 1e-10 and relinf(gp.get_alpha(), post['alpha']) < 1e-7
    gp.close()
