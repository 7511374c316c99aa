"""gpmpc_append_greedy / Engine.append_greedy / GP.append_greedy and gpmpc_create_reserve on the GPU: picks and scores
against the numpy oracle (a fresh Cholesky per step), the model afterwards against a refit of the augmented data,
determinism, handles with reserved capacity against unreserved ones, the argument and state checks, and the GP's device
and host selection paths."""
import ctypes as C

import numpy as np
import pytest

from gp_mpc_b200 import _lib as L
from oracle import gp_oracle as orc
from oracle import greedy_oracle as gro
from tests._engines import fit
from tests._util import load_fixture, relinf

pytestmark = pytest.mark.gpu


def _pool(X, n, scale, seed):
    rng = np.random.default_rng(seed)
    return X[rng.integers(0, X.shape[0], n)] + scale * rng.standard_normal((n, X.shape[1]))


def case_data(case):
    """(X, Y, hyper, Xc, Yc, n_new) of a parity case; module level so the oracle side can be checked without a GPU."""
    if case in ('tank', 'car'):
        m = load_fixture(case)
        X, Y, hyper = m['X'], m['Y'], m['hyper']
        Xc = _pool(X, 40, 0.5, 3)
        Yc = np.random.default_rng(4).standard_normal((40, Y.shape[1]))
        return X, Y, hyper, Xc, Yc, 12
    N, Nx, Ny, n, n_new = case
    p = orc.synthetic_problem(N, Nx, Ny, config_id=N + 7 * Nx + Ny)
    Xc = _pool(p['X'], n, 1.0, N + n)
    Yc = np.random.default_rng(n).standard_normal((n, Ny))
    return p['X'], p['Y'], p['hyper'], Xc, Yc, n_new


CASES = ['tank', 'car', (130, 2, 3, 65, 65), (130, 2, 1, 65, 0), (700, 5, 11, 65, 17), (700, 5, 1, 1, 1),
         (1500, 32, 1, 300, 17), (1500, 32, 3, 65, 1)]


def _preds_vs(eng, X, Y, hyper, Z, Sigma):
    post = orc.postfit(X, Y, hyper, lapack_general_solve=False)
    mo, vo = orc.gp_mean_var(X, hyper, post['alpha'], post['chol'], Z)
    Jo = orc.gp_mean_jac(X, hyper, post['alpha'], Z)
    m, v, c, J = eng.predict(Z, Sigma, L.METHOD_TA)
    assert relinf(m, mo) < 1e-6 and relinf(v, vo) < 1e-6 and relinf(J, Jo) < 1e-6
    assert relinf(c, orc.ta_cov(vo, Jo, Sigma)) < 1e-6
    m, v, c, _ = eng.predict(Z, None, L.METHOD_ME)
    assert relinf(m, mo) < 1e-6 and relinf(v, vo) < 1e-6 and relinf(c, orc.me_cov(vo)) < 1e-6
    return post


@pytest.mark.parametrize('case', CASES, ids=[str(c) for c in CASES])
def test_picks_and_model_match_the_oracle(case):
    X, Y, hyper, Xc, Yc, n_new = case_data(case)
    N = X.shape[0]
    ref = gro.greedy_select(X, hyper, Xc, n_new)
    assert np.all(ref['gap'] > 1e-8)                       # no near-tie: the picks are well defined
    eng = fit(X, Y, hyper, capacity=N + n_new)
    picked, score, ok = eng.append_greedy(Xc, Yc, n_new)
    assert ok and eng.N == N + n_new
    np.testing.assert_array_equal(picked, ref['picked'])
    if n_new:       # a score is sum_a sf2_a - |v_a|^2: its rounding is relative to the prior variances it cancels
        np.testing.assert_allclose(score, ref['score'], rtol=1e-9, atol=1e-9 * np.sum(hyper[:, X.shape[1]] ** 2))
    Xa, Ya = np.vstack([X, Xc[picked]]), np.vstack([Y, Yc[picked]])
    rng = np.random.default_rng(1)
    Z = Xa[rng.integers(0, Xa.shape[0], 5)] + 0.1 * rng.standard_normal((5, X.shape[1]))
    Sigma = 1e-4 * np.eye(X.shape[1])
    post = _preds_vs(eng, Xa, Ya, hyper, Z, Sigma)
    # car: cond(K) ~ 1e10 (its plain factorisation is held to 2e-9 / 1e-4 in test_gpu_parity); the appended rows
    # l = L^-1 k carry that conditioning once more
    tol_chol, tol_alpha = (5e-8, 1e-4) if case == 'car' else (1e-10, 1e-7)
    tol_em = 1e-4 if case == 'car' else 1e-6            # EM works from K^-1 and alpha: cond(K) eps again
    for a in range(Y.shape[1]):
        assert relinf(eng.get(L.GET_CHOL, a), post['chol'][a]) < tol_chol
        assert relinf(eng.get(L.GET_ALPHA, a), post['alpha'][a]) < tol_alpha
    # the derivative caches (Li^T, EM K^-1) follow the appends: same results as a handle fitted on the augmented data
    ref_eng = fit(Xa, Ya, hyper)
    g1, g2 = eng.predict_grad(Z, Sigma, L.METHOD_TA), ref_eng.predict_grad(Z, Sigma, L.METHOD_TA)
    for k in ('mean', 'var', 'jac', 'dvar_dz', 'dcov_dz'):
        assert relinf(g1[k], g2[k]) < 1e-6, k
    if X.shape[1] <= 8:
        e1, e2 = (e.predict(Z[:2], Sigma, L.METHOD_EM, want_jac=False) for e in (eng, ref_eng))
        assert relinf(e1[0], e2[0]) < tol_em and relinf(e1[2], e2[2]) < tol_em
        d1, d2 = eng.predict_em_grad(Z[:2], Sigma), ref_eng.predict_em_grad(Z[:2], Sigma)
        for k in ('dmean_dz', 'dcov_dSigma'):
            assert relinf(d1[k], d2[k]) < tol_em, k


def test_two_calls_give_identical_bits():
    X, Y, hyper, Xc, Yc, _ = case_data((700, 5, 3, 300, 17))
    out = []
    for _ in range(2):
        eng = fit(X, Y, hyper, capacity=X.shape[0] + 40)
        picked, score, ok = eng.append_greedy(Xc, Yc, 40)
        assert ok
        out.append((picked, score, [eng.get(L.GET_CHOL, a) for a in range(3)], [eng.get(L.GET_LINV, a) for a in range(3)]))
        eng.close()
    np.testing.assert_array_equal(out[0][0], out[1][0])
    assert out[0][1].tobytes() == out[1][1].tobytes()
    for a in range(3):
        assert out[0][2][a].tobytes() == out[1][2][a].tobytes()
        assert out[0][3][a].tobytes() == out[1][3][a].tobytes()


@pytest.mark.parametrize('N', [128, 4096])
def test_reserved_capacity_matches_an_unreserved_handle(N):
    p = orc.synthetic_problem(N, 4, 2, config_id=N + 3, H=6)
    X, Y, hyper, Z, Sigma = p['X'], p['Y'], p['hyper'], p['Z'], p['Sigma']
    plain, res = fit(X, Y, hyper), fit(X, Y, hyper, capacity=N + 300)
    assert plain.capacity == -(-N // 128) * 128 and res.capacity == -(-(N + 300) // 128) * 128
    # a larger padded size splits the recursion and the predict product's stream-K work differently: rounding only
    for a in range(2):
        assert relinf(res.get(L.GET_CHOL, a), plain.get(L.GET_CHOL, a)) < 1e-11
        assert relinf(res.get(L.GET_ALPHA, a), plain.get(L.GET_ALPHA, a)) < 1e-8
        assert relinf(res.get(L.GET_LOGDET, a), plain.get(L.GET_LOGDET, a)) < 1e-11
    _preds_vs(res, X, Y, hyper, Z, Sigma)
    for k, (u, v) in enumerate(zip(res.predict(Z, Sigma, L.METHOD_TA), plain.predict(Z, Sigma, L.METHOD_TA))):
        assert relinf(u, v) < 1e-8, k
    g1, g2 = res.predict_grad(Z, Sigma, L.METHOD_TA), plain.predict_grad(Z, Sigma, L.METHOD_TA)
    for k in ('mean', 'var', 'jac', 'dvar_dz', 'dcov_dz'):
        assert relinf(g1[k], g2[k]) < 1e-8, k
    e1, e2 = (e.predict(Z[:2], Sigma, L.METHOD_EM, want_jac=False) for e in (res, plain))
    # the EM covariance is a difference of O(sf2) terms over K^-1: held to the oracle tolerance
    assert relinf(e1[0], e2[0]) < 1e-8 and relinf(e1[2], e2[2]) < 1e-6
    d1, d2 = res.predict_em_grad(Z[:2], Sigma), plain.predict_em_grad(Z[:2], Sigma)
    assert relinf(d1['dmean_dz'], d2['dmean_dz']) < 1e-6 and relinf(d1['dcov_dSigma'], d2['dcov_dSigma']) < 1e-6
    th = hyper[1] * 1.1
    f1, gr1 = res.nlml(1, th)
    f2, gr2 = plain.nlml(1, th)
    assert abs(f1 - f2) <= 1e-9 * abs(f2) and relinf(gr1, gr2) < 1e-8
    assert abs(f1 - orc.calc_NLL(th, X, Y[:, 1], False)) <= 1e-8 * abs(f1)
    assert relinf(gr1, orc.calc_NLL_grad_analytic(th, X, Y[:, 1])) < 1e-6
    # 200 rank-1 appends fit in the reserve (gpmpc_append reports a full capacity as False)
    res.factorize()
    Xn = _pool(X, 200, 0.5, 9); Yn = np.random.default_rng(2).standard_normal((200, 2))
    for k in range(200):
        assert res.append(Xn[k], Yn[k]), k
    post = _preds_vs(res, np.vstack([X, Xn]), np.vstack([Y, Yn]), hyper, Z, Sigma)
    assert relinf(res.get(L.GET_CHOL, 0), post['chol'][0]) < 1e-10


def test_gp_selects_at_a_full_padded_size_in_one_device_call(monkeypatch):
    import gp_mpc_b200
    p = orc.synthetic_problem(4096, 4, 2, config_id=11)
    gp = gp_mpc_b200.GP(p['X'], p['Y'], hyper=dict(hyper=p['hyper']), normalize=False)
    assert gp.engine.capacity == 4096                      # no spare rows: the engine is rebuilt with a reserve
    calls = []
    real = gp_mpc_b200._lib.Engine.append_greedy
    monkeypatch.setattr(gp_mpc_b200._lib.Engine, 'append_greedy', lambda self, *a: calls.append(a[2]) or real(self, *a))
    Xc = _pool(p['X'], 256, 1.0, 5); Yc = np.zeros((256, 2))
    picked = gp.append_greedy(Xc, Yc, 64)
    assert calls == [64] and len(set(picked.tolist())) == 64 and gp.get_size()[0] == 4096 + 64
    ref = gro.greedy_select(p['X'], p['hyper'], Xc, 4)
    np.testing.assert_array_equal(picked[:4], ref['picked'])


def test_state_and_argument_errors_leave_the_model_untouched():
    X, Y, hyper, Xc, Yc, _ = case_data((130, 2, 3, 65, 65))
    lib = L.load()
    Z = X[:4] + 0.1
    ip = C.POINTER(C.c_int)
    dp = C.POINTER(C.c_double)

    def call(eng, n, n_new, xc=Xc, yc=Yc, null=None):
        picked = np.zeros(max(n_new, 1), dtype=np.int32); added = C.c_int(-7)
        ptr = {k: None if k == null else v for k, v in dict(
            X=np.ascontiguousarray(xc).ctypes.data_as(dp), Y=np.ascontiguousarray(yc).ctypes.data_as(dp),
            P=picked.ctypes.data_as(ip), A=C.byref(added)).items()}
        return lib.gpmpc_append_greedy(eng.h, n, ptr['X'], ptr['Y'], n_new, ptr['P'], None, ptr['A'])

    eng = fit(X, Y, hyper)                                # capacity 256
    before = eng.predict(Z, 1e-4 * np.eye(2), L.METHOD_TA)
    assert call(eng, 65, 66) == L.ERR_ARG                  # n_new > n
    assert call(eng, 65, -1) == L.ERR_ARG
    assert call(eng, 0, 0) == L.ERR_ARG
    for k in ('X', 'Y', 'P', 'A'):
        assert call(eng, 65, 3, null=k) == L.ERR_ARG
    big = _pool(X, 200, 1.0, 1)
    assert call(eng, 200, 127, xc=big, yc=np.zeros((200, 3))) == L.ERR_STATE      # 130 + 127 > 256
    assert 'capacity' in lib.gpmpc_last_error(eng.h).decode()
    after = eng.predict(Z, 1e-4 * np.eye(2), L.METHOD_TA)
    for u, v in zip(before, after):
        assert u.tobytes() == v.tobytes()
    assert eng.N == 130
    sharded = fit(X, Y, hyper, out_begin=1, out_count=2)
    assert call(sharded, 65, 3) == L.ERR_STATE
    fresh = L.Engine(X.shape[0], 2, 3, device=0, capacity=200)
    fresh.set_data(X, Y)
    fresh.set_hyper(hyper)
    assert call(fresh, 65, 3) == L.ERR_STATE                # not factorised
    assert 'factorize' in lib.gpmpc_last_error(fresh.h).decode()


def test_gp_device_and_host_paths_agree_on_the_car_model():
    """normalize=True: the car fixture is stored unnormalised, so the GP is given a standardisation of its own (its
    stored X, Y count as already standardised; only the pool is mapped)."""
    import gp_mpc_b200
    m = load_fixture('car')
    Ny, Nx = m['Y'].shape[1], m['X'].shape[1]
    rng = np.random.default_rng(8)
    mZ, sZ = rng.standard_normal(Nx), rng.uniform(0.5, 2.0, Nx)
    meta = dict(meanY=rng.standard_normal(Ny), stdY=rng.uniform(0.5, 2.0, Ny), meanZ=mZ, stdZ=sZ,
                meanX=mZ[:Ny], stdX=sZ[:Ny], meanU=mZ[Ny:], stdU=sZ[Ny:])

    def gp():
        return gp_mpc_b200.GP(m['X'], m['Y'], mean_func='zero', gp_method='TA', normalize=True,
                              hyper=dict(hyper=m['hyper']), meta=meta)
    Xs = _pool(m['X'], 40, 0.5, 3)
    X_new = Xs * sZ + mZ
    Y_new = np.random.default_rng(4).standard_normal((40, Ny)) * meta['stdY'] + meta['meanY']
    g_dev, g_host, g_all = gp(), gp(), gp()
    p_dev = g_dev.append_greedy(X_new, Y_new, 12, device_select=True)
    p_host = g_host.append_greedy(X_new, Y_new, 12, device_select=False)
    np.testing.assert_array_equal(p_dev, p_host)
    np.testing.assert_array_equal(p_dev, gro.greedy_select(m['X'], m['hyper'], Xs, 12)['picked'])
    g_all.update_data_all(X_new[p_dev], Y_new[p_dev])
    # cond(K) ~ 1e10: the tolerances of the car case above
    assert relinf(g_dev.get_chol(), g_all.get_chol()) < 5e-8
    assert relinf(g_dev.get_alpha(), g_all.get_alpha()) < 1e-4


def _singular_problem():
    """Training points 100 length scales apart (K = I up to 2^-1020 terms), sf = 1, sn = 0, so a pool copy of a training
    point has Schur complement sf2 + sn2 - |L^-1 k|^2 <= 0 in floating point: the K build clamps k(x, x) at sf2 and the ks
    kernel's k(x, x) is exactly sf2.  Far-away pool points have variance 1 and are picked first (ties to the lowest
    index)."""
    N = 130
    X = np.column_stack([100.0 * np.arange(N), np.zeros(N)])
    Y = np.random.default_rng(0).standard_normal((N, 2))
    hyper = np.tile([1.0, 1.0, 1.0, 0.0], (2, 1))
    far = np.column_stack([100.0 * np.arange(3), np.full(3, 1e4)])
    return X, Y, hyper, far


def _greedy_raw(eng, Xc, Yc, n_new):
    lib = L.load()
    Xc = np.ascontiguousarray(Xc, dtype=np.float64); Yc = np.ascontiguousarray(Yc, dtype=np.float64)
    picked = np.full(n_new, -1, dtype=np.int32); score = np.zeros(n_new); added = C.c_int(-7)
    rc = lib.gpmpc_append_greedy(eng.h, Xc.shape[0], Xc.ctypes.data_as(C.POINTER(C.c_double)),
                                 Yc.ctypes.data_as(C.POINTER(C.c_double)), n_new, picked.ctypes.data_as(C.POINTER(C.c_int)),
                                 score.ctypes.data_as(C.POINTER(C.c_double)), C.byref(added))
    return rc, added.value, picked, score


@pytest.mark.parametrize('where', ['last', 'earlier', 'only'])
def test_a_failed_pivot_is_reported_at_any_pick(where):
    X, Y, hyper, far = _singular_problem()
    N = X.shape[0]
    Xc = {'last': [far[0], far[1], X[5]], 'earlier': [X[5], far[0], X[7], far[1]], 'only': [X[5]]}[where]
    Xc = np.array(Xc)
    n_new = Xc.shape[0]
    Yc = np.zeros((n_new, 2))
    eng = fit(X, Y, hyper, capacity=N + n_new)
    rc, added, picked, score = _greedy_raw(eng, Xc, Yc, n_new)
    assert rc == L.ERR_NOTPD
    assert 'positive definiteness' in L.load().gpmpc_last_error(eng.h).decode()
    expect = {'last': ([0, 1, 2], 3), 'earlier': ([1, 3], 3), 'only': ([0], 1)}[where]
    assert added == expect[1]
    np.testing.assert_array_equal(picked[:len(expect[0])], expect[0])
    assert np.all(picked[added:] == -1)                   # nothing reported past the failing pick
    assert score[added - 1] <= 0.0                        # the copy's variance: no room left for it
    with pytest.raises(L.GpmpcError) as e:                # the factor is stale until the next factorisation
        eng.predict(X[:2], None, L.METHOD_ME)
    assert e.value.code == L.ERR_STATE


def test_gp_recovers_from_failed_pivots_by_refactorising():
    import gp_mpc_b200
    X, Y, hyper, far = _singular_problem()
    gp = gp_mpc_b200.GP(X, Y, hyper=dict(hyper=hyper), normalize=False)
    Xc = np.array([X[5], far[0], X[7], far[1]])
    Yc = np.random.default_rng(1).standard_normal((4, 2))
    picked = gp.append_greedy(Xc, Yc, 4)
    # far[0], far[1], then the copies: each copy's pivot fails and the GP refits (with the jitter retry) before going on
    assert picked[:2].tolist() == [1, 3] and sorted(picked[2:].tolist()) == [0, 2]
    assert gp.get_size()[0] == X.shape[0] + 4 and gp.engine.N == X.shape[0] + 4
    Xa = np.vstack([X, Xc[picked]])
    m, v, _, _ = gp.engine.predict(Xa[-6:], None, L.METHOD_ME)
    assert np.all(np.isfinite(m)) and np.all(np.isfinite(v))
    Ya = np.vstack([Y, Yc[picked]])
    # the far points are isolated training points: mean = y / (1 + sn2 + jitter), jitter <= 1e-8
    np.testing.assert_allclose(m[[2, 3]], Ya[-4:-2], rtol=1e-6, atol=1e-7)
