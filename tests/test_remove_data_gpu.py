"""gpmpc_remove / Engine.remove / GP.remove_data / GP.append_data(max_points=...) on the GPU: the model after removals
against a LAPACK refit of the remaining data, every entry point against a fresh handle fitted on that data, a sliding
window at a full padded size, reuse of the freed capacity, determinism, and the argument and state checks."""
import ctypes as C

import numpy as np
import pytest

from gp_mpc_b200 import _lib as L
from oracle import gp_oracle as orc
from oracle import greedy_oracle as gro
from tests._engines import fit, problem
from tests._util import relinf

pytestmark = pytest.mark.gpu


def _indices(where, N):
    return {'first': [0], 'last': [N - 1], '127': [127], '128': [128], 'middle': [N // 2 + 3],
            'several': [N // 3, 0, N - 1, N // 2, 5]}[where]


def _points(X, n, seed):
    rng = np.random.default_rng(seed)
    return X[rng.integers(0, X.shape[0], n)] + 0.1 * rng.standard_normal((n, X.shape[1]))


def _preds_vs(eng, X, Y, hyper, Z, Sigma, post=None):
    """TA and ME predictions against the oracle on (X, Y) (the pattern of test_append_greedy_gpu)."""
    post = post or orc.postfit(X, Y, hyper, lapack_general_solve=False)
    mo, vo = orc.gp_mean_var(X, hyper, post['alpha'], post['chol'], Z)
    Jo = orc.gp_mean_jac(X, hyper, post['alpha'], Z)
    m, v, c, J = eng.predict(Z, Sigma, L.METHOD_TA)
    assert relinf(m, mo) < 1e-6 and relinf(v, vo) < 1e-6 and relinf(J, Jo) < 1e-6
    assert relinf(c, orc.ta_cov(vo, Jo, Sigma)) < 1e-6
    m, v, c, _ = eng.predict(Z, None, L.METHOD_ME)
    assert relinf(m, mo) < 1e-6 and relinf(v, vo) < 1e-6 and relinf(c, orc.me_cov(vo)) < 1e-6
    return post


CASES = [('tank', w) for w in ('first', 'middle', 'last', 'several')] + \
        [('car', w) for w in ('first', '127', '128', 'middle', 'last', 'several')] + \
        [((1000, 8, 6), w) for w in ('first', '127', '128', 'middle', 'last', 'several')] + \
        [((4096, 4, 2), w) for w in ('first', '128', 'middle', 'last')]


@pytest.mark.parametrize('case,where', CASES, ids=['%s-%s' % c for c in CASES])
def test_removal_matches_a_refit(case, where):
    X, Y, hyper = problem(case)
    N = X.shape[0]
    idx = _indices(where, N)
    eng = fit(X, Y, hyper)
    cap = eng.capacity
    eng.remove(idx)
    assert eng.N == N - len(idx) and eng.capacity == cap
    keep = np.setdiff1d(np.arange(N), idx)
    Xk, Yk = X[keep], Y[keep]
    Z = _points(Xk, 5, 1)
    Sigma = 1e-4 * np.eye(X.shape[1])
    post = _preds_vs(eng, Xk, Yk, hyper, Z, Sigma)
    # car: cond(K) ~ 1e10 (its plain factorisation is held to 2e-9 / 1e-4 in test_gpu_parity), as for appends
    tol_chol, tol_alpha, tol_ld = (5e-8, 1e-4, 1e-6) if case == 'car' else (1e-10, 1e-7, 1e-9)
    for a in range(Y.shape[1]):
        assert relinf(eng.get(L.GET_CHOL, a), post['chol'][a]) < tol_chol
        assert relinf(eng.get(L.GET_ALPHA, a), post['alpha'][a]) < tol_alpha
        ld = 2 * np.sum(np.log(np.diag(post['chol'][a])))
        assert abs(eng.get(L.GET_LOGDET, a)[0] - ld) <= tol_ld * max(1.0, abs(ld))


@pytest.mark.parametrize('N', [129, 257])
def test_removal_across_a_padding_boundary(N):
    """129 -> 128 and 257 -> 256 points: the last 128-block becomes all identity tail (the padded size stays)."""
    X, Y, hyper = problem((N, 3, 2))
    eng = fit(X, Y, hyper)
    eng.remove([N // 2])
    assert eng.N == N - 1 and eng.capacity == -(-N // 128) * 128
    keep = np.setdiff1d(np.arange(N), [N // 2])
    post = _preds_vs(eng, X[keep], Y[keep], hyper, _points(X, 6, 2), 1e-4 * np.eye(3))
    for a in range(2):
        assert relinf(eng.get(L.GET_CHOL, a), post['chol'][a]) < 1e-10


def test_a_sharded_handle_updates_the_outputs_it_owns():
    X, Y, hyper = problem((700, 5, 4))
    eng = fit(X, Y, hyper, out_begin=1, out_count=2)
    eng.remove([600, 3, 128])
    keep = np.setdiff1d(np.arange(700), [600, 3, 128])
    post = orc.postfit(X[keep], Y[keep], hyper, lapack_general_solve=False)
    for a in (1, 2):
        assert relinf(eng.get(L.GET_CHOL, a), post['chol'][a]) < 1e-10
        assert relinf(eng.get(L.GET_ALPHA, a), post['alpha'][a]) < 1e-7


def test_every_entry_point_matches_a_fresh_handle():
    """Tolerances of test_reserved_capacity_matches_an_unreserved_handle: after removals the zero upper triangles of the
    diagonal blocks and the identity tail feed the stream-K product like a fresh factorisation's."""
    p = orc.synthetic_problem(700, 4, 2, config_id=31, H=6)
    X, Y, hyper, Z, Sigma = p['X'], p['Y'], p['hyper'], p['Z'], p['Sigma']
    idx = [699, 128, 0, 127, 350, 256]
    keep = np.setdiff1d(np.arange(700), idx)
    eng = fit(X, Y, hyper)
    # the derivative caches (Li^T, EM K^-1) are built before the removal and must not survive it
    eng.predict_grad(Z, Sigma, L.METHOD_TA)
    eng.predict_em_grad(Z[:2], Sigma)
    eng.remove(idx)
    fresh = fit(X[keep], Y[keep], hyper)
    assert eng.capacity == fresh.capacity
    for a in range(2):
        assert relinf(eng.get(L.GET_CHOL, a), fresh.get(L.GET_CHOL, a)) < 1e-11
        assert relinf(eng.get(L.GET_ALPHA, a), fresh.get(L.GET_ALPHA, a)) < 1e-8
        assert relinf(eng.get(L.GET_LOGDET, a), fresh.get(L.GET_LOGDET, a)) < 1e-11
    for meth in (L.METHOD_TA, L.METHOD_ME):
        for k, (u, v) in enumerate(zip(eng.predict(Z, Sigma, meth), fresh.predict(Z, Sigma, meth))):
            assert relinf(u, v) < 1e-8, (meth, k)
    e1, e2 = (e.predict(Z[:2], Sigma, L.METHOD_EM, want_jac=False) for e in (eng, fresh))
    assert relinf(e1[0], e2[0]) < 1e-8 and relinf(e1[2], e2[2]) < 1e-6
    g1, g2 = eng.predict_grad(Z, Sigma, L.METHOD_TA), fresh.predict_grad(Z, Sigma, L.METHOD_TA)
    for k in ('mean', 'var', 'jac', 'dvar_dz', 'dcov_dz'):
        assert relinf(g1[k], g2[k]) < 1e-8, k
    h1, h2 = eng.predict_hess(Z, Sigma, L.METHOD_TA), fresh.predict_hess(Z, Sigma, L.METHOD_TA)
    for k in ('hess', 'd2var_dz2', 'd3mean_dz3', 'd2cov_dz2'):
        assert relinf(h1[k], h2[k]) < 1e-8, k
    d1, d2 = eng.predict_em_grad(Z[:2], Sigma), fresh.predict_em_grad(Z[:2], Sigma)
    assert relinf(d1['dmean_dz'], d2['dmean_dz']) < 1e-6 and relinf(d1['dcov_dSigma'], d2['dcov_dSigma']) < 1e-6
    assert relinf(eng.posterior_cov(Z), fresh.posterior_cov(Z)) < 1e-8
    z0 = Z[:3]; U = 0.1 * np.random.default_rng(4).standard_normal((3, 5, 2)); S = np.stack([Sigma] * 3)
    for u, v in zip(eng.rollout_batch(z0, U, S, L.METHOD_TA), fresh.rollout_batch(z0, U, S, L.METHOD_TA)):
        assert relinf(u, v) < 1e-8
    f1, gr1 = eng.nlml(1, hyper[1])
    f2, gr2 = fresh.nlml(1, hyper[1])
    assert abs(f1 - f2) <= 1e-9 * abs(f2) and relinf(gr1, gr2) < 1e-8


def test_a_sliding_window_at_a_full_padded_size():
    """N = 4096 leaves no spare row: 256 cycles of remove(0) + append, then a refit of the final window."""
    Nw, cycles = 4096, 256
    p = orc.synthetic_problem(Nw + cycles, 4, 2, config_id=41)
    X, Y, hyper = p['X'], p['Y'], p['hyper']
    eng = fit(X[:Nw], Y[:Nw], hyper)
    assert eng.capacity == Nw
    for c in range(cycles):
        eng.remove([0])
        assert eng.append(X[Nw + c], Y[Nw + c]), c
    assert eng.N == Nw and eng.capacity == Nw
    Xw, Yw = X[cycles:], Y[cycles:]
    post = _preds_vs(eng, Xw, Yw, hyper, _points(Xw, 6, 3), 1e-4 * np.eye(4))
    for a in range(2):
        assert relinf(eng.get(L.GET_CHOL, a), post['chol'][a]) < 1e-9
        assert relinf(eng.get(L.GET_ALPHA, a), post['alpha'][a]) < 1e-7


def test_freed_capacity_takes_appends_and_greedy_appends():
    X, Y, hyper = problem((256, 3, 2))
    eng = fit(X, Y, hyper)
    assert eng.capacity == 256
    eng.remove([10, 200, 0, 130, 64, 255])
    Xn = _points(X, 3, 5); Yn = np.random.default_rng(6).standard_normal((3, 2))
    for k in range(3):
        assert eng.append(Xn[k], Yn[k])
    Xc = _points(X, 40, 7); Yc = np.random.default_rng(8).standard_normal((40, 2))
    keep = np.setdiff1d(np.arange(256), [10, 200, 0, 130, 64, 255])
    Xa, Ya = np.vstack([X[keep], Xn]), np.vstack([Y[keep], Yn])
    ref = gro.greedy_select(Xa, hyper, Xc, 3)
    picked, _, ok = eng.append_greedy(Xc, Yc, 3)
    assert ok and eng.N == 256
    np.testing.assert_array_equal(picked, ref['picked'])
    Xa, Ya = np.vstack([Xa, Xc[picked]]), np.vstack([Ya, Yc[picked]])
    post = _preds_vs(eng, Xa, Ya, hyper, _points(Xa, 5, 9), 1e-4 * np.eye(3))
    for a in range(2):
        assert relinf(eng.get(L.GET_CHOL, a), post['chol'][a]) < 1e-10
        assert relinf(eng.get(L.GET_ALPHA, a), post['alpha'][a]) < 1e-7
    assert not eng.append(Xn[0], Yn[0])                   # full again: gpmpc_append reports the capacity


def test_two_handles_give_identical_bits():
    X, Y, hyper = problem((1000, 8, 6))
    Z = _points(X, 7, 2)
    Xn = _points(X, 4, 3); Yn = np.random.default_rng(4).standard_normal((4, 6))
    out = []
    for _ in range(2):
        eng = fit(X, Y, hyper)
        eng.remove([999, 0, 513, 128])
        for k in range(4):
            assert eng.append(Xn[k], Yn[k])
        eng.remove([17, 640])
        res = [eng.get(w, a) for w in (L.GET_CHOL, L.GET_LINV, L.GET_ALPHA) for a in range(6)]
        res += list(eng.predict(Z, 1e-4 * np.eye(8), L.METHOD_TA))
        out.append(res)
        eng.close()
    for u, v in zip(*out):
        assert u.tobytes() == v.tobytes()


def test_state_and_argument_errors_leave_the_model_untouched():
    X, Y, hyper = problem((300, 3, 2))
    lib = L.load()
    Z = _points(X, 4, 1)
    eng = fit(X, Y, hyper)
    before = eng.predict(Z, 1e-4 * np.eye(3), L.METHOD_TA)

    def call(idx, n=None, null=False):
        a = np.ascontiguousarray(idx, dtype=np.int32)
        return lib.gpmpc_remove(eng.h, len(a) if n is None else n, None if null else a.ctypes.data_as(C.POINTER(C.c_int)))

    assert call([3], null=True) == L.ERR_ARG
    assert call([3], n=-1) == L.ERR_ARG
    for bad in ([-1], [300], [5, 7, 5], list(range(300))):
        assert call(bad) == L.ERR_ARG, bad
    assert 'leaves none' in lib.gpmpc_last_error(eng.h).decode()
    assert call([], null=True) == L.OK                    # n = 0: no-op
    assert call([4, 9], n=0) == L.OK
    with pytest.raises(L.GpmpcError) as e:
        eng.remove([2, 2])
    assert e.value.code == L.ERR_ARG and eng.N == 300
    after = eng.predict(Z, 1e-4 * np.eye(3), L.METHOD_TA)
    for u, v in zip(before, after):
        assert u.tobytes() == v.tobytes()
    fresh = L.Engine(300, 3, 2, device=0)
    fresh.set_data(X, Y)
    fresh.set_hyper(hyper)
    with pytest.raises(L.GpmpcError) as e:               # not factorised
        fresh.remove([0])
    assert e.value.code == L.ERR_STATE and 'factorize' in lib.gpmpc_last_error(fresh.h).decode()


def test_gp_keeps_a_window_at_a_full_padded_size(monkeypatch):
    import gp_mpc_b200
    p = orc.synthetic_problem(4096 + 16, 4, 2, config_id=13)
    X, Y, hyper = p['X'], p['Y'], p['hyper']
    gp = gp_mpc_b200.GP(X[:4096], Y[:4096], hyper=dict(hyper=hyper), normalize=False)
    eng = gp.engine
    assert eng.capacity == 4096
    calls = []
    Eng = gp_mpc_b200._lib.Engine
    real_rm, real_ap = Eng.remove, Eng.append
    monkeypatch.setattr(Eng, 'remove', lambda self, idx: calls.append(('remove', list(idx))) or real_rm(self, idx))
    monkeypatch.setattr(Eng, 'append', lambda self, x, y: calls.append(('append',)) or real_ap(self, x, y))
    gp.append_data(X[4096:], Y[4096:], max_points=4096)
    assert calls == [('remove', [0]), ('append',)] * 16
    assert gp.engine is eng and eng.capacity == 4096 and eng.N == 4096 and gp.get_size()[0] == 4096
    ref = gp_mpc_b200.GP(X[16:], Y[16:], hyper=dict(hyper=hyper), normalize=False)
    Zs = _points(X[16:], 8, 4)
    m1, c1 = gp.predict_batch(Zs[:, :2], Zs[:, 2:])
    m2, c2 = ref.predict_batch(Zs[:, :2], Zs[:, 2:])
    assert relinf(m1, m2) < 1e-6 and relinf(c1, c2) < 1e-6
