"""Removal of training points (GP.remove_data, GP.append_data(max_points=...)) on CPU: the numpy form of the O(N^2)
update against a LAPACK refit of the remaining data, its drift over a long sliding window, and the GP class's
bookkeeping through an oracle-backed engine that removes with that form."""
import numpy as np
import pytest
from scipy.linalg import solve_triangular

import gp_mpc_b200
from oracle import gp_oracle as orc
from oracle import remove_oracle as rmo
from tests._fake_engine import OracleEngine, problem
from tests._util import load_fixture, relinf


def _factors(X, hyper_a):
    L = np.linalg.cholesky(orc.assemble_K(X, hyper_a))
    return L, _inv(L)


def _inv(L):
    return solve_triangular(L, np.eye(L.shape[0]), lower=True)


# (chol, L^-1, alpha).  L^-1 and alpha of two factorisations of the same K differ by about cond(K) eps, even where the
# removal is exact (the last point): cond(K) ~ 6e7 for tank, ~ 7e10 for car, ~ 2e6 for the synthetic problem
TOL = {'tank': (1e-11, 5e-9, 1e-8), 'car': (1e-9, 5e-6, 1e-5), 'synthetic': (1e-11, 1e-9, 1e-9)}


@pytest.mark.parametrize('case', ['tank', 'car', 'synthetic'])
@pytest.mark.parametrize('where', ['first', 'middle', 'last', 'several'])
def test_oracle_form_matches_a_refit(case, where):
    X, Y, hyper = problem(case)
    N = X.shape[0]
    idx = {'first': [0], 'middle': [N // 2], 'last': [N - 1], 'several': [N // 3, 0, N - 1, 7, N // 2]}[where]
    keep = np.setdiff1d(np.arange(N), idx)
    post = orc.postfit(X[keep], Y[keep], hyper, lapack_general_solve=False)
    tol_chol, tol_li, tol_alpha = TOL[case]
    for a in range(Y.shape[1]):
        L, Li = _factors(X, hyper[a])
        logdet = 2 * np.sum(np.log(np.diag(L)))
        L2, Li2 = rmo.remove(L, Li, idx)
        assert np.all(np.triu(L2, 1) == 0) and np.all(np.triu(Li2, 1) == 0)
        assert relinf(L2, post['chol'][a]) < tol_chol
        assert relinf(Li2, _inv(post['chol'][a])) < tol_li
        assert relinf(rmo.alpha(Li2, Y[keep, a]), post['alpha'][a]) < tol_alpha
        if len(idx) == 1:                  # logdet' = logdet - 2 log lambda + log t_{n-1}
            i = idx[0]
            p, _, _ = rmo.coefficients(L, Li, i)
            pred = logdet - 2 * np.log(L[i, i]) + np.log1p(np.sum(p * p))
            assert abs(pred - 2 * np.sum(np.log(np.diag(L2)))) <= 1e-12 * max(1.0, abs(pred))


def test_a_long_sliding_window_does_not_drift():
    """500 cycles of remove(0) + append(next stream point) against a refit of the final window."""
    Nw, Nx, cycles = 200, 4, 500
    p = orc.synthetic_problem(Nw + cycles, Nx, 1, config_id=5)
    X, Y, hyper = p['X'], p['Y'], p['hyper'][0]
    sf2, sn2 = hyper[Nx] ** 2, hyper[Nx + 1] ** 2
    L, Li = _factors(X[:Nw], hyper)
    for c in range(cycles):
        L, Li = rmo.remove_point(L, Li, 0)
        win = X[c + 1:c + Nw]
        k = orc.covSEard(win, X[c + Nw:c + Nw + 1], hyper[:Nx], sf2)[:, 0]
        L, Li = rmo.append_point(L, Li, k, sf2 + sn2)
    win = slice(cycles, cycles + Nw)
    post = orc.postfit(X[win], Y[win], hyper[None], lapack_general_solve=False)
    assert relinf(L, post['chol'][0]) < 1e-10
    assert relinf(Li, _inv(post['chol'][0])) < 1e-9
    assert relinf(rmo.alpha(Li, Y[win, 0]), post['alpha'][0]) < 1e-7


class RemoveEngine(OracleEngine):
    """The oracle-backed engine stand-in with `remove` done by the numpy form of gpmpc_remove; records its calls."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.calls = []

    def append(self, x_new, y_new):
        self.calls.append(('append', self.N))
        return super().append(x_new, y_new)

    def remove(self, idx):
        idx = [int(k) for k in np.asarray(idx).reshape(-1)]
        self.calls.append(('remove', idx))
        keep = np.setdiff1d(np.arange(self.N), idx)
        chol, alpha, invK = [], [], []
        for k, a in enumerate(self.local_outputs):
            L = self.post['chol'][k]
            L2, Li2 = rmo.remove(L, _inv(L), idx)
            chol.append(L2); alpha.append(rmo.alpha(Li2, self.Y[keep, a])); invK.append(Li2.T @ Li2)
        self.post = dict(self.post, chol=np.array(chol), alpha=np.array(alpha), invK=np.array(invK))
        self.X, self.Y = self.X[keep], self.Y[keep]
        self.N = len(keep)


def _gp(X, Y, hyper, normalize, meta=None, factory=RemoveEngine):
    kw = dict(meta=meta) if meta is not None else {}
    return gp_mpc_b200.GP(X, Y, mean_func='zero', gp_method='TA', normalize=normalize, hyper=dict(hyper=hyper),
                          engine_factory=factory, **kw)


def _data(normalize):
    if normalize:                       # the tank fixture is stored standardised, with its meta
        m = load_fixture('tank')
        return m['X'], m['Y'], m['hyper'], m['meta']
    p = orc.synthetic_problem(150, 4, 2, config_id=23)
    return p['X'], p['Y'], p['hyper'], None


def _same_predictions(g1, g2, X):
    Ny = g1.get_size()[1]
    rng = np.random.default_rng(3)
    Z = X[rng.integers(0, X.shape[0], 6)] + 0.05 * rng.standard_normal((6, X.shape[1]))
    if g1._GP__normalize:               # predict_batch takes caller units
        meta = g1._GP__meanZ, g1._GP__stdZ
        Z = Z * meta[1] + meta[0]
    m1, c1 = g1.predict_batch(Z[:, :Ny], Z[:, Ny:])
    m2, c2 = g2.predict_batch(Z[:, :Ny], Z[:, Ny:])
    # the variances are small differences sf2 - k^T K^-1 k: relative to themselves they keep cond(K) eps
    assert relinf(m1, m2) < 1e-9 and relinf(c1, c2) < 1e-7


@pytest.mark.parametrize('normalize', [True, False])
def test_remove_data_matches_a_gp_fitted_on_the_rest(normalize):
    X, Y, hyper, meta = _data(normalize)
    N = X.shape[0]
    gp = _gp(X, Y, hyper, normalize, meta)
    eng = gp.engine
    idx = [N - 1, 3, N // 2, 0]
    gp.remove_data(idx)
    keep = np.setdiff1d(np.arange(N), idx)
    assert gp.engine is eng and eng.calls == [('remove', idx)]
    assert gp.get_size()[0] == N - 4 and eng.N == N - 4
    np.testing.assert_array_equal(gp._GP__X, X[keep])
    np.testing.assert_array_equal(gp._GP__Y, Y[keep])
    ref = _gp(X[keep], Y[keep], hyper, normalize, meta)
    assert relinf(gp.get_chol(), ref.get_chol()) < 1e-11
    assert relinf(gp.get_alpha(), ref.get_alpha()) < 1e-9
    assert relinf(gp.get_invK(), ref.get_invK()) < 1e-9
    _same_predictions(gp, ref, X)
    gp.remove_data([])                                    # no-op: the engine is not called
    assert eng.calls == [('remove', idx)] and gp.get_size()[0] == N - 4


@pytest.mark.parametrize('normalize', [True, False])
def test_append_data_keeps_a_sliding_window(normalize):
    X, Y, hyper, meta = _data(normalize)
    N = X.shape[0]
    rng = np.random.default_rng(9)
    Xs = X[rng.integers(0, N, 7)] + 0.3 * rng.standard_normal((7, X.shape[1]))
    Ys = rng.standard_normal((7, Y.shape[1]))
    X_new, Y_new = Xs, Ys
    if normalize:                       # append_data takes caller units
        X_new, Y_new = Xs * meta['stdZ'] + meta['meanZ'], Ys * meta['stdY'] + meta['meanY']
    gp = _gp(X, Y, hyper, normalize, meta)
    eng = gp.engine
    gp.append_data(X_new, Y_new, max_points=N - 2)
    # the first point makes room for three (N + 1 <= N - 2), the others for one each
    assert eng.calls == [('remove', [0, 1, 2]), ('append', N - 3)] + [('remove', [0]), ('append', N - 3)] * 6
    assert gp.engine is eng and gp.get_size()[0] == N - 2
    Xw, Yw = np.vstack([X, Xs])[-(N - 2):], np.vstack([Y, Ys])[-(N - 2):]
    np.testing.assert_allclose(gp._GP__X, Xw, rtol=0, atol=1e-12)
    ref = _gp(Xw, Yw, hyper, normalize, meta)
    assert relinf(gp.get_chol(), ref.get_chol()) < 1e-10
    assert relinf(gp.get_alpha(), ref.get_alpha()) < 1e-8
    _same_predictions(gp, ref, X)


def test_append_data_without_max_points_only_grows():
    X, Y, hyper, _ = _data(False)
    N = X.shape[0]
    gp = _gp(X, Y, hyper, False)
    gp.append_data(X[:3] + 0.1, Y[:3])
    assert gp.engine.calls == [('append', N), ('append', N + 1), ('append', N + 2)]
    assert gp.get_size()[0] == N + 3


def test_the_refit_fallback_keeps_the_window(monkeypatch):
    X, Y, hyper, _ = _data(False)
    N = X.shape[0]
    gp = _gp(X, Y, hyper, False)
    eng = gp.engine
    # the second append (at N - 1 points after its removal) loses positive definiteness
    monkeypatch.setattr(OracleEngine, 'fail_on', (0, N - 1))
    Xn, Yn = X[:4] + 0.2, Y[:4] + 1.0
    gp.append_data(Xn, Yn, max_points=N)
    assert eng.calls == [('remove', [0]), ('append', N - 1)]
    assert gp.engine is not eng                           # refitted on a new engine
    Xw, Yw = np.vstack([X[1:], Xn])[-N:], np.vstack([Y[1:], Yn])[-N:]
    np.testing.assert_array_equal(gp._GP__X, Xw)
    assert gp.get_size()[0] == N and gp.engine.N == N
    ref = _gp(Xw, Yw, hyper, False)
    assert relinf(gp.get_chol(), ref.get_chol()) < 1e-12


def test_bad_indices_raise_before_the_engine_is_touched():
    X, Y, hyper, _ = _data(False)
    N = X.shape[0]
    gp = _gp(X, Y, hyper, False)
    eng = gp.engine
    for bad in ([0.0], [1.5], [3, 3], [-1], [N], np.arange(N), [True]):
        with pytest.raises(ValueError):
            gp.remove_data(bad)
    with pytest.raises(ValueError):
        gp.append_data(X[:1], Y[:1], max_points=1)
    assert eng.calls == [] and gp.get_size()[0] == N
    gp.remove_data(np.array([2, 1], dtype=np.int32))      # any integer dtype
    assert eng.calls == [('remove', [2, 1])]
