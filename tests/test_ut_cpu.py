"""The unscented transform ('UT') without a GPU: the oracle's square root, weights and rule (tests/test_ut_gpu.py checks
the engine against it), its accuracy against Gauss-Hermite quadrature of the 'ME' mean, and the GP bookkeeping through an
oracle-backed stand-in engine."""
import numpy as np
import pytest

import gp_mpc_b200
from oracle import gp_oracle as orc
from oracle import ut_oracle as uto
from tests._fake_engine import OracleEngineWithRolloutBatch, TwoRanks, fixture_gp, sharded
from tests._util import load_fixture, relinf, trajectories

PARAMS = [(1.0, 0.0, 0.0), (0.5, 2.0, 1.0), (1e-3, 2.0, 0.0), (1.0, 0.0, -2.0), (2.0, 0.5, 3.0)]


def _spd(rng, n, H=None):
    A = rng.standard_normal(((H,) if H else ()) + (n, n))
    return A @ np.swapaxes(A, -1, -2) + 0.1 * np.eye(n)


def _feedback_cov(rng, Ny, Nu):
    """[C, C K^T; K C, K C K^T]: the rank-Ny input covariance of a feedback roll-out."""
    C = _spd(rng, Ny)
    K = rng.standard_normal((Nu, Ny))
    return np.block([[C, C @ K.T], [K @ C, K @ C @ K.T]])


@pytest.mark.parametrize('n', [1, 2, 6, 17, 32])
def test_square_root_of_a_full_rank_sigma(n):
    rng = np.random.default_rng(n)
    S = _spd(rng, n, 4)
    L = uto.sqrt_psd(S)
    assert np.array_equal(L, np.tril(L))
    assert np.abs(L @ np.swapaxes(L, 1, 2) - S).max() / np.abs(S).max() < 1e-15
    assert (np.diagonal(L, axis1=1, axis2=2) > 0).all()


@pytest.mark.parametrize('Ny,Nu', [(4, 2), (3, 2), (1, 5)])
def test_square_root_zero_columns_where_the_rank_drops(Ny, Nu):
    rng = np.random.default_rng(Ny * 10 + Nu)
    n = Ny + Nu
    open_loop = np.zeros((n, n)); open_loop[:Ny, :Ny] = _spd(rng, Ny)
    for S in (open_loop, _feedback_cov(rng, Ny, Nu)):
        L = uto.sqrt_psd(S)
        assert (L[:, Ny:] == 0).all()                       # exactly zero, not small
        assert (np.diag(L)[:Ny] > 0).all()
        assert np.abs(L @ L.T - S).max() / np.abs(S).max() < 1e-15
    assert (uto.sqrt_psd(np.zeros((n, n))) == 0).all()


@pytest.mark.parametrize('params', PARAMS)
@pytest.mark.parametrize('n', [1, 6, 32])
def test_weights_sum_to_one(n, params):
    if n + params[2] <= 0:                                  # kappa <= -n: no rule (the engine rejects it)
        return
    c, wm, wc = uto.weights(n, params)
    assert wm.size == wc.size == 2 * n + 1
    assert abs(np.sum(wm) - 1.0) < 1e-15 * max(1.0, np.abs(wm).sum())
    assert np.array_equal(wm[1:], wc[1:])
    alpha, beta, kappa = params
    assert c == pytest.approx(np.sqrt(alpha ** 2 * (n + kappa)), rel=1e-9)     # n + lambda cancels at small alpha
    assert wc[0] - wm[0] == pytest.approx(1 - alpha ** 2 + beta, abs=1e-12 * max(1.0, abs(wm[0])))
    if params == (1.0, 0.0, 0.0):                           # the symmetric cubature rule
        assert wm[0] == wc[0] == 0.0 and c == np.sqrt(n) and (wm >= 0).all()


def _identity(P):
    return P, np.zeros_like(P)


@pytest.mark.parametrize('params', PARAMS[:2] + PARAMS[3:])
def test_first_two_moments_of_a_gaussian_are_exact(params):
    """f(x) = x: the rule returns z and Sigma, for a full-rank and a rank-deficient Sigma."""
    rng = np.random.default_rng(3)
    n = 6
    Z = rng.standard_normal((3, n))
    for Sigma in (_spd(rng, n, 3), np.stack([_feedback_cov(rng, 4, 2)] * 3)):
        mean, var, cov = uto.ut(_identity, Z, Sigma, params)
        scale = np.abs(Sigma).max() * max(1.0, abs(uto.weights(n, params)[2][0]))
        assert np.abs(mean - Z).max() < 1e-14 * max(1.0, np.abs(Z).max()) * max(1.0, abs(uto.weights(n, params)[1][0]))
        assert np.abs(cov - Sigma).max() < 1e-13 * scale
        assert np.array_equal(var, np.diagonal(cov, axis1=1, axis2=2))


def test_mean_of_a_cubic_polynomial_is_exact():
    rng = np.random.default_rng(5)
    n = 5
    z = rng.standard_normal(n)
    Sigma = _spd(rng, n) * 0.3
    c0, g, A, T = rng.standard_normal(), rng.standard_normal(n), rng.standard_normal((n, n)), rng.standard_normal((n, n, n))

    def f(P):
        m = c0 + P @ g + np.einsum('hi,ij,hj->h', P, A, P) + np.einsum('hi,hj,hk,ijk->h', P, P, P, T)
        return m[:, None], np.zeros((P.shape[0], 1))

    Ezz = np.outer(z, z) + Sigma
    exact = c0 + g @ z + np.sum(A * Ezz) + np.einsum('ijk,i,j,k->', T, z, z, z) \
        + np.einsum('ijk,i,jk->', T, z, Sigma) + np.einsum('ijk,j,ik->', T, z, Sigma) + np.einsum('ijk,k,ij->', T, z, Sigma)
    for params in PARAMS[:2] + PARAMS[3:]:
        mean = uto.ut(f, z[None], Sigma, params)[0][0, 0]
        assert abs(mean - exact) < 1e-12 * (1 + abs(exact)), params


def _gauss_hermite_mean(X, hyper, alpha, chol, z, Sigma, deg=7):
    """E[mean(x)] for x ~ N(z, Sigma) by the tensor Gauss-Hermite rule of deg points per dimension."""
    x, w = np.polynomial.hermite_e.hermegauss(deg)
    w = w / w.sum()
    n = z.size
    grids = np.stack(np.meshgrid(*[x] * n, indexing='ij'), -1).reshape(-1, n)
    W = np.prod(np.stack(np.meshgrid(*[w] * n, indexing='ij'), -1).reshape(-1, n), 1)
    P = z + grids @ np.linalg.cholesky(Sigma).T
    m = orc.gp_mean_var(X, hyper, alpha, chol, P)[0]
    return W @ m


def test_ut_mean_of_the_me_mean_converges_as_sigma_to_the_fourth():
    """On the tank fixture the 'UT' mean's error against quadrature of the same 'ME' mean falls by about 16x per halving
    of the input standard deviation (O(sigma^4)); 'TA''s mean (the 'ME' mean at z) falls by about 4x (O(sigma^2))."""
    m = load_fixture('tank')
    X, hyper = m['X'], m['hyper']
    post = orc.postfit(X, m['Y'], hyper)
    z = np.array([0.3, -0.2, 0.1, 0.4, -0.5, 0.2])
    base = np.diag(hyper[0, :6] ** 2) * 0.003
    ut_err, ta_err = [], []
    for s in (1.0, 0.5, 0.25):
        Sigma = base * s * s
        gh = _gauss_hermite_mean(X, hyper, post['alpha'], post['chol'], z, Sigma)
        ut_mean = uto.ut_me(X, hyper, post['alpha'], post['chol'], z[None], Sigma)[0][0]
        ta_mean = orc.gp_mean_var(X, hyper, post['alpha'], post['chol'], z[None])[0][0]
        ut_err.append(np.abs(ut_mean - gh).max()); ta_err.append(np.abs(ta_mean - gh).max())
    for k in range(2):
        assert 14 < ut_err[k] / ut_err[k + 1] < 18, ut_err
        assert 3.7 < ta_err[k] / ta_err[k + 1] < 4.3, ta_err
    assert ut_err[0] < 0.1 * ta_err[0]


# ------------------------------------------------------------------ the GP bookkeeping
class UtEngine(OracleEngineWithRolloutBatch):
    """The stand-in engine with METHOD_UT through the oracle and set_ut_params; records the methods it was asked for and
    its roll-out calls."""
    log = None

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.ut = uto.DEFAULT_PARAMS

    def set_ut_params(self, alpha=1.0, beta=0.0, kappa=0.0):
        if not (alpha > 0 and kappa > -self.Nx):
            raise gp_mpc_b200._lib.GpmpcError(-1, 'bad UT parameters')
        self.ut = (alpha, beta, kappa)
        type(self).log.append(('set_ut_params', self.ut))

    def predict(self, Z, Sigma=None, method=1, want_cov=True, want_jac=True):
        type(self).log.append(('predict', method))
        if method != gp_mpc_b200._lib.METHOD_UT:
            return super().predict(Z, Sigma, method, want_cov, want_jac)
        Z = np.asarray(Z).reshape(-1, self.Nx)
        mean, var, cov = uto.ut(lambda P: super(UtEngine, self).predict(P, None, 0, False, False)[:2], Z,
                                np.broadcast_to(Sigma, (Z.shape[0], self.Nx, self.Nx)), self.ut)
        jac = super().predict(Z, None, 0, False, True)[3]
        return mean, var, (cov if want_cov else None), (jac if want_jac else None)

    def rollout(self, z0, U, Sigma0, method=1, scale=None):
        type(self).log.append(('rollout', method))
        return super().rollout(z0, U, Sigma0, method, scale)

    def rollout_batch(self, z0, U, Sigma0, method=1, scale=None, K=None, x_ref=None, uscale=None):
        type(self).log.append(('rollout_batch', method))
        return super().rollout_batch(z0, U, Sigma0, method, scale, K, x_ref, uscale)


@pytest.fixture(autouse=True)
def _log():
    UtEngine.log = []
    yield UtEngine.log


def test_method_mapping_and_units(_log):
    """'UT' maps to METHOD_UT; predict standardises x, u, hands the input covariance (zeros when None) to the engine and
    de-standardises the mean; cov stays in the GP's units as for 'TA'."""
    gp, m = fixture_gp('tank', UtEngine)
    gp.set_method('UT')
    st = m['meta']
    rng = np.random.default_rng(1)
    x, u = rng.standard_normal(4) * st['stdX'] + st['meanX'], rng.standard_normal(2) * st['stdU'] + st['meanU']
    Sigma = 0.01 * _spd(rng, 6)
    mean, cov = gp.predict(x, u, Sigma)
    assert ('predict', 3) in _log
    post = orc.postfit(m['X'], m['Y'], m['hyper'], lapack_general_solve=False)
    z = np.concatenate([(x - st['meanX']) / st['stdX'], (u - st['meanU']) / st['stdU']])[None]
    om, _, oc, _ = uto.ut_me(m['X'], m['hyper'], post['alpha'], post['chol'], z, Sigma)
    assert relinf(mean[:, 0], om[0] * st['stdY'] + st['meanY']) < 1e-13 and relinf(cov, oc[0]) < 1e-13
    # no input covariance: 'UT' is 'ME', up to the oracle's BLAS, whose order depends on the batch size (the variance
    # sf2 - |v|^2 cancels: its bar is relative to sf2)
    m0, c0 = gp.predict_batch(x[None], u[None])
    me_m, me_c = gp.predict_batch(x[None], u[None], method='ME')
    assert relinf(m0, me_m) < 1e-11
    assert np.abs(c0 - me_c).max() < 1e-13 * np.max(m['hyper'][:, 6] ** 2)


def test_ut_params_are_passed_and_kept(_log):
    gp, m = fixture_gp('car', UtEngine)
    with pytest.raises(ValueError, match="'UT' only"):
        gp.set_method('TA', ut_params=(0.5, 2.0, 1.0))
    gp.set_method('UT', ut_params=(0.5, 2, 1))
    assert gp.engine.ut == (0.5, 2.0, 1.0)
    X0, U, _ = trajectories('car', 1, 1, cyclic=False)
    Sigma = 0.02 * np.eye(5)
    mean, cov = gp.predict(X0[0], U[0, 0], Sigma)
    post = orc.postfit(m['X'], m['Y'], m['hyper'], lapack_general_solve=False)
    om, _, oc, _ = uto.ut_me(m['X'], m['hyper'], post['alpha'], post['chol'],
                             np.concatenate([X0[0], U[0, 0]])[None], Sigma, (0.5, 2.0, 1.0))
    assert relinf(mean[:, 0], om[0]) < 1e-13 and relinf(cov, oc[0]) < 1e-13
    gp.set_method('TA'); gp.set_method('UT')                # kept across method switches
    assert gp.engine.ut == (0.5, 2.0, 1.0)
    gp.update_data_all(m['X'][:3] + 0.01, m['Y'][:3])       # and across a new engine
    assert gp.engine.ut == (0.5, 2.0, 1.0)
    with pytest.raises(gp_mpc_b200._lib.GpmpcError):
        gp.set_method('UT', ut_params=(0.0, 0.0, 0.0))
    assert gp.engine.ut == (0.5, 2.0, 1.0)


def test_unsupported_cases_raise(_log):
    fm = load_fixture('tank')
    sh = gp_mpc_b200.GP(fm['X'], fm['Y'], normalize=False, hyper=dict(hyper=fm['hyper']), comm=TwoRanks(),
                        engine_factory=sharded(UtEngine))
    with pytest.raises(NotImplementedError, match="'UT' needs all outputs on one GPU"):
        sh.set_method('UT')
    with pytest.raises(NotImplementedError, match="'UT' needs all outputs on one GPU"):
        sh.predict_batch(np.zeros((1, 4)), np.zeros((1, 2)), method='UT')
    pm = gp_mpc_b200.GP(fm['X'], fm['Y'], normalize=False, mean_func='const', prior_mean_in_predict=True,
                        hyper=dict(hyper=np.column_stack([fm['hyper'], np.full(4, 0.1)])), engine_factory=UtEngine)
    with pytest.raises(NotImplementedError, match='prior_mean_in_predict'):
        pm.set_method('UT')
    with pytest.raises(NotImplementedError, match='prior_mean_in_predict'):
        pm.predict_batch(np.zeros((1, 4)), np.zeros((1, 2)), method='UT')
    gp, _ = fixture_gp('tank', UtEngine)
    X0, U, _ = trajectories('tank', 1, 3, cyclic=False)
    with pytest.raises(NotImplementedError):
        gp.predict_batch_grad(X0, U[:, 0], method='UT')
    with pytest.raises(NotImplementedError):
        gp.predict_batch_hess(X0, U[:, 0], method='UT')
    with pytest.raises(NotImplementedError):
        gp.rollout_grad(X0[0], U[0], method='UT')
    gp.set_method('UT')
    with pytest.raises(NotImplementedError):              # the GP's method is the default of the derivative entries
        gp.predict_batch_grad(X0, U[:, 0])
    with pytest.raises(NotImplementedError):
        gp.rollout_grad(X0[0], U[0])
    assert ('predict', 3) not in _log


def test_rollout_routes_ut_to_the_device_entries(_log):
    """rollout(methods=[..., 'UT']) runs gpmpc_rollout for one open-loop trajectory and gpmpc_rollout_batch otherwise, with
    METHOD_UT, and equals the host loop of predict(UT) calls; device_rollout=False keeps the loop.  The default methods
    are unchanged."""
    gp, m = fixture_gp('tank', UtEngine)
    X0, U, x_ref = trajectories('tank', 2, 4, cyclic=False)
    rm, rv = gp.rollout(X0[0], U[0], methods=['UT', 'TA'])
    assert ('rollout', 3) in _log and ('rollout', 1) in _log
    del _log[:]
    hm, hv = gp.rollout(X0[0], U[0], methods=['UT', 'TA'], device_rollout=False)
    assert not any(k.startswith('rollout') for k, _ in _log) and ('predict', 3) in _log
    assert relinf(rm, hm) < 1e-12 and relinf(rv, hv) < 1e-12
    for kw in (dict(), dict(feedback=True, x_ref=x_ref)):
        del _log[:]
        bm, bv = gp.rollout(X0, U, methods=['UT'], **kw)
        assert ('rollout_batch', 3) in _log
        hm, hv = gp.rollout(X0, U, methods=['UT'], device_rollout=False, **kw)
        assert relinf(bm, hm) < 1e-12 and relinf(bv, hv) < 1e-12
        assert (bv[:, :, 1:] > 0).all()
    del _log[:]
    gp.rollout(X0, U)
    assert ('rollout_batch', 3) not in _log and ('predict', 3) not in _log
    assert gp._GP__gp_method == 'TA'
