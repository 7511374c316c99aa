"""gpmpc_rollout_sample on the device (DESIGN 4.12): consistent function samples along the visited inputs, against the
predict path, the joint Cholesky draw of the visited points, exact moment matching, and GP.sample_rollout."""
import ctypes

import numpy as np
import pytest
import scipy.linalg

from gp_mpc_b200 import _lib as L
from oracle import gp_oracle as orc
from oracle import sample_oracle as so
from tests._engines import sample_engine
from tests._util import load_fixture, load_golden, relinf

pytestmark = pytest.mark.gpu

# |f - m - R eps| / sqrt(sf2) over the kept points (DESIGN 4.12): tank's slow dynamics visit strongly correlated points,
# so R has small pivots and its inverse amplifies the last-bit differences between the host's and the device's covariances
TOL = {'synthetic': 1e-8, 'tank': 1e-6}


def _inputs(m, B, Nt, seed):
    """Starts near the data and small open-loop inputs, GP input units."""
    rng = np.random.default_rng(seed)
    X = m['X']
    Nx, Ny = X.shape[1], m['Y'].shape[1]
    z0 = X[rng.integers(0, X.shape[0], B)] + 0.05 * rng.standard_normal((B, Nx))
    U = np.repeat(z0[:, None, Ny:], Nt, 1) + 0.05 * rng.standard_normal((B, Nt, Nx - Ny))
    return z0, U, rng.standard_normal((B, Nt, Ny))


def _joint_error(eng, m, samples, z_out, kept, eps, Linv=None, alpha=None):
    """max over (b, a) of |f - m - R eps| / sqrt(sf2) over the kept points, V and m from the given factor (default: the
    engine's own L^-1 and alpha)."""
    Nx, Ny = m['X'].shape[1], m['Y'].shape[1]
    Linv = [eng.get(L.GET_LINV, a) for a in range(Ny)] if Linv is None else Linv
    alpha = [eng.get(L.GET_ALPHA, a) for a in range(Ny)] if alpha is None else alpha
    err = 0.0
    for b in range(samples.shape[0]):
        for a in range(Ny):
            mu, C = so.path_moments(m['X'], m['hyper'][a], alpha[a], Linv[a], z_out[b])
            k = kept[b, :, a].astype(bool)
            d = samples[b, k, a] - so.joint_draw(mu, C, eps[b, :, a], k)
            err = max(err, np.abs(d).max() / abs(m['hyper'][a, Nx]))
    return err


@pytest.mark.parametrize('name', ['tank', 'car', 'synthetic'])
def test_step_one_is_the_predicted_mean_plus_sqrt_var_eps(name):
    eng, m = sample_engine(name)
    B = 70
    z0, U, _ = _inputs(m, B, 1, 1)
    Ny = m['Y'].shape[1]
    f0 = eng.rollout_sample(z0, U, np.zeros((B, 1, Ny)))[0][:, 0]
    f1 = eng.rollout_sample(z0, U, np.ones((B, 1, Ny)))[0][:, 0]
    mean, var, _, _ = eng.predict(z0, None, L.METHOD_ME, want_cov=False, want_jac=False)
    assert relinf(f0, mean) < 1e-12
    assert relinf((f1 - f0) ** 2, var) < 1e-8
    eng.close()


@pytest.mark.parametrize('B', [1, 64, 65, 130])
@pytest.mark.parametrize('name', ['tank', 'synthetic'])
def test_teacher_forced_joint_identity(name, B):
    """f - m = R eps over every trajectory's kept points, R = chol of the joint posterior covariance of its visited
    inputs formed on the host from the engine's own L^-1."""
    eng, m = sample_engine(name)
    z0, U, eps = _inputs(m, B, 12, B)
    samples, z_out, kept = eng.rollout_sample(z0, U, eps)
    assert np.isfinite(samples).all() and kept[:, 0].all()
    assert _joint_error(eng, m, samples, z_out, kept, eps) <= TOL[name]
    eng.close()


@pytest.mark.parametrize('name', ['tank', 'car'])
def test_joint_identity_against_a_lapack_factor(name):
    """The same identity with V and m from an independent LAPACK factor.  car: cond(K) ~ 1e10 (DESIGN 4.12)."""
    eng, m = sample_engine(name)
    Ny = m['Y'].shape[1]
    z0, U, eps = _inputs(m, 16, 12, 7)
    samples, z_out, kept = eng.rollout_sample(z0, U, eps)
    post = orc.postfit(m['X'], m['Y'], m['hyper'], lapack_general_solve=False)
    Linv = [scipy.linalg.solve_triangular(post['chol'][a], np.eye(m['X'].shape[0]), lower=True) for a in range(Ny)]
    err = _joint_error(eng, m, samples, z_out, kept, eps, Linv, post['alpha'])
    assert err <= (TOL['tank'] if name == 'tank' else 1e-5), err
    eng.close()


def test_degenerate_path_of_a_contractive_model():
    """x+ = 0.5 x learned from data: every sampled trajectory converges to a fixed point of its draw, so the conditional
    variance falls to the rounding level and later points leave the conditioning set."""
    import gp_mpc_b200
    rng = np.random.default_rng(2)
    X = rng.uniform(-2, 2, (60, 2))
    Y = 0.5 * X + 1e-3 * rng.standard_normal(X.shape)
    hyper = np.array([[3.0, 3.0, 1.0, 1e-3], [3.0, 3.0, 1.0, 1e-3]])
    m = dict(X=X, Y=Y, hyper=hyper)
    eng = gp_mpc_b200.Engine(60, 2, 2, device=0)
    eng.set_data(X, Y); eng.set_hyper(hyper); eng.factorize()
    B, Nt = 8, 60
    z0 = rng.uniform(-1.5, 1.5, (B, 2))
    eps = rng.standard_normal((B, Nt, 2))
    samples, z_out, kept = eng.rollout_sample(z0, np.zeros((B, Nt, 0)), eps)
    assert np.isfinite(samples).all()
    assert (kept == 0).any() and kept[:, 0].all()
    assert _joint_error(eng, m, samples, z_out, kept, eps) <= 1e-6
    eng.close()


def test_bit_identical_alone_in_a_batch_and_on_repeat():
    eng, m = sample_engine('synthetic')
    z0, U, eps = _inputs(m, 130, 6, 3)
    full = eng.rollout_sample(z0, U, eps)
    again = eng.rollout_sample(z0, U, eps)
    for x, y in zip(full, again):
        assert np.array_equal(x, y)
    for b in (0, 63, 64, 129):
        one = eng.rollout_sample(z0[b:b + 1], U[b:b + 1], eps[b:b + 1])
        for x, y in zip(one, full):
            assert np.array_equal(x[0], y[b]), b
    eng.close()


def test_feedback_applies_the_gain_to_each_sampled_state():
    """u_t = K (x_t - x_ref), standardised, where x_t is the sampled state: recomputed on the host."""
    import gp_mpc_b200
    m = load_fixture('tank')
    kw = dict(mean_func='zero', gp_method='TA', normalize=True, hyper=dict(hyper=m['hyper']), meta=m['meta'],
              xlb=m['xlb'], xub=m['xub'], ulb=m['ulb'], uub=m['uub'])
    gp = gp_mpc_b200.GP(m['X'], m['Y'], **kw)
    d = load_golden('derived', 'tank')
    x0, u0 = np.asarray(d['x0']), np.asarray(d['u0'])
    st = m['meta']
    A, Bm = gp.discrete_linearize(x0, u0, None)
    K = gp_mpc_b200.lqr(A, Bm, np.eye(4), np.eye(2))[0]
    x_ref = 0.9 * x0 + 0.1
    B, Nt = 32, 10
    rng = np.random.default_rng(8)
    zx = (x0 - st['meanX']) / st['stdX'] + 0.1 * rng.standard_normal((B, 4))
    z0 = np.concatenate([zx, np.tile((K @ (x0 - x_ref) - st['meanU']) / st['stdU'], (B, 1))], 1)
    scale = np.stack([st['stdY'], st['meanY'], st['meanX'], st['stdX']])
    uscale = np.stack([st['meanU'], st['stdU']])
    samples, z_out, _ = gp.engine.rollout_sample(z0, np.zeros((B, Nt, 2)), rng.standard_normal((B, Nt, 4)),
                                                 rng.standard_normal((B, Nt, 4)), scale, K, x_ref, uscale)
    x = samples * st['stdY'] + st['meanY']
    u = np.einsum('ij,btj->bti', K, x[:, :-1] - x_ref)
    assert relinf(z_out[:, 1:, 4:], (u - st['meanU']) / st['stdU']) < 1e-12
    assert relinf(z_out[:, 1:, :4], (x[:, :-1] - st['meanX']) / st['stdX']) < 1e-14
    # a different gain changes the trajectories
    s2 = gp.engine.rollout_sample(z0, np.zeros((B, Nt, 2)), np.zeros((B, Nt, 4)), None, scale, 2 * K, x_ref, uscale)[0]
    s1 = gp.engine.rollout_sample(z0, np.zeros((B, Nt, 2)), np.zeros((B, Nt, 4)), None, scale, K, x_ref, uscale)[0]
    assert relinf(s1, s2) > 1e-6
    gp.close()


def test_step_one_statistics_match_exact_moment_matching():
    """8192 draws from N(z0, Sigma0): the sample mean and covariance of step 1 lie within 5 standard errors of 'EM'."""
    eng, m = sample_engine('tank')
    d = load_golden('derived', 'tank')
    st = m['meta']
    Nx, Ny = 6, 4
    zbar = np.concatenate([(np.asarray(d['x0']) - st['meanX']) / st['stdX'], (np.asarray(d['u0']) - st['meanU']) / st['stdU']])
    A = np.random.default_rng(1).standard_normal((Nx, Nx))
    S0 = 0.02 * np.eye(Nx) + 0.005 * A @ A.T
    n = 8192
    rng = np.random.default_rng(21)
    z0 = zbar + rng.standard_normal((n, Nx)) @ np.linalg.cholesky(S0).T
    f = eng.rollout_sample(z0, np.repeat(z0[:, None, Ny:], 1, 1), rng.standard_normal((n, 1, Ny)))[0][:, 0]
    em_m, _, em_c, _ = eng.predict(zbar[None], S0, L.METHOD_EM, want_jac=False)
    mc_m, mc_c = f.mean(0), np.cov(f.T)
    se_m = np.sqrt(np.diag(mc_c) / n)
    se_c = np.sqrt((np.outer(np.diag(mc_c), np.diag(mc_c)) + mc_c ** 2) / n)
    assert (np.abs(mc_m - em_m[0]) < 5 * se_m).all(), (mc_m - em_m[0]) / se_m
    assert (np.abs(mc_c - em_c[0]) < 5 * se_c).all(), (mc_c - em_c[0]) / se_c
    eng.close()


def test_argument_and_state_errors_leave_the_model_usable():
    import gp_mpc_b200
    lib = L.load()
    eng, m = sample_engine('tank')
    Nx, Ny = 6, 4
    z0, U, eps = _inputs(m, 2, 3, 0)
    K = np.zeros((2, Ny))
    out, zo = np.zeros(2 * 3 * Ny), np.zeros(2 * 3 * Nx)
    kp = np.zeros(2 * 3 * Ny, dtype=np.int32)
    p = lambda a: None if a is None else a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    ip = kp.ctypes.data_as(ctypes.POINTER(ctypes.c_int))
    before = eng.predict(z0, None, L.METHOD_ME, want_cov=False, want_jac=False)
    rs = lambda B, Nt, z, u, e, s, k: lib.gpmpc_rollout_sample(eng.h, B, Nt, p(z), p(u), p(e), None, None, p(k), None,
                                                               None, p(s), p(zo), ip)
    assert rs(0, 3, z0, U, eps, out, None) == L.ERR_ARG
    assert rs(2, 0, z0, U, eps, out, None) == L.ERR_ARG
    assert rs(2, 3, None, U, eps, out, None) == L.ERR_ARG
    assert rs(2, 3, z0, U, None, out, None) == L.ERR_ARG
    assert rs(2, 3, z0, U, eps, None, None) == L.ERR_ARG
    assert rs(2, 3, z0, None, eps, out, None) == L.ERR_ARG                 # open loop needs U
    assert rs(2, 5000, z0, U, eps, out, None) == L.ERR_ARG                 # Nt beyond the factor's shared memory
    after = eng.predict(z0, None, L.METHOD_ME, want_cov=False, want_jac=False)
    assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])
    assert rs(2, 3, z0, None, eps, out, K) == L.OK                         # U may be NULL with K
    eng.close()
    # K with Nu = 0
    rng = np.random.default_rng(0)
    X = rng.standard_normal((20, 2)); hyper = np.array([[1., 1., 1., .1], [1., 1., 1., .1]])
    e2 = gp_mpc_b200.Engine(20, 2, 2, device=0); e2.set_data(X, X); e2.set_hyper(hyper); e2.factorize()
    z, e, o = np.zeros((1, 2)), np.zeros((1, 1, 2)), np.zeros(2)
    assert lib.gpmpc_rollout_sample(e2.h, 1, 1, p(z), None, p(e), None, None, p(np.zeros(2)), None, None, p(o), None,
                                    None) == L.ERR_ARG
    assert lib.gpmpc_rollout_sample(e2.h, 1, 1, p(z), None, p(e), None, None, None, None, None, p(o), None, None) == L.OK
    e2.close()
    # a handle that owns only some outputs
    e3 = gp_mpc_b200.Engine(m['X'].shape[0], Nx, Ny, out_begin=0, out_count=2, device=0)
    e3.set_data(m['X'], m['Y']); e3.set_hyper(m['hyper']); e3.factorize()
    b3 = e3.predict(z0, None, L.METHOD_ME, want_cov=False, want_jac=False)
    with pytest.raises(L.GpmpcError) as ex:
        e3.rollout_sample(z0, U, eps)
    assert ex.value.code == L.ERR_STATE
    a3 = e3.predict(z0, None, L.METHOD_ME, want_cov=False, want_jac=False)
    assert np.array_equal(b3[0], a3[0])
    e3.close()


def test_gp_sample_rollout_is_the_engine_fed_the_same_draws():
    """car (no normalisation): GP.sample_rollout, single and batched, equals Engine.rollout_sample with the draws of
    default_rng(seed) in the documented order."""
    import gp_mpc_b200
    m = load_fixture('car')
    gp = gp_mpc_b200.GP(m['X'], m['Y'], mean_func='zero', gp_method='TA', normalize=False, hyper=dict(hyper=m['hyper']))
    d = load_golden('derived', 'car')
    x0, u0 = np.asarray(d['x0']), np.asarray(d['u0'])
    Nx, Ny, Nt, ns = 5, 3, 6, 20
    U = np.tile(u0, (Nt, 1)) * (1 + 0.02 * np.arange(Nt)[:, None])
    X0 = np.stack([x0, 1.02 * x0])
    UB = np.stack([U, 0.98 * U])
    S0 = np.eye(Nx) * 1e-6
    S0[:Ny, :Ny] = np.diag(m['hyper'][:, Nx + 1] ** 2)
    F = np.linalg.cholesky(S0)
    for single in (True, False):
        xs, us = (x0[None], U[None]) if single else (X0, UB)
        nb = xs.shape[0]
        s = gp.sample_rollout(x0 if single else X0, U if single else UB, ns, seed=4, process_noise=True)
        rng = np.random.default_rng(4)
        n0 = rng.standard_normal((nb, ns, Nx))
        eps = rng.standard_normal((nb, ns, Nt, Ny))
        xi = rng.standard_normal((nb, ns, Nt, Ny))
        z0 = np.concatenate([xs, us[:, 0]], 1)[:, None, :] + n0 @ F.T
        f = gp.engine.rollout_sample(z0.reshape(-1, Nx), np.repeat(us, ns, 0), eps.reshape(-1, Nt, Ny),
                                     xi.reshape(-1, Nt, Ny))[0].reshape(nb, ns, Nt, Ny)
        got = s[None] if single else s
        assert got.shape == (nb, ns, Nt + 1, Ny)
        assert np.array_equal(got[:, :, 1:], f) and np.array_equal(got[:, :, 0], z0[:, :, :Ny])
    gp.close()
