"""Sampled roll-outs (DESIGN 4.12): the sequential conditioning of oracle/sample_oracle.py against the joint Cholesky
draw and exact moment matching, and GP.sample_rollout's bookkeeping (shapes, units, draw order, feedback grouping,
errors) through an oracle-backed stand-in engine.  The device path is covered by tests/test_sample_rollout_gpu.py."""
import os
import re

import numpy as np
import pytest

import gp_mpc_b200
from oracle import gp_oracle as orc
from oracle import sample_oracle as so
from tests._fake_engine import OracleEngine, TwoRanks, sample_model, sharded
from tests._util import load_fixture, load_golden, relinf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class OracleEngineWithSample(OracleEngine):
    """Adds gpmpc_rollout_sample, restated by the oracle from the stand-in's own factor; records every call."""
    calls = None

    def rollout_sample(self, z0, U, eps, xi=None, scale=None, K=None, x_ref=None, uscale=None):
        if OracleEngineWithSample.calls is not None:
            OracleEngineWithSample.calls.append(dict(B=np.shape(z0)[0], K=None if K is None else np.array(K)))
        Linv = np.stack([np.linalg.inv(L) for L in self.post['chol']])
        model = dict(X=self.X, hyper=self.hyper, alpha=self.post['alpha'])
        return so.rollout_sample(model, Linv, z0, U, np.asarray(eps), xi, scale, K, x_ref, uscale)


def _gp(name, factory=OracleEngineWithSample, **kw):
    m = sample_model(name)
    args = dict(mean_func='zero', gp_method='TA', normalize=m['normalize'], hyper=dict(hyper=m['hyper']),
                engine_factory=factory)
    if m['normalize']:
        args.update(meta=m['meta'], xlb=m['xlb'], xub=m['xub'], ulb=m['ulb'], uub=m['uub'])
    args.update(kw)
    return gp_mpc_b200.GP(m['X'], m['Y'], **args), m


def _path(m, T, rng):
    """T visited points near the data, with exact returns to earlier points (their conditional variance is zero)."""
    X = m['X']
    Z = X[rng.integers(0, X.shape[0], T)] + 0.05 * rng.standard_normal((T, X.shape[1]))
    Z[5] = Z[2]
    Z[9] = Z[4]
    return Z


@pytest.mark.parametrize('name', ['tank', 'car', 'synthetic'])
def test_sequential_conditioning_is_the_joint_cholesky_draw(name):
    m = sample_model(name)
    post = orc.postfit(m['X'], m['Y'], m['hyper'], lapack_general_solve=False)
    rng = np.random.default_rng(3)
    Z = _path(m, 12, rng)
    Nx = m['X'].shape[1]
    for a in range(m['hyper'].shape[0]):
        Linv = np.linalg.inv(post['chol'][a])
        mu, C = so.path_moments(m['X'], m['hyper'][a], post['alpha'][a], Linv, Z)
        eps = rng.standard_normal(12)
        sf2 = m['hyper'][a, Nx] ** 2
        f, kept = so.conditional_draw(mu, C, eps, sf2)
        assert not kept[5] and not kept[9] and kept[:5].all()          # the returns are skipped by the delta rule
        assert np.abs(f[kept] - so.joint_draw(mu, C, eps, kept)).max() <= 1e-8 * np.sqrt(sf2)
        # a skipped point takes the value the draw already has there
        assert abs(f[5] - f[2]) <= 1e-8 * np.sqrt(sf2) and abs(f[9] - f[4]) <= 1e-8 * np.sqrt(sf2)


def test_step_one_monte_carlo_matches_exact_moment_matching():
    """z ~ N(z0, Sigma0), f = m(z) + sqrt(var(z)) eps: the mean and covariance of f are those of 'EM'."""
    m = load_fixture('tank')
    post = orc.postfit(m['X'], m['Y'], m['hyper'], lapack_general_solve=False)
    d = load_golden('derived', 'tank')
    Nx, Ny = m['X'].shape[1], m['Y'].shape[1]
    st = m['meta']
    z0 = np.concatenate([(np.asarray(d['x0']) - st['meanX']) / st['stdX'], (np.asarray(d['u0']) - st['meanU']) / st['stdU']])
    A = np.random.default_rng(1).standard_normal((Nx, Nx))
    S0 = 0.02 * np.eye(Nx) + 0.005 * A @ A.T
    rng = np.random.default_rng(11)
    n = 8192
    Z = z0 + rng.standard_normal((n, Nx)) @ np.linalg.cholesky(S0).T
    mu, var = orc.gp_mean_var(m['X'], m['hyper'], post['alpha'], post['chol'], Z)
    f = mu + np.sqrt(var) * rng.standard_normal((n, Ny))
    em_m, em_c = orc.gp_exact_moment(m['invK'], m['X'], m['Y'], m['hyper'], z0, S0)
    mc_m, mc_c = f.mean(0), np.cov(f.T)
    se_m = np.sqrt(np.diag(mc_c) / n)
    se_c = np.sqrt((np.outer(np.diag(mc_c), np.diag(mc_c)) + mc_c ** 2) / n)
    assert (np.abs(mc_m - em_m) < 5 * se_m).all(), (mc_m - em_m) / se_m
    assert (np.abs(mc_c - em_c) < 5 * se_c).all(), (mc_c - em_c) / se_c


def test_shapes_single_and_batched():
    gp, m = _gp('tank')
    d = load_golden('derived', 'tank')
    x0, u0 = np.asarray(d['x0']), np.asarray(d['u0'])
    U = np.tile(u0, (4, 1))
    s = gp.sample_rollout(x0, U, 3, seed=0)
    assert s.shape == (3, 5, 4) and np.isfinite(s).all()
    sb = gp.sample_rollout(np.stack([x0, 1.01 * x0]), np.stack([U, U]), 2, seed=0, process_noise=True)
    assert sb.shape == (2, 2, 5, 4) and np.isfinite(sb).all()


@pytest.mark.parametrize('name', ['tank', 'car'])
def test_units_and_the_documented_draw_order(name):
    """tank normalises, car does not.  Row 0 is the drawn start in caller units; step 1 with Sigma0 = 0 is the predicted
    mean plus stdY sqrt(var) eps; the whole result is the engine's, fed the draws of default_rng(seed) in the
    documented order (initial perturbations, eps, xi)."""
    gp, m = _gp(name)
    d = load_golden('derived', name)
    x0, u0 = np.asarray(d['x0'], dtype=np.float64), np.asarray(d['u0'], dtype=np.float64)
    Nx, Ny = m['X'].shape[1], m['Y'].shape[1]
    Nt, ns = 3, 4
    U = np.tile(u0, (Nt, 1))
    s = gp.sample_rollout(x0, U, ns, seed=5, Sigma0=np.zeros((Nx, Nx)), process_noise=True)
    assert relinf(s[:, 0], np.tile(x0, (ns, 1))) < 1e-14
    rng = np.random.default_rng(5)
    rng.standard_normal((1, ns, Nx))
    eps = rng.standard_normal((1, ns, Nt, Ny))[0]
    xi = rng.standard_normal((1, ns, Nt, Ny))[0]
    mean, cov = gp.predict_batch(x0[None], u0[None], np.zeros((Nx, Nx)), 'ME')
    sd = np.sqrt(np.diag(cov[0]))
    sn = m['hyper'][:, Nx + 1]
    stdY = m['meta']['stdY'] if m['normalize'] else np.ones(Ny)
    assert relinf(s[:, 1], mean[0] + stdY * (sd * eps[:, 0] + sn * xi[:, 0])) < 1e-10
    # every step: the engine's draws, mapped to caller units
    S0 = np.eye(Nx) * 1e-6
    S0[:Ny, :Ny] = np.diag(sn ** 2)
    s2 = gp.sample_rollout(x0, U, ns, seed=9)
    rng = np.random.default_rng(9)
    n0 = rng.standard_normal((1, ns, Nx))[0]
    eps = rng.standard_normal((1, ns, Nt, Ny))[0]
    if m['normalize']:
        st = m['meta']
        zbar = np.concatenate([(x0 - st['meanX']) / st['stdX'], (u0 - st['meanU']) / st['stdU']])
        scale = np.stack([st['stdY'], st['meanY'], st['meanX'], st['stdX']])
        Ug = (U - st['meanU']) / st['stdU']
    else:
        zbar, scale, Ug = np.concatenate([x0, u0]), None, U
    z0 = zbar + n0 @ np.linalg.cholesky(S0).T
    f, z_out, kept = gp.engine.rollout_sample(z0, np.tile(Ug, (ns, 1, 1)), eps, None, scale)
    assert np.array_equal(z_out[:, 0], z0) and kept.all()
    if m['normalize']:
        f = f * st['stdY'] + st['meanY']
        z0x = z0[:, :Ny] * st['stdX'] + st['meanX']
    else:
        z0x = z0[:, :Ny]
    assert np.array_equal(s2[:, 1:], f) and np.array_equal(s2[:, 0], z0x)
    # the next input is the sampled state, re-standardised with the X scalers
    x1 = f[:, 0]
    assert relinf(z_out[:, 1, :Ny], (x1 - st['meanX']) / st['stdX'] if m['normalize'] else x1) < 1e-14


def test_feedback_runs_one_pass_per_distinct_gain():
    gp, m = _gp('tank')
    d = load_golden('derived', 'tank')
    x0, u0 = np.asarray(d['x0']), np.asarray(d['u0'])
    X0 = np.stack([x0, 1.05 * x0, x0])                   # trajectories 0 and 2 share their linearisation point
    U = np.stack([np.tile(u0, (3, 1))] * 3)
    x_ref = 0.9 * x0 + 0.1
    OracleEngineWithSample.calls = []
    try:
        s = gp.sample_rollout(X0, U, 2, seed=1, feedback=True, x_ref=x_ref)
        calls = OracleEngineWithSample.calls
    finally:
        OracleEngineWithSample.calls = None
    assert s.shape == (3, 2, 4, 4)
    assert sorted(c['B'] for c in calls) == [2, 4] and all(c['K'] is not None for c in calls)
    assert not np.array_equal(calls[0]['K'], calls[1]['K'])
    # the applied input is K (x - x_ref) of the sampled state (standardised): recompute it for trajectory 1
    A, Bm = gp.discrete_linearize(X0[1], U[1, 0], None)
    K = gp_mpc_b200.lqr(A, Bm, np.eye(4), np.eye(2))[0]
    st = m['meta']
    OracleEngineWithSample.calls = None
    rng = np.random.default_rng(1)
    n0 = rng.standard_normal((3, 2, 6))
    eps = rng.standard_normal((3, 2, 3, 4))
    S0 = np.eye(6) * 1e-6
    S0[:4, :4] = np.diag(m['hyper'][:, -1] ** 2)
    zbar = np.concatenate([(X0[1] - st['meanX']) / st['stdX'], (K @ (X0[1] - x_ref) - st['meanU']) / st['stdU']])
    z0 = zbar + n0[1] @ np.linalg.cholesky(S0).T
    f, z_out, _ = gp.engine.rollout_sample(z0, U[:2], eps[1], None, np.stack([st['stdY'], st['meanY'], st['meanX'], st['stdX']]),
                                           K, x_ref, np.stack([st['meanU'], st['stdU']]))
    x = f * st['stdY'] + st['meanY']
    assert relinf(s[1, :, 1:], x) < 1e-12
    u_app = np.einsum('ij,btj->bti', K, x[:, :-1] - x_ref)
    assert relinf(z_out[:, 1:, 4:], (u_app - st['meanU']) / st['stdU']) < 1e-12


_ShardEngine = sharded(OracleEngineWithSample)


def test_argument_errors():
    gp, m = _gp('tank')
    x0, U = np.zeros(4), np.zeros((3, 2))
    with pytest.raises(ValueError):
        gp.sample_rollout(x0, U, 0)
    with pytest.raises(ValueError):
        gp.sample_rollout(x0, np.zeros((0, 2)), 2)
    with pytest.raises(ValueError):
        gp.sample_rollout(x0, U, 2, Sigma0=np.eye(4))
    rng = np.random.default_rng(1)
    X = rng.standard_normal((20, 2)); Y = X + 0.1 * rng.standard_normal((20, 2))
    hyper = np.array([[1., 1., 1., .1], [1., 1., 1., .1]])
    auto = gp_mpc_b200.GP(X, Y, normalize=False, hyper=dict(hyper=hyper), engine_factory=OracleEngineWithSample)
    with pytest.raises(ValueError):
        auto.sample_rollout(np.zeros(2), np.zeros((3, 0)), 2, feedback=True)
    assert auto.sample_rollout(np.zeros(2), np.zeros((3, 0)), 2, seed=0).shape == (2, 4, 2)
    # sharded by output over two ranks
    sh = gp_mpc_b200.GP(m['X'], m['Y'], normalize=False, hyper=dict(hyper=m['hyper']), comm=TwoRanks(),
                        engine_factory=_ShardEngine)
    with pytest.raises(NotImplementedError, match='needs all outputs on one GPU'):
        sh.sample_rollout(x0, U, 2)
    # a prior mean added in predict
    pm = gp_mpc_b200.GP(m['X'], m['Y'], normalize=False, mean_func='const', prior_mean_in_predict=True,
                        hyper=dict(hyper=np.column_stack([m['hyper'], np.full(4, 0.1)])), engine_factory=OracleEngineWithSample)
    with pytest.raises(NotImplementedError):
        pm.sample_rollout(x0, U, 2)


def test_rollout_sample_is_declared_and_bound():
    hdr = open(os.path.join(ROOT, 'include', 'gpmpc.h')).read()
    assert re.search(r'\bint gpmpc_rollout_sample\s*\(', hdr)
    import __graft_entry__ as g
    g.build()
    L = gp_mpc_b200._lib
    assert 'gpmpc_rollout_sample' in {s[0] for s in L.SYMBOLS}
    assert L.load().gpmpc_rollout_sample is not None
