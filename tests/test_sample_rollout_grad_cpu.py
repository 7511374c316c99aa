"""Pathwise derivatives of sampled roll-outs (DESIGN 4.16): the forward-mode checker tests/_sample_grad_oracle.py against
central differences of oracle/sample_oracle.py's draws with the normals held fixed and against the joint Cholesky form,
and GP.sample_rollout_grad's bookkeeping (draws, units, shapes, feedback grouping, errors) through an oracle-backed
stand-in engine.  The device entry is covered by tests/test_sample_rollout_grad_gpu.py."""
import os
import re

import numpy as np
import pytest

import gp_mpc_b200
from oracle import gp_oracle as orc
from oracle import sample_oracle as so
from tests import _sample_grad_oracle as sgo
from tests._fake_engine import OracleEngine, TwoRanks, sample_model, sharded
from tests._util import load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# Central-difference step and bar (relative to 1 + max |derivative|).  The error of a quotient is the draw's rounding over
# the step: R^-1 enters the draw twice and tank's and car's pivots are small (cond K ~ 1e10 on car), so their draws carry
# ~1e-10 of rounding and need a step of 1e-4 (errors measured up to 8e-7 there, 7e-5 at a step of 1e-6); the
# synthetic problem resolves a step of 1e-6.
STEP = dict(tank=1e-4, car=1e-4, synthetic=1e-6)
BAR = dict(tank=5e-6, car=5e-6, synthetic=2e-5)


class OracleEngineWithSampleGrad(OracleEngine):
    """Adds gpmpc_rollout_sample and gpmpc_rollout_sample_grad, restated by the oracles from the stand-in's own factor;
    records every call of the latter."""
    calls = None

    def _factor(self):
        Linv = np.stack([np.linalg.inv(L) for L in self.post['chol']])
        return dict(X=self.X, hyper=self.hyper, alpha=self.post['alpha'], chol=self.post['chol']), Linv

    def rollout_sample(self, z0, U, eps, xi=None, scale=None, K=None, x_ref=None, uscale=None):
        model, Linv = self._factor()
        return so.rollout_sample(model, Linv, z0, U, np.asarray(eps), xi, scale, K, x_ref, uscale)

    def rollout_sample_grad(self, z0, U, eps, xi=None, scale=None, K=None, x_ref=None, uscale=None):
        if OracleEngineWithSampleGrad.calls is not None:
            OracleEngineWithSampleGrad.calls.append(dict(B=np.shape(z0)[0], K=None if K is None else np.array(K)))
        model, Linv = self._factor()
        r = sgo.rollout_sample_grad(model, Linv, z0, U, np.asarray(eps), xi, scale, K, x_ref, uscale)
        return r['samples'], r['z_out'], r['kept'], r['dsamples']


def _engine_problem(name, feedback, Nt=4, B=2, seed=0):
    """A factor and a roll-out of B trajectories in the engine's units: model, Linv, args of rollout_sample_grad."""
    m = sample_model(name)
    post = orc.postfit(m['X'], m['Y'], m['hyper'], lapack_general_solve=False)
    model = dict(X=m['X'], hyper=m['hyper'], alpha=post['alpha'], chol=post['chol'])
    Linv = np.stack([np.linalg.inv(L) for L in post['chol']])
    Ny, Nx = m['hyper'].shape[0], m['X'].shape[1]
    Nu = Nx - Ny
    rng = np.random.default_rng(seed)
    if name == 'synthetic':
        zbar = m['X'][3]
        scale = uscale = None
    else:
        d = load_golden('derived', name)
        x0, u0 = np.asarray(d['x0'], dtype=np.float64), np.asarray(d['u0'], dtype=np.float64)
        if m['normalize']:
            st = m['meta']
            zbar = np.concatenate([(x0 - st['meanX']) / st['stdX'], (u0 - st['meanU']) / st['stdU']])
            scale = np.stack([st['stdY'], st['meanY'], st['meanX'], st['stdX']])
            uscale = np.stack([st['meanU'], st['stdU']])
        else:
            zbar, scale, uscale = np.concatenate([x0, u0]), None, None
    z0 = zbar + 0.3 * rng.standard_normal((B, Nx))
    U = np.tile(zbar[Ny:], (B, Nt, 1)) + 0.3 * rng.standard_normal((B, Nt, Nu))
    eps = rng.standard_normal((B, Nt, Ny))
    xi = rng.standard_normal((B, Nt, Ny))
    K = x_ref = None
    if feedback:
        K = 0.05 * rng.standard_normal((Nu, Ny))
        x_ref = (zbar[:Ny] if scale is None else zbar[:Ny] * scale[3] + scale[2]) + 0.01
    else:
        uscale = None
    return model, Linv, dict(z0=z0, U=U, eps=eps, xi=xi, scale=scale, K=K, x_ref=x_ref, uscale=uscale)


def _perturbed(args, p, h):
    """args with parameter column p moved by h: z0[:, p], then U rows 1.. (open loop) or K row-major."""
    a = {k: (None if v is None else np.array(v, dtype=np.float64)) for k, v in args.items()}
    Nx = a['z0'].shape[1]
    if p < Nx:
        a['z0'][:, p] += h
    elif a['K'] is None:
        Nu = a['U'].shape[2]
        a['U'][:, 1 + (p - Nx) // Nu, (p - Nx) % Nu] += h
    else:
        a['K'].reshape(-1)[p - Nx] += h
    return a


@pytest.mark.parametrize('feedback', [False, True])
@pytest.mark.parametrize('name', ['tank', 'car', 'synthetic'])
def test_oracle_matches_central_differences_of_the_draws(name, feedback):
    model, Linv, args = _engine_problem(name, feedback)
    r = sgo.rollout_sample_grad(model, Linv, **args)
    sgo.assert_margin(r['d'], model['hyper'])
    s0, _, k0 = so.rollout_sample(model, Linv, **args)
    assert np.array_equal(r['kept'], k0) and np.abs(r['samples'] - s0).max() <= 1e-12 * (1 + np.abs(s0).max())
    D = r['dsamples']
    h = STEP[name]
    for p in range(D.shape[-1]):
        sp = so.rollout_sample(model, Linv, **_perturbed(args, p, h))
        sm = so.rollout_sample(model, Linv, **_perturbed(args, p, -h))
        assert np.array_equal(sp[2], k0) and np.array_equal(sm[2], k0)
        fd = (sp[0] - sm[0]) / (2 * h)
        err = np.abs(D[..., p] - fd).max() / (1.0 + np.abs(D).max())
        assert err < BAR[name], (p, err)


@pytest.mark.parametrize('name', ['tank', 'car', 'synthetic'])
def test_oracle_matches_the_joint_cholesky_form(name):
    """Teacher-forced along a fixed path Z moved in a direction dZ: the sequential recursion's df against differences of
    f_S = m_S + chol(C[S, S]) eps_S, an independent route to the same draw."""
    m = sample_model(name)
    post = orc.postfit(m['X'], m['Y'], m['hyper'], lapack_general_solve=False)
    rng = np.random.default_rng(4)
    Nx, T = m['X'].shape[1], 8
    Z = m['X'][rng.integers(0, m['X'].shape[0], T)] + m['X'].std(0) * rng.standard_normal((T, Nx))
    dZ = rng.standard_normal((T, Nx, 1))
    eps = rng.standard_normal(T)
    for a in range(m['hyper'].shape[0]):
        Linv = np.linalg.inv(post['chol'][a])
        c = sgo.Conditioner(m['X'], m['hyper'][a], post['alpha'][a], post['chol'][a], Linv, T, 1)
        df, d = np.empty(T), np.empty(T)
        for t in range(T):
            _, g, d[t], kept = c.step(Z[:t + 1], dZ[:t + 1], eps[:t + 1])
            assert kept
            df[t] = g[0]
        sgo.assert_margin(d[None], m['hyper'][a:a + 1])

        def joint(Zp):
            mu, C = so.path_moments(m['X'], m['hyper'][a], post['alpha'][a], Linv, Zp)
            return so.joint_draw(mu, C, eps, np.ones(T, dtype=bool))
        h = STEP[name]
        fd = (joint(Z + h * dZ[..., 0]) - joint(Z - h * dZ[..., 0])) / (2 * h)
        # the joint route re-factors C at every difference point: measured up to 1.1e-5 on car
        assert np.abs(df - fd).max() / (1.0 + np.abs(df).max()) < 4 * BAR[name]


def test_a_skipped_point_takes_the_branch_taken():
    """A return to an earlier point is dropped by the delta rule: its draw is the conditional mean, whose derivative is
    the derivative of the value the draw already has there."""
    m = sample_model('synthetic')
    post = orc.postfit(m['X'], m['Y'], m['hyper'], lapack_general_solve=False)
    rng = np.random.default_rng(2)
    Nx, T = m['X'].shape[1], 4
    Z = m['X'][:T] + 0.05 * rng.standard_normal((T, Nx))
    Z[3] = Z[1]
    dZ = np.zeros((T, Nx, Nx))
    dZ[1] = dZ[3] = np.eye(Nx)                           # the returning point moves with the point it returns to
    eps = rng.standard_normal(T)
    Linv = np.linalg.inv(post['chol'][0])
    c = sgo.Conditioner(m['X'], m['hyper'][0], post['alpha'][0], post['chol'][0], Linv, T, Nx)
    out = [c.step(Z[:t + 1], dZ[:t + 1], eps[:t + 1]) for t in range(T)]
    assert [o[3] for o in out] == [True, True, True, False]
    assert abs(out[3][0] - out[1][0]) < 1e-8
    assert np.abs(out[3][1] - out[1][1]).max() < 1e-6 * (1 + np.abs(out[1][1]).max())


def _gp(name, factory=OracleEngineWithSampleGrad, **kw):
    m = sample_model(name)
    args = dict(mean_func='zero', gp_method='TA', normalize=m['normalize'], hyper=dict(hyper=m['hyper']),
                engine_factory=factory)
    if m['normalize']:
        args.update(meta=m['meta'], xlb=m['xlb'], xub=m['xub'], ulb=m['ulb'], uub=m['uub'])
    args.update(kw)
    return gp_mpc_b200.GP(m['X'], m['Y'], **args), m


@pytest.mark.parametrize('feedback', [False, True])
def test_caller_units_against_differences_of_sample_rollout(feedback):
    """Same seed: the samples are sample_rollout's bit for bit, and every derivative matches central differences of
    sample_rollout in the caller's x0, u or K (the gain held fixed, as the documented chain holds it).  tank normalises,
    so the whole unit chain is exercised; car's derived start is a rest point, where the draws drop points."""
    name = 'tank'
    gp, m = _gp(name)
    d = load_golden('derived', name)
    x0, u0 = np.asarray(d['x0'], dtype=np.float64), np.asarray(d['u0'], dtype=np.float64)
    Ny, Nu, Nt, ns = m['Y'].shape[1], m['X'].shape[1] - m['Y'].shape[1], 3, 2
    U = np.tile(u0, (Nt, 1))
    kw = dict(seed=7, process_noise=True)
    if feedback:
        kw.update(feedback=True, x_ref=0.98 * x0)
    r = gp.sample_rollout_grad(x0, U, ns, **kw)
    assert np.array_equal(r['samples'], gp.sample_rollout(x0, U, ns, **kw))
    assert r['kept'].shape == (ns, Nt, Ny) and r['kept'].all()
    assert np.array_equal(r['dsamples_dx0'][:, 0], np.tile(np.eye(Ny), (ns, 1, 1)))
    hx = STEP[name] * (np.abs(x0) + 1.0)
    if feedback:
        # K is held fixed: differentiate with the gain the call used, through a stand-in that returns it for any x0
        K0 = gp._GP__lqr_gains(x0[None], U[None, 0], np.eye(Ny), np.eye(Nu))
        gp._GP__lqr_gains = lambda X0, U0, Q, R: np.repeat(K0, len(X0), 0)
        for i in range(Nu):
            for k in range(Ny):
                hk = STEP[name] * (abs(K0[0, i, k]) + 1.0)
                Kp, Km = K0.copy(), K0.copy()
                Kp[0, i, k] += hk
                Km[0, i, k] -= hk
                gp._GP__lqr_gains = lambda X0, U0, Q, R, K=Kp: np.repeat(K, len(X0), 0)
                sp = gp.sample_rollout(x0, U, ns, **kw)
                gp._GP__lqr_gains = lambda X0, U0, Q, R, K=Km: np.repeat(K, len(X0), 0)
                sm = gp.sample_rollout(x0, U, ns, **kw)
                fd = (sp - sm) / (2 * hk)
                assert np.abs(r['dsamples_dK'][..., i, k] - fd).max() < 10 * BAR[name] * (1 + np.abs(fd).max()), (i, k)
        gp._GP__lqr_gains = lambda X0, U0, Q, R: np.repeat(K0, len(X0), 0)
    for k in range(Ny):
        xp, xm = x0.copy(), x0.copy()
        xp[k] += hx[k]
        xm[k] -= hx[k]
        fd = (gp.sample_rollout(xp, U, ns, **kw) - gp.sample_rollout(xm, U, ns, **kw)) / (2 * hx[k])
        assert np.abs(r['dsamples_dx0'][..., k] - fd).max() < 10 * BAR[name] * (1 + np.abs(fd).max()), k
    if not feedback:
        for s in range(Nt):
            for i in range(Nu):
                hu = STEP[name] * (abs(U[s, i]) + 1.0)
                Up, Um = U.copy(), U.copy()
                Up[s, i] += hu
                Um[s, i] -= hu
                fd = (gp.sample_rollout(x0, Up, ns, **kw) - gp.sample_rollout(x0, Um, ns, **kw)) / (2 * hu)
                assert np.abs(r['dsamples_du'][..., s, i] - fd).max() < 10 * BAR[name] * (1 + np.abs(fd).max()), (s, i)


def test_shapes_single_and_batched():
    gp, m = _gp('tank')
    d = load_golden('derived', 'tank')
    x0, u0 = np.asarray(d['x0']), np.asarray(d['u0'])
    U = np.tile(u0, (4, 1))
    r = gp.sample_rollout_grad(x0, U, 3, seed=0)
    assert r['samples'].shape == (3, 5, 4) and r['kept'].shape == (3, 4, 4)
    assert r['dsamples_dx0'].shape == (3, 5, 4, 4) and r['dsamples_du'].shape == (3, 5, 4, 4, 2)
    X0, UU = np.stack([x0, 1.01 * x0]), np.stack([U, U])
    rb = gp.sample_rollout_grad(X0, UU, 2, seed=0, process_noise=True)
    assert rb['samples'].shape == (2, 2, 5, 4) and rb['dsamples_du'].shape == (2, 2, 5, 4, 4, 2)
    assert np.array_equal(rb['samples'], gp.sample_rollout(X0, UU, 2, seed=0, process_noise=True))
    rk = gp.sample_rollout_grad(X0, UU, 2, seed=0, feedback=True)
    assert rk['dsamples_dK'].shape == (2, 2, 5, 4, 2, 4) and 'dsamples_du' not in rk


def test_feedback_runs_one_pass_per_distinct_gain():
    gp, m = _gp('tank')
    d = load_golden('derived', 'tank')
    x0, u0 = np.asarray(d['x0']), np.asarray(d['u0'])
    X0 = np.stack([x0, 1.05 * x0, x0])
    U = np.stack([np.tile(u0, (3, 1))] * 3)
    OracleEngineWithSampleGrad.calls = []
    try:
        r = gp.sample_rollout_grad(X0, U, 2, seed=1, feedback=True, x_ref=0.9 * x0 + 0.1)
        calls = OracleEngineWithSampleGrad.calls
    finally:
        OracleEngineWithSampleGrad.calls = None
    assert r['samples'].shape == (3, 2, 4, 4)
    assert sorted(c['B'] for c in calls) == [2, 4] and all(c['K'] is not None for c in calls)
    assert np.array_equal(r['samples'], gp.sample_rollout(X0, U, 2, seed=1, feedback=True, x_ref=0.9 * x0 + 0.1))


_ShardEngine = sharded(OracleEngineWithSampleGrad)


def test_argument_errors():
    gp, m = _gp('tank')
    x0, U = np.zeros(4), np.zeros((3, 2))
    with pytest.raises(ValueError):
        gp.sample_rollout_grad(x0, U, 0)
    with pytest.raises(ValueError):
        gp.sample_rollout_grad(x0, np.zeros((0, 2)), 2)
    with pytest.raises(ValueError):
        gp.sample_rollout_grad(x0, U, 2, Sigma0=np.eye(4))
    rng = np.random.default_rng(1)
    X = rng.standard_normal((20, 2)); Y = X + 0.1 * rng.standard_normal((20, 2))
    hyper = np.array([[1., 1., 1., .1], [1., 1., 1., .1]])
    auto = gp_mpc_b200.GP(X, Y, normalize=False, hyper=dict(hyper=hyper), engine_factory=OracleEngineWithSampleGrad)
    with pytest.raises(ValueError):
        auto.sample_rollout_grad(np.zeros(2), np.zeros((3, 0)), 2, feedback=True)
    r = auto.sample_rollout_grad(np.zeros(2), np.zeros((3, 0)), 2, seed=0)
    assert r['dsamples_dx0'].shape == (2, 4, 2, 2) and r['dsamples_du'].shape == (2, 4, 2, 3, 0)
    sh = gp_mpc_b200.GP(m['X'], m['Y'], normalize=False, hyper=dict(hyper=m['hyper']), comm=TwoRanks(),
                        engine_factory=_ShardEngine)
    with pytest.raises(NotImplementedError, match='needs all outputs on one GPU'):
        sh.sample_rollout_grad(x0, U, 2)
    pm = gp_mpc_b200.GP(m['X'], m['Y'], normalize=False, mean_func='const', prior_mean_in_predict=True,
                        hyper=dict(hyper=np.column_stack([m['hyper'], np.full(4, 0.1)])),
                        engine_factory=OracleEngineWithSampleGrad)
    with pytest.raises(NotImplementedError):
        pm.sample_rollout_grad(x0, U, 2)
    plain, _ = _gp('tank', factory=OracleEngine)
    with pytest.raises(NotImplementedError, match='gpmpc_rollout_sample_grad'):
        plain.sample_rollout_grad(x0, U, 2)


def test_rollout_sample_grad_is_declared_and_bound():
    hdr = open(os.path.join(ROOT, 'include', 'gpmpc.h')).read()
    assert re.search(r'\bint gpmpc_rollout_sample_grad\s*\(', hdr)
    import __graft_entry__ as g
    g.build()
    L = gp_mpc_b200._lib
    assert 'gpmpc_rollout_sample_grad' in {s[0] for s in L.SYMBOLS}
    assert L.load().gpmpc_rollout_sample_grad is not None
