"""GP.rollout_grad(method='EM') and its checker on CPU: the forward-mode 'EM' oracle (tests/_rollout_em_grad_oracle.py)
against central differences of predict_compare_loop and against em_grad_closed at one step, and GP.rollout_grad's
caller-unit mapping through a numpy restatement of gpmpc_rollout_batch_em_grad.  The device entry is covered by
tests/test_rollout_em_grad_gpu.py."""
import os
import re

import numpy as np
import pytest

import gp_mpc_b200
from gp_mpc_b200.gp_class import _matmul_seq
from oracle import em_grad_oracle, rollout_oracle
from oracle import gp_oracle as orc
from oracle.rollout_oracle import predict_compare_loop
from tests._fake_engine import OracleEngineWithRolloutBatch, fixture_gp
from tests._rollout_em_grad_oracle import rollout_em_grad
from tests._util import central, load_fixture, relinf, trajectories

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class OracleEngineWithRolloutBatchEmGrad(OracleEngineWithRolloutBatch):
    """Adds a numpy restatement of gpmpc_rollout_batch_em_grad (include/gpmpc.h) in the GP's units: the step's primal from
    gp_exact_moment, its derivatives from em_grad_closed, the tangents by the entry's recurrence (dS carried open loop too)."""
    calls = []

    def rollout_batch_em_grad(self, z0, U, Sigma0, scale=None, K=None, x_ref=None, uscale=None):
        type(self).calls.append(np.array(z0).shape[0])
        Ny, Nx = self.Ny, self.Nx
        Nu = Nx - Ny
        Z0 = np.array(z0, dtype=np.float64).reshape(-1, Nx)
        B, Nt = Z0.shape[0], np.shape(U)[1]
        P = Nx + (Nu * Ny if K is not None else (Nt - 1) * Nu)
        means = np.zeros((B, Nt, Ny)); var = np.zeros((B, Nt, Ny)); cov = np.zeros((B, Ny, Ny))
        dmeans = np.zeros((B, Nt, Ny, P)); dvars = np.zeros((B, Nt, Ny, P))
        sY, mY, mX, sX = (np.ones(Ny), np.zeros(Ny), np.zeros(Ny), np.ones(Ny)) if scale is None else scale
        mU, sU = (np.zeros(Nu), np.ones(Nu)) if uscale is None else uscale
        xr = np.zeros(Ny) if x_ref is None else x_ref
        dK = np.zeros((Nu, Ny, P))
        if K is not None:
            for i in range(Nu):
                dK[i, :, Nx + i * Ny:Nx + (i + 1) * Ny] = np.eye(Ny)
        for b in range(B):
            z = Z0[b].copy(); S = np.array(Sigma0[b], dtype=np.float64)
            dz = np.eye(Nx, P); dS = np.zeros((Nx, Nx, P))
            for t in range(Nt):
                m, C = orc.gp_exact_moment(self.post['invK'], self.X, self.Y, self.hyper, z, S)
                g = em_grad_oracle.em_grad_closed(self.X, self.hyper, self.post['alpha'], self.post['chol'], z[None], S)
                dm = g['dmean_dz'][0] @ dz + np.einsum('ade,dep->ap', g['dmean_dSigma'][0], dS)
                dC = np.einsum('ace,ep->acp', g['dcov_dz'][0], dz) + np.einsum('acde,dep->acp', g['dcov_dSigma'][0], dS)
                means[b, t], var[b, t], cov[b] = m, np.diag(C), C
                dmeans[b, t] = dm
                dvars[b, t] = np.einsum('aap->ap', dC)
                x, dx = m * sY + mY, dm * sY[:, None]
                z[:Ny] = (x - mX) / sX
                dz = dz.copy(); dz[:Ny] = dx / sX[:, None]
                dSn = dS.copy(); dSn[:Ny, :Ny] = dC
                if K is None:
                    z[Ny:] = U[b, t + 1] if t + 1 < Nt else 0.0
                    dz[Ny:] = 0.0
                    if t + 1 < Nt:
                        dz[Ny:, Nx + t * Nu:Nx + (t + 1) * Nu] = np.eye(Nu)
                else:
                    xt = x - xr
                    z[Ny:] = (_matmul_seq(K, xt[:, None])[:, 0] - mU) / sU
                    dz[Ny:] = (K @ dx + np.einsum('ikp,k->ip', dK, xt)) / sU[:, None]
                    dxu = np.einsum('rkp,ik->rip', dC, K) + np.einsum('rk,ikp->rip', C, dK)
                    duu = (np.einsum('ikp,kc,jc->ijp', dK, C, K) + np.einsum('ik,kcp,jc->ijp', K, dC, K)
                           + np.einsum('ik,kc,jcp->ijp', K, C, dK))
                    dSn[:Ny, Ny:] = dxu; dSn[Ny:, :Ny] = np.transpose(dxu, (1, 0, 2)); dSn[Ny:, Ny:] = duu
                    S[Ny:, Ny:] = _matmul_seq(_matmul_seq(K, C), K.T)
                    S[:Ny, Ny:] = _matmul_seq(C, K.T); S[Ny:, :Ny] = S[:Ny, Ny:].T
                S[:Ny, :Ny] = C
                dS = dSn
        return means, var, cov, dmeans, dvars


def _gp(name):
    gp, m = fixture_gp(name, OracleEngineWithRolloutBatchEmGrad, gp_method='EM')
    eng = gp.engine
    model = dict(X=eng.X, Y=eng.Y, hyper=m['hyper'], alpha=eng.post['alpha'], chol=eng.post['chol'],
                 invK=eng.post['invK'], normalize=m['normalize'], meta=m.get('meta'))     # the stand-in's own factor
    return gp, model


def _case(name, nb=1, Nt=5):
    return trajectories(name, nb, Nt, cyclic=False)


def _gain(model, x0, u0):
    A, Bm = orc.discrete_linearize(model, x0, u0)
    return rollout_oracle.lqr_gain(A, Bm, np.eye(A.shape[0]), np.eye(Bm.shape[1]))[0]


def _resolvable(name):
    """The fixture's data with each output's noise level raised to at least 0.1 std(y), and its CPU factor.  At the
    fixtures' own noise (sn ~ 1e-3 std(y)) the 'EM' variance is sf2 minus nearly equal terms (car: 2e-7 against
    cond(K) ~ 1e10), which no fp64 or long-double evaluation resolves to the digits a difference quotient needs."""
    m = load_fixture(name)
    hyper = m['hyper'].copy()
    Nx = m['X'].shape[1]
    hyper[:, Nx + 1] = np.maximum(hyper[:, Nx + 1], 0.1 * m['Y'].std(0))
    post = orc.postfit(m['X'], m['Y'], hyper, lapack_general_solve=False)
    return dict(X=m['X'], Y=m['Y'], hyper=hyper, alpha=post['alpha'], chol=post['chol'], invK=post['invK'],
                normalize=m['normalize'], meta=m.get('meta'))


# (relative step, tolerance on the mean blocks, on the variance blocks), from the agreement measured with the oracle
# (relinf over each block, Nt = 5): tank at a step of 1e-3 <= 6.3e-8 (mean) and <= 1.2e-5 (var); car at 1e-4 <= 1.3e-5
# and <= 8.3e-5, limited by the rounding of predict_compare_loop's plain fp64 'EM' formula
_FD = dict(tank=(1e-3, 1e-6, 1e-4), car=(1e-4, 1e-4, 5e-4))


@pytest.mark.parametrize('feedback', [False, True])
@pytest.mark.parametrize('name', ['tank', 'car'])
def test_oracle_equals_central_differences_of_predict_compare(name, feedback, monkeypatch):
    """The forward-mode 'EM' oracle against central differences of predict_compare_loop(methods=['EM']) with the
    gain held fixed.  From step 2 on the x block of the input covariance has off-diagonal tangents, and with feedback so
    has Sigma_xu, so a factor of two on the off-diagonal Sigma derivatives would show here."""
    model = _resolvable(name)
    X0, U, x_ref = _case(name)
    x0, u = X0[0], U[0]
    K0 = _gain(model, x0, u[0]) if feedback else None
    o = rollout_em_grad(model, x0, u, feedback=feedback, x_ref=x_ref, K=K0)
    gain = [K0]
    monkeypatch.setattr(rollout_oracle, 'lqr_gain', lambda *a: (gain[0], None))

    def loop(x, uu):
        m, v = predict_compare_loop(model, x, uu, ['EM'], feedback=feedback, x_ref=x_ref)
        return m[0], v[0]

    pm, pv = loop(x0, u)
    assert np.array_equal(o['mean'], pm) and np.array_equal(o['var'], pv)        # the same arithmetic
    rel, tm, tv = _FD[name]
    worst = []
    fm, fv = central(lambda p: loop(p, u), x0, rel)
    worst += [relinf(o['dmean_dx0'], fm), relinf(o['dvar_dx0'], fv)]
    if feedback:
        def with_gain(Kp):
            gain[0] = Kp
            return loop(x0, u)
        fm, fv = central(with_gain, K0, rel)
        worst += [relinf(o['dmean_dK'], fm), relinf(o['dvar_dK'], fv)]
    else:
        fm, fv = central(lambda p: loop(x0, p), u, rel)
        worst += [relinf(o['dmean_du'], fm), relinf(o['dvar_du'], fv)]
    print('[fd] %s fb=%s %s' % (name, feedback, ['%.1e' % w for w in worst]))
    assert max(worst[0::2]) < tm and max(worst[1::2]) < tv, worst
    assert np.abs(o['dvar_dx0']).max() > 0


@pytest.mark.parametrize('name', ['tank', 'car'])
def test_one_step_is_em_grad_closed(name):
    """At Nt = 1 the derivatives are em_grad_closed's z blocks in caller units: nothing of the Sigma blocks enters."""
    _, model = _gp(name)
    X0, U, _ = _case(name, Nt=1)
    o = rollout_em_grad(model, X0[0], U[0])
    Ny, Nx = X0.shape[1], model['X'].shape[1]
    if model['normalize']:
        st = model['meta']
        sX, sU, sY = (np.asarray(st[k], dtype=np.float64) for k in ('stdX', 'stdU', 'stdY'))
        z = np.concatenate([(X0[0] - st['meanX']) / sX, (U[0, 0] - st['meanU']) / sU])
    else:
        sX, sU, sY = np.ones(Ny), np.ones(Nx - Ny), np.ones(Ny)
        z = np.concatenate([X0[0], U[0, 0]])
    S = np.eye(Nx) * 1e-6
    S[:Ny, :Ny] = np.diag(model['hyper'][:, Nx + 1] ** 2)
    g = em_grad_oracle.em_grad_closed(model['X'], model['hyper'], model['alpha'], model['chol'], z[None], S)
    dcv = np.einsum('aae->ae', g['dcov_dz'][0])
    assert relinf(o['dmean_dx0'][1], g['dmean_dz'][0][:, :Ny] / sX * sY[:, None]) < 1e-14
    assert relinf(o['dmean_du'][1, :, 0], g['dmean_dz'][0][:, Ny:] / sU * sY[:, None]) < 1e-14
    assert relinf(o['dvar_dx0'][1], dcv[:, :Ny] / sX * (sY ** 2)[:, None]) < 1e-14
    assert relinf(o['dvar_du'][1, :, 0], dcv[:, Ny:] / sU * (sY ** 2)[:, None]) < 1e-14


@pytest.mark.parametrize('feedback', [False, True])
@pytest.mark.parametrize('name', ['tank', 'car'])
def test_rollout_grad_mapping_equals_the_oracle(name, feedback):
    """GP.rollout_grad(method='EM') through the restated entry: the scalers of z0, u_0 = K (x0 - x_ref) in z0's tail, stdY
    and stdY^2 on the outputs; B = 1 and a batch of two; with feedback one pass per distinct gain, here two distinct gains
    and then one gain shared by both trajectories."""
    gp, model = _gp(name)
    X0, U, x_ref = _case(name, nb=2)
    kw = dict(feedback=feedback, x_ref=x_ref if feedback else None)
    calls = OracleEngineWithRolloutBatchEmGrad.calls
    del calls[:]
    r = gp.rollout_grad(X0, U, method='EM', **kw)
    assert calls == ([1, 1] if feedback else [2])
    Ny, Nu, Nt = X0.shape[1], U.shape[2], U.shape[1]
    keys = ('dmean_dK', 'dvar_dK') if feedback else ('dmean_du', 'dvar_du')
    assert r[keys[0]].shape == ((2, Nt + 1, Ny, Nu, Ny) if feedback else (2, Nt + 1, Ny, Nt, Nu))
    for b in range(2):
        K = _gain(model, X0[b], U[b, 0]) if feedback else None
        o = rollout_em_grad(model, X0[b], U[b], feedback=feedback, x_ref=x_ref, K=K)
        for k in ('mean', 'var', 'dmean_dx0', 'dvar_dx0') + keys:
            assert relinf(r[k][b], o[k]) < 1e-10, (k, b, relinf(r[k][b], o[k]))
        s = gp.rollout_grad(X0[b], U[b], method='EM', **kw)
        for k in s:
            assert relinf(s[k], r[k][b]) < 1e-13, (k, b)
    assert np.array_equal(r['dmean_dx0'][:, 0], np.tile(np.eye(Ny), (2, 1, 1))) and not r['dvar_dx0'][:, 0].any()
    assert not r[keys[0]][:, 0].any() and not r[keys[1]][:, 0].any()
    if feedback:                                        # one linearisation point: one gain, one pass of two trajectories
        X0[1] = X0[0]; U[1, 0] = U[0, 0]
        del calls[:]
        r2 = gp.rollout_grad(X0, U, method='EM', **kw)
        assert calls == [2]
        for k in r2:
            assert np.array_equal(r2[k][0], r2[k][1]), k


def test_default_method_and_autonomous_model():
    """method defaults to the GP's gp_method ('EM' here); Nu = 0 has only the start as parameter."""
    gp, model = _gp('tank')
    X0, U, _ = _case('tank', Nt=3)
    r = gp.rollout_grad(X0[0], U[0])
    o = rollout_em_grad(model, X0[0], U[0])
    assert relinf(r['dmean_du'], o['dmean_du']) < 1e-10
    rng = np.random.default_rng(1)
    X = rng.standard_normal((20, 2)); Y = X + 0.1 * rng.standard_normal((20, 2))
    hyper = np.array([[1., 1., 1., .1], [1., 1., 1., .1]])
    auto = gp_mpc_b200.GP(X, Y, normalize=False, hyper=dict(hyper=hyper), engine_factory=OracleEngineWithRolloutBatchEmGrad)
    a = auto.rollout_grad(np.array([0.3, -0.2]), np.zeros((4, 0)), method='EM')
    e = auto.engine
    m = dict(X=e.X, Y=e.Y, hyper=hyper, alpha=e.post['alpha'], chol=e.post['chol'], invK=e.post['invK'], normalize=False)
    o = rollout_em_grad(m, np.array([0.3, -0.2]), np.zeros((4, 0)))
    assert a['dmean_du'].shape == (5, 2, 4, 0)
    assert relinf(a['dmean_dx0'], o['dmean_dx0']) < 1e-10 and relinf(a['dvar_dx0'], o['dvar_dx0']) < 1e-10


def test_rollout_batch_em_grad_is_declared_and_bound():
    hdr = open(os.path.join(ROOT, 'include', 'gpmpc.h')).read()
    assert re.search(r'\bint gpmpc_rollout_batch_em_grad\s*\(', hdr)
    import __graft_entry__ as g
    g.build()
    L = gp_mpc_b200._lib
    assert 'gpmpc_rollout_batch_em_grad' in {s[0] for s in L.SYMBOLS}
    assert L.load().gpmpc_rollout_batch_em_grad is not None
    assert hasattr(gp_mpc_b200.Engine, 'rollout_batch_em_grad')
