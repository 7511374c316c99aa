"""GP.rollout_grad and its checker on CPU: the forward-mode oracle (oracle/rollout_grad_oracle.py) against central
differences of predict_compare_loop, and GP.rollout_grad's caller-unit mapping through a numpy restatement of
gpmpc_rollout_batch_grad.  The device entry is covered by tests/test_rollout_grad_gpu.py."""
import os
import re

import numpy as np
import pytest

import gp_mpc_b200
from gp_mpc_b200.gp_class import _matmul_seq
from oracle import hess_oracle, rollout_oracle
from oracle.rollout_grad_oracle import rollout_grad
from oracle.rollout_oracle import predict_compare_loop
from tests._fake_engine import OracleEngine, OracleEngineWithRolloutBatch, TwoRanks, fixture_gp, sharded
from tests._util import central, load_fixture, relinf, trajectories

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class OracleEngineWithRolloutBatchGrad(OracleEngineWithRolloutBatch):
    """Adds a numpy restatement of gpmpc_rollout_batch_grad (include/gpmpc.h): the primal is rollout_batch's, the tangents
    follow the entry's recurrences in the GP's units with J, dvar / dz, dcov / dz from hess_oracle.predict_grad_closed."""

    def rollout_batch_grad(self, z0, U, Sigma0, method=1, scale=None, K=None, x_ref=None, uscale=None):
        means, var, cov = self.rollout_batch(z0, U, Sigma0, method, scale, K, x_ref, uscale)
        Ny, Nx = self.Ny, self.Nx
        Nu = Nx - Ny
        Z0 = np.array(z0, dtype=np.float64).reshape(-1, Nx)
        B, Nt = Z0.shape[0], np.shape(U)[1]
        P = Nx + (Nu * Ny if K is not None else (Nt - 1) * Nu)
        dmeans = np.zeros((B, Nt, Ny, P)); dvars = np.zeros((B, Nt, Ny, P))
        ta = method == gp_mpc_b200._lib.METHOD_TA
        sY, mY, mX, sX = (np.ones(Ny), np.zeros(Ny), np.zeros(Ny), np.ones(Ny)) if scale is None else scale
        mU, sU = (np.zeros(Nu), np.ones(Nu)) if uscale is None else uscale
        xr = np.zeros(Ny) if x_ref is None else x_ref
        for b in range(B):
            z = Z0[b].copy(); S = np.array(Sigma0[b], dtype=np.float64)
            dz = np.eye(Nx, P); dS = np.zeros((Nx, Nx, P))
            for t in range(Nt):
                g = hess_oracle.predict_grad_closed(self.X, self.hyper, self.post['alpha'], self.post['chol'], z[None], S,
                                                    'TA' if ta else 'ME')
                J, m = g['dmean'][0], g['mean'][0]
                dm = J @ dz
                if ta:
                    C = np.diag(g['var'][0]) + J @ S @ J.T
                    dC = np.einsum('ace,ep->acp', g['dcov'][0], dz) + np.einsum('ae,efp,cf->acp', J, dS, J)
                else:
                    C = np.diag(g['var'][0])
                    dC = np.zeros((Ny, Ny, P)); dC[np.arange(Ny), np.arange(Ny)] = g['dvar'][0] @ dz
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
                    dK = np.zeros((Nu, Ny, P))
                    for i in range(Nu):
                        dK[i, :, Nx + i * Ny:Nx + (i + 1) * Ny] = np.eye(Ny)
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


def _gp(name, factory=OracleEngineWithRolloutBatchGrad):
    gp, m = fixture_gp(name, factory)
    model = dict(X=m['X'], Y=m['Y'], hyper=m['hyper'], alpha=gp.get_alpha(), chol=gp.get_chol(),
                 normalize=m['normalize'], meta=m.get('meta'))          # the stand-in engine's own factor
    return gp, model


def _case(name, nb=1, Nt=6):
    return trajectories(name, nb, Nt, cyclic=False)


def _gain(model, x0, u0):
    A, Bm = rollout_oracle.orc.discrete_linearize(model, x0, u0)
    return rollout_oracle.lqr_gain(A, Bm, np.eye(A.shape[0]), np.eye(Bm.shape[1]))[0]


# (relative step, tolerance on the mean blocks, on the variance blocks), from the agreement measured with the oracle
# (relinf over each block).  tank at a step of 1e-4: <= 4e-7 (mean), <= 1.5e-5 (var); smaller steps are limited by the
# rounding of the roll-out (2.6e-6 / 1e-3 at 1e-6).  car at 3e-6: <= 4.9e-5 (mean) and, for 'ME' open loop, 2.2e-3 (var):
# its variances are small differences sf2 - |L^-1 k|^2, and larger steps meet the curvature (0.7 at 1e-4)
_FD = dict(tank=(1e-4, 1e-6, 5e-5), car=(3e-6, 1e-4, 5e-3))


@pytest.mark.parametrize('feedback', [False, True])
@pytest.mark.parametrize('method', ['TA', 'ME'])
@pytest.mark.parametrize('name', ['tank', 'car'])
def test_oracle_equals_central_differences_of_predict_compare(name, method, feedback, monkeypatch):
    """rollout_grad_oracle's forward mode against central differences of predict_compare_loop itself, with the gain held
    fixed (lqr_gain stubbed to return it) so that x0 and K can be perturbed on their own."""
    gp, model = _gp(name, OracleEngine)
    X0, U, x_ref = _case(name)
    x0, u = X0[0], U[0]
    K0 = _gain(model, x0, u[0]) if feedback else None
    o = rollout_grad(model, x0, u, method, feedback=feedback, x_ref=x_ref, K=K0)
    gain = [K0]
    monkeypatch.setattr(rollout_oracle, 'lqr_gain', lambda *a: (gain[0], None))

    def loop(x, uu):
        m, v = predict_compare_loop(model, x, uu, [method], feedback=feedback, x_ref=x_ref)
        return m[0], v[0]

    pm, pv = loop(x0, u)
    assert relinf(o['mean'], pm) < 1e-12 and relinf(o['var'], pv) < 1e-10       # J: another summation order than gp_mean_jac
    rel, tm, tv = _FD[name]
    fm, fv = central(lambda p: loop(p, u), x0, rel)
    assert relinf(o['dmean_dx0'], fm) < tm and relinf(o['dvar_dx0'], fv) < tv
    if feedback:
        def with_gain(Kp):
            gain[0] = Kp
            return loop(x0, u)
        fm, fv = central(with_gain, K0, rel)
        assert relinf(o['dmean_dK'], fm) < tm and relinf(o['dvar_dK'], fv) < tv
    else:
        fm, fv = central(lambda p: loop(x0, p), u, rel)
        assert relinf(o['dmean_du'], fm) < tm and relinf(o['dvar_du'], fv) < tv
    assert np.abs(o['dvar_dx0']).max() > 0                     # the variance really depends on the start


@pytest.mark.parametrize('feedback', [False, True])
@pytest.mark.parametrize('method', ['TA', 'ME'])
@pytest.mark.parametrize('name', ['tank', 'car'])
def test_rollout_grad_mapping_equals_the_oracle(name, method, feedback):
    """GP.rollout_grad through the restated entry: the scalers of z0, u_0 = K (x0 - x_ref) in z0's tail, stdY and stdY^2
    on the outputs, one pass per distinct gain; single and batched shapes; mean / var are GP.rollout's."""
    gp, model = _gp(name)
    X0, U, x_ref = _case(name, nb=2)
    kw = dict(feedback=feedback, x_ref=x_ref if feedback else None)
    r = gp.rollout_grad(X0, U, method=method, **kw)
    rm, rv = gp.rollout(X0, U, methods=[method], **kw)
    assert np.array_equal(r['mean'], rm[0]) and np.array_equal(r['var'], rv[0])
    Ny, Nu, Nt = X0.shape[1], U.shape[2], U.shape[1]
    keys = ('dmean_dK', 'dvar_dK') if feedback else ('dmean_du', 'dvar_du')
    assert not any(k in r for k in (('dmean_du', 'dvar_du') if feedback else ('dmean_dK', 'dvar_dK')))
    assert r['dmean_dx0'].shape == (2, Nt + 1, Ny, Ny)
    assert r[keys[0]].shape == ((2, Nt + 1, Ny, Nu, Ny) if feedback else (2, Nt + 1, Ny, Nt, Nu))
    for b in range(2):
        o = rollout_grad(model, X0[b], U[b], method, feedback=feedback, x_ref=x_ref)
        for k in ('mean', 'var', 'dmean_dx0', 'dvar_dx0') + keys:
            assert relinf(r[k][b], o[k]) < 1e-10, (k, b)
        s = gp.rollout_grad(X0[b], U[b], method=method, **kw)
        for k in s:
            assert relinf(s[k], r[k][b]) < 1e-13, (k, b)
    assert np.array_equal(r['dmean_dx0'][:, 0], np.tile(np.eye(Ny), (2, 1, 1))) and not r['dvar_dx0'][:, 0].any()
    assert not r[keys[0]][:, 0].any() and not r[keys[1]][:, 0].any()


def test_default_method_and_autonomous_model():
    """method defaults to the GP's gp_method; Nu = 0 has only the start as parameter."""
    gp, model = _gp('tank')
    X0, U, _ = _case('tank')
    gp.set_method('ME')
    r = gp.rollout_grad(X0[0], U[0])
    o = rollout_grad(model, X0[0], U[0], 'ME')
    assert relinf(r['dmean_du'], o['dmean_du']) < 1e-10
    rng = np.random.default_rng(1)
    X = rng.standard_normal((20, 2)); Y = X + 0.1 * rng.standard_normal((20, 2))
    hyper = np.array([[1., 1., 1., .1], [1., 1., 1., .1]])
    auto = gp_mpc_b200.GP(X, Y, normalize=False, hyper=dict(hyper=hyper), engine_factory=OracleEngineWithRolloutBatchGrad)
    a = auto.rollout_grad(np.array([0.3, -0.2]), np.zeros((5, 0)), method='TA')
    m = dict(X=X, Y=Y, hyper=hyper, alpha=auto.get_alpha(), chol=auto.get_chol(), normalize=False)
    o = rollout_grad(m, np.array([0.3, -0.2]), np.zeros((5, 0)), 'TA')
    assert a['dmean_du'].shape == (6, 2, 5, 0)
    assert relinf(a['dmean_dx0'], o['dmean_dx0']) < 1e-10 and relinf(a['dvar_dx0'], o['dvar_dx0']) < 1e-10


_ShardEngine = sharded(OracleEngineWithRolloutBatchGrad)


def test_not_implemented_cases():
    gp, m = _gp('tank')
    X0, U, _ = _case('tank')
    with pytest.raises(NotImplementedError, match="'ME' and 'TA'"):
        gp.rollout_grad(X0[0], U[0], method='EM')
    with pytest.raises(ValueError):
        gp.rollout_grad(X0[0], np.zeros((0, 2)))
    fm = load_fixture('tank')
    sh = gp_mpc_b200.GP(fm['X'], fm['Y'], normalize=False, hyper=dict(hyper=fm['hyper']), comm=TwoRanks(),
                        engine_factory=_ShardEngine)
    with pytest.raises(NotImplementedError, match='needs all outputs on one GPU'):
        sh.rollout_grad(X0[0], U[0])
    pm = gp_mpc_b200.GP(fm['X'], fm['Y'], normalize=False, mean_func='const', prior_mean_in_predict=True,
                        hyper=dict(hyper=np.column_stack([fm['hyper'], np.full(4, 0.1)])),
                        engine_factory=OracleEngineWithRolloutBatchGrad)
    with pytest.raises(NotImplementedError, match='prior_mean_in_predict'):
        pm.rollout_grad(X0[0], U[0])


def test_rollout_batch_grad_is_declared_and_bound():
    hdr = open(os.path.join(ROOT, 'include', 'gpmpc.h')).read()
    assert re.search(r'\bint gpmpc_rollout_batch_grad\s*\(', hdr)
    import __graft_entry__ as g
    g.build()
    L = gp_mpc_b200._lib
    assert 'gpmpc_rollout_batch_grad' in {s[0] for s in L.SYMBOLS}
    assert L.load().gpmpc_rollout_batch_grad is not None
