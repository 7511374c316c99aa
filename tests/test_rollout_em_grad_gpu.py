"""gpmpc_rollout_batch_em_grad on the device: the roll-out of gpmpc_rollout_batch_em bit for bit, plus the forward-mode
derivatives of every step's mean and variance w.r.t. the start, the inputs or the feedback gain, chained on the engine's
own gpmpc_predict_em_grad blocks, against central differences of gpmpc_rollout_batch_em and against the forward-mode 'EM'
oracle of tests/_rollout_em_grad_oracle.py with the CPU factor."""
import ctypes

import numpy as np
import pytest

from gp_mpc_b200 import _lib as L
from oracle import gp_oracle as orc
from oracle.rollout_oracle_ld import feedback_inputs64
from tests._em_cases import feedback_sigma
from tests._engines import lqr_gain
from tests._rollout_em_grad_oracle import rollout_em_grad
from tests._util import assert_same, load_fixture, relinf, trajectories

pytestmark = pytest.mark.gpu


def _gp(name, sn_floor=None):
    """A GP on the device and the CPU model of the same data (its own Cholesky factor) for the oracle.  sn_floor raises each
    output's noise level to at least sn_floor std(y) (see _FD_TOL)."""
    import gp_mpc_b200
    if name == 'synthetic':
        from bench import WORKLOADS, make_workload
        wl = WORKLOADS['c2']
        w = make_workload(wl['N'], wl['Nx'], wl['Ny'], wl['cfg'], wl['H'])
        m = dict(X=w['X'], Y=w['Y'], hyper=w['hyper'].copy(), normalize=False, Z=w['Z'])
    else:
        m = dict(load_fixture(name))
        m['hyper'] = m['hyper'].copy()
    Nx = m['X'].shape[1]
    if sn_floor is not None:
        m['hyper'][:, Nx + 1] = np.maximum(m['hyper'][:, Nx + 1], sn_floor * m['Y'].std(0))
    kw = dict(mean_func='zero', gp_method='EM', normalize=m['normalize'], hyper=dict(hyper=m['hyper']))
    if m['normalize']:
        kw.update(meta=m['meta'], xlb=m['xlb'], xub=m['xub'], ulb=m['ulb'], uub=m['uub'])
    return gp_mpc_b200.GP(m['X'], m['Y'], **kw), m


def _model(m):
    post = orc.postfit(m['X'], m['Y'], m['hyper'], lapack_general_solve=False)
    return dict(X=m['X'], Y=m['Y'], hyper=m['hyper'], alpha=post['alpha'], chol=post['chol'], invK=post['invK'],
                normalize=m['normalize'], meta=m.get('meta'))


def _case(name, m, nb, Nt):
    if name == 'synthetic':
        Ny = m['Y'].shape[1]
        rows = m['Z'][np.arange(nb) % m['Z'].shape[0]]
        X0 = rows[:, :Ny]
        U = np.repeat(rows[:, None, Ny:], Nt, 1) * (1 + 0.01 * np.arange(Nt)[None, :, None])
        return X0, U, 0.5 * X0[0]
    return trajectories(name, nb, Nt, cyclic=True)


def _inputs(m, X0, U, K=None, x_ref=None):
    """The engine's arguments as GP.rollout forms them: z0, U and Sigma0 in GP units, and the policy keywords."""
    Ny, Nx = X0.shape[1], m['X'].shape[1]
    Nu = Nx - Ny
    un = U if K is None else np.stack([K @ (x - x_ref) for x in X0])[:, None, :]
    scale = uscale = None
    zx = X0
    if m['normalize']:
        st = m['meta']
        zx = (X0 - st['meanX']) / st['stdX']
        un = (un - st['meanU']) / st['stdU']
        scale = np.stack([st['stdY'], st['meanY'], st['meanX'], st['stdX']])
        uscale = np.stack([st['meanU'], st['stdU']])
    S = np.tile(np.eye(Nx) * 1e-6, (X0.shape[0], 1, 1))
    S[:, :Ny, :Ny] = np.diag(m['hyper'][:, Nx + 1] ** 2)
    pol = dict(scale=scale)
    if K is not None:
        pol.update(K=K, x_ref=x_ref, uscale=uscale)
    return np.concatenate([zx, un[:, 0, :Nu]], 1), (un if K is None else U), S, pol


@pytest.mark.parametrize('B', [1, 3, 5])
@pytest.mark.parametrize('name', ['tank', 'car', 'synthetic'])
def test_rollout_is_rollout_batch_em_bit_for_bit(name, B):
    """means, vars, cov_last equal gpmpc_rollout_batch_em's, open loop and with feedback, with em_points = 2 so that chunk
    boundaries fall inside the batch; the derivatives are finite and have the documented shape."""
    gp, m = _gp(name)
    eng = gp.engine
    eng.set_option('em_points', 2)
    X0, U, x_ref = _case(name, m, B, 4)
    Ny, Nx = X0.shape[1], m['X'].shape[1]
    Nu = Nx - Ny
    K = lqr_gain(gp, X0, U)
    for fb in (False, True):
        z0, Ug, S, pol = _inputs(m, X0, U, K if fb else None, x_ref)
        ref = eng.rollout_batch_em(z0, Ug, S, **pol)
        got = eng.rollout_batch_em_grad(z0, Ug, S, **pol)
        assert_same(ref, got[:3])
        P = Nx + (Nu * Ny if fb else 3 * Nu)
        assert got[3].shape == got[4].shape == (B, 4, Ny, P)
        assert np.isfinite(got[3]).all() and np.isfinite(got[4]).all()
    gp.close()


@pytest.mark.parametrize('name', ['tank', 'car'])
def test_one_trajectory_equals_its_row_and_calls_repeat(name):
    """Trajectory b alone equals row b of a batch bit for bit; two identical calls, and calls under other em_points caps,
    give identical bits."""
    gp, m = _gp(name)
    eng = gp.engine
    X0, U, x_ref = _case(name, m, 5, 5)
    K = lqr_gain(gp, X0, U)
    for fb in (False, True):
        z0, Ug, S, pol = _inputs(m, X0, U, K if fb else None, x_ref)
        eng.set_option('em_points', 0)
        full = eng.rollout_batch_em_grad(z0, Ug, S, **pol)
        assert_same(full, eng.rollout_batch_em_grad(z0, Ug, S, **pol))
        for cap in (1, 2):
            eng.set_option('em_points', cap)
            assert_same(full, eng.rollout_batch_em_grad(z0, Ug, S, **pol))
        eng.set_option('em_points', 0)
        for b in (0, 3):
            one = eng.rollout_batch_em_grad(z0[b:b + 1], Ug[b:b + 1], S[b:b + 1], **pol)
            assert_same([x[b] for x in full], [x[0] for x in one])
    gp.close()


def _chain(eng, z0, U, S0, means, covs, scale=None, K=None, x_ref=None, uscale=None):
    """The entry's recurrence in numpy on Engine.predict_em_grad's blocks at the engine's own (z_t, Sigma_t): z_t from
    feedback_inputs64 of the engine's means, Sigma_t from the cov_last of its t-step prefix (covs[t-1])."""
    B, Nx = z0.shape
    Ny = means.shape[2]
    Nu, Nt = Nx - Ny, means.shape[1]
    P = Nx + (Nu * Ny if K is not None else (Nt - 1) * Nu)
    sY, mY, _, sX = (np.ones(Ny), np.zeros(Ny), None, np.ones(Ny)) if scale is None else scale
    sU = np.ones(Nu) if uscale is None else uscale[1]
    xr = np.zeros(Ny) if x_ref is None else x_ref
    dK = np.zeros((Nu, Ny, P))
    if K is not None:
        for i in range(Nu):
            dK[i, :, Nx + i * Ny:Nx + (i + 1) * Ny] = np.eye(Ny)
    dmeans = np.zeros((B, Nt, Ny, P)); dvars = np.zeros((B, Nt, Ny, P))
    dz = np.tile(np.eye(Nx, P), (B, 1, 1)); dS = np.zeros((B, Nx, Nx, P))
    for t in range(Nt):
        if t == 0:
            z, S = z0, S0
        else:
            z = feedback_inputs64(means[:, t - 1], scale, K, x_ref, uscale, U[:, t] if K is None else None)
            S = np.stack([feedback_sigma(S0[b], covs[t - 1][b], K) for b in range(B)])
        g = eng.predict_em_grad(z, S)
        for b in range(B):
            dm = g['dmean_dz'][b] @ dz[b] + np.einsum('ade,dep->ap', g['dmean_dSigma'][b], dS[b])
            dC = np.einsum('ace,ep->acp', g['dcov_dz'][b], dz[b]) + np.einsum('acde,dep->acp', g['dcov_dSigma'][b], dS[b])
            dmeans[b, t] = dm
            dvars[b, t] = np.einsum('aap->ap', dC)
            C = g['cov'][b]
            dx = dm * sY[:, None]
            dzn = np.zeros((Nx, P)); dzn[:Ny] = dx / sX[:, None]
            dSn = dS[b].copy(); dSn[:Ny, :Ny] = dC
            if K is None:
                if t + 1 < Nt:
                    dzn[Ny:, Nx + t * Nu:Nx + (t + 1) * Nu] = np.eye(Nu)
            else:
                xt = means[b, t] * sY + mY - xr
                dzn[Ny:] = (K @ dx + np.einsum('ikp,k->ip', dK, xt)) / sU[:, None]
                dxu = np.einsum('rkp,ik->rip', dC, K) + np.einsum('rk,ikp->rip', C, dK)
                duu = (np.einsum('ikp,kc,jc->ijp', dK, C, K) + np.einsum('ik,kcp,jc->ijp', K, dC, K)
                       + np.einsum('ik,kc,jcp->ijp', K, C, dK))
                dSn[:Ny, Ny:] = dxu; dSn[Ny:, :Ny] = np.transpose(dxu, (1, 0, 2)); dSn[Ny:, Ny:] = duu
            dz[b], dS[b] = dzn, dSn
    return dmeans, dvars


# measured on an H100 80GB HBM3 at 700 W (relinf over each block, Nt = 4, B = 3): <= 2.2e-15 (car with feedback), <= 1.5e-15
# otherwise; the numpy chain sums in other orders than the tangent kernel
_CHAIN_TOL = 1e-13


@pytest.mark.parametrize('fb', [False, True])
@pytest.mark.parametrize('name', ['tank', 'car', 'synthetic'])
def test_chain_on_the_engines_own_derivatives(name, fb):
    """The tangent kernel alone: dmeans / dvars against the recurrence chained in numpy on Engine.predict_em_grad's blocks
    at the engine's own step inputs (a prefix roll-out's cov_last is the full roll-out's step, bit for bit)."""
    gp, m = _gp(name)
    eng = gp.engine
    X0, U, x_ref = _case(name, m, 3, 4)
    K = lqr_gain(gp, X0, U) if fb else None
    z0, Ug, S, pol = _inputs(m, X0, U, K, x_ref)
    means, _, _, dm, dv = eng.rollout_batch_em_grad(z0, Ug, S, **pol)
    covs = [eng.rollout_batch_em(z0, Ug[:, :t], S, **pol)[2] for t in range(1, 4)]
    cm, cv = _chain(eng, z0, Ug, S, means, covs, **pol)
    em, ev = relinf(dm, cm), relinf(dv, cv)
    print('[chain] %s fb=%s dmeans %.2e dvars %.2e' % (name, fb, em, ev))
    assert em < _CHAIN_TOL and ev < _CHAIN_TOL, (em, ev)
    gp.close()


# measured on an H100 80GB HBM3 at 700 W (central differences at a relative step of 1e-4, Nt = 6, relinf over each block):
# tank 3.4e-10 (dmeans) and 2.2e-8 (dvars), synthetic 3.5e-8 and 1.9e-6.  tank runs with its noise level raised to 0.1 std(y):
# at the fixture's own sn (~3e-3) its 'EM' variance is sf2 minus nearly equal terms, which fp64 does not resolve to the
# digits a difference quotient needs.
_FD_TOL = dict(mean=1e-7, var=1e-5)


@pytest.mark.parametrize('fb', [False, True])
@pytest.mark.parametrize('name', ['tank', 'synthetic'])
def test_derivatives_equal_central_differences_on_the_device(name, fb):
    """dmeans / dvars against central differences of gpmpc_rollout_batch_em on the same device in every parameter: z0, then
    the U rows 1..Nt-1 open loop or the entries of K with feedback.  No CPU factor is involved."""
    gp, m = _gp(name, sn_floor=0.1 if name == 'tank' else None)
    eng = gp.engine
    Nt = 6
    X0, U, x_ref = _case(name, m, 2, Nt)
    K = lqr_gain(gp, X0, U) if fb else None
    z0, Ug, S, pol = _inputs(m, X0, U, K, x_ref)
    Ny, Nx = X0.shape[1], z0.shape[1]
    Nu = Nx - Ny
    _, _, _, dm, dv = eng.rollout_batch_em_grad(z0, Ug, S, **pol)
    P = dm.shape[-1]
    assert P == Nx + (Nu * Ny if fb else (Nt - 1) * Nu)
    fm = np.zeros_like(dm); fv = np.zeros_like(dv)
    rel = 1e-4
    for p in range(P):
        zp, zm, Up, Um = z0.copy(), z0.copy(), Ug.copy(), Ug.copy()
        pp, pm = dict(pol), dict(pol)
        if p < Nx:
            h = rel * np.maximum(1.0, np.abs(z0[:, p]))
            zp[:, p] += h; zm[:, p] -= h
        elif not fb:
            r, i = 1 + (p - Nx) // Nu, (p - Nx) % Nu
            h = rel * np.maximum(1.0, np.abs(Ug[:, r, i]))
            Up[:, r, i] += h; Um[:, r, i] -= h
        else:
            i, k = (p - Nx) // Ny, (p - Nx) % Ny
            h = np.full(2, rel * max(1.0, abs(K[i, k])))
            pp['K'] = K.copy(); pp['K'][i, k] += h[0]
            pm['K'] = K.copy(); pm['K'][i, k] -= h[0]
        mp, vp, _ = eng.rollout_batch_em(zp, Up, S, **pp)
        mm, vm, _ = eng.rollout_batch_em(zm, Um, S, **pm)
        fm[..., p] = (mp - mm) / (2 * h[:, None, None])
        fv[..., p] = (vp - vm) / (2 * h[:, None, None])
    em, ev = relinf(dm, fm), relinf(dv, fv)
    print('[fd] %s fb=%s dmeans %.2e dvars %.2e' % (name, fb, em, ev))
    assert em < _FD_TOL['mean'] and ev < _FD_TOL['var'], (em, ev)
    gp.close()


# (mean blocks, variance blocks), measured on an H100 80GB HBM3 at 700 W, worst block: tank 2.9e-8 and 2.0e-3, synthetic
# 4.2e-9 and 6.3e-5, car (noise raised) 5.3e-8 and 2.6e-7.  The oracle's primal is the reference's plain fp64 'EM' formula,
# whose variance loses digits to the beta beta^T - K^-1 cancellation, and the next step's Sigma carries that into the
# derivatives.  At car's own noise level that variance is not resolved at all (0.99 on the variance blocks), so car runs
# with its noise raised to 0.1 std(y).
_ORACLE_TOL = dict(tank=(1e-7, 5e-3), car=(1e-6, 1e-5), synthetic=(1e-7, 2e-4))


@pytest.mark.parametrize('fb', [False, True])
@pytest.mark.parametrize('name', ['tank', 'car', 'synthetic'])
def test_rollout_grad_equals_the_oracle(name, fb):
    """GP.rollout_grad(method='EM') in caller units against the 'EM' oracle with the CPU factor and the same gain; its mean /
    var are GP.rollout(methods=['EM'])'s bit for bit."""
    gp, m = _gp(name, sn_floor=0.1 if name == 'car' else None)
    model = _model(m)
    nb, Nt = (1, 3) if name == 'synthetic' else (2, 4)
    X0, U, x_ref = _case(name, m, nb, Nt)
    kw = dict(feedback=fb, x_ref=x_ref if fb else None)
    r = gp.rollout_grad(X0, U, method='EM', **kw)
    rm, rv = gp.rollout(X0, U, methods=['EM'], **kw)
    assert np.array_equal(r['mean'], rm[0]) and np.array_equal(r['var'], rv[0])
    keys = ('dmean_dx0', 'dvar_dx0') + (('dmean_dK', 'dvar_dK') if fb else ('dmean_du', 'dvar_du'))
    worst = dict(mean=0.0, var=0.0)
    for b in range(nb):
        K = gp._GP__lqr_gains(X0[b:b + 1], U[b:b + 1, 0], np.eye(X0.shape[1]), np.eye(U.shape[2]))[0] if fb else None
        o = rollout_em_grad(model, X0[b], U[b], feedback=fb, x_ref=x_ref, K=K)
        for k in keys:
            w = 'var' if 'var' in k else 'mean'
            worst[w] = max(worst[w], relinf(r[k][b], o[k]))
    print('[oracle] %s fb=%s mean %.2e var %.2e' % (name, fb, worst['mean'], worst['var']))
    assert worst['mean'] < _ORACLE_TOL[name][0] and worst['var'] < _ORACLE_TOL[name][1], worst
    gp.close()


def test_autonomous_model_has_the_start_as_only_parameter():
    """Nu = 0: P = Nx; GP.rollout_grad against the oracle with the CPU factor."""
    import gp_mpc_b200
    rng = np.random.default_rng(12)
    X = rng.uniform(-2, 2, (40, 2))
    Y = np.column_stack([X[:, 0] + 0.1 * X[:, 1], X[:, 1] + 0.1 * (-X[:, 0] + (1 - X[:, 0] ** 2) * X[:, 1])])
    Y = Y + 2e-2 * rng.standard_normal(Y.shape)
    hyper = np.column_stack([np.full((2, 2), 1.5), np.full(2, 1.2), np.full(2, 0.05)])
    gp = gp_mpc_b200.GP(X, Y, normalize=False, gp_method='EM', hyper=dict(hyper=hyper))
    X0 = np.array([[1.0, 0.5], [-0.5, 1.5]])
    out = gp.engine.rollout_batch_em_grad(X0, np.zeros((2, 8, 0)), np.tile(np.eye(2) * 1e-3, (2, 1, 1)))
    assert out[3].shape == (2, 8, 2, 2)
    assert_same(gp.engine.rollout_batch_em(X0, np.zeros((2, 8, 0)), np.tile(np.eye(2) * 1e-3, (2, 1, 1))), out[:3])
    model = _model(dict(X=X, Y=Y, hyper=hyper, normalize=False))
    r = gp.rollout_grad(X0, np.zeros((2, 8, 0)), method='EM')
    assert r['dmean_du'].shape == (2, 9, 2, 8, 0)
    worst = 0.0
    for b in range(2):
        o = rollout_em_grad(model, X0[b], np.zeros((8, 0)))
        worst = max(worst, relinf(r['dmean_dx0'][b], o['dmean_dx0']), relinf(r['dvar_dx0'][b], o['dvar_dx0']))
    print('[autonomous] %.2e' % worst)
    assert worst < 1e-6, worst
    gp.close()


def test_error_codes():
    import gp_mpc_b200
    lib = L.load()
    p = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    gp, m = _gp('tank')
    eng = gp.engine
    Nx, Ny = 6, 4
    z0 = m['X'][:2].copy(); U = np.zeros((2, 3, 2)); S = np.tile(np.eye(Nx) * 1e-3, (2, 1, 1))
    out = np.full(2 * 3 * Ny * 64, 7.0)
    o = p(out)
    rg = lambda B, Nt, z, u, s, mo, dmo, dvo: lib.gpmpc_rollout_batch_em_grad(eng.h, B, Nt, z, u, s, None, None, None,
                                                                               None, mo, mo, None, dmo, dvo)
    assert rg(0, 3, p(z0), p(U), p(S), o, o, o) == L.ERR_ARG          # B < 1
    assert rg(2, 0, p(z0), p(U), p(S), o, o, o) == L.ERR_ARG          # Nt < 1
    assert rg(2, 3, None, p(U), p(S), o, o, o) == L.ERR_ARG           # z0
    assert rg(2, 3, p(z0), None, p(S), o, o, o) == L.ERR_ARG          # U, open loop
    assert rg(2, 3, p(z0), p(U), None, o, o, o) == L.ERR_ARG          # Sigma0
    assert rg(2, 3, p(z0), p(U), p(S), None, o, o) == L.ERR_ARG       # means / vars
    assert rg(2, 3, p(z0), p(U), p(S), o, None, o) == L.ERR_ARG       # dmeans
    assert rg(2, 3, p(z0), p(U), p(S), o, o, None) == L.ERR_ARG       # dvars
    assert (out == 7.0).all()                                         # checked before any work
    # Sigma + Lambda not positive definite at step 0 for trajectory 1: ERR_ARG naming both; a correct call afterwards
    good = eng.rollout_batch_em_grad(z0, U, S)
    bad = S.copy()
    bad[1, 0, 0] = -1e3
    with pytest.raises(L.GpmpcError) as e:
        eng.rollout_batch_em_grad(z0, U, bad)
    assert e.value.code == L.ERR_ARG and 'step 0' in str(e.value) and 'trajectory 1' in str(e.value)
    assert_same(good, eng.rollout_batch_em_grad(z0, U, S))
    # gpmpc_rollout_batch_grad keeps rejecting 'EM'
    assert lib.gpmpc_rollout_batch_grad(eng.h, L.METHOD_EM, 2, 3, p(z0), p(U), p(S), None, None, None, None, o, o, None,
                                        o, o) == L.ERR_ARG
    gp.close()
    # not factorised
    e2 = gp_mpc_b200.Engine(m['X'].shape[0], Nx, Ny, device=0)
    e2.set_data(m['X'], m['Y']); e2.set_hyper(m['hyper'])
    with pytest.raises(L.GpmpcError) as e:
        e2.rollout_batch_em_grad(z0, U, S)
    assert e.value.code == L.ERR_STATE
    e2.close()
    # a handle that owns only some outputs
    e3 = gp_mpc_b200.Engine(m['X'].shape[0], Nx, Ny, out_begin=0, out_count=2, device=0)
    e3.set_data(m['X'], m['Y']); e3.set_hyper(m['hyper']); e3.factorize()
    with pytest.raises(L.GpmpcError) as e:
        e3.rollout_batch_em_grad(z0, U, S)
    assert e.value.code == L.ERR_STATE
    e3.close()
