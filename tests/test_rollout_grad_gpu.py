"""gpmpc_rollout_batch_grad on the device: the roll-out of gpmpc_rollout_batch bit for bit, plus the forward-mode
derivatives of every step's mean and variance w.r.t. the start, the inputs or the feedback gain, against central
differences of gpmpc_rollout_batch and against oracle/rollout_grad_oracle.py with the CPU factor."""
import ctypes

import numpy as np
import pytest

from gp_mpc_b200 import _lib as L
from oracle import gp_oracle as orc
from oracle.rollout_grad_oracle import rollout_grad
from tests._engines import lqr_gain
from tests._fake_engine import fixture_gp
from tests._util import relinf, trajectories

pytestmark = pytest.mark.gpu


def _gp(name):
    """A GP on the device and the CPU model of the same data (its own Cholesky factor) for the oracle."""
    import gp_mpc_b200
    if name == 'synthetic':
        from bench import WORKLOADS, make_workload
        wl = WORKLOADS['c2']
        w = make_workload(wl['N'], wl['Nx'], wl['Ny'], wl['cfg'], wl['H'])
        m = dict(X=w['X'], Y=w['Y'], hyper=w['hyper'], normalize=False, Z=w['Z'])
        gp = gp_mpc_b200.GP(w['X'], w['Y'], normalize=False, hyper=dict(hyper=w['hyper']))
    else:
        gp, m = fixture_gp(name)
    return gp, m


def _model(m):
    post = orc.postfit(m['X'], m['Y'], m['hyper'], lapack_general_solve=False)
    return dict(X=m['X'], Y=m['Y'], hyper=m['hyper'], alpha=post['alpha'], chol=post['chol'],
                normalize=m['normalize'], meta=m.get('meta'))


def _case(name, m, nb, Nt):
    if name == 'synthetic':
        Ny = m['Y'].shape[1]
        rows = m['Z'][np.arange(nb) % m['Z'].shape[0]]
        X0 = rows[:, :Ny] * (1 + 0.002 * (np.arange(nb) // m['Z'].shape[0]))[:, None]
        U = np.repeat(rows[:, None, Ny:], Nt, 1) * (1 + 0.01 * np.arange(Nt)[None, :, None])
        return X0, U, 0.5 * X0[0]
    return trajectories(name, nb, Nt, cyclic=True)


def _inputs(gp, m, X0, U, K=None, x_ref=None):
    """The engine's arguments as GP.rollout forms them: z0, U and Sigma0 in GP units, scale, uscale."""
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
    return np.concatenate([zx, un[:, 0, :Nu]], 1), (un if K is None else U), S, scale, uscale


@pytest.mark.parametrize('B', [1, 3, 64, 65, 130])
@pytest.mark.parametrize('name', ['tank', 'car', 'synthetic'])
def test_rollout_is_rollout_batch_bit_for_bit(name, B):
    """means, vars, cov_last equal gpmpc_rollout_batch's for 'TA' and 'ME', open loop and with feedback, across the 64-point
    chunks of the predict pass; the derivatives are finite and have the documented shape."""
    gp, m = _gp(name)
    eng = gp.engine
    X0, U, x_ref = _case(name, m, B, 4)
    Ny, Nx = X0.shape[1], m['X'].shape[1]
    Nu = Nx - Ny
    K = lqr_gain(gp, X0, U)
    for meth in (L.METHOD_TA, L.METHOD_ME):
        for fb in (False, True):
            z0, Ug, S, scale, uscale = _inputs(gp, m, X0, U, K if fb else None, x_ref)
            args = (z0, Ug, S, meth, scale) + ((K, x_ref, uscale) if fb else ())
            ref = eng.rollout_batch(*args)
            got = eng.rollout_batch_grad(*args)
            for x, y in zip(ref, got[:3]):
                assert np.array_equal(x, y), (meth, fb)
            P = Nx + (Nu * Ny if fb else 3 * Nu)
            assert got[3].shape == got[4].shape == (B, 4, Ny, P)
            assert np.isfinite(got[3]).all() and np.isfinite(got[4]).all()
    gp.close()


@pytest.mark.parametrize('name', ['tank', 'car'])
def test_one_trajectory_equals_its_row_and_calls_repeat(name):
    """Trajectory b alone equals row b of a batch bit for bit (every sum in a fixed order, one CTA per trajectory), and two
    identical calls give identical bits."""
    gp, m = _gp(name)
    eng = gp.engine
    X0, U, x_ref = _case(name, m, 5, 6)
    K = lqr_gain(gp, X0, U)
    for meth in (L.METHOD_TA, L.METHOD_ME):
        for fb in (False, True):
            z0, Ug, S, scale, uscale = _inputs(gp, m, X0, U, K if fb else None, x_ref)
            extra = (K, x_ref, uscale) if fb else ()
            full = eng.rollout_batch_grad(z0, Ug, S, meth, scale, *extra)
            again = eng.rollout_batch_grad(z0, Ug, S, meth, scale, *extra)
            for x, y in zip(full, again):
                assert np.array_equal(x, y)
            for b in (0, 3):
                one = eng.rollout_batch_grad(z0[b:b + 1], Ug[b:b + 1], S[b:b + 1], meth, scale, *extra)
                for x, y in zip(full, one):
                    assert np.array_equal(x[b], y[0]), (meth, fb, b)
    gp.close()


# measured on an H100 80GB HBM3 at 700 W (central differences at a step of 1e-5 relative, Nt = 8, batch-inf-norm relative over
# each block): tank 8.5e-7 (dmeans) and <= 9.9e-5 (dvars: its variances are small differences sf2 - |L^-1 k|^2, so the
# quotient carries their rounding), synthetic <= 1.2e-7 and <= 1.5e-7
_FD_TOL = dict(mean=2e-6, var=4e-4)


@pytest.mark.parametrize('meth', ['TA', 'ME'])
@pytest.mark.parametrize('name', ['tank', 'synthetic'])
def test_derivatives_equal_central_differences_on_the_device(name, meth):
    """Open loop, Nt = 8: dmeans / dvars against central differences of gpmpc_rollout_batch on the same device in every
    parameter (z0, then U rows 1..Nt-1); no CPU factor is involved."""
    gp, m = _gp(name)
    eng = gp.engine
    method = L.METHOD_TA if meth == 'TA' else L.METHOD_ME
    X0, U, _ = _case(name, m, 2, 8)
    z0, Ug, S, scale, _ = _inputs(gp, m, X0, U)
    Ny, Nx, Nt = X0.shape[1], z0.shape[1], 8
    Nu = Nx - Ny
    _, _, _, dm, dv = eng.rollout_batch_grad(z0, Ug, S, method, scale)
    P = Nx + (Nt - 1) * Nu
    fm = np.zeros_like(dm); fv = np.zeros_like(dv)
    rel = 1e-5
    for p in range(P):
        zp, zm, Up, Um = z0.copy(), z0.copy(), Ug.copy(), Ug.copy()
        if p < Nx:
            h = rel * np.maximum(1.0, np.abs(z0[:, p]))
            zp[:, p] += h; zm[:, p] -= h
        else:
            r, i = 1 + (p - Nx) // Nu, (p - Nx) % Nu
            h = rel * np.maximum(1.0, np.abs(Ug[:, r, i]))
            Up[:, r, i] += h; Um[:, r, i] -= h
        mp, vp, _ = eng.rollout_batch(zp, Up, S, method, scale)
        mm, vm, _ = eng.rollout_batch(zm, Um, S, method, scale)
        fm[..., p] = (mp - mm) / (2 * h[:, None, None])
        fv[..., p] = (vp - vm) / (2 * h[:, None, None])
    em, ev = relinf(dm, fm), relinf(dv, fv)
    print('[fd] %s %s dmeans %.2e dvars %.2e' % (name, meth, em, ev))
    assert em < _FD_TOL['mean'] and ev < _FD_TOL['var'], (em, ev)
    gp.close()


# measured on an H100 80GB HBM3 at 700 W, worst block: tank <= 4.0e-9, synthetic <= 2.1e-10; car (cond K ~ 1e10, the factors
# differing by ~1e-16 cond(K)^1/2 and the closed loop amplifying single roundings, DESIGN.md 4.11) 4.2e-5 for 'ME' open loop,
# <= 1.1e-6 otherwise
_ORACLE_TOL = dict(tank=1e-7, synthetic=1e-7, car=1e-4)


@pytest.mark.parametrize('fb', [False, True])
@pytest.mark.parametrize('meth', ['TA', 'ME'])
@pytest.mark.parametrize('name', ['tank', 'car', 'synthetic'])
def test_rollout_grad_equals_the_oracle(name, meth, fb):
    """GP.rollout_grad in caller units against the forward-mode oracle with the CPU factor and the same gain; its mean / var
    are GP.rollout's bit for bit."""
    gp, m = _gp(name)
    model = _model(m)
    X0, U, x_ref = _case(name, m, 3, 6)
    kw = dict(feedback=fb, x_ref=x_ref if fb else None)
    r = gp.rollout_grad(X0, U, method=meth, **kw)
    rm, rv = gp.rollout(X0, U, methods=[meth], **kw)
    assert np.array_equal(r['mean'], rm[0]) and np.array_equal(r['var'], rv[0])
    keys = ('dmean_dx0', 'dvar_dx0') + (('dmean_dK', 'dvar_dK') if fb else ('dmean_du', 'dvar_du'))
    worst = 0.0
    for b in range(3):
        K = gp._GP__lqr_gains(X0[b:b + 1], U[b:b + 1, 0], np.eye(X0.shape[1]), np.eye(U.shape[2]))[0] if fb else None
        o = rollout_grad(model, X0[b], U[b], meth, feedback=fb, x_ref=x_ref, K=K)
        for k in keys:
            worst = max(worst, relinf(r[k][b], o[k]))
    print('[oracle] %s %s fb=%s %.2e' % (name, meth, fb, worst))
    assert worst < _ORACLE_TOL[name], worst
    gp.close()


def test_autonomous_model_has_the_start_as_only_parameter():
    """Nu = 0: P = Nx; against the oracle with the CPU factor."""
    import gp_mpc_b200
    rng = np.random.default_rng(12)
    X = rng.uniform(-2, 2, (40, 2))
    Y = np.column_stack([X[:, 0] + 0.1 * X[:, 1], X[:, 1] + 0.1 * (-X[:, 0] + (1 - X[:, 0] ** 2) * X[:, 1])])
    Y = Y + 2e-2 * rng.standard_normal(Y.shape)
    hyper = np.column_stack([np.full((2, 2), 1.5), np.full(2, 1.2), np.full(2, 0.05)])
    gp = gp_mpc_b200.GP(X, Y, normalize=False, gp_method='TA', hyper=dict(hyper=hyper))
    X0 = np.array([[1.0, 0.5], [-0.5, 1.5]])
    out = gp.engine.rollout_batch_grad(X0, np.zeros((2, 10, 0)), np.tile(np.eye(2) * 1e-3, (2, 1, 1)))
    assert out[3].shape == (2, 10, 2, 2)
    model = _model(dict(X=X, Y=Y, hyper=hyper, normalize=False))
    for meth in ('TA', 'ME'):
        r = gp.rollout_grad(X0, np.zeros((2, 10, 0)), method=meth)
        assert r['dmean_du'].shape == (2, 11, 2, 10, 0)
        for b in range(2):
            o = rollout_grad(model, X0[b], np.zeros((10, 0)), meth)
            assert relinf(r['dmean_dx0'][b], o['dmean_dx0']) < 1e-7 and relinf(r['dvar_dx0'][b], o['dvar_dx0']) < 1e-7
    gp.close()


def test_error_codes_leave_the_model_unchanged():
    import gp_mpc_b200
    lib = L.load()
    gp, m = _gp('tank')
    eng = gp.engine
    Nx, Ny = 6, 4
    Zp = 0.3 * np.random.default_rng(3).standard_normal((7, Nx))
    before = eng.predict(Zp, np.eye(Nx) * 1e-4, L.METHOD_TA)
    z0 = np.zeros((2, Nx)); U = np.zeros((2, 3, 2)); S = np.tile(np.eye(Nx) * 1e-3, (2, 1, 1))
    K = np.zeros((2, Ny)); out = np.zeros(2 * 3 * Ny * 64)
    p = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    rg = lambda meth, B, Nt, z, u, s, k, mo, vo, dmo, dvo: lib.gpmpc_rollout_batch_grad(
        eng.h, meth, B, Nt, z, u, s, None, k, None, None, mo, vo, None, dmo, dvo)
    o = p(out)
    assert rg(L.METHOD_EM, 2, 3, p(z0), p(U), p(S), None, o, o, o, o) == L.ERR_ARG
    assert rg(L.METHOD_TA, 0, 3, p(z0), p(U), p(S), None, o, o, o, o) == L.ERR_ARG        # B < 1
    assert rg(L.METHOD_TA, 2, 0, p(z0), p(U), p(S), None, o, o, o, o) == L.ERR_ARG        # Nt < 1
    assert rg(L.METHOD_TA, 2, 3, None, p(U), p(S), None, o, o, o, o) == L.ERR_ARG         # z0
    assert rg(L.METHOD_TA, 2, 3, p(z0), None, p(S), None, o, o, o, o) == L.ERR_ARG        # U, open loop
    assert rg(L.METHOD_TA, 2, 3, p(z0), p(U), None, None, o, o, o, o) == L.ERR_ARG        # Sigma0
    assert rg(L.METHOD_TA, 2, 3, p(z0), p(U), p(S), None, None, o, o, o) == L.ERR_ARG     # means
    assert rg(L.METHOD_TA, 2, 3, p(z0), p(U), p(S), None, o, o, None, o) == L.ERR_ARG     # dmeans
    assert rg(L.METHOD_TA, 2, 3, p(z0), p(U), p(S), None, o, o, o, None) == L.ERR_ARG     # dvars
    assert rg(L.METHOD_TA, 2, 3, p(z0), None, p(S), p(K), o, o, o, o) == L.OK             # U may be NULL with K
    after = eng.predict(Zp, np.eye(Nx) * 1e-4, L.METHOD_TA)
    for x, y in zip(before, after):
        assert np.array_equal(x, y)
    # K with Nu = 0
    rng = np.random.default_rng(0)
    X = rng.standard_normal((20, 2)); hyper = np.array([[1., 1., 1., .1], [1., 1., 1., .1]])
    e2 = gp_mpc_b200.Engine(20, 2, 2, device=0); e2.set_data(X, X); e2.set_hyper(hyper)
    z = np.zeros((1, 2)); S2 = np.eye(2)[None] * 1e-3; K0 = np.zeros(2); o2 = np.zeros(8)
    assert lib.gpmpc_rollout_batch_grad(e2.h, L.METHOD_ME, 1, 1, p(z), None, p(S2), None, None, None, None,
                                        p(o2), p(o2), None, p(o2), p(o2)) == L.ERR_STATE           # not factorised
    e2.factorize()
    assert lib.gpmpc_rollout_batch_grad(e2.h, L.METHOD_ME, 1, 1, p(z), None, p(S2), None, p(K0), None, None,
                                        p(o2), p(o2), None, p(o2), p(o2)) == L.ERR_ARG
    e2.close()
    # a handle that owns only some outputs
    e3 = gp_mpc_b200.Engine(m['X'].shape[0], Nx, Ny, out_begin=0, out_count=2, device=0)
    e3.set_data(m['X'], m['Y']); e3.set_hyper(m['hyper']); e3.factorize()
    with pytest.raises(L.GpmpcError) as e:
        e3.rollout_batch_grad(z0, U, S, L.METHOD_TA)
    assert e.value.code == L.ERR_STATE
    e3.close()
    gp.close()
