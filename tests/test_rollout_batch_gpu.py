"""gpmpc_rollout_batch on the device: B trajectories per predict pass, open loop and with LQR feedback (reference
gp_class.py:770-804, mpc_class.py:956-976), against GP.rollout's host loop and the predict_compare restatement."""
import ctypes

import numpy as np
import pytest

from gp_mpc_b200 import _lib as L
from oracle.rollout_oracle import predict_compare_loop
from tests._fake_engine import fixture_gp
from tests._util import relinf, trajectories

pytestmark = pytest.mark.gpu


def _scalers(m, X0, U):
    """GP input units of the starts and inputs, and the [stdY|meanY|meanX|stdX], [meanU|stdU] maps (None without normalize)."""
    if not m['normalize']:
        return X0, U, None, None
    st = m['meta']
    return ((X0 - st['meanX']) / st['stdX'], (U - st['meanU']) / st['stdU'],
            np.stack([st['stdY'], st['meanY'], st['meanX'], st['stdX']]), np.stack([st['meanU'], st['stdU']]))


@pytest.mark.parametrize('B', [1, 3, 64, 65, 130])
@pytest.mark.parametrize('name', ['tank', 'car'])
def test_batched_open_loop_equals_the_host_loop(name, B):
    """B trajectories in one predict pass per step (two 64-point chunks above 64) equal the per-step host loop."""
    gp, m = fixture_gp(name)
    X0, U, _ = trajectories(name, B, 4, cyclic=True)
    rm, rv = gp.rollout(X0, U, methods=['TA', 'ME'])
    hm, hv = gp.rollout(X0, U, methods=['TA', 'ME'], device_rollout=False)
    assert rm.shape == (2, B, 5, m['Y'].shape[1])
    for b in range(B):
        assert relinf(rm[:, b], hm[:, b]) < 1e-12 and relinf(rv[:, b], hv[:, b]) < 1e-12, b
    assert (rv[:, :, 1:] > 0).all()
    gp.close()


@pytest.mark.parametrize('name', ['tank', 'car'])
def test_single_entry_is_the_batch_of_one_bit_for_bit(name):
    gp, m = fixture_gp(name)
    eng = gp.engine
    X0, U, _ = trajectories(name, 3, 6, cyclic=True)
    Ny = X0.shape[1]
    zx, un, scale, _ = _scalers(m, X0, U)
    z0 = np.concatenate([zx, un[:, 0]], 1)
    S = np.tile(np.eye(z0.shape[1]) * 1e-6, (3, 1, 1))
    S[:, :Ny, :Ny] = np.diag(m['hyper'][:, -1] ** 2)
    for meth in (L.METHOD_TA, L.METHOD_ME):
        a = eng.rollout(z0[0], un[0], S[0], meth, scale)
        b = eng.rollout_batch(z0[:1], un[:1], S[:1], meth, scale)
        for x, y in zip(a, b):
            assert np.array_equal(x, y[0])
        c1 = eng.rollout_batch(z0, un, S, meth, scale)
        c2 = eng.rollout_batch(z0, un, S, meth, scale)
        for x, y in zip(c1, c2):
            assert np.array_equal(x, y)
    gp.close()


@pytest.mark.parametrize('B', [1, 5])
@pytest.mark.parametrize('name', ['tank', 'car'])
def test_device_feedback_equals_host_loop_and_predict_compare(name, B):
    """GP.rollout(feedback=True) on the device (the gain of each trajectory's (x0, u[0]); u_t = K (mean_t - x_ref), input
    blocks K cov K^T, cov K^T) against the host loop (1e-12) and predict_compare's restatement with the CPU factor (1e-6,
    as every GPU-against-oracle comparison here)."""
    gp, m = fixture_gp(name)
    X0, U, x_ref = trajectories(name, B, 8, cyclic=True)
    rm, rv = gp.rollout(X0, U, methods=['TA', 'ME'], feedback=True, x_ref=x_ref)
    hm, hv = gp.rollout(X0, U, methods=['TA', 'ME'], feedback=True, x_ref=x_ref, device_rollout=False)
    assert relinf(rm, hm) < 1e-12 and relinf(rv, hv) < 1e-12
    for b in range(B):
        om, ov = predict_compare_loop(m, X0[b], U[b], ['TA', 'ME'], feedback=True, x_ref=x_ref)
        assert relinf(rm[:, b], om) < 1e-6 and relinf(rv[:, b], ov) < 1e-5
    gp.close()


@pytest.mark.parametrize('name', ['tank', 'car'])
def test_shared_gain_batch_equals_one_trajectory_at_a_time(name):
    """One gain for B = 5 different starts in a single pass (five CTAs of the feedback kernel) equals five B = 1 passes."""
    gp, m = fixture_gp(name)
    eng = gp.engine
    X0, U, x_ref = trajectories(name, 5, 7, cyclic=True)
    Ny, Nu = X0.shape[1], U.shape[2]
    A, Bm = gp.discrete_linearize(X0[0], U[0, 0], None)
    import gp_mpc_b200
    K = gp_mpc_b200.lqr(A, Bm, np.eye(Ny), np.eye(Nu))[0]
    zx, u0, scale, uscale = _scalers(m, X0, np.stack([K @ (x - x_ref) for x in X0]))
    z0 = np.concatenate([zx, u0], 1)
    S = np.tile(np.eye(Ny + Nu) * 1e-6, (5, 1, 1))
    mb, vb, cb = eng.rollout_batch(z0, U, S, L.METHOD_TA, scale, K, x_ref, uscale)
    for b in range(5):
        m1, v1, c1 = eng.rollout_batch(z0[b:b + 1], U[b:b + 1], S[b:b + 1], L.METHOD_TA, scale, K, x_ref, uscale)
        assert relinf(mb[b], m1[0]) < 1e-12 and relinf(vb[b], v1[0]) < 1e-12 and relinf(cb[b], c1[0]) < 1e-12
    gp.close()


def test_batched_autonomous_system():
    """Nu = 0 (van_der_pol.py): a batch of starts, 'ME', equals sequential GP.predict calls."""
    import gp_mpc_b200
    rng = np.random.default_rng(12)
    X = rng.uniform(-2, 2, (40, 2))
    Y = np.column_stack([X[:, 0] + 0.1 * X[:, 1], X[:, 1] + 0.1 * (-X[:, 0] + (1 - X[:, 0] ** 2) * X[:, 1])])
    Y = Y + 2e-2 * rng.standard_normal(Y.shape)
    hyper = np.column_stack([np.full((2, 2), 1.5), np.full(2, 1.2), np.full(2, 0.05)])
    gp = gp_mpc_b200.GP(X, Y, normalize=False, gp_method='ME', hyper=dict(hyper=hyper))
    X0 = np.array([[1.0, 0.5], [-0.5, 1.5], [0.2, -1.0]])
    rm, rv = gp.rollout(X0, np.zeros((3, 20, 0)), methods=['ME'])
    assert rm.shape == (1, 3, 21, 2)
    for b in range(3):
        x = X0[b]
        for t in range(20):
            mean, _ = gp.predict(x, [], np.zeros((2, 2)))
            x = np.array(mean).flatten()
            assert relinf(rm[0, b, t + 1], x) < 1e-12
    assert (rv[0, :, 1:] > 0).all()
    gp.close()


def test_argument_checks():
    import gp_mpc_b200
    lib = L.load()
    gp, m = fixture_gp('tank')
    eng = gp.engine
    Nx, Ny = 6, 4
    z0 = np.zeros((2, Nx)); U = np.zeros((2, 3, 2)); S = np.tile(np.eye(Nx) * 1e-3, (2, 1, 1))
    K = np.zeros((2, Ny)); out = np.zeros(2 * 3 * Ny)
    p = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    with pytest.raises(L.GpmpcError) as e:
        eng.rollout_batch(z0, U, S, L.METHOD_EM)
    assert e.value.code == L.ERR_ARG
    rb = lambda *a: lib.gpmpc_rollout_batch(eng.h, *a)
    assert rb(L.METHOD_TA, 0, 3, p(z0), p(U), p(S), None, None, None, None, p(out), p(out), None) == L.ERR_ARG   # B < 1
    assert rb(L.METHOD_TA, 2, 0, p(z0), p(U), p(S), None, None, None, None, p(out), p(out), None) == L.ERR_ARG   # Nt < 1
    assert rb(L.METHOD_TA, 2, 3, None, p(U), p(S), None, None, None, None, p(out), p(out), None) == L.ERR_ARG     # z0
    assert rb(L.METHOD_TA, 2, 3, p(z0), None, p(S), None, None, None, None, p(out), p(out), None) == L.ERR_ARG    # U, open loop
    assert rb(L.METHOD_TA, 2, 3, p(z0), p(U), None, None, None, None, None, p(out), p(out), None) == L.ERR_ARG    # Sigma0
    assert rb(L.METHOD_TA, 2, 3, p(z0), p(U), p(S), None, None, None, None, None, p(out), None) == L.ERR_ARG      # means
    assert rb(L.METHOD_TA, 2, 3, p(z0), None, p(S), None, p(K), None, None, p(out), p(out), None) == L.OK         # U may be NULL with K
    gp.close()
    # K with Nu = 0
    rng = np.random.default_rng(0)
    X = rng.standard_normal((20, 2)); hyper = np.array([[1., 1., 1., .1], [1., 1., 1., .1]])
    e2 = gp_mpc_b200.Engine(20, 2, 2, device=0); e2.set_data(X, X); e2.set_hyper(hyper); e2.factorize()
    z = np.zeros((1, 2)); S2 = np.eye(2)[None] * 1e-3; K0 = np.zeros(2); o2 = np.zeros(2)
    assert lib.gpmpc_rollout_batch(e2.h, L.METHOD_ME, 1, 1, p(z), None, p(S2), None, p(K0), None, None, p(o2), p(o2), None) == L.ERR_ARG
    assert lib.gpmpc_rollout_batch(e2.h, L.METHOD_ME, 1, 1, p(z), None, p(S2), None, None, None, None, p(o2), p(o2), None) == L.OK
    e2.close()
    # a handle that owns only some outputs
    e3 = gp_mpc_b200.Engine(m['X'].shape[0], Nx, Ny, out_begin=0, out_count=2, device=0)
    e3.set_data(m['X'], m['Y']); e3.set_hyper(m['hyper']); e3.factorize()
    with pytest.raises(L.GpmpcError) as e:
        e3.rollout_batch(z0, U, S, L.METHOD_TA)
    assert e.value.code == L.ERR_STATE
    e3.close()


def test_default_methods_run_em_on_the_host_and_ta_me_on_the_device():
    """GP.rollout(feedback=True) with the reference's default methods ['EM', 'TA', 'ME']: 'EM' takes the host loop, 'TA' and
    'ME' the batched entry, and the result equals the all-host loop ('EM' bit for bit)."""
    gp, m = fixture_gp('tank')
    X0, U, x_ref = trajectories('tank', 2, 5, cyclic=True)
    eng = gp.engine
    calls = []
    real = eng.rollout_batch

    def spy(*a, **k):
        calls.append(a[3] if len(a) > 3 else k.get('method'))
        return real(*a, **k)

    eng.rollout_batch = spy
    rm, rv = gp.rollout(X0, U, feedback=True, x_ref=x_ref)
    del eng.rollout_batch
    hm, hv = gp.rollout(X0, U, feedback=True, x_ref=x_ref, device_rollout=False)
    assert sorted(set(calls)) == [L.METHOD_ME, L.METHOD_TA] and L.METHOD_EM not in calls
    assert rm.shape == (3, 2, 6, 4)
    assert np.array_equal(rm[0], hm[0]) and np.array_equal(rv[0], hv[0])
    assert relinf(rm, hm) < 1e-12 and relinf(rv, hv) < 1e-12
    gp.close()
