"""gpmpc_rollout_batch_em: exact moment matching ('EM') roll-outs on the device, one batched EM forward over the B
trajectories per step, against GP.rollout's host loop of gpmpc_predict(EM, H = 1) calls (bit for bit), against itself
under different chunkings, and step by step against the long-double EM formula of test_em_shapes_gpu.py on the engine's
own inputs."""
import ctypes

import numpy as np
import pytest

from gp_mpc_b200 import _lib as L
from oracle import gp_oracle as orc
from oracle.rollout_oracle_ld import feedback_inputs64
from tests._em_cases import EM_TOL, em_errors, em_terms, engine_factor, feedback_sigma, tma_on_device
from tests._engines import require
from tests._fake_engine import fixture_gp
from tests._util import assert_same, trajectories

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('B', [1, 3, 65])
@pytest.mark.parametrize('name', ['tank', 'car'])
def test_open_loop_equals_the_host_loop_bit_for_bit(name, B):
    """B = 65 runs as one chunk; B = 1 also as the single trajectory x0:(Ny,), which GP.rollout sends as B = 1."""
    gp, m = fixture_gp(name)
    X0, U, _ = trajectories(name, B, 4, cyclic=True)
    assert_same(gp.rollout(X0, U, methods=['EM']), gp.rollout(X0, U, methods=['EM'], device_rollout=False))
    if B == 1:
        assert_same(gp.rollout(X0[0], U[0], methods=['EM']), gp.rollout(X0[0], U[0], methods=['EM'], device_rollout=False))
    gp.close()


@pytest.mark.parametrize('B', [1, 5])
@pytest.mark.parametrize('name', ['tank', 'car'])
def test_feedback_equals_the_host_loop_bit_for_bit(name, B):
    """A gain per trajectory (one engine pass each), and one gain shared by all (a single pass of B trajectories)."""
    gp, m = fixture_gp(name)
    X0, U, x_ref = trajectories(name, B, 6, cyclic=True)
    kw = dict(methods=['EM'], feedback=True, x_ref=x_ref)
    assert_same(gp.rollout(X0, U, **kw), gp.rollout(X0, U, device_rollout=False, **kw))
    X0[:] = X0[0]; U[:, 0] = U[0, 0]                       # one linearisation point: one gain
    assert_same(gp.rollout(X0, U, **kw), gp.rollout(X0, U, device_rollout=False, **kw))
    gp.close()


def test_autonomous_system_equals_the_host_loop():
    import gp_mpc_b200
    rng = np.random.default_rng(12)
    X = rng.uniform(-2, 2, (40, 2))
    Y = np.column_stack([X[:, 0] + 0.1 * X[:, 1], X[:, 1] + 0.1 * (-X[:, 0] + (1 - X[:, 0] ** 2) * X[:, 1])])
    Y = Y + 2e-2 * rng.standard_normal(Y.shape)
    hyper = np.column_stack([np.full((2, 2), 1.5), np.full(2, 1.2), np.full(2, 0.05)])
    gp = gp_mpc_b200.GP(X, Y, normalize=False, gp_method='EM', hyper=dict(hyper=hyper))
    X0 = np.array([[1.0, 0.5], [-0.5, 1.5], [0.2, -1.0]])
    rm, rv = gp.rollout(X0, np.zeros((3, 12, 0)), methods=['EM'])
    assert_same((rm, rv), gp.rollout(X0, np.zeros((3, 12, 0)), methods=['EM'], device_rollout=False))
    assert rm.shape == (1, 3, 13, 2) and (rv[0, :, 1:] > 0).all()
    gp.close()


def test_predict_em_points_do_not_depend_on_the_chunk():
    """gpmpc_predict(EM) at H = 7 equals seven H = 1 calls with the em_points cap at 1, 3 and unlimited; the same for
    gpmpc_predict_em_grad at H = 5."""
    gp, m = fixture_gp('car')
    eng = gp.engine
    rng = np.random.default_rng(3)
    Nx = m['X'].shape[1]
    Z = m['X'][:7] + 0.05 * rng.standard_normal((7, Nx))
    A = rng.standard_normal((7, Nx, Nx))
    S = 1e-3 * np.eye(Nx) + 1e-3 * A @ np.swapaxes(A, 1, 2)
    alone = [eng.predict(Z[h:h + 1], S[h], L.METHOD_EM, want_jac=False) for h in range(7)]
    galone = [eng.predict_em_grad(Z[h:h + 1], S[h]) for h in range(5)]
    for cap in (1, 3, 0):
        eng.set_option('em_points', cap)
        batch = eng.predict(Z, S, L.METHOD_EM, want_jac=False)
        for h in range(7):
            for i in range(3):
                assert np.array_equal(alone[h][i][0], batch[i][h]), (cap, h, i)
        gb = eng.predict_em_grad(Z[:5], S[:5])
        for h in range(5):
            for k, v in gb.items():
                assert np.array_equal(galone[h][k][0], v[h]), (cap, h, k)
    gp.close()


def _engine_case(name, B, Nt, feedback):
    """The fixture's engine and the engine-unit inputs of a roll-out: z0, U, Sigma0, scale and the policy."""
    gp, m = fixture_gp(name)
    X0, U, x_ref = trajectories(name, B, Nt, cyclic=True)
    Ny, Nu = X0.shape[1], U.shape[2]
    st = m.get('meta')
    scale = np.stack([st['stdY'], st['meanY'], st['meanX'], st['stdX']]) if m['normalize'] else None
    uscale = np.stack([st['meanU'], st['stdU']]) if m['normalize'] else None
    K = 0.05 * np.random.default_rng(5).standard_normal((Nu, Ny)) if feedback else None
    u0 = U[:, 0] if K is None else np.stack([K @ (x - x_ref) for x in X0])
    if m['normalize']:
        X0 = (X0 - st['meanX']) / st['stdX']; u0 = (u0 - st['meanU']) / st['stdU']; U = (U - st['meanU']) / st['stdU']
    S = np.tile(np.eye(Ny + Nu) * 1e-6, (B, 1, 1))
    S[:, :Ny, :Ny] = np.diag(m['hyper'][:, -1] ** 2)
    return gp, np.concatenate([X0, u0], 1), U, S, dict(scale=scale, K=K, x_ref=x_ref if feedback else None,
                                                       uscale=uscale if feedback else None)


@pytest.mark.parametrize('feedback', [False, True])
@pytest.mark.parametrize('name', ['tank', 'car'])
def test_rollout_does_not_depend_on_b_chunk_or_row_and_a_prefix_is_a_prefix(name, feedback):
    gp, z0, U, S, pol = _engine_case(name, 5, 4, feedback)
    eng = gp.engine
    full = eng.rollout_batch_em(z0, U, S, **pol)
    for cap in (1, 3):
        eng.set_option('em_points', cap)
        assert_same(full, eng.rollout_batch_em(z0, U, S, **pol))
    eng.set_option('em_points', 0)
    for b in (0, 3):
        one = eng.rollout_batch_em(z0[b:b + 1], U[b:b + 1], S[b:b + 1], **pol)
        assert_same([x[b] for x in full], [x[0] for x in one])
    rev = eng.rollout_batch_em(z0[::-1].copy(), U[::-1].copy(), S[::-1].copy(), **pol)
    assert_same([x[::-1] for x in rev], full)
    prefix = eng.rollout_batch_em(z0, U[:, :3], S, **pol)
    assert_same((prefix[0], prefix[1]), (full[0][:, :3], full[1][:, :3]))
    gp.close()


# name -> (N, Nx, Ny): 17 pair tiles against 18 trace tiles; Npad 3072 puts the trace product on the TMA feed
LD_CASES = {'partial': (1030, 8, 6), 'tma': (3000, 6, 2)}


@pytest.mark.parametrize('feedback', [False, True])
@pytest.mark.parametrize('name', list(LD_CASES))
def test_every_step_against_long_double(name, feedback):
    """Step t of every trajectory against the long-double formula at the engine's own input of that step: z from
    feedback_inputs64 of the engine's means, Sigma from the cov_last of the engine's t-step prefix, so each comparison is
    single-step and keeps test_em_shapes_gpu's bar (errors over the sums of |terms|)."""
    import gp_mpc_b200
    if name == 'tma':
        require(tma_on_device(), 'the TMA feed')
    N, Nx, Ny = LD_CASES[name]
    Nu, B, Nt = Nx - Ny, 2, 3
    p = orc.synthetic_problem(N, Nx, Ny, config_id=700 + Nx, H=B)
    hyper = p['hyper'].copy()
    hyper[:, Nx + 1] = 0.3
    eng = gp_mpc_b200.Engine(N, Nx, Ny, device=0)
    eng.set_data(p['X'], p['Y']); eng.set_hyper(hyper)
    assert not eng.factorize().any()
    alpha, kinv = engine_factor(eng, Ny)
    rng = np.random.default_rng(9)
    z0 = p['Z']
    U = 0.3 * rng.standard_normal((B, Nt, Nu))
    K = 0.1 * rng.standard_normal((Nu, Ny)) if feedback else None
    S0 = np.tile(0.05 * np.diag(hyper[0, :Nx] ** 2), (B, 1, 1))
    pol = dict(K=K, x_ref=0.1 * np.ones(Ny) if feedback else None)
    means, _, _ = eng.rollout_batch_em(z0, U, S0, **pol)
    covs = [eng.rollout_batch_em(z0, U[:, :t], S0, **pol)[2] for t in range(1, Nt)]
    worst = dict(mean=0.0, cov=0.0)
    for t in range(Nt):
        z = z0 if t == 0 else feedback_inputs64(means[:, t - 1], None, K, pol['x_ref'], None, U[:, t])
        for b in range(B):
            S = S0[b] if t == 0 else feedback_sigma(S0[b], covs[t - 1][b], K)
            one = eng.predict(z[b:b + 1], S, L.METHOD_EM, want_jac=False)
            assert np.array_equal(one[0][0], means[b, t])          # the engine's step is its predict at these inputs
            ref = orc.gp_exact_moment(kinv, p['X'], p['Y'], hyper, z[b], S, extended=True, beta=alpha)
            e = em_errors(one[0][0], one[2][0], ref, em_terms(p['X'], hyper, alpha, kinv, z[b], S))
            worst = {k: max(worst[k], e[k]) for k in worst}
    eng.close()
    assert worst['mean'] < EM_TOL[0] and worst['cov'] < EM_TOL[1], worst


def test_error_codes():
    import gp_mpc_b200
    lib = L.load()
    p = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    # Ny = 45 (every model with Nu >= 0 has Ny <= Nx <= 32)
    q = orc.synthetic_problem(130, 3, 45, config_id=545, H=1)
    e1 = gp_mpc_b200.Engine(130, 3, 45, device=0)
    e1.set_data(q['X'], q['Y']); e1.set_hyper(q['hyper']); e1.factorize()
    with pytest.raises(L.GpmpcError) as e:
        e1.rollout_batch_em(np.zeros((1, 3)), np.zeros((1, 2, 0)), np.eye(3)[None] * 1e-3)
    assert e.value.code == L.ERR_ARG
    e1.close()
    gp, m = fixture_gp('tank')
    eng = gp.engine
    Nx, Ny = 6, 4
    z0 = np.zeros((2, Nx)); U = np.zeros((2, 3, 2)); S = np.tile(np.eye(Nx) * 1e-3, (2, 1, 1))
    out = np.zeros(2 * 3 * Ny)
    rb = lambda *a: lib.gpmpc_rollout_batch_em(eng.h, *a)
    assert rb(0, 3, p(z0), p(U), p(S), None, None, None, None, p(out), p(out), None) == L.ERR_ARG       # B < 1
    assert rb(2, 0, p(z0), p(U), p(S), None, None, None, None, p(out), p(out), None) == L.ERR_ARG       # Nt < 1
    assert rb(2, 3, None, p(U), p(S), None, None, None, None, p(out), p(out), None) == L.ERR_ARG         # z0
    assert rb(2, 3, p(z0), None, p(S), None, None, None, None, p(out), p(out), None) == L.ERR_ARG        # U, open loop
    assert rb(2, 3, p(z0), p(U), None, None, None, None, None, p(out), p(out), None) == L.ERR_ARG        # Sigma0
    assert rb(2, 3, p(z0), p(U), p(S), None, None, None, None, None, p(out), None) == L.ERR_ARG          # means
    assert rb(2, 3, p(z0), p(U), p(S), None, None, None, None, p(out), None, None) == L.ERR_ARG          # vars
    # an indefinite Sigma0: ERR_ARG naming step 0, and the handle stays usable
    Z = m['X'][:2]
    before = eng.predict(Z, S[0], L.METHOD_EM, want_jac=False)
    bad = S.copy()
    bad[1, 0, 0] = -1e3
    with pytest.raises(L.GpmpcError) as e:
        eng.rollout_batch_em(z0, U, bad)
    assert e.value.code == L.ERR_ARG and 'step 0' in str(e.value)
    assert_same(before, eng.predict(Z, S[0], L.METHOD_EM, want_jac=False))
    gp.close()
    # a handle that owns only some outputs
    e3 = gp_mpc_b200.Engine(m['X'].shape[0], Nx, Ny, out_begin=0, out_count=2, device=0)
    e3.set_data(m['X'], m['Y']); e3.set_hyper(m['hyper']); e3.factorize()
    with pytest.raises(L.GpmpcError) as e:
        e3.rollout_batch_em(z0, U, S)
    assert e.value.code == L.ERR_STATE
    e3.close()
