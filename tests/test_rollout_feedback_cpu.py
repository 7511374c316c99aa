"""GP.rollout's closed-loop branch (reference gp_class.py:770-804 with the LQR gain of mpc_class.py:956-976) and
batches of trajectories, on CPU through the oracle-backed stand-in engine.  The device path is covered by
tests/test_rollout_batch_gpu.py."""
import os
import re

import numpy as np
import pytest

import gp_mpc_b200
from oracle.rollout_oracle import predict_compare_loop
from tests._fake_engine import OracleEngine, OracleEngineWithRolloutBatch, fixture_gp
from tests._util import relinf, trajectories

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gp(name, factory=OracleEngine):
    gp, m = fixture_gp(name, factory)
    model = dict(X=m['X'], Y=m['Y'], hyper=m['hyper'], alpha=gp.get_alpha(), chol=gp.get_chol(),
                 normalize=m['normalize'], meta=m.get('meta'))          # the stand-in engine's own factor
    return gp, model


def _case(name, nb=1, Nt=8):
    return trajectories(name, nb, Nt, cyclic=False)


@pytest.mark.parametrize('name', ['tank', 'car'])
def test_feedback_host_loop_equals_predict_compare(name):
    """The host loop with feedback restates gp_class.py:770-804: per method the gain of the linearisation at (x0, u[0]),
    u_t = K (mean_t - x_ref) and the input blocks K cov K^T, cov K^T; the covariance is shared across methods."""
    gp, model = _gp(name)
    X0, U, x_ref = _case(name)
    rm, rv = gp.rollout(X0[0], U[0], methods=['TA', 'ME'], feedback=True, x_ref=x_ref)
    om, ov = predict_compare_loop(model, X0[0], U[0], ['TA', 'ME'], feedback=True, x_ref=x_ref)
    assert rm.shape == om.shape == (2, 9, X0.shape[1])
    assert relinf(rm, om) < 1e-12 and relinf(rv, ov) < 1e-12
    # the input really is fed back: the open-loop roll-out from the same start differs
    rm_open, _ = gp.rollout(X0[0], U[0], methods=['TA', 'ME'])
    assert relinf(rm_open, rm) > 1e-6
    # Q, R reach the gain
    rq, _ = gp.rollout(X0[0], U[0], methods=['ME'], feedback=True, x_ref=x_ref, R=10 * np.eye(U.shape[2]))
    oq, _ = predict_compare_loop(model, X0[0], U[0], ['ME'], feedback=True, x_ref=x_ref, R=10 * np.eye(U.shape[2]))
    assert relinf(rq, oq) < 1e-12 and relinf(rq, rm[1:]) > 1e-9


@pytest.mark.parametrize('name', ['tank', 'car'])
def test_lqr_stabilises_and_solves_the_riccati_equation(name):
    gp, _ = _gp(name)
    X0, U, _ = _case(name)
    A, B = gp.discrete_linearize(X0[0], U[0, 0], None)
    rng = np.random.default_rng(4)
    for Q, R in ((np.eye(A.shape[0]), np.eye(B.shape[1])),
                 (np.diag(rng.uniform(0.5, 2.0, A.shape[0])), np.diag(rng.uniform(0.1, 5.0, B.shape[1])))):
        K, P, E = gp_mpc_b200.lqr(A, B, Q, R)
        assert K.shape == (B.shape[1], A.shape[0])
        assert np.all(np.abs(np.linalg.eigvals(A + B @ K)) < 1) and np.allclose(np.sort_complex(E),
                                                                            np.sort_complex(np.linalg.eigvals(A + B @ K)))
        res = A.T @ P @ A - P - A.T @ P @ B @ np.linalg.solve(R + B.T @ P @ B, B.T @ P @ A) + Q
        assert np.abs(res).max() / max(1.0, np.abs(P).max()) < 1e-10
        assert np.abs(K + np.linalg.solve(R + B.T @ P @ B, B.T @ P @ A)).max() < 1e-10 * max(1.0, np.abs(K).max())


@pytest.mark.parametrize('feedback', [False, True])
@pytest.mark.parametrize('factory', [OracleEngine, OracleEngineWithRolloutBatch])
def test_batch_equals_single_rollouts(factory, feedback):
    """x0:(B,Ny), u:(B,Nt,Nu) gives (methods, B, Nt+1, Ny); trajectory b is the single roll-out of x0[b], u[b], on the
    host loop (OracleEngine) and through the batched entry (its numpy restatement)."""
    gp, _ = _gp('tank', factory)
    X0, U, x_ref = _case('tank', nb=3, Nt=6)
    kw = dict(methods=['TA', 'ME'], feedback=feedback, x_ref=x_ref if feedback else None)
    rm, rv = gp.rollout(X0, U, **kw)
    assert rm.shape == rv.shape == (2, 3, 7, 4)
    for b in range(3):
        sm, sv = gp.rollout(X0[b], U[b], **kw)
        assert relinf(rm[:, b], sm) < 1e-12 and relinf(rv[:, b], sv) < 1e-12
    hm, hv = gp.rollout(X0, U, device_rollout=False, **kw)
    assert relinf(rm, hm) < 1e-12 and relinf(rv, hv) < 1e-12


@pytest.mark.parametrize('name', ['tank', 'car'])
def test_feedback_device_mapping_equals_the_host_loop(name):
    """With an engine that restates gpmpc_rollout_batch in numpy, the device mapping (first input K (x0 - x_ref) standardised,
    [meanU | stdU], one pass per distinct gain, the final input blocks formed from cov_last) reproduces the host loop, also for
    a second method that starts from the first one's input blocks."""
    gp, model = _gp(name, OracleEngineWithRolloutBatch)
    X0, U, x_ref = _case(name, nb=2)
    X0[1] = X0[0]; U[1, 0] = U[0, 0]                       # same linearisation point: one pass with B = 2
    rm, rv = gp.rollout(X0, U, methods=['TA', 'ME', 'TA'], feedback=True, x_ref=x_ref)
    hm, hv = gp.rollout(X0, U, methods=['TA', 'ME', 'TA'], feedback=True, x_ref=x_ref, device_rollout=False)
    assert relinf(rm, hm) < 1e-12 and relinf(rv, hv) < 1e-12
    om, ov = predict_compare_loop(model, X0[0], U[0], ['TA', 'ME', 'TA'], feedback=True, x_ref=x_ref)
    assert relinf(rm[:, 0], om) < 1e-12 and relinf(rv[:, 0], ov) < 1e-12
    assert not np.array_equal(rv[0], rv[2])                # the second 'TA' starts from the blocks 'ME' left


def test_rollout_feedback_needs_inputs():
    rng = np.random.default_rng(1)
    X = rng.standard_normal((20, 2)); Y = X + 0.1 * rng.standard_normal((20, 2))
    gp = gp_mpc_b200.GP(X, Y, normalize=False, hyper=dict(hyper=np.array([[1., 1., 1., .1], [1., 1., 1., .1]])),
                        engine_factory=OracleEngine)
    with pytest.raises(ValueError):
        gp.rollout(np.zeros(2), np.zeros((3, 0)), methods=['ME'], feedback=True)
    rm, rv = gp.rollout(np.zeros((2, 2)), np.zeros((2, 3, 0)), methods=['ME'])          # autonomous batch
    assert rm.shape == (1, 2, 4, 2)


def test_rollout_batch_is_declared_and_bound():
    hdr = open(os.path.join(ROOT, 'include', 'gpmpc.h')).read()
    assert re.search(r'\bint gpmpc_rollout_batch\s*\(', hdr)
    assert 'gp_class.py:770-804' in hdr and 'mpc_class.py:956-976' in hdr
    import __graft_entry__ as g
    g.build()
    L = gp_mpc_b200._lib
    assert 'gpmpc_rollout_batch' in {s[0] for s in L.SYMBOLS}
    assert L.load().gpmpc_rollout_batch is not None
