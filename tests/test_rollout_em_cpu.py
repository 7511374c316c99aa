"""GP.rollout's routing of 'EM' to gpmpc_rollout_batch_em, on CPU through the oracle-backed stand-in engine: the arguments
the GP hands the engine (scalers, one pass per distinct gain, B = 1 for a single trajectory) and the models that keep the
host loop.  The device path is covered by tests/test_rollout_em_gpu.py."""
import os
import re

import numpy as np
import pytest

import gp_mpc_b200
from tests._fake_engine import OracleEngineWithRollout, OracleEngineWithRolloutBatch, TwoRanks, fixture_gp, sharded
from tests._util import relinf, trajectories

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class RecordingEmEngine(OracleEngineWithRolloutBatch):
    """Adds gpmpc_rollout_batch_em as the numpy restatement of the batched roll-out with method 'EM', and records every
    call's arguments."""
    calls = None

    def rollout_batch_em(self, z0, U, Sigma0, scale=None, K=None, x_ref=None, uscale=None):
        type(self).calls.append(dict(z0=np.array(z0), U=np.array(U), Sigma0=np.array(Sigma0), scale=scale, K=K,
                                     x_ref=x_ref, uscale=uscale))
        return self.rollout_batch(z0, U, Sigma0, 2, scale, K, x_ref, uscale)


_ShardEngine = sharded(RecordingEmEngine)


@pytest.fixture(autouse=True)
def _calls():
    RecordingEmEngine.calls = []
    yield RecordingEmEngine.calls


def _gp(name, factory=RecordingEmEngine, **extra):
    return fixture_gp(name, factory, **extra)


def _case(name, nb, Nt=5):
    return trajectories(name, nb, Nt, cyclic=False)


def test_single_open_loop_trajectory_is_one_call_of_b_1(_calls):
    gp, m = _gp('tank')
    X0, U, _ = _case('tank', 1)
    rm, rv = gp.rollout(X0[0], U[0], methods=['EM'])
    assert len(_calls) == 1
    c = _calls[0]
    st = m['meta']
    assert c['z0'].shape == (1, 6) and c['U'].shape == (1, 5, 2) and c['Sigma0'].shape == (1, 6, 6)
    assert np.array_equal(c['scale'], np.stack([st['stdY'], st['meanY'], st['meanX'], st['stdX']]))
    assert c['K'] is None
    assert relinf(c['z0'][0], np.concatenate([(X0[0] - st['meanX']) / st['stdX'], (U[0, 0] - st['meanU']) / st['stdU']])) < 1e-15
    assert np.array_equal(c['Sigma0'][0][:4, :4], np.diag(m['hyper'][:, -1] ** 2))
    hm, hv = gp.rollout(X0[0], U[0], methods=['EM'], device_rollout=False)
    assert len(_calls) == 1
    assert relinf(rm, hm) < 1e-12 and relinf(rv, hv) < 1e-12


def test_feedback_makes_one_call_per_distinct_gain(_calls):
    gp, m = _gp('tank')
    X0, U, x_ref = _case('tank', 3)
    X0[2] = X0[0]; U[2, 0] = U[0, 0]                       # trajectories 0 and 2 share a gain
    kw = dict(methods=['EM'], feedback=True, x_ref=x_ref)
    rm, rv = gp.rollout(X0, U, **kw)
    assert sorted(c['z0'].shape[0] for c in _calls) == [1, 2]
    st = m['meta']
    for c in _calls:
        assert c['K'].shape == (2, 4) and np.array_equal(c['x_ref'], x_ref)
        assert np.array_equal(c['uscale'], np.stack([st['meanU'], st['stdU']]))
    shared = next(c for c in _calls if c['z0'].shape[0] == 2)
    assert np.array_equal(shared['z0'][0], shared['z0'][1])
    hm, hv = gp.rollout(X0, U, device_rollout=False, **kw)
    assert relinf(rm, hm) < 1e-12 and relinf(rv, hv) < 1e-12


def test_default_methods_send_em_to_its_entry(_calls):
    gp, _ = _gp('car')
    X0, U, _ = _case('car', 2)
    gp.rollout(X0, U)
    assert len(_calls) == 1 and _calls[0]['z0'].shape[0] == 2 and _calls[0]['scale'] is None


def test_host_loop_models(_calls):
    """device_rollout=False, a prior mean added in predict and an engine without the entry keep the host loop; a model
    sharded by output has no 'EM' at all."""
    X0, U, _ = _case('tank', 2)
    gp, m = _gp('tank')
    gp.rollout(X0, U, methods=['EM'], device_rollout=False)
    pm, _ = _gp('tank', mean_func='const', prior_mean_in_predict=True, normalize=False, meta=None,
                hyper=dict(hyper=np.column_stack([m['hyper'], np.full(4, 0.1)])))
    pm.rollout(X0, U, methods=['EM'])
    old, _ = _gp('tank', OracleEngineWithRollout)
    old.rollout(X0, U, methods=['EM'])
    sh, _ = _gp('tank', _ShardEngine, comm=TwoRanks(), normalize=False, meta=None)
    with pytest.raises(NotImplementedError, match='needs all outputs on one GPU'):
        sh.rollout(X0, U, methods=['EM'])
    assert _calls == []


def test_rollout_batch_em_is_declared_and_bound():
    hdr = open(os.path.join(ROOT, 'include', 'gpmpc.h')).read()
    assert re.search(r'\bint gpmpc_rollout_batch_em\s*\(', hdr)
    import __graft_entry__ as g
    g.build()
    L = gp_mpc_b200._lib
    assert 'gpmpc_rollout_batch_em' in {s[0] for s in L.SYMBOLS}
    assert L.load().gpmpc_rollout_batch_em is not None
