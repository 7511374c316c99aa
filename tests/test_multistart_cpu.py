"""Multi-start hyper-parameter fits ('starts': 'lhs') on CPU: the lockstep driver of optimize.train_gp_b200 over an
oracle-backed engine whose nlml_batch loops over the oracle, checked against single-start fits from each start."""
import threading

import numpy as np
import pytest
from scipy.optimize import minimize, rosen, rosen_der

from gp_mpc_b200.optimize import _Lockstep, bounds_and_init, lhs_starts, train_gp_b200
from oracle import gp_oracle as orc
from tests._fake_engine import OracleEngine
from tests._util import GOLDEN, load_fixture

NOTPD = -5


class BatchEngine(OracleEngine):
    """OracleEngine with nlml_batch.  Every nlml / nlml_batch call of every instance goes to the class log (the fit
    creates scratch engines of this type); `fail(call, row)` marks rows NOTPD."""
    log, lock, fail = [], threading.Lock(), None

    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        self.device = 0

    @classmethod
    def reset(cls, fail=None):
        cls.log, cls.fail = [], fail

    def nlml(self, a, theta, grad=True):
        with BatchEngine.lock:
            BatchEngine.log.append(('nlml', a, np.array(theta)))
        return OracleEngine.nlml(self, a, theta, grad)

    def nlml_batch(self, a, thetas, grad=True):
        thetas = np.array(thetas)
        with BatchEngine.lock:
            k = sum(1 for e in BatchEngine.log if e[0] == 'batch' and e[1] == a)
            BatchEngine.log.append(('batch', a, thetas.copy()))
        S = len(thetas)
        nll, g, st = np.empty(S), np.empty(thetas.shape), np.zeros(S, dtype=np.int32)
        for i, th in enumerate(thetas):
            try:
                if BatchEngine.fail is not None and BatchEngine.fail(k, i):
                    raise np.linalg.LinAlgError('not positive definite')
                r = OracleEngine.nlml(self, a, th, grad)
            except np.linalg.LinAlgError:
                nll[i], g[i], st[i] = np.nan, np.nan, NOTPD
                continue
            nll[i], g[i] = r if grad else (r, 0.0)
        return nll, (g if grad else None), st


def _engine(X, Y, out_begin=0, out_count=None):
    e = BatchEngine(X.shape[0], X.shape[1], Y.shape[1], out_begin, out_count)
    e.set_data(X, Y)
    return e


def _tank():
    m = load_fixture('tank')
    return m['X'], m['Y']


def _two_optima():
    z = np.load(GOLDEN + '/multistart_two_optima.npz')
    return z['X'], z['Y']


def _calls(kind, a):
    return [e[2] for e in BatchEngine.log if e[0] == kind and e[1] == a]


def _solo_runs(X, Y, a, x0, opts):
    """Single-start fit of output a from each row of x0: (its evaluated thetas, its row)."""
    out = []
    for x in x0:
        BatchEngine.reset()
        hyp = np.zeros((Y.shape[1], X.shape[1] + 2))
        hyp[a] = x
        row = train_gp_b200(_engine(X, Y, a, 1), X, Y, hyper_init=hyp, optimizer_opts=opts, verbose=False)[0]
        out.append((_calls('nlml', a), row))
    return out


@pytest.mark.parametrize('jac', ['analytic', 'fd'])
def test_every_start_follows_its_single_start_fit_and_batches_list_live_starts_in_order(jac):
    X, Y = _tank()
    a, S = 1, 3
    bounds, init = bounds_and_init(X, Y[:, a])
    x0 = lhs_starts(init, bounds, S, 0, a)
    solo = _solo_runs(X, Y, a, x0, {'jac': jac})
    BatchEngine.reset()
    row = train_gp_b200(_engine(X, Y, a, 1), X, Y, multistart=S, optimizer_opts={'starts': 'lhs', 'jac': jac},
                        verbose=False)[0]
    batches = _calls('batch', a)
    assert not _calls('nlml', a)
    assert len(batches) == max(len(seq) for seq, _ in solo)
    for k, b in enumerate(batches):
        expect = np.array([seq[k] for seq, _ in solo if k < len(seq)])
        assert np.array_equal(b, expect), k
    # start 0 is today's single-start fit; the chosen row is the solo fit of the start with the lowest final NLML
    plain = train_gp_b200(_engine(X, Y, a, 1), X, Y, optimizer_opts={'jac': jac}, verbose=False)[0]
    assert np.array_equal(solo[0][1], plain)
    final = [orc.calc_NLL(r, X, Y[:, a], lapack_general_solve=False) for _, r in solo]
    assert np.array_equal(row, solo[int(np.argmin(final))][1])


def test_same_seed_same_bits_and_other_seed_other_starts():
    X, Y = _tank()
    opts = {'starts': 'lhs', 'seed': 5}
    r1 = train_gp_b200(_engine(X, Y, 2, 1), X, Y, multistart=3, optimizer_opts=opts, verbose=False)
    BatchEngine.reset()
    r2 = train_gp_b200(_engine(X, Y, 2, 1), X, Y, multistart=3, optimizer_opts=opts, verbose=False)
    first5 = _calls('batch', 2)[0]
    assert np.array_equal(r1, r2)
    BatchEngine.reset()
    train_gp_b200(_engine(X, Y, 2, 1), X, Y, multistart=3, optimizer_opts={'starts': 'lhs', 'seed': 6}, verbose=False)
    first6 = _calls('batch', 2)[0]
    assert np.array_equal(first5[0], first6[0])
    assert not np.any(first5[1:] == first6[1:])


def test_starts_lie_in_the_bounds_are_distinct_and_depend_on_seed_and_output_only():
    X, Y = _tank()
    for a in range(Y.shape[1]):
        for fixed in (False, True):
            bounds, init = bounds_and_init(X, Y[:, a], fixed)
            x0 = lhs_starts(init, bounds, 8, 3, a)
            assert np.array_equal(x0[0], init)
            assert np.all(x0[1:] >= bounds[:, 0]) and np.all(x0[1:] <= bounds[:, 1])
            assert len({tuple(r) for r in x0}) == 8
            assert np.array_equal(x0, lhs_starts(init, bounds, 8, 3, a))
        # the hypercube is a function of (seed, a): another output's starts, mapped from this init, differ
        assert not np.array_equal(lhs_starts(init, bounds, 4, 3, a), lhs_starts(init, bounds, 4, 3, a + 1))
    # sequential, parallel and output-sharded fits agree bit for bit
    opts = {'starts': 'lhs', 'seed': 2}
    par = train_gp_b200(_engine(X, Y), X, Y, multistart=3, optimizer_opts=opts, verbose=False)
    seq = train_gp_b200(_engine(X, Y), X, Y, multistart=3, optimizer_opts=dict(opts, parallel_fits=False),
                        verbose=False)
    shard = np.vstack([train_gp_b200(_engine(X, Y, b, 2), X, Y, multistart=3, optimizer_opts=opts, verbose=False)
                       for b in (0, 2)])
    assert np.array_equal(par, seq) and np.array_equal(par, shard)


def test_without_starts_multistart_is_one_run_and_no_batch_call():
    X, Y = _tank()
    BatchEngine.reset()
    r4 = train_gp_b200(_engine(X, Y), X, Y, multistart=4, verbose=False)
    assert not [e for e in BatchEngine.log if e[0] == 'batch']
    r1 = train_gp_b200(_engine(X, Y), X, Y, multistart=1, verbose=False)
    assert np.array_equal(r4, r1)


def test_a_notpd_start_is_abandoned_and_the_others_still_win(capsys):
    X, Y = _tank()
    a, S = 0, 4
    bounds, init = bounds_and_init(X, Y[:, a])
    x0 = lhs_starts(init, bounds, S, 0, a)
    solo = _solo_runs(X, Y, a, x0, None)
    BatchEngine.reset(fail=lambda k, i: k == 2 and i == 1)        # start 1 at its third evaluation
    row = train_gp_b200(_engine(X, Y, a, 1), X, Y, multistart=S, optimizer_opts={'starts': 'lhs'})[0]
    batches = _calls('batch', a)
    assert len(batches[2]) == S and all(len(b) <= S - 1 for b in batches[3:])
    assert '1 abandoned' in capsys.readouterr().out
    final = [orc.calc_NLL(r, X, Y[:, a], lapack_general_solve=False) if s != 1 else np.inf
             for s, (_, r) in enumerate(solo)]
    assert np.array_equal(row, solo[int(np.argmin(final))][1])


def test_every_start_notpd_raises_what_a_single_start_fit_raises():
    X, Y = _tank()
    BatchEngine.reset(fail=lambda k, i: True)
    with pytest.raises(np.linalg.LinAlgError):
        train_gp_b200(_engine(X, Y, 0, 1), X, Y, multistart=3, optimizer_opts={'starts': 'lhs'}, verbose=False)


@pytest.mark.parametrize('opts', [{'starts': 'lhs', 'objective': 'loo'}, {'starts': 'lhs', 'fit_mean': True},
                                  {'starts': 'sobol'}])
def test_unsupported_combinations_raise_before_any_engine_call(opts):
    X, Y = _tank()
    BatchEngine.reset()
    with pytest.raises(ValueError):
        train_gp_b200(_engine(X, Y), X, Y, meanFunc='const', multistart=4, optimizer_opts=opts, verbose=False)
    assert not BatchEngine.log


def test_two_optima_data_set_improves_strictly():
    """On this data set start 0 (the reference's) ends in a local optimum whose NLML is about 4.8 above the one an LHS
    start reaches."""
    X, Y = _two_optima()
    one = train_gp_b200(_engine(X, Y), X, Y, verbose=False)[0]
    four = train_gp_b200(_engine(X, Y), X, Y, multistart=4, optimizer_opts={'starts': 'lhs'}, verbose=False)[0]
    f1 = orc.calc_NLL(one, X, Y[:, 0], lapack_general_solve=False)
    f4 = orc.calc_NLL(four, X, Y[:, 0], lapack_general_solve=False)
    assert f4 < f1 - 1.0, (f1, f4)


class _RosenEngine:
    """nlml_batch over the Rosenbrock function, in row order."""

    def nlml_batch(self, a, thetas, grad=True):
        return (np.array([rosen(t) for t in thetas]), np.array([rosen_der(t) for t in thetas]),
                np.zeros(len(thetas), dtype=np.int32))


def test_lockstep_solves_return_their_solo_bits():
    """Six bounded SLSQP solves behind one lockstep group, each from its own start, return the bits of the same solve
    run alone."""
    rng = np.random.default_rng(0)
    x0 = rng.uniform(-2, 2, (6, 4))
    bounds = [(-1.5, 2.0)] * 4
    solo = [minimize(lambda x: (rosen(x), rosen_der(x)), x, method='SLSQP', jac=True, bounds=bounds, tol=1e-12)
            for x in x0]
    group, out = _Lockstep(_RosenEngine(), 0, 6, True), [None] * 6

    def solve(s):
        try:
            out[s] = minimize(lambda x: group.evaluate(s, x), x0[s], method='SLSQP', jac=True, bounds=bounds, tol=1e-12)
        finally:
            group.leave(s)

    threads = [threading.Thread(target=solve, args=(s,)) for s in range(6)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for r, q in zip(out, solo):
        assert np.array_equal(r.x, q.x) and r.fun == q.fun and r.nit == q.nit
