"""Greedy max-variance selection (GP.append_greedy) on CPU: the oracle against a numpy restatement of the incremental
downdate the CUDA path runs, the host selection path of the GP class through an oracle-backed engine without a device
selection, standardisation, argument checks, and two gloo ranks with sharded outputs."""
import os

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

import gp_mpc_b200
from oracle import gp_oracle as orc
from oracle import greedy_oracle as gro
from tests._fake_engine import OracleEngine
from tests._util import free_port, load_fixture


class HostSelectEngine(OracleEngine):
    """The oracle-backed engine stand-in; like every engine without `append_greedy` it sends GP.append_greedy down
    the host path (one predict and one append per pick)."""


def _downdate_select(X, hyper, Xc, n_new):
    """The per-step arithmetic of gpmpc_append_greedy in numpy: V = L^-1 k(X, C) once, then per pick the candidate's
    own column l, lambda = sqrt(sf2 + sn2 - |l|^2), w = (k(x*, C) - l^T V) / lambda appended to V, var -= w^2."""
    Ny, Nx = hyper.shape[0], X.shape[1]
    Vs, var = [], np.zeros((Ny, Xc.shape[0]))
    for a in range(Ny):
        L = np.linalg.cholesky(orc.assemble_K(X, hyper[a]))
        V = np.linalg.solve(L, orc.covSEard(X, Xc, hyper[a, :Nx], hyper[a, Nx] ** 2))
        Vs.append(V)
        var[a] = hyper[a, Nx] ** 2 - np.sum(V * V, 0)
    active = np.ones(Xc.shape[0], dtype=bool)
    picked, score = [], []
    for _ in range(n_new):
        s = var[0].copy()
        for a in range(1, Ny):
            s += var[a]
        s[~active] = -np.inf
        c = int(np.argmax(s))
        picked.append(c); score.append(s[c]); active[c] = False
        for a in range(Ny):
            sf2, sn2 = hyper[a, Nx] ** 2, hyper[a, Nx + 1] ** 2
            l = Vs[a][:, c].copy()
            lam = np.sqrt(sf2 + sn2 - l @ l)
            w = (orc.covSEard(Xc[c:c + 1], Xc, hyper[a, :Nx], sf2)[0] - l @ Vs[a]) / lam
            Vs[a] = np.vstack([Vs[a], w])
            var[a] -= w * w
    return np.array(picked), np.array(score)


def _problem(N, Nx, Ny, n, seed):
    p = orc.synthetic_problem(N, Nx, Ny, config_id=seed)
    rng = np.random.default_rng(seed)
    Xc = p['X'][rng.integers(0, N, n)] + 0.7 * rng.standard_normal((n, Nx))
    Yc = rng.standard_normal((n, Ny))
    return p['X'], p['Y'], p['hyper'], Xc, Yc


@pytest.mark.parametrize('N,Nx,Ny,n,n_new', [(30, 2, 1, 20, 20), (50, 3, 3, 40, 12), (80, 5, 2, 65, 17)])
def test_oracle_matches_the_downdate_formula(N, Nx, Ny, n, n_new):
    X, _, hyper, Xc, _ = _problem(N, Nx, Ny, n, N + Nx)
    ref = gro.greedy_select(X, hyper, Xc, n_new)
    pk, sc = _downdate_select(X, hyper, Xc, n_new)
    assert np.all(ref['gap'][:-1] > 1e-8)
    np.testing.assert_array_equal(ref['picked'], pk)
    np.testing.assert_allclose(sc, ref['score'], rtol=1e-12, atol=1e-14)
    assert np.all(np.diff(ref['score']) <= 1e-12 * ref['score'][0])         # a pick never raises the maximum


def _fixture_gp(name, **kw):
    m = load_fixture(name)
    args = dict(mean_func='zero', gp_method='TA', normalize=m['normalize'], hyper=dict(hyper=m['hyper']),
                engine_factory=HostSelectEngine)
    if m['normalize']:
        args.update(meta=m['meta'], xlb=m['xlb'], xub=m['xub'], ulb=m['ulb'], uub=m['uub'])
    args.update(kw)
    return gp_mpc_b200.GP(m['X'], m['Y'], **args), m


def test_host_path_picks_what_the_oracle_picks_in_the_gp_units():
    gp, m = _fixture_gp('tank')
    assert m['normalize']
    meta = m['meta']
    X, hyper = m['X'], m['hyper']
    rng = np.random.default_rng(11)
    n = 25
    Xs_pool = X[rng.integers(0, X.shape[0], n)] + 0.5 * rng.standard_normal((n, X.shape[1]))
    Ys_pool = rng.standard_normal((n, m['Y'].shape[1]))
    # the caller's units: GP.append_greedy standardises with meanZ / stdZ and meanY / stdY
    X_new = Xs_pool * meta['stdZ'] + meta['meanZ']
    Y_new = Ys_pool * meta['stdY'] + meta['meanY']
    ref = gro.greedy_select(X, hyper, Xs_pool, 8)
    assert np.all(ref['gap'] > 1e-8)
    N0 = gp.get_size()[0]
    picked = gp.append_greedy(X_new, Y_new, 8)
    np.testing.assert_array_equal(picked, ref['picked'])
    assert gp.get_size()[0] == N0 + 8
    post = orc.postfit(np.vstack([X, Xs_pool[picked]]), np.vstack([m['Y'], Ys_pool[picked]]), hyper,
                       lapack_general_solve=False)
    np.testing.assert_allclose(gp.get_chol(), post['chol'], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(gp.get_alpha(), post['alpha'], rtol=1e-8, atol=1e-10)


def test_no_op_and_argument_errors():
    gp, m = _fixture_gp('tank')
    N0 = gp.get_size()[0]
    X_new = m['X'][:3] + 0.1; Y_new = m['Y'][:3]
    assert gp.append_greedy(X_new, Y_new, 0).size == 0
    assert gp.get_size()[0] == N0
    with pytest.raises(ValueError):
        gp.append_greedy(X_new, Y_new, 4)
    with pytest.raises(ValueError):
        gp.append_greedy(X_new, Y_new, -1)
    with pytest.raises(ValueError):
        gp.append_greedy(X_new, Y_new[:2])
    with pytest.raises(NotImplementedError, match='append_greedy'):
        gp.update_data(X_new, Y_new)


def _worker(rank, world, port, q):
    os.environ['MASTER_ADDR'] = '127.0.0.1'; os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        X, Y, hyper, Xc, Yc = _problem(40, 4, 3, 20, 9)
        # the full stand-in: it has no append_greedy either, and sharded outputs take the host path anyway
        gp = gp_mpc_b200.GP(X, Y, hyper=dict(hyper=hyper), normalize=False, engine_factory=OracleEngine)
        eng = gp.engine
        first = gp.append_greedy(Xc[:10], Yc[:10], 4)
        # only rank 1 "loses positive definiteness" on the 2nd append of the next call: the refit is collective
        OracleEngine.fail_on = (1, 45)
        second = gp.append_greedy(Xc[10:], Yc[10:], 3)
        OracleEngine.fail_on = None
        q.put((rank, (eng.out_begin, eng.out_count), first, second, gp.get_size()[0], gp.get_chol()))
    finally:
        dist.destroy_process_group()


def test_two_ranks_with_sharded_outputs_pick_the_same_points():
    world = 2
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for pr in procs:
        pr.start()
    res = sorted([q.get(timeout=240) for _ in range(world)], key=lambda t: t[0])
    for pr in procs:
        pr.join(timeout=60)
        assert pr.exitcode == 0
    assert [r[1] for r in res] == [(0, 2), (2, 1)]
    X, Y, hyper, Xc, Yc = _problem(40, 4, 3, 20, 9)
    ref1 = gro.greedy_select(X, hyper, Xc[:10], 4)
    X1 = np.vstack([X, Xc[:10][ref1['picked']]])
    ref2 = gro.greedy_select(X1, hyper, Xc[10:], 3)
    assert np.all(ref1['gap'] > 1e-8) and np.all(ref2['gap'] > 1e-8)
    X2 = np.vstack([X1, Xc[10:][ref2['picked']]])
    Y2 = np.vstack([Y, Yc[:10][ref1['picked']], Yc[10:][ref2['picked']]])
    post = orc.postfit(X2, Y2, hyper, lapack_general_solve=False)
    for r in res:
        np.testing.assert_array_equal(r[2], ref1['picked'])
        np.testing.assert_array_equal(r[3], ref2['picked'])
        assert r[4] == 47
        np.testing.assert_allclose(r[5], post['chol'], rtol=1e-12, atol=1e-14)


class DeviceSelectEngine(OracleEngine):
    """An oracle-backed stand-in WITH a device selection: `append_greedy` appends the oracle's picks.  `fail_rank`
    makes that rank alone report a lost positive definiteness at the 2nd pick of its first call (2 points in, ok
    False), as gpmpc_append_greedy does with GPMPC_ERR_NOTPD."""
    fail_rank = None

    def __init__(self, N, Nx, Ny, out_begin=0, out_count=None, device=0, capacity=None):
        super().__init__(N, Nx, Ny, out_begin, out_count, device)
        self.capacity = -(-max(N, capacity or 0) // 128) * 128

    def append_greedy(self, Xc, Yc, n_new):
        ref = gro.greedy_select(self.X, self.hyper[list(self.local_outputs)], Xc, n_new)
        k, ok = n_new, True
        if DeviceSelectEngine.fail_rank is not None and dist.get_rank() == DeviceSelectEngine.fail_rank and n_new > 2:
            DeviceSelectEngine.fail_rank = None
            k, ok = 2, False
        picked = ref['picked'][:k]
        self.X = np.vstack([self.X, Xc[picked]]); self.Y = np.vstack([self.Y, Yc[picked]])
        self.N += k
        if ok:
            self.factorize()
        return picked, ref['score'][:k], ok


def _replicated_worker(rank, world, port, q):
    os.environ['MASTER_ADDR'] = '127.0.0.1'; os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        X, Y, hyper, Xc, Yc = _problem(40, 3, 1, 20, 6)        # Ny = 1 < world: every rank holds the whole model
        gp = gp_mpc_b200.GP(X, Y, hyper=dict(hyper=hyper), normalize=False, engine_factory=DeviceSelectEngine)
        DeviceSelectEngine.fail_rank = 1
        picked = gp.append_greedy(Xc, Yc, 6)
        q.put((rank, picked, gp.get_size()[0], gp.engine.N, gp.get_chol()))
    finally:
        dist.destroy_process_group()


def test_replicated_ranks_make_the_refit_decision_together():
    """'points' mode: every rank selects on its own engine; a NOTPD on one rank only must make every rank keep the
    common picks, refit and go on (no hang in the refit's barrier, the same model everywhere)."""
    world = 2
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_replicated_worker, args=(r, world, port, q)) for r in range(world)]
    for pr in procs:
        pr.start()
    res = sorted([q.get(timeout=240) for _ in range(world)], key=lambda t: t[0])
    for pr in procs:
        pr.join(timeout=60)
        assert pr.exitcode == 0
    X, Y, hyper, Xc, Yc = _problem(40, 3, 1, 20, 6)
    ref = gro.greedy_select(X, hyper, Xc, 6)
    assert np.all(ref['gap'] > 1e-8)
    post = orc.postfit(np.vstack([X, Xc[ref['picked']]]), np.vstack([Y, Yc[ref['picked']]]), hyper,
                       lapack_general_solve=False)
    for r in res:
        np.testing.assert_array_equal(r[1], ref['picked'])
        assert r[2] == r[3] == 46
        np.testing.assert_allclose(r[4], post['chol'], rtol=1e-12, atol=1e-14)
