"""world_size-2 tests of the N>1 host path on CPU (gloo): output partitioning, NCCL-id
broadcast, per-rank training + hyper all-gather, gathered prediction, and the 'points'
fallback when there are fewer outputs than ranks.  The engine is the oracle-backed stand-in
(tests/_fake_engine.py); on the GPU box the same GP code drives libgpmpc + NCCL."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import gp_oracle as orc
from tests._util import free_port


def _worker(rank, world, port, case, q):
    os.environ['MASTER_ADDR'] = '127.0.0.1'; os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        import gp_mpc_b200
        from tests._fake_engine import OracleEngine
        if case == 'outputs':
            p = orc.synthetic_problem(40, 4, 3, config_id=5, H=9)        # Ny=3 over 2 ranks: [0,2) and [2,3)
        else:
            p = orc.synthetic_problem(40, 3, 1, config_id=6, H=9)        # Ny=1 < world: replicate, split points
        Ny = p['Y'].shape[1]; Nx = p['X'].shape[1]
        hyper = dict(hyper=p['hyper'], invK=None, alpha=None, chol=None, length_scale=None, signal_var=None,
                     noise_var=None, mean=None)
        gp = gp_mpc_b200.GP(p['X'], p['Y'], hyper=hyper, normalize=False, engine_factory=OracleEngine)
        eng = gp.engine
        info = dict(rank=rank, begin=eng.out_begin, count=eng.out_count, uid_ok=(eng.uid == b'u' * 128) if case == 'outputs' else True)
        mean, cov = gp.predict_batch(p['Z'][:, :Ny], p['Z'][:, Ny:], p['Sigma'])
        chol = gp.get_chol()
        # sequential roll-out across ranks: one collective predict per step (the device-resident path needs all outputs on
        # one handle, so sharded models keep the host loop); default methods drop 'EM' when outputs are sharded
        roll = gp.rollout(p['Z'][0, :Ny], np.tile(p['Z'][:1, Ny:], (4, 1)), methods=['TA', 'ME'])
        # training path: every rank fits its own outputs, rows are gathered
        gp2 = gp_mpc_b200.GP(p['X'], p['Y'], normalize=False, engine_factory=OracleEngine,
                             optimizer_opts={'maxiter': 30})
        hy = np.column_stack([gp2.get_hyper_parameters()['length_scale'],
                              np.sqrt(gp2.get_hyper_parameters()['signal_var']),
                              np.sqrt(gp2.get_hyper_parameters()['noise_var'])])
        extra = {}
        if case == 'outputs':
            # ADVICE r1: only rank 1 "loses positive definiteness" on the 2nd appended point; the
            # refit fallback is a collective, so the decision must be collective (no hang, same N)
            OracleEngine.fail_on = (1, 41)
            rng = np.random.default_rng(3)
            Xn = rng.standard_normal((3, Nx)); Yn = rng.standard_normal((3, Ny))
            gp.append_data(Xn, Yn)
            OracleEngine.fail_on = None
            extra['N_after'] = gp.get_size()[0]
            extra['chol_after'] = gp.get_chol()
            extra['Xn'], extra['Yn'] = Xn, Yn
            try:
                gp.set_method('EM')
                extra['em'] = 'accepted'
            except NotImplementedError:
                extra['em'] = 'rejected'
        extra['roll'] = roll
        info.update(extra)
        q.put((rank, info, mean, cov, chol, hy))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('case', ['outputs', 'points'])
def test_two_ranks(case):
    world = 2
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, case, q)) for r in range(world)]
    for pr in procs:
        pr.start()
    res = sorted([q.get(timeout=240) for _ in range(world)], key=lambda t: t[0])
    for pr in procs:
        pr.join(timeout=60)
        assert pr.exitcode == 0
    if case == 'outputs':
        p = orc.synthetic_problem(40, 4, 3, config_id=5, H=9)
        assert [(r[1]['begin'], r[1]['count']) for r in res] == [(0, 2), (2, 1)]
    else:
        p = orc.synthetic_problem(40, 3, 1, config_id=6, H=9)
        assert [(r[1]['begin'], r[1]['count']) for r in res] == [(0, 1), (0, 1)]
    assert all(r[1]['uid_ok'] for r in res)
    post = orc.postfit(p['X'], p['Y'], p['hyper'], lapack_general_solve=False)
    mo, vo = orc.gp_mean_var(p['X'], p['hyper'], post['alpha'], post['chol'], p['Z'])
    co = orc.ta_cov(vo, orc.gp_mean_jac(p['X'], p['hyper'], post['alpha'], p['Z']), p['Sigma'])
    for r in res:
        np.testing.assert_allclose(r[2], mo, rtol=1e-10, atol=1e-12)        # every rank holds all outputs
        np.testing.assert_allclose(r[3], co, rtol=1e-9, atol=1e-14)
        np.testing.assert_allclose(r[4], post['chol'], rtol=1e-12, atol=1e-14)
    np.testing.assert_array_equal(res[0][5], res[1][5])                     # gathered hypers identical
    # the roll-out of the sharded / point-split model equals the single-process one
    import gp_mpc_b200
    from tests._fake_engine import OracleEngine
    Ny = p['Y'].shape[1]
    gp1 = gp_mpc_b200.GP(p['X'], p['Y'], hyper=dict(hyper=p['hyper']), normalize=False, engine_factory=OracleEngine)
    rm1, rv1 = gp1.rollout(p['Z'][0, :Ny], np.tile(p['Z'][:1, Ny:], (4, 1)), methods=['TA', 'ME'])
    for r in res:
        np.testing.assert_allclose(r[1]['roll'][0], rm1, rtol=1e-10, atol=1e-12)
        np.testing.assert_allclose(r[1]['roll'][1], rv1, rtol=1e-9, atol=1e-14)
    assert res[0][5].shape == (p['Y'].shape[1], p['X'].shape[1] + 2)
    # and equal to what one process fits (rank-local fits are independent per output)
    for a in range(p['Y'].shape[1]):
        assert orc.calc_NLL(res[0][5][a], p['X'], p['Y'][:, a]) < orc.calc_NLL(orc.train_bounds_init(p['X'], p['Y'][:, a])[1], p['X'], p['Y'][:, a])
    if case == 'outputs':
        for r in res:
            assert r[1]['N_after'] == 43 and r[1]['em'] == 'rejected'
        Xa = np.vstack([p['X'], res[0][1]['Xn']]); Ya = np.vstack([p['Y'], res[0][1]['Yn']])
        post = orc.postfit(Xa, Ya, p['hyper'], lapack_general_solve=False)
        for r in res:
            np.testing.assert_allclose(r[1]['chol_after'], post['chol'], rtol=1e-12, atol=1e-14)
