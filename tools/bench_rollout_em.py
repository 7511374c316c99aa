"""'EM' roll-outs on the device (gpmpc_rollout_batch_em) against GP.rollout's host loop of gpmpc_predict(EM, H = 1)
calls at a bench.py workload, and gpmpc_predict(EM) at the workload's H across two builds of the library.

    python tools/bench_rollout_em.py [--workload c2|c3|c5] [--batches 1,8,32,64] [--nt 10] [--reps 3]
    python tools/bench_rollout_em.py --predict [--dump out.npz] [--root TREE]
    python tools/bench_rollout_em.py --ab OLD_TREE,NEW_TREE [--rounds 3] [--dump-dir DIR]

Roll-outs: one JSON line per B.  Both sides are host-timed whole calls (every copy and synchronisation inside), open loop,
starts and inputs drawn from the workload's test points: `device_ms_per_step` is the median of --reps calls of
Engine.rollout_batch_em after one warm-up, over Nt; `host_ms_per_step` one GP.rollout(device_rollout=False) over Nt;
`*_ms_per_point_step` divide by B as well.  `bits_equal_host_loop`: the two give the same means and variances bit for
bit.

--predict: one JSON line, gpmpc_predict(EM) at the workload's H with its shared Sigma, host-timed, median of 20 calls after
3; with --dump the EM outputs of the tank and car fixtures (gpmpc_predict(EM), gpmpc_predict_em_grad and
gpmpc_predict_em_hess at three points, per-point Sigma) go to an npz.  --root imports the package (and so its built
library) from another checkout of the repository, e.g. an older commit.  --ab runs --predict on each of two checkouts in
turn, --rounds times alternating, and reports whether every dumped array is identical between the two."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if '--root' in sys.argv:                 # before the imports below: the package and its library come from that tree
    ROOT = os.path.abspath(sys.argv[sys.argv.index('--root') + 1])
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from bench import WORKLOADS, make_workload  # noqa: E402


def _card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else None
    except (OSError, subprocess.SubprocessError):
        return None


def _engine(w, N, Nx, Ny):
    import gp_mpc_b200
    eng = gp_mpc_b200.Engine(N, Nx, Ny, device=0)
    eng.set_data(w['X'], w['Y'])
    eng.set_hyper(w['hyper'])
    eng.factorize()
    return eng


def rollouts(args):
    import gp_mpc_b200
    wl = WORKLOADS[args.workload]
    N, Nx, Ny = wl['N'], wl['Nx'], wl['Ny']
    w = make_workload(N, Nx, Ny, wl['cfg'], wl['H'])
    Nt = args.nt
    gp = gp_mpc_b200.GP(w['X'], w['Y'], normalize=False, hyper=dict(hyper=w['hyper']), device=0)
    eng = gp.engine
    rng = np.random.default_rng(5)
    Bs = [int(b) for b in args.batches.split(',')]
    rows = w['Z'][rng.integers(0, w['Z'].shape[0], max(Bs))]
    X0 = rows[:, :Ny]
    U = np.repeat(rows[:, None, Ny:], Nt, 1) * (1 + 0.01 * np.arange(Nt)[None, :, None])
    S0 = np.tile(np.eye(Nx) * 1e-6, (max(Bs), 1, 1))
    S0[:, :Ny, :Ny] = np.diag(w['hyper'][:, Nx + 1] ** 2)
    for B in Bs:
        z0 = np.concatenate([X0[:B], U[:B, 0]], 1)
        eng.rollout_batch_em(z0, U[:B], S0[:B])
        times = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            dm, dv, _ = eng.rollout_batch_em(z0, U[:B], S0[:B])
            times.append((time.perf_counter() - t0) * 1e3)
        dev = float(np.median(times)) / Nt
        t0 = time.perf_counter()
        hm, hv = gp.rollout(X0[:B], U[:B], methods=['EM'], device_rollout=False)
        host = (time.perf_counter() - t0) * 1e3 / Nt
        same = bool(np.array_equal(dm, hm[0, :, 1:]) and np.array_equal(dv, hv[0, :, 1:]))
        print(json.dumps(dict(metric='rollout_batch_em', workload=args.workload, N=N, Nx=Nx, Ny=Ny, Nt=Nt, B=B,
                              device_ms_per_step=round(dev, 3), host_ms_per_step=round(host, 3),
                              device_ms_per_point_step=round(dev / B, 4), host_ms_per_point_step=round(host / B, 4),
                              speedup=round(host / dev, 2), bits_equal_host_loop=same, reps=args.reps, card=_card())),
              flush=True)
    gp.close()


def _fixture_outputs():
    """EM outputs of the tank and car fixtures at three points with one Sigma each."""
    import gp_mpc_b200
    from gp_mpc_b200 import _lib as L
    from tests._util import load_fixture
    out = {}
    for name in ('tank', 'car'):
        m = load_fixture(name)
        N, Nx = m['X'].shape
        Ny = m['Y'].shape[1]
        eng = gp_mpc_b200.Engine(N, Nx, Ny, device=0)
        eng.set_data(m['X'], m['Y']); eng.set_hyper(m['hyper']); eng.factorize()
        rng = np.random.default_rng(11)
        Z = m['X'][:3] + 0.05 * rng.standard_normal((3, Nx))
        A = rng.standard_normal((3, Nx, Nx))
        S = 1e-3 * np.eye(Nx) + 1e-3 * A @ np.swapaxes(A, 1, 2)
        for k, v in zip(('mean', 'var', 'cov'), eng.predict(Z, S, L.METHOD_EM, want_jac=False)):
            out['%s_predict_%s' % (name, k)] = v
        for k, v in eng.predict_em_grad(Z, S).items():
            out['%s_grad_%s' % (name, k)] = v
        for k, v in eng.predict_em_hess(Z, S).items():
            out['%s_hess_%s' % (name, k)] = v
        eng.close()
    return out


def predict(args):
    from gp_mpc_b200 import _lib as L
    wl = WORKLOADS[args.workload]
    N, Nx, Ny, H = wl['N'], wl['Nx'], wl['Ny'], wl['H']
    w = make_workload(N, Nx, Ny, wl['cfg'], H)
    eng = _engine(w, N, Nx, Ny)
    for _ in range(3):
        eng.predict(w['Z'], w['Sigma'], L.METHOD_EM, want_jac=False)
    times = []
    for _ in range(20):
        t0 = time.perf_counter()
        eng.predict(w['Z'], w['Sigma'], L.METHOD_EM, want_jac=False)
        times.append((time.perf_counter() - t0) * 1e3)
    eng.close()
    if args.dump:
        np.savez(args.dump, **_fixture_outputs())
    print(json.dumps(dict(metric='predict_em', workload=args.workload, H=H, lib=L.LIB_PATH,
                          ms_median=round(float(np.median(times)), 3), ms_min=round(float(np.min(times)), 3),
                          card=_card())), flush=True)


def ab(args):
    trees = args.ab.split(',')
    args.dump_dir = args.dump_dir or tempfile.mkdtemp()
    os.makedirs(args.dump_dir, exist_ok=True)
    for r in range(args.rounds):
        for i, tree in enumerate(trees):
            dump = os.path.join(args.dump_dir, 'em_%d.npz' % i)
            subprocess.run([sys.executable, os.path.abspath(__file__), '--predict', '--workload', args.workload,
                            '--root', tree] + (['--dump', dump] if r == 0 else []), check=True)
    a, b = (np.load(os.path.join(args.dump_dir, 'em_%d.npz' % i)) for i in range(2))
    diff = sorted(k for k in a.files if not np.array_equal(a[k], b[k]))
    print(json.dumps(dict(metric='em_outputs_identical', arrays=len(a.files), identical=not diff, differing=diff)),
          flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='c2', choices=sorted(WORKLOADS))
    ap.add_argument('--batches', default='1,8,32,64')
    ap.add_argument('--nt', type=int, default=10)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--predict', action='store_true')
    ap.add_argument('--dump', default=None)
    ap.add_argument('--ab', default=None)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--dump-dir', default=None)
    ap.add_argument('--root', default=None)
    args = ap.parse_args()
    if args.ab:
        ab(args)
    elif args.predict:
        predict(args)
    else:
        rollouts(args)


if __name__ == '__main__':
    main()
