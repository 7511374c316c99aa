"""Batched open-loop roll-outs (gpmpc_rollout_batch) at a bench.py workload: B trajectories of Nt steps, one predict pass
over all B per step.  Prints one JSON line per B.

    python tools/bench_rollout_batch.py [--workload c2|c3|c5] [--batches 1,8,32,64] [--nt 10] [--reps 5] [--warmup 2]

`device_ms_per_step`: CUDA events on the engine's stream around one call (the H2D copy, the Nt predict passes with their
feedback kernels and the D2H copy), divided by Nt; the median of `--reps` calls after `--warmup` calls.
`traj_steps_per_s` = B / device_ms_per_step * 1e3; `ratio_to_b1` is device_ms_per_step over that of B = 1.
`parity_vs_host_loop`: trajectories 0 and B-1 against GP.rollout's host loop (one gpmpc_predict call per step),
batch-inf-norm relative over mean and variance, method TA."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
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


def _relinf(a, b):
    den = np.abs(b).max()
    return float(np.abs(a - b).max() / (den if den > 0 else 1.0))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='c2', choices=sorted(WORKLOADS))
    ap.add_argument('--batches', default='1,8,32,64')
    ap.add_argument('--nt', type=int, default=10)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    args = ap.parse_args()
    import torch
    import gp_mpc_b200
    from gp_mpc_b200 import _lib as L

    wl = WORKLOADS[args.workload]
    N, Nx, Ny = wl['N'], wl['Nx'], wl['Ny']
    w = make_workload(N, Nx, Ny, wl['cfg'], wl['H'])
    Nu, Nt = Nx - Ny, args.nt
    gp = gp_mpc_b200.GP(w['X'], w['Y'], normalize=False, hyper=dict(hyper=w['hyper']), device=0)
    eng = gp.engine
    stream = torch.cuda.ExternalStream(eng.stream())
    rng = np.random.default_rng(5)
    Bmax = max(int(b) for b in args.batches.split(','))
    rows = w['Z'][rng.integers(0, w['Z'].shape[0], Bmax)]           # starts and inputs drawn from the workload's test points
    X0 = rows[:, :Ny]
    U = np.repeat(rows[:, None, Ny:], Nt, 1) * (1 + 0.01 * np.arange(Nt)[None, :, None])
    S0 = np.tile(np.eye(Nx) * 1e-6, (Bmax, 1, 1))
    S0[:, :Ny, :Ny] = np.diag(w['hyper'][:, Nx + 1] ** 2)
    t_b1 = None
    for B in (int(b) for b in args.batches.split(',')):
        z0 = np.concatenate([X0[:B], U[:B, 0]], 1)

        def call():
            return eng.rollout_batch(z0, U[:B], S0[:B], L.METHOD_TA)

        for _ in range(args.warmup):
            call()
        times = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            call()
            e1.record(stream)
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
        ms = float(np.median(times)) / Nt
        t_b1 = ms if B == 1 else t_b1
        pick = [0, B - 1] if B > 1 else [0]
        dm, dv = gp.rollout(X0[:B], U[:B], methods=['TA'])
        hm, hv = gp.rollout(X0[pick], U[pick], methods=['TA'], device_rollout=False)
        parity = max(_relinf(dm[:, pick], hm), _relinf(dv[:, pick], hv))
        line = dict(metric='rollout_batch', workload=args.workload, N=N, Nx=Nx, Ny=Ny, Nu=Nu, Nt=Nt, B=B, method='TA',
                    device_ms_per_step=round(ms, 4), traj_steps_per_s=round(B / ms * 1e3, 1),
                    ratio_to_b1=round(ms / t_b1, 3) if t_b1 else None, parity_vs_host_loop=parity,
                    reps=args.reps, card=_card())
        print(json.dumps(line), flush=True)
    gp.close()


if __name__ == '__main__':
    main()
