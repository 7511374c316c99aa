"""Forward-mode roll-out derivatives (gpmpc_rollout_batch_grad) against the roll-out alone (gpmpc_rollout_batch) and
against the P + 1 roll-outs a forward difference needs, on bench.py's synthetic problem.  Prints the card, then one JSON
line per (workload, feedback, B).

    python tools/bench_rollout_grad.py [--workloads c2,c5] [--batches 1,8,64] [--nt 10] [--reps 5] [--warmup 2]

Method 'TA'.  Open loop: P = Nx + (Nt-1) Nu parameters; feedback (one gain for the batch, the LQR gain of the first start):
P = Nx + Nu Ny.  `grad_ms_per_step` / `rollout_ms_per_step`: CUDA events on the engine's stream around one call (the H2D
copy, the Nt steps and the D2H copy), divided by Nt; median of `--reps` calls after `--warmup` calls.  `fd_ms` = (P + 1)
times the median rollout_batch call: what a forward difference over every parameter would spend on the device."""
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


def _time(stream, call, reps, warmup):
    import torch
    for _ in range(warmup):
        call()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        call()
        e1.record(stream)
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workloads', default='c2,c5')
    ap.add_argument('--batches', default='1,8,64')
    ap.add_argument('--nt', type=int, default=10)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    args = ap.parse_args()
    import torch
    import gp_mpc_b200
    from gp_mpc_b200 import _lib as L

    print(json.dumps(dict(card=_card())), flush=True)
    Nt = args.nt
    for wname in args.workloads.split(','):
        wl = WORKLOADS[wname]
        N, Nx, Ny = wl['N'], wl['Nx'], wl['Ny']
        Nu = Nx - Ny
        w = make_workload(N, Nx, Ny, wl['cfg'], wl['H'])
        gp = gp_mpc_b200.GP(w['X'], w['Y'], normalize=False, hyper=dict(hyper=w['hyper']), device=0)
        eng = gp.engine
        stream = torch.cuda.ExternalStream(eng.stream())
        rng = np.random.default_rng(5)
        Bmax = max(int(b) for b in args.batches.split(','))
        rows = w['Z'][rng.integers(0, w['Z'].shape[0], Bmax)]
        X0 = rows[:, :Ny]
        U = np.repeat(rows[:, None, Ny:], Nt, 1) * (1 + 0.01 * np.arange(Nt)[None, :, None])
        S0 = np.tile(np.eye(Nx) * 1e-6, (Bmax, 1, 1))
        S0[:, :Ny, :Ny] = np.diag(w['hyper'][:, Nx + 1] ** 2)
        A, Bm = gp.discrete_linearize(X0[0], U[0, 0], None)
        K = gp_mpc_b200.lqr(A, Bm, np.eye(Ny), np.eye(Nu))[0]
        x_ref = np.zeros(Ny)
        for fb in (False, True):
            for B in (int(b) for b in args.batches.split(',')):
                u0 = np.stack([K @ x for x in X0[:B]]) if fb else U[:B, 0]
                z0 = np.concatenate([X0[:B], u0], 1)
                a = (z0, U[:B], S0[:B], L.METHOD_TA, None) + ((K, x_ref, None) if fb else ())
                P = Nx + (Nu * Ny if fb else (Nt - 1) * Nu)
                t_grad = _time(stream, lambda: eng.rollout_batch_grad(*a), args.reps, args.warmup)
                t_roll = _time(stream, lambda: eng.rollout_batch(*a), args.reps, args.warmup)
                line = dict(metric='rollout_batch_grad', workload=wname, N=N, Nx=Nx, Ny=Ny, Nu=Nu, Nt=Nt, B=B, P=P,
                            method='TA', feedback=fb, grad_ms_per_step=round(t_grad / Nt, 4),
                            rollout_ms_per_step=round(t_roll / Nt, 4), ratio=round(t_grad / t_roll, 2),
                            fd_ms=round((P + 1) * t_roll, 3), grad_ms=round(t_grad, 3),
                            speedup_vs_fd=round((P + 1) * t_roll / t_grad, 1), reps=args.reps)
                print(json.dumps(line), flush=True)
        gp.close()


if __name__ == '__main__':
    main()
