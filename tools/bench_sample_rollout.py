"""Sampled roll-outs (gpmpc_rollout_sample) against propagated-moment roll-outs (gpmpc_rollout_batch, 'TA') for the same
B trajectories of Nt steps.  Prints one JSON line per (N, B) with the card's name, power limit and SM clock.

    python tools/bench_sample_rollout.py [--sizes 1024,4096,16384] [--batches 64,256] [--nt 30] [--reps 3] [--warmup 1]

Synthetic problem of bench.py (Nx = 10, Ny = 8, so Nu = 2).  `sample_ms_per_step` / `rollout_batch_ms_per_step`: CUDA
events on the engine's stream around one call (H2D copy, the Nt steps, D2H copy and the host-side reordering), divided by
Nt; the median of `--reps` calls after `--warmup` calls.  `v_store_gb`: the device store of solved rows the sampled call
keeps (Ny Nt B Npad doubles)."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from bench import make_workload  # noqa: E402


def _card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else None
    except (OSError, subprocess.SubprocessError):
        return None


def _time(stream, fn, reps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fn()
        e1.record(stream)
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', default='1024,4096,16384')
    ap.add_argument('--batches', default='64,256')
    ap.add_argument('--nt', type=int, default=30)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    args = ap.parse_args()
    import torch
    import gp_mpc_b200
    from gp_mpc_b200 import _lib as L

    Nx, Ny, Nt = 10, 8, args.nt
    card = _card()
    for N in (int(s) for s in args.sizes.split(',')):
        w = make_workload(N, Nx, Ny, 5, 64)
        eng = gp_mpc_b200.Engine(N, Nx, Ny, device=0)
        eng.set_data(w['X'], w['Y']); eng.set_hyper(w['hyper']); eng.factorize()
        stream = torch.cuda.ExternalStream(eng.stream())
        rng = np.random.default_rng(5)
        for B in (int(b) for b in args.batches.split(',')):
            rows = w['X'][rng.integers(0, N, B)]
            z0 = rows + 0.05 * rng.standard_normal((B, Nx))
            U = np.repeat(z0[:, None, Ny:], Nt, 1)
            eps = rng.standard_normal((B, Nt, Ny))
            S0 = np.tile(np.eye(Nx) * 1e-6, (B, 1, 1))
            S0[:, :Ny, :Ny] = np.diag(w['hyper'][:, Nx + 1] ** 2)
            ms_s = _time(stream, lambda: eng.rollout_sample(z0, U, eps), args.reps, args.warmup) / Nt
            ms_r = _time(stream, lambda: eng.rollout_batch(z0, U, S0, L.METHOD_TA), args.reps, args.warmup) / Nt
            kept = eng.rollout_sample(z0, U, eps)[2]
            line = dict(metric='rollout_sample', N=N, Nx=Nx, Ny=Ny, B=B, Nt=Nt,
                        sample_ms_per_step=round(ms_s, 4), rollout_batch_ms_per_step=round(ms_r, 4),
                        ratio=round(ms_s / ms_r, 3), kept_fraction=float(kept.mean()),
                        v_store_gb=round(8.0 * Ny * Nt * B * eng.capacity / 1e9, 3), reps=args.reps, card=card)
            print(json.dumps(line), flush=True)
        eng.close()
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
