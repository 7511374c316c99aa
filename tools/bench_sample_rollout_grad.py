"""Pathwise derivatives of sampled roll-outs (gpmpc_rollout_sample_grad) against the sampled roll-out alone
(gpmpc_rollout_sample) and against the P + 1 sample calls of the difference quotient it replaces, for the same B
trajectories of Nt steps.  Prints one JSON line per (N, B) with the card's name, power limit and SM clock.

    python tools/bench_sample_rollout_grad.py [--sizes 1000,4096,16384] [--batches 16,64] [--nt 30] [--reps 3] [--warmup 1]

Synthetic problem of bench.py (Nx = 10, Ny = 8, so Nu = 2; open loop, P = Nx + (Nt-1) Nu = 68 at Nt = 30).
`grad_ms_per_step` / `sample_ms_per_step`: CUDA events on the engine's stream around one call (H2D copy, the Nt steps, D2H
copy and the host-side reordering), divided by Nt; the median of `--reps` calls after `--warmup` calls.
`quotient_ms_per_step` = (P + 1) sample_ms_per_step, the forward differences of P + 1 sample calls.  `extra_gb`: the
device memory the derivatives add (beta store, U = L^-1^T, dR, the tangent history), from the header's formulas.  At
N = 16384 the beta and V stores grow with B Nt: B = 256 with Nt = 30 does not fit beside the factor on an 80 GB card."""
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
    ap.add_argument('--sizes', default='1000,4096,16384')
    ap.add_argument('--batches', default='16,64')
    ap.add_argument('--nt', type=int, default=30)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    args = ap.parse_args()
    import torch
    import gp_mpc_b200

    Nx, Ny, Nt = 10, 8, args.nt
    Nu = Nx - Ny
    P = Nx + (Nt - 1) * Nu
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
            ms_g = _time(stream, lambda: eng.rollout_sample_grad(z0, U, eps), args.reps, args.warmup) / Nt
            ms_s = _time(stream, lambda: eng.rollout_sample(z0, U, eps), args.reps, args.warmup) / Nt
            ref, got = eng.rollout_sample(z0, U, eps), eng.rollout_sample_grad(z0, U, eps)
            npad = eng.capacity
            extra = 8.0 * (Ny * Nt * B * npad + Ny * npad * npad + Ny * B * P * Nt * Nt + Nt * B * P * Nx) / 1e9
            line = dict(metric='rollout_sample_grad', N=N, Nx=Nx, Ny=Ny, B=B, Nt=Nt, P=P,
                        grad_ms_per_step=round(ms_g, 4), sample_ms_per_step=round(ms_s, 4),
                        quotient_ms_per_step=round((P + 1) * ms_s, 3), grad_over_sample=round(ms_g / ms_s, 3),
                        quotient_over_grad=round((P + 1) * ms_s / ms_g, 2),
                        draws_bit_identical=all(bool(np.array_equal(x, y)) for x, y in zip(ref, got[:3])),
                        kept_fraction=float(got[2].mean()), extra_gb=round(extra, 3), reps=args.reps, card=card)
            print(json.dumps(line), flush=True)
        eng.close()
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
