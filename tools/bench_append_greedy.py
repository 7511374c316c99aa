"""Greedy max-variance selection: the device path (gpmpc_append_greedy, one call) against the host path (per pick a
predict of the pool's variances and one rank-1 append, GP.append_greedy(device_select=False)).  Prints one JSON line
per N.

    python tools/bench_append_greedy.py [--sizes 1024,4096,16384] [--ny 8] [--nx 10] [--pool 1024] [--picks 64]
                                        [--host-picks 16] [--reps 3]

`device_ms_per_pick`: CUDA events on the engine's stream around one Engine.append_greedy call (pool copy, pool V and
variances, the picks, alpha), divided by the picks; the median of `--reps` calls, each on a freshly factorised handle
with the capacity reserved (one untimed call first).  `host_ms_per_pick`: wall clock of the host path over
`--host-picks` picks, divided by them, on an engine with room reserved for them as well, so none of its rank-1 appends
falls back to a refit (without a reserve, N = 4096 and 16384 have no spare row and the first append refits).  `bytes_per_pick`: per output 8 Nk^2 / 2 (the lower triangle of L^-1 read for
the new row) + 8 n Nk (the pool's V read by the downdate), Nk the training size halfway through the selection;
`hbm_share` relates that traffic per device pick to the H100 SXM data-sheet bandwidth of 3.35 TB/s.
`picks_equal_host`: the host path's picks equal the first `--host-picks` device picks."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from bench import make_workload  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def _card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else None
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', default='1024,4096,16384')
    ap.add_argument('--ny', type=int, default=8)
    ap.add_argument('--nx', type=int, default=10)
    ap.add_argument('--pool', type=int, default=1024)
    ap.add_argument('--picks', type=int, default=64)
    ap.add_argument('--host-picks', type=int, default=16)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    import torch
    import gp_mpc_b200
    from gp_mpc_b200 import _lib as L

    card = _card()
    Ny, Nx, n, k = args.ny, args.nx, args.pool, args.picks
    for N in (int(s) for s in args.sizes.split(',')):
        w = make_workload(N, Nx, Ny, 5, 1)
        rng = np.random.default_rng(3)
        Xc = w['X'][rng.integers(0, N, n)] + 0.5 * rng.standard_normal((n, Nx))
        Yc = rng.standard_normal((n, Ny))

        def fresh():
            eng = L.Engine(N, Nx, Ny, device=0, capacity=N + k)
            eng.set_data(w['X'], w['Y'])
            eng.set_hyper(w['hyper'])
            eng.factorize()
            return eng

        times, picked = [], None
        for rep in range(args.reps + 1):
            eng = fresh()
            stream = torch.cuda.ExternalStream(eng.stream())
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            p, _, ok = eng.append_greedy(Xc, Yc, k)
            e1.record(stream)
            e1.synchronize()
            assert ok
            if rep:
                times.append(e0.elapsed_time(e1))
            picked = p if picked is None else picked
            assert np.array_equal(p, picked)
            eng.close()
        dev_ms = float(np.median(times)) / k
        def reserved(*a, **kw):
            kw.setdefault('capacity', N + args.host_picks)
            return L.Engine(*a, **kw)

        gp = gp_mpc_b200.GP(w['X'], w['Y'], normalize=False, hyper=dict(hyper=w['hyper']), device=0,
                            engine_factory=reserved)
        t0 = time.perf_counter()
        hp = gp.append_greedy(Xc, Yc, args.host_picks, device_select=False)
        host_ms = (time.perf_counter() - t0) * 1e3 / args.host_picks
        gp.close()
        Nk = N + k // 2
        nbytes = Ny * (8.0 * Nk * Nk / 2 + 8.0 * n * Nk)
        line = dict(metric='append_greedy', N=N, Nx=Nx, Ny=Ny, pool=n, picks=k, host_picks=args.host_picks,
                    device_ms_per_pick=round(dev_ms, 4), host_ms_per_pick=round(host_ms, 3),
                    speedup=round(host_ms / dev_ms, 1), bytes_per_pick=nbytes,
                    hbm_share=round(nbytes / (dev_ms * 1e-3) / HBM_BYTES_PER_S, 3),
                    picks_equal_host=bool(np.array_equal(hp, picked[:args.host_picks])), reps=args.reps, card=card)
        print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
