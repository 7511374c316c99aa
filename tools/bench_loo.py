"""Leave-one-out cross-validation (gpmpc_loo, gpmpc_loo_nlpp) against the marginal likelihood it sits beside
(gpmpc_nlml).  Prints one JSON line per size.

    python tools/bench_loo.py [--sizes 1024:10:8,4096:10:8,8192:8:1] [--reps 10] [--numpy-max 4096]

Each size is N:Nx:Ny (8192:8:1 is the C4 shape).  Every time is a host clock (perf_counter) around calls that end in a
device synchronise, the median of `--reps` calls after one untimed call of the same kind:
  loo_ms                     one Engine.loo() on a factorised handle (all Ny outputs);
  loo_nlpp_ms / _grad_ms     one Engine.loo_nlpp(0, theta) without / with the gradient;
  nlml_ms / nlml_grad_ms     one Engine.nlml(0, theta) without / with the gradient, on the same handle;
  numpy_loo_ms               the closed form in numpy (LAPACK Cholesky, triangular inverse, column norms) for one
                             output, N <= --numpy-max.
`loo_bytes`: the least traffic of the column-norm pass, 4 N^2 bytes per output (the lower triangle of L^-1 read once);
`loo_hbm_share` relates it to the H100 SXM data-sheet bandwidth of 3.35 TB/s (the whole call, launches and copies
included, so it is a lower bound on the kernel's share).  `card`: name, power limit and max SM clock, read in the same
run."""
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


def _timed(fn, reps):
    ts = []
    for _ in range(reps + 1):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts[1:])) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', default='1024:10:8,4096:10:8,8192:8:1')
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--numpy-max', type=int, default=4096)
    args = ap.parse_args()
    from gp_mpc_b200 import _lib as L
    from oracle import loo_oracle as lo

    card = _card()
    for size in args.sizes.split(','):
        N, Nx, Ny = (int(s) for s in size.split(':'))
        w = make_workload(N, Nx, Ny, 5, 1)
        eng = L.Engine(N, Nx, Ny, device=0)
        eng.set_data(w['X'], w['Y'])
        eng.set_hyper(w['hyper'])
        eng.factorize()
        loo_ms = _timed(eng.loo, args.reps)
        theta = w['hyper'][0]
        line = dict(metric='loo', N=N, Nx=Nx, Ny=Ny, loo_ms=round(loo_ms, 4))
        line['loo_bytes'] = 4.0 * N * N * Ny
        line['loo_hbm_share'] = round(line['loo_bytes'] / (loo_ms * 1e-3) / HBM_BYTES_PER_S, 3)
        for key, fn in (('loo_nlpp_ms', lambda: eng.loo_nlpp(0, theta, grad=False)),
                        ('loo_nlpp_grad_ms', lambda: eng.loo_nlpp(0, theta, grad=True)),
                        ('nlml_ms', lambda: eng.nlml(0, theta, grad=False)),
                        ('nlml_grad_ms', lambda: eng.nlml(0, theta, grad=True))):
            line[key] = round(_timed(fn, args.reps), 3)
        line['loo_over_nlml'] = round(line['loo_nlpp_ms'] / line['nlml_ms'], 2)
        line['loo_grad_over_nlml_grad'] = round(line['loo_nlpp_grad_ms'] / line['nlml_grad_ms'], 2)
        if N <= args.numpy_max:
            line['numpy_loo_ms'] = round(_timed(lambda: lo.closed_form(w['X'], w['Y'][:, 0], theta), 2), 1)
        line.update(reps=args.reps, card=card)
        eng.close()
        print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
