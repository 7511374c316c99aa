"""gpmpc_nlml_batch against sequential gpmpc_nlml calls, and multi-start fit wall time.

1. One nlml_batch call of S rows against S nlml calls (S = 1, 4, 16), with and without the gradient, at N = 1000, 2048,
   4096, 8192 and Nx = 8.  Both entries synchronise the device before they return, so host timing covers the work; each
   figure is the median of `--reps` repeats after one warm-up call of the same shape.
2. The fit at C2 (N = 1000, Nx = 8, Ny = 6): multistart=1 against multistart=8 with 'starts': 'lhs', wall time, the
   final NLML per output and how many outputs improved.
Prints one JSON object, with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import gp_mpc_b200                                    # noqa: E402
from gp_mpc_b200.optimize import train_gp_b200        # noqa: E402
from bench import make_workload                       # noqa: E402


def _card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'unknown'


def _median_s(f, reps):
    f()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        f()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', type=int, nargs='+', default=[1000, 2048, 4096, 8192])
    ap.add_argument('--starts', type=int, nargs='+', default=[1, 4, 16])
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--no-fit', action='store_true')
    args = ap.parse_args()
    out = {'card': _card(), 'calls_ms': {}}
    for N in args.sizes:
        w = make_workload(N, 8, 1, 4, 30)
        eng = gp_mpc_b200.Engine(N, 8, 1, device=0)
        eng.set_data(w['X'], w['Y'])
        rng = np.random.default_rng(N)
        for S in args.starts:
            th = np.tile(w['hyper'][0], (S, 1)) * 2.0 ** rng.uniform(-0.5, 0.5, (S, 10))
            th[:, 9] = 10.0 ** rng.uniform(-3, -2, S)
            for grad in (True, False):
                batch = _median_s(lambda: eng.nlml_batch(0, th, grad=grad), args.reps)
                seq = _median_s(lambda: [eng.nlml(0, t, grad=grad) for t in th], args.reps)
                out['calls_ms']['N=%d S=%d grad=%d' % (N, S, grad)] = {
                    'batch': batch * 1e3, 'sequential': seq * 1e3, 'sequential/batch': seq / batch}
        eng.close()
    if not args.no_fit:
        w = make_workload(1000, 8, 6, 4, 30)
        X, Y = w['X'], w['Y']
        fits = {}
        for S, opts in ((1, None), (8, {'starts': 'lhs'})):
            eng = gp_mpc_b200.Engine(1000, 8, 6, device=0)
            eng.set_data(X, Y)
            t0 = time.perf_counter()
            rows = train_gp_b200(eng, X, Y, multistart=S, optimizer_opts=opts, verbose=False)
            secs = time.perf_counter() - t0
            fits[S] = (secs, [eng.nlml(a, rows[a], grad=False) for a in range(6)])
            eng.close()
        out['fit_C2'] = {'multistart=1_s': fits[1][0], 'multistart=8_lhs_s': fits[8][0],
                         'nlml_multistart=1': fits[1][1], 'nlml_multistart=8_lhs': fits[8][1],
                         'outputs_improved': int(sum(b < a for a, b in zip(fits[1][1], fits[8][1])))}
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
