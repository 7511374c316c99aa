"""Removal of training points (gpmpc_remove) against the refit it replaces.  Prints one JSON line per N.

    python tools/bench_remove.py [--sizes 1024,4096,16384] [--ny 8] [--nx 10] [--reps 5] [--parity-max 4096]

Every time is a host clock (perf_counter) around calls that end in a device synchronise, the median of `--reps` calls
after one untimed call of the same kind, on one handle without a reserve (N = 4096 and 16384 have no spare row):
  remove_first_ms / remove_mid_ms  one Engine.remove([i]) at i = 0 / N/2 (an untimed append restores N after each);
  window_step_ms                   one remove([0]) + append(next point), the sliding-window step at a constant N;
  refit_ms                         one Engine.factorize() of the same model (K build, potrf, trtri, alpha): what a
                                   window step costs without a removal once the padded size is full.
`bytes_first` / `bytes_mid`: the least traffic of one removal, over all outputs: 16 (N^2 - i^2) bytes per output (the
lower triangles of L and L^-1 in rows > i, read once and written once) plus 8 N^2 (L^-1 read twice for alpha);
`hbm_share_*` relates them to the H100 SXM data-sheet bandwidth of 3.35 TB/s.  `chol_err` / `alpha_err`: relative
inf-norm difference of outputs 0 and Ny-1 from a LAPACK refit of the data the handle holds after the timed removals
and appends (N <= --parity-max).  `card`: name, power limit and max SM clock, read in the same run."""
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


def _relinf(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', default='1024,4096,16384')
    ap.add_argument('--ny', type=int, default=8)
    ap.add_argument('--nx', type=int, default=10)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--parity-max', type=int, default=4096)
    args = ap.parse_args()
    from gp_mpc_b200 import _lib as L
    from oracle import gp_oracle as orc

    card = _card()
    Ny, Nx, reps = args.ny, args.nx, args.reps
    for N in (int(s) for s in args.sizes.split(',')):
        w = make_workload(N, Nx, Ny, 5, 1)
        rng = np.random.default_rng(3)
        n_stream = 3 * (reps + 1)
        Xs = w['X'][rng.integers(0, N, n_stream)] + 0.3 * rng.standard_normal((n_stream, Nx))
        Ys = rng.standard_normal((n_stream, Ny))
        eng = L.Engine(N, Nx, Ny, device=0)
        eng.set_data(w['X'], w['Y'])
        eng.set_hyper(w['hyper'])
        eng.factorize()
        X, Y = w['X'].copy(), w['Y'].copy()          # the data the handle holds
        nxt = [0]

        def remove(i):
            nonlocal X, Y
            t0 = time.perf_counter()
            eng.remove([i])
            dt = time.perf_counter() - t0
            X, Y = np.delete(X, i, 0), np.delete(Y, i, 0)
            return dt

        def append():
            nonlocal X, Y
            k = nxt[0]
            nxt[0] += 1
            t0 = time.perf_counter()
            assert eng.append(Xs[k], Ys[k])
            dt = time.perf_counter() - t0
            X, Y = np.vstack([X, Xs[k]]), np.vstack([Y, Ys[k]])
            return dt

        def timed(step):
            ts = [step() for _ in range(reps + 1)][1:]
            return float(np.median(ts)) * 1e3

        def remove_then_refill(i):
            dt = remove(i)
            append()
            return dt

        first = timed(lambda: remove_then_refill(0))
        mid = timed(lambda: remove_then_refill(N // 2))
        window = timed(lambda: remove(0) + append())
        parity = {}
        if N <= args.parity_max:
            outs = [0, Ny - 1]
            post = orc.postfit(X, Y[:, outs], w['hyper'][outs], lapack_general_solve=False)
            parity['chol_err'] = max(_relinf(eng.get(L.GET_CHOL, a), post['chol'][k]) for k, a in enumerate(outs))
            parity['alpha_err'] = max(_relinf(eng.get(L.GET_ALPHA, a), post['alpha'][k]) for k, a in enumerate(outs))

        def refit():
            t0 = time.perf_counter()
            eng.factorize()
            return time.perf_counter() - t0

        refit_ms = timed(refit)
        line = dict(metric='remove', N=N, Nx=Nx, Ny=Ny, remove_first_ms=round(first, 3), remove_mid_ms=round(mid, 3),
                    window_step_ms=round(window, 3), refit_ms=round(refit_ms, 2),
                    refit_over_window_step=round(refit_ms / window, 1))
        for tag, i, ms in (('first', 0, first), ('mid', N // 2, mid)):
            nbytes = Ny * (16.0 * (N * N - i * i) + 8.0 * N * N)
            line['bytes_' + tag] = nbytes
            line['hbm_share_' + tag] = round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 3)
        line.update(parity, reps=reps, card=card)
        eng.close()
        print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
