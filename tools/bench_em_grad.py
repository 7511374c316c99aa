"""'EM' first derivatives (gpmpc_predict_em_grad) at a bench.py workload: the time of one host call next to the 'EM'
prediction it extends, the one-time cost of the K^-1 cache, and parity against the closed forms.  Prints one JSON line.

    python tools/bench_em_grad.py [--workload c2|c3|c5] [--steps K] [--warmup W] [--points P]

Both calls are host-timed (H2D, D2H and synchronisation inside, mean of K calls after W warm-up calls), Sigma shared by
the H points.  `first_call_ms` is the first gpmpc_predict_em_grad after gpmpc_factorize, which also builds the per-output
K^-1 cache; `kinv_cache_ms` is that call minus the steady-state one.  `em_grad_parity_vs_oracle` compares the first P
points with oracle/em_grad_oracle.em_grad_closed fed with the engine's own alpha and Cholesky factor (gpmpc_get),
batch-inf-norm relative."""
import argparse
import json
import os
import subprocess
import sys
import time

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='c2', choices=sorted(WORKLOADS))
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--points', type=int, default=2)
    args = ap.parse_args()
    import gp_mpc_b200
    from gp_mpc_b200 import _lib as L
    from oracle import em_grad_oracle as emo

    wl = WORKLOADS[args.workload]
    N, Nx, Ny, H = wl['N'], wl['Nx'], wl['Ny'], wl['H']
    w = make_workload(N, Nx, Ny, wl['cfg'], H)
    eng = gp_mpc_b200.Engine(N, Nx, Ny, 0, Ny, device=0)
    eng.set_data(w['X'], w['Y'])
    eng.set_hyper(w['hyper'])
    eng.factorize()
    Z, S = w['Z'], w['Sigma']

    def timed(fn):
        t0 = time.perf_counter()
        out = fn()
        return (time.perf_counter() - t0) * 1e3, out

    for _ in range(args.warmup):
        eng.predict(Z, S, L.METHOD_EM, want_jac=False)
    ms_first, _ = timed(lambda: eng.predict_em_grad(Z, S))
    for _ in range(args.warmup):
        eng.predict_em_grad(Z, S)
    ms_em = sum(timed(lambda: eng.predict(Z, S, L.METHOD_EM, want_jac=False))[0] for _ in range(args.steps)) / args.steps
    ms_g = 0.0
    for _ in range(args.steps):
        dt, g = timed(lambda: eng.predict_em_grad(Z, S))
        ms_g += dt / args.steps
    P = min(H, args.points)
    alpha = np.stack([eng.get(L.GET_ALPHA, a) for a in range(Ny)])
    chol = np.stack([eng.get(L.GET_CHOL, a) for a in range(Ny)])
    eng.close()
    ref = emo.em_grad_closed(w['X'], w['hyper'], alpha, chol, Z[:P], S)

    def rel(x, y):
        return float(np.abs(x - y).max() / max(np.abs(y).max(), 1e-300))

    par = {k: rel(g[k][:P], ref[k]) for k in ('dmean_dz', 'dmean_dSigma', 'dcov_dz', 'dcov_dSigma')}
    ok = par['dmean_dz'] < 1e-6 and par['dmean_dSigma'] < 1e-6 and par['dcov_dz'] < 1e-5 and par['dcov_dSigma'] < 1e-5
    par.update(max=max(par.values()), ok=bool(ok), points=P)
    print(json.dumps({'workload': wl['name'], 'method': 'EM', 'N': N, 'Nx': Nx, 'Ny': Ny, 'H': H, 'gpu': _card(),
                      'predict_em_ms_per_call': ms_em, 'em_grad_ms_per_call': ms_g,
                      'ratio_to_predict_em': ms_g / ms_em, 'first_call_ms': ms_first, 'kinv_cache_ms': ms_first - ms_g,
                      'em_grad_parity_vs_oracle': par}), flush=True)


if __name__ == '__main__':
    main()
