"""'EM' second derivatives (gpmpc_predict_em_hess) at a bench.py workload: the time of one host call next to
gpmpc_predict_em_grad and the 'EM' prediction it extends, the first call after gpmpc_factorize, and parity against the
closed forms.  Prints one JSON line.

    python tools/bench_em_hess.py [--workload c2|c3|c5] [--steps K] [--warmup W] [--points P]

`--nx16` runs N=1000, Nx=16, Ny=2, H=10 instead.  All calls are host-timed (H2D, D2H and synchronisation inside, mean of K calls after W warm-up calls), Sigma shared by
the H points.  `first_call_ms` is the first gpmpc_predict_em_hess after gpmpc_factorize, which also builds the
per-output K^-1 cache.  `em_hess_device_kernel_ms` sums the kernels of one call (torch.profiler), the rest of the call
is host work and copies.  `em_hess_parity_vs_oracle` compares the first P points with
oracle/em_hess_oracle.em_hess_closed fed with the engine's own alpha and Cholesky factor (gpmpc_get), batch-inf-norm
relative."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from bench import WORKLOADS, make_workload  # noqa: E402
from tools.bench_em_grad import _card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='c2', choices=sorted(WORKLOADS))
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--points', type=int, default=2)
    ap.add_argument('--nx16', action='store_true', help='N=1000, Nx=16, Ny=2, H=10 instead of the workload')
    args = ap.parse_args()
    import gp_mpc_b200
    from gp_mpc_b200 import _lib as L
    from oracle import em_hess_oracle as emh

    wl = dict(WORKLOADS[args.workload])
    if args.nx16:
        wl.update(N=1000, Nx=16, Ny=2, H=10, name='N=1000 Nx=16 Ny=2 H=10')
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
    ms_first, _ = timed(lambda: eng.predict_em_hess(Z, S))
    for _ in range(args.warmup):
        eng.predict_em_grad(Z, S)
        eng.predict_em_hess(Z, S)

    def mean_ms(fn):
        return sum(timed(fn)[0] for _ in range(args.steps)) / args.steps

    ms_em = mean_ms(lambda: eng.predict(Z, S, L.METHOD_EM, want_jac=False))
    ms_g = mean_ms(lambda: eng.predict_em_grad(Z, S))
    ms_h = 0.0
    for _ in range(args.steps):
        dt, o = timed(lambda: eng.predict_em_hess(Z, S))
        ms_h += dt / args.steps
    # device share: the kernels of one call (torch.profiler, CUDA activity); the rest of the call is host work and copies
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.predict_em_hess(Z, S)
        torch.cuda.synchronize()
    dev_ms = sum(e.device_time_total for e in prof.key_averages() if e.device_time_total > 0 and 'emcpy' not in e.key
                 and 'emset' not in e.key) / 1e3
    P = min(H, args.points)
    alpha = np.stack([eng.get(L.GET_ALPHA, a) for a in range(Ny)])
    chol = np.stack([eng.get(L.GET_CHOL, a) for a in range(Ny)])
    eng.close()
    par = None
    if P > 0:               # --points 0 skips the long-double oracle (minutes at Nx = 16, N = 1000)
        ref = emh.em_hess_closed(w['X'], w['hyper'], alpha, chol, Z[:P], S)

        def rel(x, y):
            return float(np.abs(x - y).max() / max(np.abs(y).max(), 1e-300))

        par = {k: rel(o[k][:P], ref[k]) for k in emh.KEYS}
        ok = all(par[k] < 1e-5 for k in emh.KEYS[:3]) and all(par[k] < 1e-4 for k in emh.KEYS[3:])
        par.update(max=max(par.values()), ok=bool(ok), points=P)
    print(json.dumps({'workload': wl['name'], 'method': 'EM', 'N': N, 'Nx': Nx, 'Ny': Ny, 'H': H, 'gpu': _card(),
                      'predict_em_ms_per_call': ms_em, 'em_grad_ms_per_call': ms_g, 'em_hess_ms_per_call': ms_h,
                      'ratio_to_em_grad': ms_h / ms_g, 'first_call_ms': ms_first,
                      'em_hess_device_kernel_ms': dev_ms, 'em_hess_host_and_copy_ms': ms_h - dev_ms,
                      'em_hess_parity_vs_oracle': par}), flush=True)


if __name__ == '__main__':
    main()
