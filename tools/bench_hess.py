"""Second derivatives of the prediction (gpmpc_predict_hess) at a bench.py workload: the time of one host call next to the
predict step, and its parity against the closed forms on an independent CPU factor.  Prints one JSON line.

    python tools/bench_hess.py [--workload c5|c3|c2] [--steps K] [--warmup W] [--points P]

The predict step is timed as bench.py times it (device pointers, CUDA events on the engine's stream, method TA, all outputs on
one GPU); the Hessian call is host-timed (H2D, D2H and synchronisation inside, mean of K calls after W warm-up calls).
`hess_parity_vs_oracle` compares outputs 0 and Ny-1 on the first P points with oracle/hess_oracle.predict_hess, batch-inf-norm
relative, on np.linalg.cholesky factors of the expansion-form K (oracle.gp_oracle.factor_large)."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from bench import WORKLOADS, make_workload  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='c5', choices=sorted(WORKLOADS))
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--points', type=int, default=4)
    args = ap.parse_args()
    import torch
    import gp_mpc_b200
    from gp_mpc_b200 import _lib as L
    from oracle import gp_oracle as orc
    from oracle import hess_oracle as hor

    wl = WORKLOADS[args.workload]
    N, Nx, Ny, H = wl['N'], wl['Nx'], wl['Ny'], wl['H']
    w = make_workload(N, Nx, Ny, wl['cfg'], H)
    eng = gp_mpc_b200.Engine(N, Nx, Ny, 0, Ny, device=0)
    eng.set_data(w['X'], w['Y'])
    eng.set_hyper(w['hyper'])
    eng.factorize()

    # predict step as bench.py measures it
    st = torch.cuda.ExternalStream(eng.stream())
    dZ = torch.from_numpy(w['Z']).cuda(); dS = torch.from_numpy(w['Sigma']).cuda()
    d_mean = torch.empty(H, Ny, dtype=torch.float64, device='cuda'); d_var = torch.empty_like(d_mean)
    d_cov = torch.empty(H, Ny, Ny, dtype=torch.float64, device='cuda')
    d_jac = torch.empty(H, Ny, Nx, dtype=torch.float64, device='cuda')
    torch.cuda.synchronize()

    def step_dev():
        eng.predict_device(L.METHOD_TA, H, dZ.data_ptr(), dS.data_ptr(), 0, d_mean.data_ptr(), d_var.data_ptr(),
                           d_cov.data_ptr(), d_jac.data_ptr(), sync=False)

    for _ in range(args.warmup):
        step_dev()
    eng.synchronize()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
    with torch.cuda.stream(st):
        for e0, e1 in evs:
            e0.record(st); step_dev(); e1.record(st)
    eng.synchronize()
    ms_step = sum(e0.elapsed_time(e1) for e0, e1 in evs) / args.steps
    for _ in range(args.warmup):
        eng.predict(w['Z'], w['Sigma'], L.METHOD_TA)
    t0 = time.perf_counter()
    for _ in range(args.steps):
        eng.predict(w['Z'], w['Sigma'], L.METHOD_TA)
    ms_e2e = (time.perf_counter() - t0) / args.steps * 1e3

    for _ in range(args.warmup):
        eng.predict_hess(w['Z'], w['Sigma'], L.METHOD_TA)
    t0 = time.perf_counter()
    for _ in range(args.steps):
        gh = eng.predict_hess(w['Z'], w['Sigma'], L.METHOD_TA)
    ms_h = (time.perf_counter() - t0) / args.steps * 1e3
    eng.close()

    outs = sorted({0, Ny - 1})
    P = min(H, args.points)
    facs = [orc.factor_large(w['X'], w['Y'][:, a], w['hyper'][a]) for a in outs]
    ho = hor.predict_hess(w['X'], w['hyper'][outs], [f['alpha'] for f in facs], [f['chol'] for f in facs],
                          w['Z'][:P], w['Sigma'], 'TA')

    def rel(x, y):
        return float(np.abs(x - y).max() / max(np.abs(y).max(), 1e-300))

    par = {'d2var': rel(gh['d2var_dz2'][:P, outs], ho['d2var']), 'd3mean': rel(gh['d3mean_dz3'][:P, outs], ho['d3mean']),
           'd2cov': rel(gh['d2cov_dz2'][:P][:, outs][:, :, outs], ho['d2cov'])}
    par.update(max=max(par.values()), tol=1e-6, ok=bool(max(par.values()) < 1e-6), outputs_checked=outs, points=P)
    print(json.dumps({'workload': wl['name'], 'method': 'TA', 'gpu': torch.cuda.get_device_name(0),
                      'hess_ms_per_call': ms_h, 'predict_ms_per_step': ms_step, 'predict_e2e_ms_per_call': ms_e2e,
                      'ratio_to_predict_step': ms_h / ms_step, 'ratio_to_predict_e2e': ms_h / ms_e2e,
                      'hess_parity_vs_oracle': par}), flush=True)


if __name__ == '__main__':
    main()
