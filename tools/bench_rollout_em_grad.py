"""Derivatives of 'EM' roll-outs on the device (gpmpc_rollout_batch_em_grad) against the roll-out alone
(gpmpc_rollout_batch_em) and against the P + 1 roll-outs of the forward difference quotient it replaces, at a bench.py
workload.

    python tools/bench_rollout_em_grad.py [--workload c2|c3] [--batches 1,8,32] [--nt 10] [--reps 3] [--step 1e-7]

One JSON line per B, open loop, starts and inputs drawn from the workload's test points.  Every time is a host-timed
whole call (every copy and synchronisation inside), the median of --reps calls after one warm-up, over Nt:
`grad_ms_per_step` for Engine.rollout_batch_em_grad, `rollout_ms_per_step` for Engine.rollout_batch_em and
`quotient_ms_per_step` for the P + 1 calls of Engine.rollout_batch_em that forward differences need (P = Nx + (Nt-1) Nu
parameters per trajectory, all B trajectories perturbed in one call); `*_per_point_step` divide by B as well.
`quotient_parity`: relinf of the quotient's dmeans and dvars against the entry's (relative step --step).  `card`: the
GPU's name, power limit and maximum SM clock, read in the same run."""
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


def _timed(f, reps):
    f()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        r = f()
        times.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(times)), r


def _relinf(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='c2', choices=['c2', 'c3'])
    ap.add_argument('--batches', default='1,8,32')
    ap.add_argument('--nt', type=int, default=10)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--step', type=float, default=1e-7)
    args = ap.parse_args()
    import gp_mpc_b200
    wl = WORKLOADS[args.workload]
    N, Nx, Ny = wl['N'], wl['Nx'], wl['Ny']
    Nu, Nt = Nx - Ny, args.nt
    w = make_workload(N, Nx, Ny, wl['cfg'], wl['H'])
    eng = gp_mpc_b200.Engine(N, Nx, Ny, device=0)
    eng.set_data(w['X'], w['Y']); eng.set_hyper(w['hyper']); eng.factorize()
    rng = np.random.default_rng(5)
    Bs = [int(b) for b in args.batches.split(',')]
    rows = w['Z'][rng.integers(0, w['Z'].shape[0], max(Bs))]
    U = np.repeat(rows[:, None, Ny:], Nt, 1) * (1 + 0.01 * np.arange(Nt)[None, :, None])
    S0 = np.tile(np.eye(Nx) * 1e-6, (max(Bs), 1, 1))
    S0[:, :Ny, :Ny] = np.diag(w['hyper'][:, Nx + 1] ** 2)
    P = Nx + (Nt - 1) * Nu
    card = _card()
    for B in Bs:
        z0, Ub, S = rows[:B].copy(), U[:B].copy(), S0[:B]
        t_grad, (_, _, _, dm, dv) = _timed(lambda: eng.rollout_batch_em_grad(z0, Ub, S), args.reps)
        t_roll, _ = _timed(lambda: eng.rollout_batch_em(z0, Ub, S), args.reps)

        def quotient():
            m0, v0, _ = eng.rollout_batch_em(z0, Ub, S)
            fm, fv = np.zeros_like(dm), np.zeros_like(dv)
            for p in range(P):
                zp, Up = z0.copy(), Ub.copy()
                if p < Nx:
                    h = args.step * np.maximum(1.0, np.abs(z0[:, p])); zp[:, p] += h
                else:
                    r, i = 1 + (p - Nx) // Nu, (p - Nx) % Nu
                    h = args.step * np.maximum(1.0, np.abs(Ub[:, r, i])); Up[:, r, i] += h
                mp, vp, _ = eng.rollout_batch_em(zp, Up, S)
                fm[..., p] = (mp - m0) / h[:, None, None]
                fv[..., p] = (vp - v0) / h[:, None, None]
            return fm, fv
        t_fd, (fm, fv) = _timed(quotient, args.reps)
        print(json.dumps(dict(metric='rollout_batch_em_grad', workload=args.workload, N=N, Nx=Nx, Ny=Ny, Nt=Nt, B=B, P=P,
                              grad_ms_per_step=round(t_grad / Nt, 3), rollout_ms_per_step=round(t_roll / Nt, 3),
                              quotient_ms_per_step=round(t_fd / Nt, 3),
                              grad_ms_per_point_step=round(t_grad / Nt / B, 4),
                              rollout_ms_per_point_step=round(t_roll / Nt / B, 4),
                              quotient_ms_per_point_step=round(t_fd / Nt / B, 4),
                              speedup_vs_quotient=round(t_fd / t_grad, 2),
                              quotient_parity=dict(dmeans=_relinf(fm, dm), dvars=_relinf(fv, dv)), step=args.step,
                              reps=args.reps, card=card)), flush=True)
    eng.close()


if __name__ == '__main__':
    main()
