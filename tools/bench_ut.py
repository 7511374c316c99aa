"""The unscented transform ('UT') against 'TA' and 'EM' at bench.py's workloads: gpmpc_predict per method, and
gpmpc_rollout_batch('UT') against gpmpc_rollout_batch('TA').

    python tools/bench_ut.py [--workloads c2,c3,c5] [--reps 20] [--rounds 3] [--em-points c5:1] [--B 64] [--nt 30]

One JSON line per case.  Every timing is a host clock around whole calls, which synchronise (copies included), on one
handle that owns every output (C5 on a single GPU).  Each case runs one warm-up call, then --rounds rounds in which the
methods take turns, --reps calls each; `ms_median` is the median over all of a method's calls, `spread` the ratio of the
slowest to the fastest round median.  'EM' at C5 costs seconds per call, so --em-points caps its point count per workload
(default c5:1) and its line gives the time per point as well.  Roll-outs: B trajectories of Nt steps, open loop, starts
and inputs drawn from the workload's test points; --reps / 10 calls per round (one call runs all Nt steps)."""
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


def _timed(fn, reps):
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        out.append((time.perf_counter() - t0) * 1e3)
    return out


def _alternate(calls, reps, rounds):
    """{name: fn} -> {name: (all times, round medians)}, one warm-up call each, then the names in turn per round."""
    for fn in calls.values():
        fn()
    res = {k: ([], []) for k in calls}
    for _ in range(rounds):
        for k, fn in calls.items():
            t = _timed(fn, reps)
            res[k][0].extend(t); res[k][1].append(float(np.median(t)))
    return res


def _stats(times, medians):
    return dict(ms_median=round(float(np.median(times)), 4), ms_min=round(float(np.min(times)), 4),
                spread=round(max(medians) / min(medians), 3))


def run(name, args, card):
    import gp_mpc_b200
    from gp_mpc_b200 import _lib as L
    wl = WORKLOADS[name]
    N, Nx, Ny, H = wl['N'], wl['Nx'], wl['Ny'], wl['H']
    w = make_workload(N, Nx, Ny, wl['cfg'], H)
    eng = gp_mpc_b200.Engine(N, Nx, Ny, device=0)
    eng.set_data(w['X'], w['Y']); eng.set_hyper(w['hyper']); eng.factorize()
    Z, S = w['Z'], w['Sigma']
    head = dict(workload=name, N=N, Nx=Nx, Ny=Ny, card=card)
    res = _alternate({'UT': lambda: eng.predict(Z, S, L.METHOD_UT),
                      'TA': lambda: eng.predict(Z, S, L.METHOD_TA)}, args.reps, args.rounds)
    for meth, (t, med) in res.items():
        print(json.dumps(dict(metric='predict', method=meth, H=H, **_stats(t, med), **head)), flush=True)
    He = min(H, args.em_points.get(name, H))
    t, med = _alternate({'EM': lambda: eng.predict(Z[:He], S, L.METHOD_EM, want_jac=False)},
                        max(1, args.reps // (10 if He < H else 1)), args.rounds)['EM']
    st = _stats(t, med)
    print(json.dumps(dict(metric='predict', method='EM', H=He, ms_per_point=round(st['ms_median'] / He, 4), **st,
                          **head)), flush=True)
    # roll-outs: B trajectories, Nt steps, open loop
    B, Nt, Nu = args.B, args.nt, Nx - Ny
    rng = np.random.default_rng(5)
    rows = Z[rng.integers(0, H, B)]
    U = np.repeat(rows[:, None, Ny:], Nt, 1) * (1 + 0.01 * np.arange(Nt)[None, :, None])
    S0 = np.tile(np.eye(Nx) * 1e-6, (B, 1, 1))
    S0[:, :Ny, :Ny] = np.diag(w['hyper'][:, Nx + 1] ** 2)
    z0 = np.concatenate([rows[:, :Ny], U[:, 0]], 1)
    res = _alternate({m: (lambda m=m: eng.rollout_batch(z0, U, S0, m)) for m in (L.METHOD_UT, L.METHOD_TA)},
                     max(1, args.reps // 10), args.rounds)
    for m, (t, med) in res.items():
        st = _stats(t, med)
        print(json.dumps(dict(metric='rollout_batch', method={L.METHOD_UT: 'UT', L.METHOD_TA: 'TA'}[m], B=B, Nt=Nt, Nu=Nu,
                              ms_per_step=round(st['ms_median'] / Nt, 4), **st, **head)), flush=True)
    eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workloads', default='c2,c3,c5')
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--em-points', default='c5:1', help='workload:points caps of the EM timing, comma separated')
    ap.add_argument('--B', type=int, default=64)
    ap.add_argument('--nt', type=int, default=30)
    args = ap.parse_args()
    args.em_points = {k: int(v) for k, v in (p.split(':') for p in args.em_points.split(',') if p)}
    card = _card()
    for name in args.workloads.split(','):
        run(name, args, card)


if __name__ == '__main__':
    main()
