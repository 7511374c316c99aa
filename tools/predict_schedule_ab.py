"""A/B of the predict product alone (PROF_TRIGEMM) between builds of libgpmpc.so, alternating in one session.

Each round runs every library once, in a child process of its own (GPMPC_LIB), on the C5 model (N=16384, Nx=10, 8
outputs): the product's mean time over --reps launches at each H of --hs, then at H=50 on each grid size of --ctas.
Prints the card's name, power limit and maximum SM clock first, then one line per (round, library) and a min-max
summary per library.
    python tools/predict_schedule_ab.py --lib parent=/path/libgpmpc.so --lib new=gp-mpc_b200/lib/libgpmpc.so
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def child(args):
    sys.path.insert(0, ROOT)
    import gp_mpc_b200
    from gp_mpc_b200 import _lib as L
    from bench import make_workload
    w = make_workload(args.n, 10, 8, 5, 50)
    eng = gp_mpc_b200.Engine(args.n, 10, 8, device=0)
    eng.set_data(w['X'], w['Y'])
    eng.set_hyper(w['hyper'])
    eng.factorize()
    eng.predict(w['Z'], w['Sigma'], L.METHOD_TA)
    res = {'H%d' % H: eng.profile(L.PROF_TRIGEMM, n=H, reps=args.reps) for H in args.hs}
    for c in args.ctas:
        eng.set_option('predict_ctas', c)
        res['H50_ctas%d' % c] = eng.profile(L.PROF_TRIGEMM, n=50, reps=args.reps)
    eng.set_option('predict_ctas', 0)
    eng.close()
    print('RESULT ' + json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--lib', action='append', default=[], help='NAME=PATH of a libgpmpc.so (repeatable)')
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--reps', type=int, default=30)
    ap.add_argument('--n', type=int, default=16384)
    ap.add_argument('--hs', default='1,8,32,50,56,64')
    ap.add_argument('--ctas', default='128', help='grid sizes timed at H=50 besides the automatic one ("" for none)')
    ap.add_argument('--child', action='store_true')
    args = ap.parse_args()
    args.hs = [int(x) for x in args.hs.split(',') if x]
    args.ctas = [int(x) for x in args.ctas.split(',') if x]
    if args.child:
        return child(args)
    libs = [kv.split('=', 1) for kv in args.lib] or [['tree', os.path.join(ROOT, 'gp-mpc_b200', 'lib', 'libgpmpc.so')]]
    print(subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip(), flush=True)
    runs = {name: [] for name, _ in libs}
    for r in range(args.rounds):
        for name, path in libs:
            env = dict(os.environ, GPMPC_LIB=os.path.abspath(path))
            cmd = [sys.executable, os.path.abspath(__file__), '--child', '--n', str(args.n), '--reps', str(args.reps),
                   '--hs', ','.join(map(str, args.hs)), '--ctas', ','.join(map(str, args.ctas))]
            out = subprocess.run(cmd, env=env, capture_output=True, text=True, check=True).stdout
            res = json.loads(next(l for l in out.splitlines() if l.startswith('RESULT '))[7:])
            runs[name].append(res)
            print('round %d %-8s ' % (r, name) + '  '.join('%s %.4f' % kv for kv in res.items()), flush=True)
    for name, rs in runs.items():
        print('%-8s ' % name + '  '.join('%s %.4f-%.4f ms' % (k, min(x[k] for x in rs), max(x[k] for x in rs))
                                         for k in rs[0]), flush=True)


if __name__ == '__main__':
    main()
