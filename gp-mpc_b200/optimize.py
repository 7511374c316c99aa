"""Hyper-parameter fit driver on top of the CUDA engine.

Mirrors ``train_gp_numpy`` (reference optimize.py:359-503): per output, SLSQP
from the reference's initial point and bounds, then the post-fit block (K ->
chol -> alpha) -- except that every NLML evaluation is one call into
libgpmpc (`gpmpc_nlml`: K build + tensor-core Cholesky + logdet, on the GPU)
and, by default, SLSQP receives the ANALYTIC gradient from the same call instead
of the reference's forward differences (optimize.py:466-467).  ``jac='fd'``
reproduces the reference's finite-difference trajectory (each FD probe is again
a GPU NLML evaluation).

``optimizer_opts={'starts': 'lhs', 'seed': s}`` with ``multistart=S > 1`` fits each
output from S starting points (start 0 the reference's, the rest a Latin hypercube,
``lhs_starts``) as S SLSQP solves in lockstep: every round's objective values come
from one `gpmpc_nlml_batch` call.
"""
from __future__ import annotations

import threading
import time

import numpy as np


from .mean_functions import count_mean_params, mean_bounds, mean_design


def bounds_and_init(X, y, fixed_bounds=False):
    """Bounds / start of optimize.py:433-451 for the zero-mean model.
    ``lb[:Nx] = 1-2`` (= -1) is the reference's typo for 1e-2 (SURVEY q7); it is
    replicated unless ``fixed_bounds``."""
    N, Nx = X.shape
    num_hyp = Nx + 2
    lb = -np.inf * np.ones(num_hyp)
    ub = np.inf * np.ones(num_hyp)
    lb[:Nx] = 1e-2 if fixed_bounds else 1 - 2
    ub[:Nx] = 2e2
    lb[Nx] = 1e-8
    ub[Nx] = 1e2
    lb[Nx + 1] = 10 ** -10
    ub[Nx + 1] = 10 ** -2
    init = np.zeros(num_hyp)
    init[:Nx] = np.std(X, 0)
    init[Nx] = np.std(y)
    init[Nx + 1] = 1e-5
    return np.hstack((lb.reshape(num_hyp, 1), ub.reshape(num_hyp, 1))), init


def lhs_starts(init, bounds, S, seed, a):
    """S starting points of output a: row 0 is init, rows 1..S-1 a Latin hypercube u in [0,1)^(Nx+2) seeded by (seed, a)
    alone, mapped to ell_d, sf = init * 10^(2u-1) (one decade either side of the reference's start) and
    sn = 10^(-6+4u), then clipped into the bounds (DESIGN section 4.15)."""
    from scipy.stats import qmc
    init = np.asarray(init, dtype=np.float64)
    d = init.size
    starts = np.tile(init, (S, 1))
    if S > 1:
        u = qmc.LatinHypercube(d=d, rng=np.random.default_rng(np.random.SeedSequence([int(seed), int(a)]))).random(S - 1)
        starts[1:, :d - 1] = init[:d - 1] * 10.0 ** (2.0 * u[:, :d - 1] - 1.0)
        starts[1:, d - 1] = 10.0 ** (-6.0 + 4.0 * u[:, d - 1])
        starts[1:] = np.clip(starts[1:], bounds[:d, 0], bounds[:d, 1])
    return starts


def fit_objective(optimizer_opts):
    """The objective optimizer_opts['objective'] selects, checked before any engine call:
    'nlml' (default), the negative log marginal likelihood (gpmpc_nlml, R&W eq. 5.9), or
    'loo', the negative leave-one-out log predictive probability (gpmpc_loo_nlpp, R&W eqs. 5.10-5.13), which is more
    robust than the marginal likelihood when the SE kernel is misspecified.  'loo' does not fit mean parameters.
    optimizer_opts['starts'] = 'lhs' (multi-start from a Latin hypercube) works with 'nlml' and without fit_mean."""
    opts = optimizer_opts or {}
    objective = opts.get('objective', 'nlml')
    if objective not in ('nlml', 'loo'):
        raise ValueError("optimizer_opts['objective'] must be 'nlml' or 'loo', got %r" % (objective,))
    if objective == 'loo' and opts.get('fit_mean', False):
        raise ValueError("optimizer_opts: objective 'loo' cannot fit mean parameters (fit_mean=True)")
    starts = opts.get('starts')
    if starts not in (None, 'lhs'):
        raise ValueError("optimizer_opts['starts'] must be 'lhs', got %r" % (starts,))
    if starts == 'lhs' and objective == 'loo':
        raise ValueError("optimizer_opts: 'starts': 'lhs' supports objective 'nlml' only")
    if starts == 'lhs' and opts.get('fit_mean', False):
        raise ValueError("optimizer_opts: 'starts': 'lhs' cannot fit mean parameters (fit_mean=True)")
    return objective


class _Abandoned(Exception):
    """Raised inside a start's objective when its evaluation reported NOTPD: that start's solve stops."""


class _Lockstep:
    """S SLSQP solves of one output, one thread each, sharing every objective evaluation round.  Each start posts its theta
    and waits; the last live start to post evaluates every posted row, in start order, with one nlml_batch call and
    hands the results back.  A start that finishes leaves, and the rounds go on without it.  Each start's values are
    those gpmpc_nlml gives it alone, so its trajectory is the one a single-start SLSQP from its point follows."""

    def __init__(self, eng, a, S, grad):
        self.eng, self.a, self.grad = eng, a, grad
        self.cv = threading.Condition()
        self.live = set(range(S))
        self.posted, self.results = {}, {}

    def _run(self):
        order = sorted(self.posted)
        try:
            nll, g, status = self.eng.nlml_batch(self.a, np.array([self.posted[s] for s in order]), grad=self.grad)
            for i, s in enumerate(order):
                self.results[s] = ((float(nll[i]), g[i].copy()) if self.grad else float(nll[i]), int(status[i]))
        except Exception as e:          # every waiting start re-raises it
            for s in order:
                self.results[s] = e
        self.posted.clear()
        self.cv.notify_all()

    def evaluate(self, s, theta):
        with self.cv:
            self.posted[s] = np.array(theta, dtype=np.float64)
            if set(self.posted) == self.live:
                self._run()
            while s not in self.results:
                self.cv.wait()
            r = self.results.pop(s)
        if isinstance(r, Exception):
            raise r
        value, status = r
        if status < 0:
            raise _Abandoned()
        return value

    def leave(self, s):
        with self.cv:
            self.live.discard(s)
            if self.posted and set(self.posted) == self.live:
                self._run()


def train_gp_b200(engine, X, Y, meanFunc='zero', hyper_init=None, multistart=1,
                  optimizer_opts=None, verbose=True):
    """Fit the outputs owned by `engine`; returns hyper rows for those outputs
    (shape (out_count, Nx+2)) -- the caller gathers them across ranks."""
    from scipy.optimize import minimize

    # 'const' / 'linear' / 'polynomial' add h_m mean parameters to every hyper row
    # (optimize.py:402-417).  In the reference's NUMERIC path (the default, and the one mirrored
    # here) the objective ignores them (calc_NLL_numpy reads hyper[:Nx+2] only, optimize.py:337-340;
    # "only support a zero-mean function", :377-379), their bounds are set after `bounds` was built
    # (:435-460) and therefore never reach SLSQP, so they stay at their initial value 0 and the
    # fitted prior mean is identically zero.  That behaviour is the default here: zero columns.
    # optimizer_opts={'fit_mean': True} instead fits them jointly with the kernel parameters on the
    # objective of the reference's CasADi/IPOPT twin (calc_NLL, optimize.py:22-97: NLL of the
    # residual y - m(X)), with the mean bounds of optimize.py:452-459; the extra gradient block is
    # d NLL / d params = -Phi^T alpha (m = Phi params is linear in its parameters).
    h_m = count_mean_params(meanFunc, X.shape[1])
    N, Nx = X.shape
    options = {'disp': False, 'maxiter': 10000}
    jac_mode = 'analytic'
    fixed_bounds = False
    fit_mean = False
    parallel_fits = True
    starts, seed = None, 0
    objective = fit_objective(optimizer_opts)
    if optimizer_opts is not None:
        optimizer_opts = dict(optimizer_opts)
        starts = optimizer_opts.pop('starts', None)
        seed = int(optimizer_opts.pop('seed', 0))
        jac_mode = optimizer_opts.pop('jac', jac_mode)
        fixed_bounds = bool(optimizer_opts.pop('fixed_bounds', False))
        fit_mean = bool(optimizer_opts.pop('fit_mean', False)) and h_m > 0
        parallel_fits = bool(optimizer_opts.pop('parallel_fits', True))
        optimizer_opts.pop('objective', None)
        options.update(optimizer_opts)
    if jac_mode not in ('analytic', 'fd'):
        raise ValueError("optimizer_opts['jac'] must be 'analytic' or 'fd'")

    if verbose:
        print('\n________________________________________')
        print('# Optimizing hyperparameters (N=%d)' % N)
        print('----------------------------------------')
    rows = np.zeros((engine.out_count, Nx + 2 + h_m))
    # without 'starts', multistart re-runs from the SAME init (optimize.py:462-469, q8): identical results, so one run
    # decides
    S = int(multistart) if starts == 'lhs' else 1

    def fit_starts(eng, a, bounds, init):
        """S lockstep SLSQP solves of output a from lhs_starts; returns (best row, (winner, best, worst, abandoned))."""
        grad = jac_mode == 'analytic'
        x0 = lhs_starts(init, bounds, S, seed, a)
        group = _Lockstep(eng, a, S, grad)
        res, errors = [None] * S, [None] * S

        def solve(s):
            try:
                res[s] = minimize(lambda th: group.evaluate(s, th), x0[s], method='SLSQP', jac=grad, options=options,
                                  bounds=bounds, tol=1e-12)
            except _Abandoned:
                pass
            except Exception as e:
                errors[s] = e
            finally:
                group.leave(s)

        threads = [threading.Thread(target=solve, args=(s,)) for s in range(S)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        for e in errors:
            if e is not None:
                raise e
        final = [r.fun if r is not None and np.isfinite(r.fun) else np.inf for r in res]
        win = int(np.argmin(final))             # the first of equal values: ties go to the lowest start
        if not np.isfinite(final[win]):
            raise np.linalg.LinAlgError('gpmpc_nlml_batch: output %d: K not positive definite even with jitter at every '
                                        'one of its %d starts' % (a, S))
        done = [f for f in final if np.isfinite(f)]
        return res[win].x, (win, final[win], max(done), S - len(done))

    def fit_one(eng, a):
        """SLSQP for output a on `eng` (any engine that owns a); returns (hyper row, seconds, multi-start summary)."""
        bounds, init = bounds_and_init(X, Y[:, a], fixed_bounds)
        if hyper_init is not None:
            init = np.asarray(hyper_init, dtype=np.float64)[a, :Nx + 2].copy()
        if fit_mean:
            from ._lib import GET_ALPHA_NLML
            Phi = mean_design(X, meanFunc)
            bounds = np.vstack([bounds, mean_bounds(Y[:, a], Nx, meanFunc)])
            init = np.concatenate([init[:Nx + 2], np.zeros(h_m) if hyper_init is None
                                   else np.asarray(hyper_init, dtype=np.float64)[a, Nx + 2:Nx + 2 + h_m]])
            init = np.clip(init, bounds[:, 0], bounds[:, 1])

        def fun(theta):
            if fit_mean:
                eng.set_y(a, Y[:, a] - Phi @ theta[Nx + 2:])
                if jac_mode != 'analytic':
                    return eng.nlml(a, theta[:Nx + 2], grad=False)
                nll, g = eng.nlml(a, theta[:Nx + 2], grad=True)
                return nll, np.concatenate([g, -Phi.T @ eng.get(GET_ALPHA_NLML, a)])
            if jac_mode == 'analytic':
                return eng.nlml(a, theta, grad=True)
            return eng.nlml(a, theta, grad=False)

        t0 = time.time()
        if S > 1:
            x, info = fit_starts(eng, a, bounds, init)
            return x, time.time() - t0, info
        if objective == 'loo':
            # SLSQP runs on theta / scale with sn measured in units of its upper bound: dNLPP/dsn is ~1e5 times the other
            # components where sn ~ 1e-3, and unscaled the quasi-Newton steps stall far from a stationary point
            # (DESIGN section 4.13).  Same bounds and initial point in theta.
            scale = np.ones(Nx + 2)
            scale[Nx + 1] = bounds[Nx + 1, 1]

            def fun_loo(x):
                if jac_mode != 'analytic':
                    return eng.loo_nlpp(a, x * scale, grad=False)
                f, g = eng.loo_nlpp(a, x * scale, grad=True)
                return f, g * scale

            res = minimize(fun_loo, init / scale, method='SLSQP', jac=(jac_mode == 'analytic'), options=options,
                           bounds=bounds / scale[:, None], tol=1e-12)
            return np.clip(res.x * scale, bounds[:, 0], bounds[:, 1]), time.time() - t0, None
        res = minimize(fun, init, method='SLSQP', jac=(jac_mode == 'analytic'), options=options,
                       bounds=bounds, tol=1e-12)
        if fit_mean:
            eng.set_y(a, Y[:, a])
        return res.x, time.time() - t0, None

    def fit_scratch(a):
        """fit_one on a scratch engine of output a, closed afterwards: a multi-start pass's slabs never stay on the
        caller's handle."""
        w = type(engine)(engine.N, Nx, engine.Ny, a, 1, getattr(engine, 'device', 0))
        try:
            w.set_data(X, Y)
            return fit_one(w, a)
        finally:
            w.close()

    outs = list(engine.local_outputs)
    workers = None
    if parallel_fits and len(outs) > 1 and hasattr(engine, 'device'):
        # The per-output fits are independent (optimize.py:433 loops over them) and each NLML evaluation
        # is latency-bound below N ~ 8192 (its potrf recursion leaves most SMs idle): run them
        # concurrently, one scratch engine (own CUDA streams) and one host thread per output.  ctypes
        # releases the GIL inside the library calls.  Falls back to the sequential loop when the
        # scratch engines do not fit in device memory.
        try:
            workers = []
            for a in outs:
                w = type(engine)(engine.N, Nx, engine.Ny, a, 1, engine.device)
                w.set_data(X, Y)
                workers.append(w)
        except Exception:
            for w in workers or []:
                w.close()
            workers = None
    if workers and S > 1:
        # the workers share the GPU: cap each one's nlml_batch pass so that all of them fit in the free memory.  A pass
        # entry holds two Npad^2 slabs and the recursion's workspaces (about 2/3 Npad^2): 3 Npad^2 doubles bound it.
        try:
            import torch
            free = torch.cuda.mem_get_info(engine.device)[0]
        except Exception:
            free = None
        if free is not None:
            npad = -(-engine.N // 128) * 128
            cap = max(1, int(0.9 * free) // (len(workers) * 3 * npad * npad * 8))
            if cap < S:
                for w in workers:
                    w.set_option('nlml_batch_max', cap)
    if workers:
        from concurrent.futures import ThreadPoolExecutor
        try:
            with ThreadPoolExecutor(max_workers=len(outs)) as ex:
                futs = [ex.submit(fit_one, w, a) for w, a in zip(workers, outs)]
                results = [f.result() for f in futs]
        finally:
            for w in workers:
                w.close()
    elif S > 1:
        results = [fit_scratch(a) for a in outs]
    else:
        results = [fit_one(engine, a) for a in outs]
    for k, (a, (x, secs, info)) in enumerate(zip(outs, results)):
        if verbose and info is not None:
            print("* State %d:  %f s  (start %d of %d wins: NLML %.6g, worst %.6g, %d abandoned)"
                  % (a, secs, info[0], S, info[1], info[2], info[3]))
        elif verbose:
            print("* State %d:  %f s" % (a, secs))
        rows[k, :len(x)] = x
    if verbose:
        print('----------------------------------------')
    return rows
