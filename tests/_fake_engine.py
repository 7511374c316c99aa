"""CPU stand-ins for gp_mpc_b200.Engine, for the tests of the host-side logic without a GPU: the world_size-2 gloo tests
of the multi-GPU logic (partitioning, id broadcast, hyper gather, result assembly), the GP class and the roll-outs; and
the fixture GPs and problems those tests build on them.  The numerics come from the oracle; the product never imports
this."""
import numpy as np
import torch.distributed as dist

import gp_mpc_b200
from gp_mpc_b200.gp_class import _matmul_seq
from oracle import gp_oracle as orc
from tests._util import load_fixture


class OracleEngine:
    def __init__(self, N, Nx, Ny, out_begin=0, out_count=None, device=0):
        self.N, self.Nx, self.Ny = N, Nx, Ny
        self.out_begin = out_begin
        self.out_count = Ny - out_begin if out_count is None else out_count
        self.rank, self.world = 0, 1
        self.uid = None
        self.closed = False

    @property
    def local_outputs(self):
        return range(self.out_begin, self.out_begin + self.out_count)

    @staticmethod
    def comm_unique_id():
        return b'u' * 128

    def comm_init(self, uid, rank, world):
        assert uid == b'u' * 128 and len(uid) == 128        # the id broadcast by rank 0 arrived intact
        self.rank, self.world, self.uid = rank, world, uid

    def set_data(self, X, Y):
        self.X, self.Y = np.array(X), np.array(Y)

    def set_hyper(self, hyper):
        self.hyper = np.array(hyper)

    def set_y(self, a, y):
        self.Y[:, a] = np.asarray(y)

    def set_option(self, name, value):
        pass

    def factorize(self, jitter=1e-8):
        rows = list(self.local_outputs)
        self.post = orc.postfit(self.X, self.Y[:, rows], self.hyper[rows], lapack_general_solve=False)
        return np.zeros(self.out_count, dtype=np.int32)

    def nlml(self, a, theta, grad=True):
        f = orc.calc_NLL(theta, self.X, self.Y[:, a], lapack_general_solve=False)
        return (f, orc.calc_NLL_grad_analytic(theta, self.X, self.Y[:, a])) if grad else f

    def get(self, what, a):
        k = a - self.out_begin
        return {0: self.post['chol'][k], 1: self.post['alpha'][k], 2: self.post['invK'][k]}[what]

    def predict(self, Z, Sigma=None, method=1, want_cov=True, want_jac=True):
        rows = list(self.local_outputs)
        Z = np.asarray(Z).reshape(-1, self.Nx)
        m, v = orc.gp_mean_var(self.X, self.hyper[rows], self.post['alpha'], self.post['chol'], Z)
        J = orc.gp_mean_jac(self.X, self.hyper[rows], self.post['alpha'], Z)
        if self.world > 1:                                   # what ncclAllGather does in libgpmpc
            parts = [None] * self.world
            dist.all_gather_object(parts, (self.out_begin, m, v, J))
            parts.sort(key=lambda t: t[0])
            m = np.concatenate([p[1] for p in parts], 1); v = np.concatenate([p[2] for p in parts], 1)
            J = np.concatenate([p[3] for p in parts], 1)
        cov = None
        if want_cov:
            cov = orc.ta_cov(v, J, Sigma) if (method == 1 and Sigma is not None) else orc.me_cov(v)
        return m, v, cov, (J if want_jac else None)

    # rank-1 append stand-in: refits with the oracle; `fail_on` = (rank, N) simulates ONE rank losing
    # positive definiteness (what gpmpc_append reports as GPMPC_ERR_NOTPD -> Engine.append False)
    fail_on = None

    def append(self, x_new, y_new):
        if OracleEngine.fail_on is not None and (self.rank, self.N) == tuple(OracleEngine.fail_on):
            return False
        self.X = np.vstack([self.X, np.asarray(x_new).reshape(1, -1)])
        self.Y = np.vstack([self.Y, np.asarray(y_new).reshape(1, -1)])
        self.N += 1
        self.factorize()
        return True

    def close(self):
        self.closed = True


class OracleEngineWithRollout(OracleEngine):
    """Adds a numpy restatement of gpmpc_rollout (include/gpmpc.h): the feedback arithmetic of
    rollout_feedback_kernel in the same operation order, the predict step from the oracle."""

    def rollout(self, z0, U, Sigma0, method=1, scale=None):
        Ny, Nx = self.Ny, self.Nx
        Nu = Nx - Ny
        U = np.asarray(U, dtype=np.float64).reshape(-1, Nu) if Nu > 0 else np.zeros((np.shape(U)[0], 0))
        Nt = U.shape[0]
        z = np.asarray(z0, dtype=np.float64).copy(); Sg = np.asarray(Sigma0, dtype=np.float64).copy()
        means = np.empty((Nt, Ny)); var = np.empty((Nt, Ny)); cov = None
        for t in range(Nt):
            m, v, cov, _ = self.predict(z.reshape(1, -1), Sg, method, True, False)
            means[t] = m[0]; var[t] = np.diag(cov[0])
            if t + 1 < Nt:
                zx = m[0]
                if scale is not None:
                    zx = ((zx * scale[0] + scale[1]) - scale[2]) / scale[3]
                z = np.concatenate([zx, U[t + 1]])
                Sg[:Ny, :Ny] = cov[0]
        return means, var, cov[0]



class OracleEngineWithRolloutBatch(OracleEngineWithRollout):
    """Adds a numpy restatement of gpmpc_rollout_batch (include/gpmpc.h): one predict step for all trajectories, then
    rollout_feedback_kernel's update per trajectory."""

    def rollout_batch(self, z0, U, Sigma0, method=1, scale=None, K=None, x_ref=None, uscale=None):
        Ny, Nx = self.Ny, self.Nx
        Nu = Nx - Ny
        Z = np.array(z0, dtype=np.float64).reshape(-1, Nx)
        B, Nt = Z.shape[0], np.shape(U)[1]
        S = np.array(Sigma0, dtype=np.float64).reshape(B, Nx, Nx)
        means = np.empty((B, Nt, Ny)); var = np.empty((B, Nt, Ny)); cov = None
        for t in range(Nt):
            # every trajectory's point on its own, as the device computes each point independently of the others
            parts = [self.predict(Z[b:b + 1], S[b], method, True, False) for b in range(B)]
            m = np.concatenate([p[0] for p in parts]); cov = np.concatenate([p[2] for p in parts])
            means[:, t] = m
            var[:, t] = np.diagonal(cov, axis1=1, axis2=2)
            if t + 1 == Nt:
                break
            x = m if scale is None else m * scale[0] + scale[1]
            Z[:, :Ny] = x if scale is None else (x - scale[2]) / scale[3]
            for b in range(B):
                if K is None:
                    Z[b, Ny:] = U[b, t + 1]
                else:
                    ub = _matmul_seq(K, (x[b] - (0.0 if x_ref is None else x_ref))[:, None])[:, 0]
                    Z[b, Ny:] = ub if uscale is None else (ub - uscale[0]) / uscale[1]
                    cov_xu = _matmul_seq(cov[b], K.T)
                    S[b, Ny:, Ny:] = _matmul_seq(_matmul_seq(K, cov[b]), K.T)
                    S[b, Ny:, :Ny] = cov_xu.T
                    S[b, :Ny, Ny:] = cov_xu
                S[b, :Ny, :Ny] = cov[b]
        return means, var, cov


class TwoRanks:
    """A two-rank communicator stand-in: enough for a GP sharded by output to be built on one process."""
    rank, world = 0, 2

    def broadcast_object(self, obj, src=0):
        return obj

    def allgather_object(self, obj):
        return [obj, obj]

    def barrier(self):
        pass


def sharded(base):
    """base with a comm_init that only records its rank and world: with TwoRanks, a GP sharded by output is built on one
    process."""
    class ShardEngine(base):
        def comm_init(self, uid, rank, world):
            self.rank, self.world = rank, world
    return ShardEngine


def fixture_gp(name, factory=None, **kw):
    """A GP of a stored fixture with its hyper-parameters (the engine factorises), and the fixture; factory replaces the
    device engine, kw override GP's arguments."""
    m = load_fixture(name)
    args = dict(mean_func='zero', gp_method='TA', normalize=m['normalize'], hyper=dict(hyper=m['hyper']))
    if factory is not None:
        args['engine_factory'] = factory
    if m['normalize']:
        args.update(meta=m['meta'], xlb=m['xlb'], xub=m['xub'], ulb=m['ulb'], uub=m['uub'])
    args.update(kw)
    return gp_mpc_b200.GP(m['X'], m['Y'], **args), m


def sample_model(name):
    """The model dict of a fixture, or of the synthetic problem of the sampled roll-out tests."""
    if name == 'synthetic':
        p = orc.synthetic_problem(150, 5, 3, config_id=2)
        p['hyper'][:, :5] = 1.5
        return dict(X=p['X'], Y=p['Y'], hyper=p['hyper'], normalize=False)
    return load_fixture(name)


def problem(case):
    """X, Y, hyper of a stored fixture ('tank', 'car') or of a small synthetic problem."""
    if case in ('tank', 'car'):
        m = load_fixture(case)
        return m['X'], m['Y'], m['hyper']
    p = orc.synthetic_problem(300, 5, 2, config_id=17)
    return p['X'], p['Y'], p['hyper']
