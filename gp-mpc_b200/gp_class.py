"""``GP`` -- the host-side mirror of the reference's ``gp_mpc.gp_class.GP``
(gp_class.py:20-861) whose arithmetic runs in libgpmpc (hand-written sm_90a CUDA).

Same constructor, method names, argument meaning, return shapes, printed banners
and error types as the reference; what changes is where the numbers are made:

  reference                                          here
  -------------------------------------------------  ----------------------------------
  train_gp_numpy + SLSQP/FD  (optimize.py:359-503)   optimize.train_gp_b200 -> gpmpc_nlml
  post-fit chol/alpha/invK   (optimize.py:479-494)   gpmpc_factorize / gpmpc_get
  build_gp / build_TA_cov    (gp_functions.py:72-173) gpmpc_predict (ME / TA, batched)
  GP.covSEard / GP.covar     (gp_class.py:314-381)   gpmpc_build_K / gpmpc_predict

Host work kept in numpy is exactly what the reference keeps on the host:
standardisation of a handful of numbers (gp_class.py:253-262), JSON I/O.
There is no CPU fallback for the dense algebra.
"""
from __future__ import annotations

import json
import os

import numpy as np
import scipy.linalg

from . import _lib
from .comm import Comm
from .mean_functions import mean_function, mean_jacobian
from .optimize import fit_objective, train_gp_b200
from .partition import choose_mode, output_block, point_block

_GPU_METHODS = {'ME': _lib.METHOD_ME, 'TA': _lib.METHOD_TA, 'EM': _lib.METHOD_EM, 'UT': _lib.METHOD_UT}
_KNOWN_METHODS = ('ME', 'TA', 'EM', 'UT', 'old_ME', 'old_TA')      # gp_class.py:197-205, and the unscented transform
_SIGMA_METHODS = ('TA', 'EM', 'UT')                                # the methods that read the input covariance


def _matmul_seq(A, B):
    """A @ B with every sum in index order and separate multiplies and adds, as rollout_feedback_kernel forms the
    feedback products.  BLAS's order and use of fused multiply-adds differ between builds, and a closed loop amplifies
    one rounding step (1e-10 on the car model), so the host loop and the device roll-out share this order."""
    out = np.zeros((A.shape[0], B.shape[1]))
    for k in range(A.shape[1]):
        out = out + A[:, k:k + 1] * B[k:k + 1, :]
    return out


def lqr(A, B, Q, R):
    """ Infinite-horizon discrete-time LQR for x[k+1] = A x[k] + B u[k], u[k] = K x[k] (the reference's
    ``lqr``, mpc_class.py:956-976): P solves the discrete algebraic Riccati equation and
    K = -(R + B^T P B)^-1 B^T P A.  Returns K (Nu, Ny), P and the eigenvalues of A + B K. """
    A = np.asarray(A, dtype=np.float64); B = np.asarray(B, dtype=np.float64)
    P = scipy.linalg.solve_discrete_are(A, B, np.asarray(Q, dtype=np.float64), np.asarray(R, dtype=np.float64))
    BtP = B.T @ P
    K = -np.linalg.solve(R + BtP @ B, BtP @ A)
    return K, P, np.linalg.eigvals(A + B @ K)


def _sqrt_psd(S):
    """F with F F^T = S: the Cholesky factor, or for a singular S the eigenvalue square root (zero on its null space)."""
    try:
        return np.linalg.cholesky(S)
    except np.linalg.LinAlgError:
        w, V = np.linalg.eigh(S)
        return V * np.sqrt(np.clip(w, 0.0, None))[None, :]


def _is_symbolic(v):
    """CasADi SX/MX arguments (mpc_class.py:390-412 calls predict with MX symbols)."""
    return type(v).__module__.split('.')[0] == 'casadi' and type(v).__name__ in ('MX', 'SX')


class GP:
    def __init__(self, X, Y, mean_func="zero", gp_method="TA",
                 optimizer_opts=None, hyper=None, normalize=True, multistart=1,
                 xlb=None, xub=None, ulb=None, uub=None, meta=None,
                 optimize_nummeric=True, device=None, comm=None, engine_factory=None,
                 prior_mean_in_predict=False):
        """ Initialize and optimize GP model  (reference gp_class.py:21-75)

        Extra keyword arguments (not in the reference): ``device`` (CUDA ordinal,
        default $LOCAL_RANK or 0), ``comm`` (a ``Comm``; default: the initialised
        torch.distributed world, else single process), ``engine_factory`` (tests),
        ``prior_mean_in_predict``: the reference fits alpha on y - m(X) (optimize.py:492-494) but
        never adds the prior mean m(z) back when predicting (build_gp is always called without
        meanFunc, gp_class.py:69-71; SURVEY q2).  False (default) replicates that; True adds m(z)
        to the predicted mean and d m/d z to the Jacobian / Taylor covariance.
        """
        X = np.array(X, dtype=np.float64).copy()
        Y = np.array(Y, dtype=np.float64).copy()
        if X.ndim != 2 or Y.ndim != 2 or X.shape[0] != Y.shape[0]:
            raise ValueError('X must be (N, Nx) and Y (N, Ny) with the same N')
        self.__X = X
        self.__Y = Y
        self.__Ny = Y.shape[1]
        self.__Nx = X.shape[1]
        self.__N = X.shape[0]
        self.__Nu = self.__Nx - self.__Ny            # gp_class.py:36 (q5)

        self.__gp_method = gp_method
        self.__mean_func = mean_func
        self.__normalize = normalize
        self.__comm = comm if comm is not None else Comm()
        self.__device = int(device if device is not None else os.environ.get('LOCAL_RANK', 0))
        self.__engine_factory = engine_factory or _lib.Engine
        self.__engine = None
        self.__invK = None
        self.__prior_mean_in_predict = bool(prior_mean_in_predict)
        self.__ut_params = None                      # (alpha, beta, kappa) of 'UT'; None: the engine's defaults
        self.__xlb = self.__xub = self.__ulb = self.__uub = None

        if meta is not None:                         # gp_class.py:42-50
            self.__meanY = np.array(meta['meanY'])
            self.__stdY = np.array(meta['stdY'])
            self.__meanZ = np.array(meta['meanZ'])
            self.__stdZ = np.array(meta['stdZ'])
            self.__meanX = np.array(meta['meanX'])
            self.__stdX = np.array(meta['stdX'])
            self.__meanU = np.array(meta['meanU'])
            self.__stdU = np.array(meta['stdU'])
        if xlb is not None:                          # kept so load_model -> save_model round-trips
            self.__xlb, self.__xub = np.array(xlb), np.array(xub)
            self.__ulb, self.__uub = np.array(ulb), np.array(uub)

        """ Optimize hyperparameters """
        if hyper is None:
            self.optimize(X=X, Y=Y, opts=optimizer_opts, mean_func=mean_func,
                          xlb=xlb, xub=xub, ulb=ulb, uub=uub,
                          multistart=multistart, normalize=normalize,
                          optimize_nummeric=optimize_nummeric)
        else:
            # gp_class.py:58-66: a saved model carries (hyper, invK, alpha, chol).  The stored
            # X,Y are already standardised (:697-698) and are not re-standardised.  The factors
            # are recomputed on the GPU from (X, hyper): L^-1, which the predict kernels need,
            # is not part of the saved model.
            self.__hyper = np.array(hyper['hyper'], dtype=np.float64)
            self.__set_hyper_views()
            self.__refit()

        self.set_method(gp_method)

    # ------------------------------------------------------------------ engine plumbing
    def __set_hyper_views(self):
        Nx = self.__Nx                               # gp_class.py:139-142 (q1)
        self.__hyper_length_scales = self.__hyper[:, :Nx]
        self.__hyper_signal_variance = self.__hyper[:, Nx] ** 2
        self.__hyper_noise_variance = self.__hyper[:, Nx + 1] ** 2
        self.__hyper_mean = self.__hyper[:, (Nx + 1):]

    def __build_engine(self, capacity=None):
        """capacity: training points to reserve room for (append_greedy); passed to the factory only when given."""
        if self.__engine is not None:
            self.__engine.close()
        c = self.__comm
        self.__mode = choose_mode(self.__Ny, c.world)
        if self.__mode == 'outputs':
            b, n = output_block(self.__Ny, c.rank, c.world)
        else:
            b, n = 0, self.__Ny
        kw = {} if capacity is None else dict(capacity=int(capacity))
        self.__engine = self.__engine_factory(self.__N, self.__Nx, self.__Ny, b, n, self.__device, **kw)
        self.__engine.set_data(self.__X, self.__Y)
        if self.__ut_params is not None:
            self.__engine.set_ut_params(*self.__ut_params)
        if c.world > 1 and self.__mode == 'outputs':
            uid = self.__engine_factory.comm_unique_id() if c.rank == 0 else None
            uid = c.broadcast_object(uid, src=0)
            self.__engine.comm_init(uid, c.rank, c.world)
            # fused epilogue + all-gather over NVLink peer memory (CUDA IPC); NCCL stays the fallback
            if hasattr(self.__engine, 'peer_export') and os.environ.get('GPMPC_NO_PEER', '0') != '1':
                self.__attach_peers(c)

    def __attach_peers(self, c):
        """CUDA-IPC exchange blocks for the fused epilogue/all-gather.  The decision is collective:
        if any rank cannot export or map a peer block (no P2P, IPC disabled in the container),
        every rank falls back to the NCCL gather."""
        eng = self.__engine
        try:
            mine = eng.peer_export(int(os.environ.get('GPMPC_PEER_HCAP', 256)))
        except Exception:
            mine = None
        handles = c.allgather_object(mine)
        ok = all(hd is not None for hd in handles)
        if ok:
            try:
                eng.peer_attach(handles)
            except Exception:
                ok = False
        if not all(c.allgather_object(ok)):
            eng.set_option('peer', 0)

    def __has_prior_mean(self):
        return self.__mean_func != 'zero' and self.__hyper.shape[1] > self.__Nx + 2

    def __engine_targets(self, X, Y):
        """The targets the engine factorises: the residual Y - m(X) under a prior mean (alpha = K^-1 (y - m(X)),
        optimize.py:492-494), else Y."""
        if not self.__has_prior_mean():
            return Y
        return Y - np.column_stack([mean_function(self.__hyper[a], X, self.__mean_func) for a in range(self.__Ny)])

    def __factorize(self):
        if self.__has_prior_mean():
            T = self.__engine_targets(self.__X, self.__Y)
            for a in self.__engine.local_outputs:
                self.__engine.set_y(a, T[:, a])
        self.__engine.set_hyper(self.__hyper)
        info = self.__engine.factorize(1e-8)
        for k, a in enumerate(self.__engine.local_outputs):
            if info[k] == 1:                         # optimize.py:486
                print("K matrix is not positive definit, adding jitter!")
        self.__invK = None
        # ranks factorise independently (a jitter retry on one rank can take seconds at large N):
        # line them up again before the first predict step's peer exchange starts its timeout clock
        if self.__comm.world > 1:
            self.__comm.barrier()

    def __refit(self, capacity=None):
        """A new engine on the current X, Y, factorised at the current hyper-parameters."""
        self.__build_engine(capacity)
        self.__factorize()

    def __set_data(self, X, Y):
        self.__X, self.__Y, self.__N = X, Y, X.shape[0]
        self.__invK = None

    @property
    def engine(self):
        return self.__engine

    # ------------------------------------------------------------------ training
    def optimize(self, X=None, Y=None, opts=None, mean_func='zero',
                 xlb=None, xub=None, ulb=None, uub=None,
                 multistart=1, normalize=True, warm_start=False,
                 optimize_nummeric=True):
        """reference gp_class.py:78-142.  opts={'objective': 'loo'} fits the leave-one-out predictive probability
        instead of the marginal likelihood (optimize.fit_objective)."""
        fit_objective(opts)
        self.__mean_func = mean_func
        self.__normalize = normalize

        if normalize and X is not None:              # :85-99  (population std, ddof=0)
            self.__xlb = np.array(xlb)
            self.__xub = np.array(xub)
            self.__ulb = np.array(ulb)
            self.__uub = np.array(uub)
            self.__meanY = np.mean(Y, 0)
            self.__stdY = np.std(Y, 0)
            self.__meanZ = np.mean(X, 0)
            self.__stdZ = np.std(X, 0)
            self.__meanX = np.mean(X[:, :self.__Ny], 0)
            self.__stdX = np.std(X[:, :self.__Ny], 0)
            self.__meanU = np.mean(X[:, self.__Ny:], 0)
            self.__stdU = np.std(X[:, self.__Ny:], 0)

        if X is not None:                            # :101-117
            X = np.array(X).copy()
            self.__X = self.standardize(X, self.__meanZ, self.__stdZ) if normalize else X.copy()
        if Y is not None:
            Y = np.array(Y).copy()
            self.__Y = self.standardize(Y, self.__meanY, self.__stdY) if (normalize and X is not None) else Y.copy()
        self.__N = self.__X.shape[0]

        hyp_init = self.__hyper if warm_start else None
        self.__build_engine()
        # optimize_nummeric=False selects the CasADi/IPOPT twin in the reference
        # (optimize.py:100-294, same objective with AD gradients).  Here both settings use the
        # GPU NLML with its analytic gradient under SLSQP.
        rows = train_gp_b200(self.__engine, self.__X, self.__Y, meanFunc=self.__mean_func,
                             optimizer_opts=opts, multistart=multistart, hyper_init=hyp_init)
        blocks = self.__comm.allgather_object((self.__engine.out_begin, rows))
        hyper = np.zeros((self.__Ny, blocks[0][1].shape[1]))      # Nx+2 (+ mean parameters, all zero)
        for b, r in blocks:
            hyper[b:b + len(r)] = r
        self.__hyper = hyper
        self.__lam_x = 0
        self.__set_hyper_views()
        self.__factorize()

    def validate(self, X_test, Y_test):
        """ Validate GP model with test data  (reference gp_class.py:145-190; one batched
        GPU predict instead of the per-row Python loop) """
        Y_test = np.array(Y_test, dtype=np.float64).copy()
        X_test = np.array(X_test, dtype=np.float64).copy()
        if self.__normalize:
            Y_test = self.standardize(Y_test, self.__meanY, self.__stdY)
            X_test = self.standardize(X_test, self.__meanZ, self.__stdZ)

        mean, var = self.__predict_std(X_test, None, 'ME', want_cov=False, want_jac=False)[:2]
        var = var + self.noise_variance()[None, :]                      # :161
        return self.__report_validation(Y_test, mean, var, '# Validation of GP model ', 'Num test samples')

    def validate_loo(self):
        """ Validate the GP model without a test set: validate's SMSE and MNLP, in the GP's standardised space, with
        every training point predicted from the other N-1 (leave-one-out cross-validation, Rasmussen & Williams
        section 5.4.2) in place of test predictions.  MNLP is the LOO NLPP over N.  Returns (SMSE, MNLP) per output. """
        mean, var = self.__loo_std()
        return self.__report_validation(self.__Y, mean, var, '# Leave-one-out validation of GP model ',
                                        'Num left-out samples')

    def __report_validation(self, Y_test, mean, var, title, count_label):
        """The error measures of the reference's validate (gp_class.py:145-190) and its banner; var includes sn2."""
        N, Ny = Y_test.shape
        loss = np.sum((Y_test - mean) ** 2, 0) / N
        NLP = np.sum(0.5 * np.log(2 * np.pi * var) + ((Y_test - mean) ** 2) / (2 * var), 0)
        SMSE = loss / np.std(Y_test, 0)                                 # :166 (q15)
        MNLP = NLP / N

        print('\n________________________________________')
        print(title)
        print('----------------------------------------')
        print('* Num training samples: ' + str(self.__N))
        print('* %s: %d' % (count_label, N))
        print('----------------------------------------')
        print('* Mean squared error: ')
        for i in range(Ny):
            print('\t- State %d: %f' % (i + 1, loss[i]))
        print('----------------------------------------')
        print('* Standardized mean squared error:')
        for i in range(Ny):
            print('\t* State %d: %f' % (i + 1, SMSE[i]))
        print('----------------------------------------')
        print('* Mean Negative log Probability:')
        for i in range(Ny):
            print('\t* State %d: %f' % (i + 1, MNLP[i]))
        print('----------------------------------------\n')

        self.__SMSE = np.max(SMSE)
        return np.array(SMSE).flatten(), np.array(MNLP).flatten()

    # ------------------------------------------------------------------ prediction
    def set_method(self, gp_method='TA', ut_params=None):
        """ Select wich GP function to use  (reference gp_class.py:193-242)

            'ME': Mean Equivalence (normal GP), 'TA': 1st order Taylor Approximation and
            'EM': exact moment matching run on the GPU.  The deprecated 'old_ME'/'old_TA' are
            valid names in the reference but out of scope here (SURVEY section 2).
            'UT' (not in the reference): the unscented transform, 'ME' evaluated at the 2 Nx + 1 sigma points of the
            input distribution and recombined (include/gpmpc.h, GPMPC_METHOD_UT); its mean moves with the input
            covariance and is exact for mean functions up to cubic.  ut_params = (alpha, beta, kappa) sets its
            parameters and is kept for later 'UT' calls; until given, the engine's defaults (1, 0, 0) apply.
        """
        if gp_method not in _KNOWN_METHODS:
            raise NameError('No GP method called: ' + gp_method)        # gp_class.py:237
        if gp_method not in _GPU_METHODS:
            raise NotImplementedError("gp_method %r is not implemented by the GPU engine "
                                      "(available: 'ME', 'TA', 'EM', 'UT')" % gp_method)
        if gp_method == 'UT':
            self.__check_ut()
            if ut_params is not None:
                alpha, beta, kappa = (float(v) for v in ut_params)
                self.__engine.set_ut_params(alpha, beta, kappa)
                self.__ut_params = (alpha, beta, kappa)
        elif ut_params is not None:
            raise ValueError("ut_params applies to gp_method 'UT' only (got %r)" % gp_method)
        if gp_method == 'EM' and self.__sharded_outputs():
            # exact moment matching couples every pair of outputs (gp_functions.py:394-412): it
            # needs all Ny factors on one GPU, which the by-output sharding does not provide
            raise NotImplementedError("gp_method 'EM' needs all outputs on one GPU; this GP is sharded by "
                                      "output over %d ranks (use 'TA'/'ME', or build the GP with a "
                                      "single-process Comm)" % self.__comm.world)
        self.__gp_method = gp_method

    def __sharded_outputs(self):
        return self.__comm.world > 1 and getattr(self, '_GP__mode', 'outputs') == 'outputs'

    def __check_ut(self):
        """The cases 'UT' does not cover: outputs sharded over ranks, and a prior mean added in predict."""
        if self.__sharded_outputs():
            # the recombination couples every pair of outputs at the same sigma points
            raise NotImplementedError("gp_method 'UT' needs all outputs on one GPU; this GP is sharded by output over "
                                      "%d ranks (use 'TA'/'ME', or build the GP with a single-process Comm)"
                                      % self.__comm.world)
        if self.__prior_mean_in_predict and self.__has_prior_mean():
            raise NotImplementedError("gp_method 'UT' transforms the zero-mean posterior the engine holds; "
                                      "prior_mean_in_predict with a prior mean function is not supported")

    def __predict_std(self, Z, Sigma, method, want_cov=True, want_jac=True):
        """Batched predict in the GP's standardised space.  Z:(H,Nx)."""
        Z = np.ascontiguousarray(Z, dtype=np.float64).reshape(-1, self.__Nx)
        c = self.__comm
        if method == 'UT':
            self.__check_ut()
        add_pm = self.__prior_mean_in_predict and self.__has_prior_mean() and method != 'EM'
        need_jac = want_jac or add_pm
        if c.world > 1 and self.__mode == 'points':
            b, n = point_block(Z.shape[0], c.rank, c.world)
            Sg = Sigma[b:b + n] if (Sigma is not None and np.ndim(Sigma) == 3) else Sigma
            part = self.__engine.predict(Z[b:b + n], Sg, _GPU_METHODS[method], want_cov, need_jac) if n else None
            parts = [p for p in c.allgather_object(part) if p is not None]
            out = tuple(None if parts[0][k] is None else np.concatenate([p[k] for p in parts], 0)
                        for k in range(4))
        else:
            out = self.__engine.predict(Z, Sigma, _GPU_METHODS[method], want_cov, need_jac)
        if add_pm:
            out = self.__add_prior_mean(Z, Sigma, method, out, want_cov, want_jac)
        return out

    def __add_prior_mean(self, Z, Sigma, method, out, want_cov, want_jac):
        """flag-gated fix of SURVEY q2: mean += m(z), J += dm/dz, and for 'TA' the J Sigma J^T term is
        rebuilt with the full Jacobian (O(H Ny Nx^2) host work)."""
        mean, var, cov, jac = out
        M = np.column_stack([mean_function(self.__hyper[a], Z, self.__mean_func) for a in range(self.__Ny)])
        Jm = np.stack([mean_jacobian(self.__hyper[a], Z, self.__mean_func) for a in range(self.__Ny)], 1)
        mean = mean + M
        if jac is not None:
            jfull = jac + Jm
            if cov is not None and method == 'TA' and Sigma is not None:
                S = np.broadcast_to(np.asarray(Sigma, dtype=np.float64), (Z.shape[0], self.__Nx, self.__Nx)) \
                    if np.ndim(Sigma) == 2 else np.asarray(Sigma, dtype=np.float64)
                cov = cov + np.einsum('had,hde,hbe->hab', jfull, S, jfull) - np.einsum('had,hde,hbe->hab', jac, S, jac)
            jac = jfull
        return mean, var, cov, (jac if want_jac else None)

    def predict_batch(self, x, u, cov=None, method=None):
        """Horizon batch: x:(H,Ny) u:(H,Nu) cov:(Nx,Nx)|(H,Nx,Nx)|None ->
        mean:(H,Ny) (de-standardised), cov:(H,Ny,Ny) (standardised units, q4).
        This is the entry a batched MPC shooting loop (mpc_class.py:361-423) calls: one GPU
        pass for all nodes instead of Nt symbolic graph copies."""
        method = method or self.__gp_method
        x = np.asarray(x, dtype=np.float64).reshape(-1, self.__Ny)
        u = np.asarray(u, dtype=np.float64).reshape(x.shape[0], self.__Nu)
        if self.__normalize:
            x = self.standardize(x, self.__meanX, self.__stdX)
            u = self.standardize(u, self.__meanU, self.__stdU)
        Z = np.hstack([x, u])
        if cov is None and method in _SIGMA_METHODS:
            cov = np.zeros((self.__Nx, self.__Nx))      # no input uncertainty: TA reduces to diag(var)
        mean, var, c, _ = self.__predict_std(Z, cov if method in _SIGMA_METHODS else None, method, True, False)
        if self.__normalize:
            mean = self.inverse_mean(mean, self.__meanY, self.__stdY)
        return mean, c

    def predict_batch_grad(self, x, u, cov=None, method=None):
        """predict_batch plus the first derivatives CasADi's AD extracts from the symbolic GP when nlpsol
        differentiates the MPC's NLP (mpc_class.py:390-412, :496-513): a dict with
            mean (H,Ny)           de-standardised, as predict_batch
            cov  (H,Ny,Ny)        standardised units (q4)
            dmean_dz (H,Ny,Nx)    d mean / d [x,u] in the CALLER's units (chain rule through the scalers)
            dcov_dz  (H,Ny,Ny,Nx) d cov / d [x,u]  (cov itself is not rescaled, so only 1/stdZ enters)
            dcov_dSigma_factor (H,Ny,Nx)  J with d cov[a][b] / d Sigma[d][e] = J[a][d] J[b][e] ('TA')
        With method 'EM' (gpmpc_predict_em_grad) the covariance of the input enters the mean as well, and the dict
        holds mean, cov, dmean_dz, dcov_dz and, for Sigma in the GP's (standardised) input space,
            dmean_dSigma (H,Ny,Nx,Nx)     d mean / d Sigma[d][e], de-standardised (carries stdY)
            dcov_dSigma  (H,Ny,Ny,Nx,Nx)  d cov / d Sigma[d][e] (cov and Sigma both standardised: unscaled)
        each entry of Sigma varied with the others fixed (exactly symmetric in d, e).
        This is what a casadi.Callback's Jacobian function returns; the same
        numbers are available to `casadi.external` through gp_b200 / jac_gp_b200 (include/gpmpc_casadi.h)."""
        method = method or self.__gp_method
        if method not in ('ME', 'TA', 'EM'):
            raise NotImplementedError("derivatives are available for gp_method 'ME', 'TA' and 'EM'")
        if self.__comm.world > 1 and self.__mode == 'outputs':
            raise NotImplementedError('predict_batch_grad needs all outputs on one GPU (build the GP with a single-process Comm)')
        x = np.asarray(x, dtype=np.float64).reshape(-1, self.__Ny)
        u = np.asarray(u, dtype=np.float64).reshape(x.shape[0], self.__Nu)
        if self.__normalize:
            x = self.standardize(x, self.__meanX, self.__stdX)
            u = self.standardize(u, self.__meanU, self.__stdU)
        Z = np.hstack([x, u])
        if method == 'EM':
            return self.__em_grad_units(self.__engine.predict_em_grad(Z, np.zeros((self.__Nx, self.__Nx)) if cov is None else cov))
        if cov is None and method == 'TA':
            cov = np.zeros((self.__Nx, self.__Nx))
        g = self.__engine.predict_grad(Z, cov if method == 'TA' else None, _GPU_METHODS[method])
        mean, jac, dcov = g['mean'], g['jac'], g['dcov_dz']
        out = dict(cov=g['cov'], dcov_dSigma_factor=jac.copy())
        if self.__normalize:
            mean = self.inverse_mean(mean, self.__meanY, self.__stdY)
            jac = jac * self.__stdY[None, :, None] / self.__stdZ[None, None, :]
            dcov = dcov / self.__stdZ[None, None, None, :]
        out.update(mean=mean, dmean_dz=jac, dcov_dz=dcov)
        return out

    def __em_grad_units(self, g):
        """predict_batch_grad's 'EM' dict from the engine's: mean and the z-derivatives in the caller's units."""
        mean, dmz, dmS, dcz = g['mean'], g['dmean_dz'], g['dmean_dSigma'], g['dcov_dz']
        if self.__normalize:
            mean = self.inverse_mean(mean, self.__meanY, self.__stdY)
            dmz = dmz * self.__stdY[None, :, None] / self.__stdZ[None, None, :]
            dmS = dmS * self.__stdY[None, :, None, None]
            dcz = dcz / self.__stdZ[None, None, None, :]
        return dict(mean=mean, cov=g['cov'], dmean_dz=dmz, dcov_dz=dcz, dmean_dSigma=dmS, dcov_dSigma=g['dcov_dSigma'])

    def predict_batch_em_hess(self, x, u, cov=None):
        """'EM' second derivatives for IPOPT's exact Hessian (gpmpc_predict_em_hess): predict_batch_grad(..., method='EM')'s
        dict (the same bits) plus, for z = [x,u] in the CALLER's units and Sigma in the GP's (standardised) input space,
            d2mean_dz2       (H,Ny,Nx,Nx)          d dmean_dz[a][d] / dz_e             (stdY_a / (stdZ_d stdZ_e))
            d2mean_dSigma_dz (H,Ny,Nx,Nx,Nx)       d dmean_dSigma[a][d][e] / dz_f      (stdY_a / stdZ_f)
            d2mean_dSigma2   (H,Ny,Nx,Nx,Nx,Nx)    d dmean_dSigma[a][d][e] / dSigma[f][g]   (stdY_a)
            d2cov_dz2        (H,Ny,Ny,Nx,Nx)       d dcov_dz[a][b][d] / dz_e           (1 / (stdZ_d stdZ_e))
            d2cov_dSigma_dz  (H,Ny,Ny,Nx,Nx,Nx)    d dcov_dSigma[a][b][d][e] / dz_f    (1 / stdZ_f)
            d2cov_dSigma2    (H,Ny,Ny,Nx,Nx,Nx,Nx) d dcov_dSigma[a][b][d][e] / dSigma[f][g]
        (cov stays standardised, as in predict_batch_grad).  Errors as predict_batch_grad; Nx <= 16."""
        if self.__comm.world > 1 and self.__mode == 'outputs':
            raise NotImplementedError('predict_batch_em_hess needs all outputs on one GPU (build the GP with a single-process Comm)')
        x = np.asarray(x, dtype=np.float64).reshape(-1, self.__Ny)
        u = np.asarray(u, dtype=np.float64).reshape(x.shape[0], self.__Nu)
        if self.__normalize:
            x = self.standardize(x, self.__meanX, self.__stdX)
            u = self.standardize(u, self.__meanU, self.__stdU)
        Z = np.hstack([x, u])
        g = self.__engine.predict_em_hess(Z, np.zeros((self.__Nx, self.__Nx)) if cov is None else cov)
        out = self.__em_grad_units(g)
        h = {k: g[k] for k in ('d2mean_dz2', 'd2mean_dSigma_dz', 'd2mean_dSigma2', 'd2cov_dz2', 'd2cov_dSigma_dz', 'd2cov_dSigma2')}
        if self.__normalize:
            sy, iz = self.__stdY, 1.0 / self.__stdZ
            h['d2mean_dz2'] = h['d2mean_dz2'] * sy[None, :, None, None] * iz[None, None, :, None] * iz[None, None, None, :]
            h['d2mean_dSigma_dz'] = h['d2mean_dSigma_dz'] * sy[None, :, None, None, None] * iz[None, None, None, None, :]
            h['d2mean_dSigma2'] = h['d2mean_dSigma2'] * sy[None, :, None, None, None, None]
            h['d2cov_dz2'] = h['d2cov_dz2'] * iz[None, None, None, :, None] * iz[None, None, None, None, :]
            h['d2cov_dSigma_dz'] = h['d2cov_dSigma_dz'] * iz[None, None, None, None, None, :]
        out.update(h)
        return out

    def predict_batch_hess(self, x, u, cov=None, method=None):
        """predict_batch_grad plus the second derivatives IPOPT's default exact Hessian makes CasADi extract
        from the symbolic GP (mpc_class.py:496-513).  Adds, in the CALLER's units for z = [x,u]:
            d2mean_dz2 (H,Ny,Nx,Nx)       d^2 mean_a / dz_d dz_e = hess * stdY_a / (stdZ_d stdZ_e)
            d2cov_dz2  (H,Ny,Ny,Nx,Nx)    d^2 cov[a][b] / dz_f dz_g  (cov is not rescaled: 1/(stdZ_f stdZ_g))
            dcov_dSigma_hess (H,Ny,Nx,Nx) hess_a[d][f] / stdZ_f, so that for 'TA' (Sigma in the GP's input space)
                d^2 cov[a][b] / dz_f dSigma[d][e] = dcov_dSigma_hess[a,d,f] J[b,e] + J[a,d] dcov_dSigma_hess[b,e,f]
                with J = dcov_dSigma_factor;  d^2 cov / dSigma^2 = 0.
        Methods 'ME' and 'TA', errors as predict_batch_grad.  The same numbers reach `casadi.external` through
        jac_jac_gp_b200 (include/gpmpc_casadi.h)."""
        method = method or self.__gp_method
        if method not in ('ME', 'TA'):
            raise NotImplementedError("derivatives are available for gp_method 'ME' and 'TA'")
        if self.__comm.world > 1 and self.__mode == 'outputs':
            raise NotImplementedError('predict_batch_hess needs all outputs on one GPU (build the GP with a single-process Comm)')
        x = np.asarray(x, dtype=np.float64).reshape(-1, self.__Ny)
        u = np.asarray(u, dtype=np.float64).reshape(x.shape[0], self.__Nu)
        if self.__normalize:
            x = self.standardize(x, self.__meanX, self.__stdX)
            u = self.standardize(u, self.__meanU, self.__stdU)
        Z = np.hstack([x, u])
        if cov is None and method == 'TA':
            cov = np.zeros((self.__Nx, self.__Nx))
        g = self.__engine.predict_hess(Z, cov if method == 'TA' else None, _GPU_METHODS[method])
        mean, jac, dcov, hess, d2cov = g['mean'], g['jac'], g['dcov_dz'], g['hess'], g['d2cov_dz2']
        out = dict(cov=g['cov'], dcov_dSigma_factor=jac.copy())
        dS_hess = hess.copy()
        if self.__normalize:
            sz = self.__stdZ
            mean = self.inverse_mean(mean, self.__meanY, self.__stdY)
            jac = jac * self.__stdY[None, :, None] / sz[None, None, :]
            dcov = dcov / sz[None, None, None, :]
            hess = hess * self.__stdY[None, :, None, None] / (sz[:, None] * sz[None, :])[None, None]
            d2cov = d2cov / (sz[:, None] * sz[None, :])[None, None, None]
            dS_hess = dS_hess / sz[None, None, None, :]
        out.update(mean=mean, dmean_dz=jac, dcov_dz=dcov, d2mean_dz2=hess, d2cov_dz2=d2cov, dcov_dSigma_hess=dS_hess)
        return out

    def predict(self, x, u, cov):
        """ Predict future state  (reference gp_class.py:245-263)

        # Arguments:
            x: State vector (Nx x 1)
            u: Input vector (Nu x 1)
            cov: Covariance matrix of input z=[x, u] (Nx+nu x Nx+Nu)
        # Returns mean (Ny,1) [de-standardised] and cov (Ny,Ny) [NOT rescaled, q4]
        """
        if _is_symbolic(x) or _is_symbolic(u) or _is_symbolic(cov):
            raise NotImplementedError(
                'symbolic (CasADi MX/SX) predict: bind the engine with casadi.external("gp_b200", libgpmpc.so) or wrap '
                'GP.predict_batch / predict_batch_grad in a casadi.Callback as described in INTEGRATION.md section 3 '
                '(SURVEY 8f row 1); CasADi is not installed in this build, so that last Python step is not exercised here')
        x = np.asarray(x, dtype=np.float64).reshape(-1)
        u = np.asarray(u, dtype=np.float64).reshape(-1)
        mean, c = self.predict_batch(x.reshape(1, -1), u.reshape(1, -1),
                                     None if cov is None else np.asarray(cov, dtype=np.float64))
        return mean.reshape(self.__Ny, 1), c[0]

    def rollout(self, x0, u, methods=None, device_rollout=True, feedback=False, x_ref=None, Q=None, R=None):
        """ The numeric multi-step prediction of ``predict_compare`` (reference gp_class.py:746-804)
        without the plotting / plant simulation: for every method, propagate (mean, covariance)
        through ``predict`` over the input sequence u:(Nt,Nu), starting from x0 with covariance
        diag(sn2) (+1e-6 on the inputs).  Returns mean, var of shape (len(methods), Nt+1, Ny); var
        is rescaled by stdY^2 when normalize (:795-796).

        feedback=True is the reference's closed-loop branch (:770-804): the GP is linearised at
        (x0, u[0]) (``discrete_linearize``), ``lqr(A, B, Q, R)`` gives K, and every step applies
        u_t = K (mean_t - x_ref) with the input covariance blocks Sigma_uu = K cov K^T and
        Sigma_xu = cov K^T; u then only sets Nt and the linearisation point.  Defaults as in the
        reference: Q = I_Ny, R = I_Nu, x_ref = 0.  Like the reference, K (caller units) acts on the
        GP's standardised covariance (q4).

        A batch x0:(B,Ny) with u:(B,Nt,Nu) gives mean, var of shape (len(methods), B, Nt+1, Ny);
        trajectory b is what x0[b], u[b] give alone (its own covariance chain and, with feedback,
        its own gain).  On a single handle every method runs on the device (gpmpc_rollout_batch for
        'ME' / 'TA' / 'UT', gpmpc_rollout_batch_em for 'EM': one predict pass over all trajectories per
        step, one pass per distinct gain with feedback); sharded models, prior_mean_in_predict and
        device_rollout=False keep the host loop."""
        Ny = self.__Ny
        X0, U, single, Nt = self.__trajectories(x0, u)
        nb = X0.shape[0]
        if feedback:
            Q, R, x_ref = self.__feedback_defaults('rollout', Q, R, x_ref)
        if methods is None:                             # gp_class.py:747 default; 'EM' only where it can run
            methods = ['TA', 'ME'] if self.__sharded_outputs() else ['EM', 'TA', 'ME']
        methods = list(methods)
        mean = np.zeros((len(methods), nb, Nt + 1, Ny))
        var = np.zeros((len(methods), nb, Nt + 1, Ny))
        # one input covariance per trajectory, shared across methods as in the reference: with feedback, method i+1
        # starts from the Sigma_uu / Sigma_xu blocks that method i left behind (gp_class.py:764, :797-801)
        covar = self.__initial_covar(nb)
        covar_x0 = covar[:, :Ny, :Ny].copy()
        keep = self.__gp_method
        # a single handle: all Nt steps run on the device, same arithmetic as the loop below
        on_device = (device_rollout and self.__comm.world == 1
                     and not (self.__prior_mean_in_predict and self.__has_prior_mean()))
        for i, meth in enumerate(methods):
            self.set_method(meth)
            covar[:, :Ny, :Ny] = covar_x0
            mean[i, :, 0, :] = X0
            K = self.__lqr_gains(X0, U[:, 0], Q, R) if feedback else None      # once per method, as the reference
            if on_device and Nt > 0 and self.__rollout_device(i, meth, X0, U, covar, K, x_ref, single, mean, var):
                continue
            for b in range(nb):
                mean_t = X0[b]
                cv = covar[b]
                for t in range(1, Nt + 1):
                    u_t = _matmul_seq(K[b], (mean_t - x_ref)[:, None])[:, 0] if feedback else U[b, t - 1, :]
                    mean_t, covar_x = self.predict(mean_t, u_t, cv)
                    mean_t = np.array(mean_t).reshape(Ny)
                    mean[i, b, t, :] = mean_t
                    var[i, b, t, :] = np.diag(covar_x)
                    if self.__normalize:
                        var[i, b, t, :] = self.inverse_variance(var[i, b, t, :])
                    if feedback:
                        self.__feedback_blocks(cv, K[b], covar_x)
                    cv[:Ny, :Ny] = covar_x
        self.set_method(keep)
        if single:
            return mean[:, 0], var[:, 0]
        return mean, var

    def __lqr_gains(self, X0, U0, Q, R):
        """The reference's K = lqr(discrete_linearize(x0, u[0]))[0] for every trajectory: (B, Nu, Ny)."""
        Ks = []
        for b in range(X0.shape[0]):
            A, Bm = self.discrete_linearize(X0[b], U0[b], None)
            Ks.append(lqr(A, Bm, Q, R)[0])
        return np.stack(Ks)

    def __trajectories(self, x0, u):
        """The roll-outs' shapes: x0:(Ny,) with u:(Nt,Nu), or a batch x0:(B,Ny) with u:(B,Nt,Nu) -> X0 (B,Ny), U (B,Nt,Nu),
        single, Nt.  With Nu = 0, u only sets Nt."""
        Ny, Nu = self.__Ny, self.__Nu
        x0 = np.asarray(x0, dtype=np.float64)
        single = x0.ndim < 2
        X0 = x0.reshape(1, Ny) if single else x0.reshape(-1, Ny)
        nb = X0.shape[0]
        u = np.asarray(u, dtype=np.float64)
        if single:
            U = (u.reshape(-1, Nu) if Nu > 0 else np.zeros((u.shape[0] if u.ndim else 0, 0)))[None]   # Nu = 0: Nt = len(u)
        else:
            U = u.reshape(nb, -1, Nu) if Nu > 0 else np.zeros((nb, u.shape[1] if u.ndim > 1 else 0, 0))
        return X0, U, single, U.shape[1]

    def __feedback_defaults(self, fn, Q, R, x_ref):
        """Q, R, x_ref of a feedback roll-out with the reference's defaults Q = I, R = I, x_ref = 0 (gp_class.py:760-766);
        fn names the caller in the error for a model without inputs."""
        Ny, Nu = self.__Ny, self.__Nu
        if Nu == 0:
            raise ValueError('%s(feedback=True) needs a model with inputs (Nu > 0)' % fn)
        return (np.eye(Ny) if Q is None else np.asarray(Q, dtype=np.float64),
                np.eye(Nu) if R is None else np.asarray(R, dtype=np.float64),
                np.zeros(Ny) if x_ref is None else np.asarray(x_ref, dtype=np.float64).reshape(Ny))

    def __initial_covar(self, nb):
        """The roll-outs' initial input covariance for each of nb trajectories: diag(sn2) on x, 1e-6 on u."""
        Nx, Ny = self.__Nx, self.__Ny
        covar = np.tile(np.eye(Nx) * 1e-6, (nb, 1, 1))
        covar[:, :Ny, :Ny] = np.diag(self.__hyper[:, Nx + 1] ** 2)
        return covar

    def __engine_start(self, X0, U, K, x_ref):
        """The engine's view of a roll-out: z0 = [x0, u_0] with u_0 = U[:, 0] open loop or K (x0 - x_ref) with feedback, and
        U, both in the GP's input units, with scale = [stdY | meanY | meanX | stdX] and uscale = [meanU | stdU], the scalers
        the engine applies between steps (None without normalize)."""
        u0 = U[:, 0] if K is None else np.stack([_matmul_seq(K[b], (X0[b] - x_ref)[:, None])[:, 0] for b in range(len(X0))])
        if not self.__normalize:
            return np.concatenate([X0, u0], 1), U, None, None
        zx = self.standardize(X0, self.__meanX, self.__stdX)
        z0 = np.concatenate([zx, self.standardize(u0, self.__meanU, self.__stdU)], 1)
        scale = np.stack([self.__stdY, self.__meanY, self.__meanX, self.__stdX])
        return z0, self.standardize(U, self.__meanU, self.__stdU), scale, np.stack([self.__meanU, self.__stdU])

    @staticmethod
    def __gain_groups(K, nb):
        """A roll-out's engine passes as (trajectories, gain): all nb open loop (K None), else one pass per distinct gain."""
        if K is None:
            return [(np.arange(nb), None)]
        groups = {}
        for b in range(nb):
            groups.setdefault(K[b].tobytes(), []).append(b)
        return [(np.array(g), K[g[0]]) for g in groups.values()]

    def __feedback_blocks(self, cv, K, covar_x):
        """gp_class.py:797-801: the input blocks of the next step's covariance under u = K x."""
        Ny = self.__Ny
        cov_xu = _matmul_seq(covar_x, K.T)
        cv[Ny:, Ny:] = _matmul_seq(_matmul_seq(K, covar_x), K.T)
        cv[Ny:, :Ny] = cov_xu.T
        cv[:Ny, Ny:] = cov_xu

    def __rollout_device(self, i, meth, X0, U, covar, K, x_ref, single, mean, var):
        """Method i of every trajectory on the device; False when the engine has no roll-out entry for the case."""
        eng = self.__engine
        em = meth == 'EM'
        use_single = not em and single and K is None and hasattr(eng, 'rollout')   # gpmpc_rollout, the one open-loop trajectory
        if not (use_single or hasattr(eng, 'rollout_batch_em' if em else 'rollout_batch')):
            return False
        z0, Ug, scale, uscale = self.__engine_start(X0, U, K, x_ref)
        method = _GPU_METHODS[meth]
        if em:                                          # gpmpc_rollout_batch_em, a single trajectory as B = 1
            parts = [(g,) + tuple(eng.rollout_batch_em(z0[g], Ug[g], covar[g], scale, Kg, x_ref, uscale))
                     for g, Kg in self.__gain_groups(K, len(X0))]
        elif use_single:
            parts = [(np.arange(1),) + tuple(r[None] for r in eng.rollout(z0[0], Ug[0], covar[0], method, scale))]
        else:
            parts = [(g,) + tuple(eng.rollout_batch(z0[g], Ug[g], covar[g], method, scale, Kg, x_ref, uscale))
                     for g, Kg in self.__gain_groups(K, len(X0))]
        for g, m_std, v_std, c_last in parts:
            mean[i, g, 1:, :] = self.inverse_mean(m_std, self.__meanY, self.__stdY) if self.__normalize else m_std
            var[i, g, 1:, :] = self.inverse_variance(v_std) if self.__normalize else v_std
            for k, b in enumerate(g):
                if K is not None:
                    self.__feedback_blocks(covar[b], K[b], c_last[k])
                covar[b, :self.__Ny, :self.__Ny] = c_last[k]
        return True

    def rollout_grad(self, x0, u, method=None, feedback=False, x_ref=None, Q=None, R=None):
        """ ``rollout`` for one method with the exact derivatives of every step's mean and variance w.r.t. what produced
        the trajectory: the start x0 and, open loop, the inputs u, or with feedback=True the gain K.  Forward-mode
        tangents run on the device beside the roll-out (gpmpc_rollout_batch_grad for 'ME' and 'TA',
        gpmpc_rollout_batch_em_grad for 'EM'), so one call replaces the P + 1 roll-outs of a difference quotient and carries
        no truncation error.  'EM' needs an engine with that entry; its tangents carry the input covariance as well, since
        the exact moment-matched mean depends on it.

        Shapes follow ``rollout``: x0:(Ny,) with u:(Nt,Nu), or a batch x0:(B,Ny) with u:(B,Nt,Nu), which adds a leading B
        axis to every array below.  Returns a dict in caller units:
          mean, var (Nt+1, Ny)             ``rollout(x0, u, methods=[method], ...)``'s arrays for this method
          dmean_dx0, dvar_dx0 (Nt+1, Ny, Ny)   row 0 is the identity and zero
          open loop:  dmean_du, dvar_du (Nt+1, Ny, Nt, Nu)      d mean[t] / d u[s, i]
          feedback:   dmean_dK, dvar_dK (Nt+1, Ny, Nu, Ny)      d mean[t] / d K[i, k]
        The initial covariance, the gain per trajectory (the LQR gain of the linearisation at (x0, u[0]); defaults Q = I,
        R = I, x_ref = 0) and the grouping of trajectories by distinct gain are ``rollout``'s.  With feedback the gain is
        held fixed: its own dependence on x0 through ``discrete_linearize`` and the Riccati equation is not
        differentiated, so dmean_dx0 is the derivative of the closed loop under that fixed K, including u_0 = K (x0 - x_ref).
        method defaults to the GP's gp_method. """
        meth = self.__gp_method if method is None else method
        eng = self.__engine
        if not (meth in ('ME', 'TA') or (meth == 'EM' and hasattr(eng, 'rollout_batch_em_grad'))):
            raise NotImplementedError("rollout_grad differentiates gp_method 'ME' and 'TA' (got %r)" % (meth,))
        if self.__comm.world > 1:
            raise NotImplementedError('rollout_grad needs all outputs on one GPU (build the GP with a single-process Comm)')
        if self.__prior_mean_in_predict and self.__has_prior_mean():
            raise NotImplementedError('rollout_grad differentiates the zero-mean posterior the engine holds; '
                                      'prior_mean_in_predict with a prior mean function is not supported')
        Ny = self.__Ny
        X0, U, single, Nt = self.__trajectories(x0, u)
        nb = X0.shape[0]
        if Nt < 1:
            raise ValueError('rollout_grad needs at least one step')
        if feedback:
            Q, R, x_ref = self.__feedback_defaults('rollout_grad', Q, R, x_ref)
        K = self.__lqr_gains(X0, U[:, 0], Q, R) if feedback else None
        covar = self.__initial_covar(nb)
        z0, Ug, scale, uscale = self.__engine_start(X0, U, K, x_ref)
        sY = self.__stdY if self.__normalize else np.ones(Ny)
        P = self.__params(Nt, K)
        m_std = np.empty((nb, Nt, Ny)); v_std = np.empty((nb, Nt, Ny))
        Dm = np.empty((nb, Nt, Ny, P)); Dv = np.empty((nb, Nt, Ny, P))
        for g, Kg in self.__gain_groups(K, nb):
            if meth == 'EM':
                r = eng.rollout_batch_em_grad(z0[g], Ug[g], covar[g], scale, Kg, x_ref, uscale)
            else:
                r = eng.rollout_batch_grad(z0[g], Ug[g], covar[g], _GPU_METHODS[meth], scale, Kg, x_ref, uscale)
            m_std[g], v_std[g], _, Dm[g], Dv[g] = r
        # caller units: mean = m stdY + meanY, var = v stdY^2; z0 = [(x0 - meanX) / stdX, (u_0 - meanU) / stdU]
        Dm = Dm * sY[None, None, :, None]
        Dv = Dv * (sY ** 2)[None, None, :, None]
        out = dict(mean=np.zeros((nb, Nt + 1, Ny)), var=np.zeros((nb, Nt + 1, Ny)))
        out['mean'][:, 0] = X0
        out['mean'][:, 1:] = self.inverse_mean(m_std, self.__meanY, self.__stdY) if self.__normalize else m_std
        out['var'][:, 1:] = self.inverse_variance(v_std) if self.__normalize else v_std
        for key, D in (('mean', Dm), ('var', Dv)):
            d_x0, d_p = self.__caller_derivs(D, X0, K, x_ref, key == 'mean')
            out['d%s_%s' % (key, 'du' if K is None else 'dK')] = d_p
            out['d%s_dx0' % key] = d_x0
        if single:
            return {k: v[0] for k, v in out.items()}
        return out

    def __params(self, Nt, K):
        """P, the engine's derivative columns of a roll-out: [z0 | U rows 1 .. Nt-1] open loop, [z0 | K row-major] with K."""
        Nu = self.__Nu
        return self.__Nx + (Nu * self.__Ny if K is not None else (Nt - 1) * Nu)

    def __caller_derivs(self, D, X0, K, x_ref, identity):
        """The engine's derivative columns D (n, Nt, Ny, P) of a quantity already in caller units, for trajectories that
        start at X0 (n, Ny) with gains K (n, Nu, Ny) or None, w.r.t. the caller's parameters: d_x0 (n, Nt+1, Ny, Ny), row 0
        the identity if ``identity`` else zero, and d_u (n, Nt+1, Ny, Nt, Nu) open loop or d_K (n, Nt+1, Ny, Nu, Ny).  The
        engine's columns are z0 = [(x0 - meanX) / stdX, (u_0 - meanU) / stdU], then U rows 1.. or K row-major."""
        Nx, Ny, Nu = self.__Nx, self.__Ny, self.__Nu
        sX, sU = (self.__stdX, self.__stdU) if self.__normalize else (np.ones(Ny), np.ones(Nu))
        nb, Nt = D.shape[0], D.shape[1]
        d_x0 = np.zeros((nb, Nt + 1, Ny, Ny))
        if identity:
            d_x0[:, 0] = np.eye(Ny)
        d_x0[:, 1:] = D[..., :Ny] / sX
        d_u0 = D[..., Ny:Nx] / sU                        # w.r.t. u_0 in caller units (nb, Nt, Ny, Nu)
        if K is None:
            d_u = np.zeros((nb, Nt + 1, Ny, Nt, Nu))
            d_u[:, 1:, :, 0, :] = d_u0
            d_u[:, 1:, :, 1:, :] = (D[..., Nx:] / np.tile(sU, Nt - 1)).reshape(nb, Nt, Ny, Nt - 1, Nu)
            return d_x0, d_u
        # u_0 = K (x0 - x_ref): both x0 and K enter z0's tail
        d_x0[:, 1:] += np.einsum('btai,bik->btak', d_u0, K)
        d_K = np.zeros((nb, Nt + 1, Ny, Nu, Ny))
        d_K[:, 1:] = D[..., Nx:].reshape(nb, Nt, Ny, Nu, Ny)
        d_K[:, 1:] += d_u0[..., :, None] * (X0 - x_ref)[:, None, None, None, :]
        return d_x0, d_K

    def sample_rollout(self, x0, u, n_samples, seed=None, Sigma0=None, feedback=False, x_ref=None, Q=None, R=None,
                       process_noise=False):
        """ Monte Carlo trajectories of the learned dynamics (gpmpc_rollout_sample): each sample is one draw f of the
        GP posterior evaluated along the states that draw visits, x_{t+1} = f(x_t, u_t), with f(z_t) conditioned on the
        values the same draw took at z_0 .. z_{t-1}.  This is the ground truth the propagated moments of ``rollout``
        ('TA', 'ME', 'EM') approximate for the model.

        Shapes follow ``rollout``: x0:(Ny,) with u:(Nt,Nu) returns (n_samples, Nt+1, Ny); x0:(B,Ny) with u:(B,Nt,Nu)
        returns (B, n_samples, Nt+1, Ny).  Caller units; row 0 holds the drawn initial states.

        The first GP input z_0 = [x0, u_0] (standardised when normalize) is drawn from N(z_0, Sigma0).  Sigma0 is
        (Nx,Nx) or (B,Nx,Nx) in the GP's input units; by default it is ``rollout``'s initial covariance, diag(sn2) on x
        and 1e-6 on u, so that step 1 of the samples is distributed exactly as the 'EM' prediction of step 1 says.
        feedback=True applies u_t = K (x_t - x_ref) with ``rollout``'s LQR gain per trajectory (defaults Q = I, R = I,
        x_ref = 0) to every sampled state; u then only sets Nt and the linearisation point.  process_noise=True adds
        sn_a xi to every sampled state (the draw itself stays conditioned on the latent f).

        ``numpy.random.default_rng(seed)`` draws, in this order: the initial perturbations n (B, n_samples, Nx), with
        z_0 = mean + n F^T and F = cholesky(Sigma0) (for a singular Sigma0 the eigenvalue square root); then the function
        draws eps (B, n_samples, Nt, Ny); then, with process_noise, xi (B, n_samples, Nt, Ny).

        With normalize=True every sampled state is re-standardised with the X scalers before the next step, as
        ``rollout`` does with the mean.  ``rollout`` feeds the Y-standardised covariance as the input covariance of the
        next step (q4), so differences between the spread of the samples and its propagated variances at t >= 2 can
        come from that quirk as well as from the approximations. """
        d = self.__sample_setup('sample_rollout', x0, u, n_samples, seed, Sigma0, feedback, x_ref, Q, R, process_noise)
        nb, ns, Nt, Ny = d['nb'], d['ns'], d['Nt'], self.__Ny
        samp = np.empty((nb * ns, Nt, Ny))
        for r, Kg in d['passes']:
            samp[r] = self.__engine.rollout_sample(d['z0'][r], d['U'][r], d['eps'][r], None if d['xi'] is None else d['xi'][r],
                                                   d['scale'], Kg, d['x_ref'], d['uscale'])[0]
        out = self.__sample_states(d, samp)
        return out[0] if d['single'] else out

    def sample_rollout_grad(self, x0, u, n_samples, seed=None, Sigma0=None, feedback=False, x_ref=None, Q=None, R=None,
                            process_noise=False):
        """ ``sample_rollout`` with the pathwise derivatives of every sampled state, the draws held fixed (the
        reparameterisation gradient of a Monte Carlo objective over them, as scenario MPC and PILCO-style policy search
        use), w.r.t. the start x0 and, open loop, the inputs u, or with feedback=True the gain K (gpmpc_rollout_sample_grad:
        forward-mode tangents beside the draws on the device, one call instead of the P + 1 calls of a difference
        quotient, exact on either side of the rule that drops a point from the conditioning set).

        Arguments, draws (same seed: the same samples, bit for bit) and shapes follow ``sample_rollout``; a batch x0:(B,Ny)
        adds a leading B axis to every array below.  Returns a dict in caller units:
          samples (n_samples, Nt+1, Ny)                    ``sample_rollout``'s array
          kept (n_samples, Nt, Ny)                         1 where the step's point entered its draw's conditioning set
          dsamples_dx0 (n_samples, Nt+1, Ny, Ny)           row 0 is the identity
          open loop:  dsamples_du (n_samples, Nt+1, Ny, Nt, Nu)   d samples[t] / d u[s, i]
          feedback:   dsamples_dK (n_samples, Nt+1, Ny, Nu, Ny)   d samples[t] / d K[i, k]
        The drawn start is z_0 = zbar + F n with Sigma0 (and so F) held fixed, so it moves with zbar = [x0, u_0].  As in
        ``rollout_grad`` the gain is held fixed at the LQR gain (not differentiated through the Riccati equation), and
        u_0 = K (x0 - x_ref) is differentiated w.r.t. both x0 and K.  Where a draw drops a point (kept = 0) the derivative is
        that of the branch taken. """
        if not hasattr(self.__engine, 'rollout_sample_grad'):
            raise NotImplementedError('sample_rollout_grad needs an engine with gpmpc_rollout_sample_grad')
        d = self.__sample_setup('sample_rollout_grad', x0, u, n_samples, seed, Sigma0, feedback, x_ref, Q, R, process_noise)
        nb, ns, Nt, Ny = d['nb'], d['ns'], d['Nt'], self.__Ny
        K = d['K']
        P = self.__params(Nt, K)
        samp = np.empty((nb * ns, Nt, Ny)); kept = np.empty((nb * ns, Nt, Ny), dtype=np.int32)
        D = np.empty((nb * ns, Nt, Ny, P))
        for r, Kg in d['passes']:
            samp[r], _, kept[r], D[r] = self.__engine.rollout_sample_grad(
                d['z0'][r], d['U'][r], d['eps'][r], None if d['xi'] is None else d['xi'][r], d['scale'], Kg, d['x_ref'],
                d['uscale'])
        if self.__normalize:
            D = D * self.__stdY[None, None, :, None]
        # the chain through zbar: every draw of trajectory b starts at X0[b] with gain K[b]
        d_x0, d_p = self.__caller_derivs(D, np.repeat(d['X0'], ns, 0), None if K is None else np.repeat(K, ns, 0),
                                         d['x_ref'], True)
        out = dict(samples=self.__sample_states(d, samp), kept=kept.reshape(nb, ns, Nt, Ny),
                   dsamples_dx0=d_x0.reshape((nb, ns) + d_x0.shape[1:]))
        out['dsamples_du' if K is None else 'dsamples_dK'] = d_p.reshape((nb, ns) + d_p.shape[1:])
        if d['single']:
            return {k: v[0] for k, v in out.items()}
        return out

    def __sample_setup(self, fn, x0, u, n_samples, seed, Sigma0, feedback, x_ref, Q, R, process_noise):
        """The checks, gains and draws of a sampled roll-out (``sample_rollout``'s documented order) and the engine's view
        of them, flattened to rows b n_samples + j: a dict with X0, single, nb, ns, Nt, K, x_ref, z0, U, eps, xi, scale,
        uscale and passes, the engine passes as (rows, gain).  fn names the caller in errors."""
        if self.__sharded_outputs():
            raise NotImplementedError('%s needs all outputs on one GPU (build the GP with a single-process Comm)' % fn)
        if self.__prior_mean_in_predict and self.__has_prior_mean():
            raise NotImplementedError('%s draws from the zero-mean posterior the engine holds; '
                                      'prior_mean_in_predict with a prior mean function is not supported' % fn)
        Nx, Ny = self.__Nx, self.__Ny
        X0, U, single, Nt = self.__trajectories(x0, u)
        nb, ns = X0.shape[0], int(n_samples)
        if ns < 1 or Nt < 1:
            raise ValueError('%s needs n_samples >= 1 and at least one step (got %d, %d)' % (fn, ns, Nt))
        if feedback:
            Q, R, x_ref = self.__feedback_defaults(fn, Q, R, x_ref)
        if Sigma0 is None:
            S0 = self.__initial_covar(nb)
        else:
            S0 = np.asarray(Sigma0, dtype=np.float64)
            if S0.shape not in ((Nx, Nx), (nb, Nx, Nx)):
                raise ValueError('Sigma0 must be (%d, %d) or (%d, %d, %d)' % (Nx, Nx, nb, Nx, Nx))
            S0 = np.broadcast_to(S0, (nb, Nx, Nx))
        K = self.__lqr_gains(X0, U[:, 0], Q, R) if feedback else None
        zbar, Ug, scale, uscale = self.__engine_start(X0, U, K, x_ref)
        rng = np.random.default_rng(seed)
        n0 = rng.standard_normal((nb, ns, Nx))
        eps = rng.standard_normal((nb, ns, Nt, Ny))
        xi = rng.standard_normal((nb, ns, Nt, Ny)) if process_noise else None
        z0 = np.stack([zbar[b] + n0[b] @ _sqrt_psd(S0[b]).T for b in range(nb)])        # (nb, ns, Nx)
        rows = lambda g: (np.asarray(g)[:, None] * ns + np.arange(ns)[None, :]).reshape(-1)
        return dict(X0=X0, single=single, nb=nb, ns=ns, Nt=Nt, K=K, x_ref=x_ref, z0=z0.reshape(nb * ns, Nx),
                    U=np.repeat(Ug, ns, 0), eps=eps.reshape(nb * ns, Nt, Ny),
                    xi=None if xi is None else xi.reshape(nb * ns, Nt, Ny), scale=scale, uscale=uscale,
                    passes=[(rows(g), Kg) for g, Kg in self.__gain_groups(K, nb)])

    def __sample_states(self, d, samp):
        """The sampled states (nb, ns, Nt+1, Ny) in caller units: row 0 the drawn starts, then the engine's draws samp."""
        nb, ns, Nt, Ny = d['nb'], d['ns'], d['Nt'], self.__Ny
        out = np.empty((nb * ns, Nt + 1, Ny))
        out[:, 0] = d['z0'][:, :Ny]
        out[:, 1:] = samp
        if self.__normalize:
            out[:, 0] = self.inverse_mean(out[:, 0], self.__meanX, self.__stdX)
            out[:, 1:] = self.inverse_mean(out[:, 1:], self.__meanY, self.__stdY)
        return out.reshape(nb, ns, Nt + 1, Ny)

    def get_size(self):
        """ (N, Ny, Nu)  (reference gp_class.py:266-274) """
        return self.__N, self.__Ny, self.__Nu

    def get_hyper_parameters(self):
        """ reference gp_class.py:277-290 """
        return dict(length_scale=self.__hyper_length_scales, signal_var=self.__hyper_signal_variance,
                    noise_var=self.__hyper_noise_variance, mean=self.__hyper_mean)

    def print_hyper_parameters(self):
        """ Print out all hyperparameters  (reference gp_class.py:293-312) """
        print('\n________________________________________')
        print('# Hyper-parameters')
        print('----------------------------------------')
        print('* Num samples:', self.__N)
        print('* Ny:', self.__Ny)
        print('* Nu:', self.__Nu)
        print('* Normalization:', self.__normalize)
        for state in range(self.__Ny):
            print('----------------------------------------')
            print('* Lengthscale: ', state)
            for i in range(self.__Ny + self.__Nu):
                print(('-- l{a}: {l}').format(a=i, l=self.__hyper_length_scales[state, i]))
            print('* Signal variance: ', state)
            print('-- sf2:', self.__hyper_signal_variance[state])
            print('* Noise variance: ', state)
            print('-- sn2:', self.__hyper_noise_variance[state])
        print('----------------------------------------')

    def covSEard(self, X, Z, ell, sf2):
        """ GP Squared Exponential Kernel k(X,Z)  (reference gp_class.py:314-350).
        Same argument handling and ValueError; evaluated by the engine's K-build kernel
        on a scratch handle (X and Z stacked, off-diagonal block returned). """
        X = np.asarray(X, dtype=np.float64); Z = np.asarray(Z, dtype=np.float64)
        X = X.reshape(1, -1) if X.ndim == 1 else X
        Z = Z.reshape(1, -1) if Z.ndim == 1 else Z
        n1, D = X.shape
        n2, D2 = Z.shape
        if D != D2:
            raise ValueError('Input dimensions are not the same! D_x=' + str(D) + ', D_z=' + str(D2))
        hyp = np.concatenate([np.asarray(ell, dtype=np.float64).reshape(-1), [np.sqrt(sf2), 0.0]])[None, :]
        eng = self.__engine_factory(n1 + n2, D, 1, 0, 1, self.__device)
        try:
            eng.set_data(np.vstack([X, Z]), np.zeros((n1 + n2, 1)))
            eng.set_hyper(hyp)
            K = eng.build_K(0)
        finally:
            eng.close()
        return K[:n1, n1:].copy()

    def covar(self, X_new):
        """ Compute covariance of input data  (reference gp_class.py:353-381)

        # Arguments:
            X_new: Input matrix or vector of size (n x D), in the GP's (standardised) space.
        # Returns:
            covar: (D x (n x n)) -- the reference allocates D = input-dimension slabs and fills
                   the first Ny with  kss - v^T v  (q12); (D x n) for a 1-D input.
        """
        X_new = np.asarray(X_new, dtype=np.float64)
        one_d = X_new.ndim == 1
        Z = X_new.reshape(1, -1) if one_d else X_new
        n, D = Z.shape
        eng = self.__engine
        mine = [(eng.out_begin, eng.posterior_cov(Z))]
        if self.__comm.world > 1 and self.__mode == 'outputs':
            mine = self.__comm.allgather_object(mine[0])
        covar = np.zeros((D, n) if one_d else (D, n, n))
        for b, blk in mine:
            for k in range(blk.shape[0]):
                covar[b + k] = blk[k].reshape(n) if one_d else blk[k]
        return covar

    def loo_predict(self):
        """ Leave-one-out predictions of the training points: point i predicted by the GP on the other N-1, from the
        current factorisation in O(N^2) per output (gpmpc_loo).  Returns mean (N, Ny), in caller units
        (de-standardised like predict_batch), and var (N, Ny), the variance of the noisy target in the GP's output
        units (standardised, q4).  With a prior mean the mean is y_i - alpha_i / c_i, the prior mean included.
        Combine with remove_data to drop points the rest of the data does not explain. """
        mean, var = self.__loo_std()
        if self.__normalize:
            mean = self.inverse_mean(mean, self.__meanY, self.__stdY)
        return mean, var

    def __loo_std(self):
        """LOO mean and variance (N, Ny) in the standardised space, gathered over ranks in 'outputs' mode."""
        eng = self.__engine
        m, v, _ = eng.loo()
        mine = [(eng.out_begin, m, v)]
        if self.__comm.world > 1 and self.__mode == 'outputs':
            mine = self.__comm.allgather_object(mine[0])
        mean, var = np.zeros((self.__N, self.__Ny)), np.zeros((self.__N, self.__Ny))
        for b, mb, vb in mine:
            mean[:, b:b + mb.shape[0]] = mb.T
            var[:, b:b + vb.shape[0]] = vb.T
        if self.__has_prior_mean():                  # the engine factorised the residual y - m(X)
            mean += np.column_stack([mean_function(self.__hyper[a], self.__X, self.__mean_func)
                                     for a in range(self.__Ny)])
        return mean, var

    def update_data_all(self, X_new, Y_new):
        """ Update training data with all new observations  (reference gp_class.py:474-550):
        append, keep the hyper-parameters, rebuild chol / alpha on the GPU. """
        X_new = np.array(X_new, dtype=np.float64).copy()
        Y_new = np.array(Y_new, dtype=np.float64).copy()
        if self.__normalize:
            Y_new = self.standardize(Y_new, self.__meanY, self.__stdY)
            X_new = self.standardize(X_new, self.__meanZ, self.__stdZ)
        print('\n________________________________________')
        print('# Updating training data with ' + str(X_new.shape[0]) + ' new samples')
        print('----------------------------------------')
        self.__set_data(np.vstack([self.__X, X_new]), np.vstack([self.__Y, Y_new]))
        self.__refit()
        self.set_method(self.__gp_method)

    def remove_data(self, indices):
        """ Drop the training points ``indices`` (distinct row indices into the current training set, any order) with
        the O(N^2) rank-1 update of L, L^-1 and alpha: no refit, hyper-parameters kept, the freed rows are append
        capacity again.  Raises ValueError on a bad index (non-integer, repeated, out of range, or no point left)
        before the model is touched.  In 'outputs' mode every rank passes the same indices. """
        idx = np.asarray(indices).reshape(-1)
        if idx.size and not np.issubdtype(idx.dtype, np.integer):
            raise ValueError('indices must be integers, got dtype %s' % idx.dtype)
        idx = idx.astype(np.int64)
        if np.unique(idx).size != idx.size:
            raise ValueError('indices must be unique')
        if idx.size and (idx.min() < 0 or idx.max() >= self.__N):
            raise ValueError('indices must be in [0, %d)' % self.__N)
        if idx.size >= self.__N:
            raise ValueError('removing %d of %d points leaves none' % (idx.size, self.__N))
        if idx.size == 0:
            return
        self.__engine.remove(idx)
        self.__set_data(np.delete(self.__X, idx, axis=0), np.delete(self.__Y, idx, axis=0))

    def append_data(self, X_new, Y_new, max_points=None):
        """ Add observations one at a time with the O(N^2) rank-1 update of L, L^-1 and alpha
        (what the reference's ``update_data``, gp_class.py:384-471, set out to do); hyper-
        parameters are kept.  Falls back to a full refactorisation (``update_data_all``) when the
        padded capacity is exhausted or an update loses positive definiteness.

        max_points: a sliding window.  Before each point the oldest points (row 0, 1, ...) are removed with
        ``remove_data`` so that at most max_points remain after the append: N stays constant once the window is
        full, so a model at its full padded size keeps updating without a refit.  The refit fallback also keeps only
        the newest max_points points.  None (default): the model only grows. """
        X_new = np.array(X_new, dtype=np.float64).reshape(-1, self.__Nx)
        Y_new = np.array(Y_new, dtype=np.float64).reshape(-1, self.__Ny)
        if max_points is not None:
            max_points = int(max_points)
            if max_points < 2:                       # one old point at least stays beside each new one
                raise ValueError('max_points must be >= 2, got %d' % max_points)
        Xs, Ys = X_new, Y_new
        if self.__normalize:
            Ys = self.standardize(Y_new, self.__meanY, self.__stdY)
            Xs = self.standardize(X_new, self.__meanZ, self.__stdZ)
        Ts = self.__engine_targets(Xs, Ys)
        for k in range(Xs.shape[0]):
            if max_points is not None and self.__N + 1 > max_points:
                self.remove_data(np.arange(self.__N + 1 - max_points))
            ok = self.__engine.append(Xs[k], Ts[k])
            if self.__comm.world > 1:
                # the fallback below runs collectives (engine rebuild): the decision must be collective
                # too -- a rank that alone lost positive definiteness would otherwise hang the others
                ok = all(self.__comm.allgather_object(bool(ok)))
            if not ok:
                X, Y = np.vstack([self.__X, Xs[k:]]), np.vstack([self.__Y, Ys[k:]])
                if max_points is not None:           # the window: the newest max_points
                    X, Y = X[-max_points:], Y[-max_points:]
                self.__set_data(X, Y)
                self.__refit()
                return
            self.__set_data(np.vstack([self.__X, Xs[k:k + 1]]), np.vstack([self.__Y, Ys[k:k + 1]]))

    def replace_data_all(self, X_new, Y_new):
        """ Replace training data with new observations  (reference gp_class.py:553-626) """
        X_new = np.array(X_new, dtype=np.float64).copy()
        Y_new = np.array(Y_new, dtype=np.float64).copy()
        if self.__normalize:
            Y_new = self.standardize(Y_new, self.__meanY, self.__stdY)
            X_new = self.standardize(X_new, self.__meanZ, self.__stdZ)
        print('\n________________________________________')
        print('# Replacing training data with ' + str(X_new.shape[0]) + ' new samples')
        print('----------------------------------------')
        self.__set_data(X_new, Y_new)
        self.__refit()
        self.set_method(self.__gp_method)

    def update_data(self, X_new, Y_new, N_new=None):
        """reference gp_class.py:384-471 is self-declared broken ("NOT working as intended",
        :397; SURVEY q14).  Not replicated."""
        raise NotImplementedError('GP.update_data is broken in the reference (gp_class.py:397); use append_greedy '
                                  '(max-variance selection), update_data_all or replace_data_all')

    def append_greedy(self, X_new, Y_new, N_new=None, device_select=True):
        """ Grow the model by the N_new points of the pool (X_new, Y_new) with the highest combined posterior variance
        (sum over outputs, noise free), chosen one at a time after the previous choice has been absorbed: what the
        reference's ``update_data`` (gp_class.py:384-471) set out to do, with its argmin / sqrt(k - |l|) fixed (SURVEY
        q14).  Hyper-parameters are kept.  Returns the picked row indices into X_new, in selection order (ties go to
        the lowest index).

        device_select: the whole selection runs in one device call (gpmpc_append_greedy) when this rank's engine owns
        every output; the engine is rebuilt once with enough reserved capacity first if needed.  Otherwise (outputs
        sharded over ranks, or False) each step predicts the pool's variances and appends the best point with
        ``append_data``; every rank makes the same choice. """
        X_new = np.array(X_new, dtype=np.float64).reshape(-1, self.__Nx)
        Y_new = np.array(Y_new, dtype=np.float64).reshape(-1, self.__Ny)
        n = X_new.shape[0]
        if Y_new.shape[0] != n:
            raise ValueError('X_new and Y_new must have the same number of rows')
        N_new = n if N_new is None else int(N_new)
        if not 0 <= N_new <= n:
            raise ValueError('N_new must be in [0, %d], got %d' % (n, N_new))
        if N_new == 0:
            return np.zeros(0, dtype=np.int64)
        Xs, Ys = X_new, Y_new
        if self.__normalize:                         # gp_class.py:406-408
            Ys = self.standardize(Y_new, self.__meanY, self.__stdY)
            Xs = self.standardize(X_new, self.__meanZ, self.__stdZ)
        eng = self.__engine
        on_device = (device_select and hasattr(eng, 'append_greedy') and not self.__sharded_outputs()
                     and eng.out_count == self.__Ny)
        picked = self.__greedy_device(Xs, Ys, N_new) if on_device else self.__greedy_host(X_new, Y_new, Xs, N_new)
        return np.asarray(picked, dtype=np.int64)

    def __greedy_device(self, Xs, Ys, N_new):
        Yr = self.__engine_targets(Xs, Ys)
        remaining = np.arange(Xs.shape[0])
        picked = []
        while len(picked) < N_new:
            need = N_new - len(picked)
            if self.__engine.capacity - self.__engine.N < need:
                self.__refit(capacity=self.__N + need)
            idx, _, ok = self.__engine.append_greedy(Xs[remaining], Yr[remaining], need)
            if self.__comm.world > 1:
                # replicated engines ('points' mode): the kept picks and the refit decision are collective, so a rank
                # that alone lost positive definiteness cannot leave the others in __factorize's barrier
                res = self.__comm.allgather_object((idx.tolist(), bool(ok)))
                k = min(len(r[0]) for r in res)
                if any(r[0][:k] != res[0][0][:k] for r in res):
                    raise RuntimeError('append_greedy: ranks selected different points')
                if not all(r[1] and len(r[0]) == k for r in res):
                    idx, ok = idx[:k], False          # every rank keeps the common picks and refits on them
            sel = remaining[idx]
            self.__set_data(np.vstack([self.__X, Xs[sel]]), np.vstack([self.__Y, Ys[sel]]))
            picked.extend(sel.tolist())
            remaining = np.delete(remaining, idx)
            if not ok:
                # positive definiteness lost at the last pick (it is in X): refactorise, the jitter policy applies there
                need = N_new - len(picked)
                self.__refit(capacity=self.__N + need if need else None)
        return picked

    def __greedy_host(self, X_new, Y_new, Xs, N_new):
        remaining = np.arange(Xs.shape[0])
        picked = []
        for _ in range(N_new):
            # gathered over ranks: every rank holds every output's variance and makes the same choice
            var = self.__predict_std(Xs[remaining], None, 'ME', want_cov=False, want_jac=False)[1]
            score = var[:, 0].copy()
            for a in range(1, self.__Ny):            # outputs in order, as the device pick sums them
                score += var[:, a]
            j = int(np.argmax(score))                # first maximum: ties to the lowest index
            c = int(remaining[j])
            self.append_data(X_new[c:c + 1], Y_new[c:c + 1])      # its refit decision is collective
            picked.append(c)
            remaining = np.delete(remaining, j)
        return picked

    def standardize(self, Y, mean, std):
        return (Y - mean) / std                      # gp_class.py:629-630

    def normalize(self, u, lb, ub):
        return (u - lb) / (ub - lb)                  # gp_class.py:632-633

    def inverse_mean(self, x, mean, std):
        """ Inverse standardization of the mean  (gp_class.py:635-638) """
        return (x * std) + mean

    def inverse_variance(self, variance):
        """ Inverse standardization of the variance  (gp_class.py:640-644) """
        return variance * self.__stdY ** 2

    def discrete_linearize(self, x0, u0, cov0):
        """ Linearize the GP around the operating point  x[k+1] = Ax[k] + Bu[k]
        (reference gp_class.py:647-661): Jacobian of the predicted mean in standardised
        space, inputs standardised when normalize, outputs not rescaled.  The reference
        differentiates the ACTIVE method's mean; for 'ME'/'TA' that is the posterior-mean Jacobian
        returned here, for 'EM' (mean depends on the input covariance) the reference's A, B differ --
        this engine always linearises the 'ME' mean. """
        x0 = np.asarray(x0, dtype=np.float64).reshape(-1)
        u0 = np.asarray(u0, dtype=np.float64).reshape(-1)
        if self.__normalize:
            x0 = self.standardize(x0, self.__meanX, self.__stdX)
            u0 = self.standardize(u0, self.__meanU, self.__stdU)
        J = self.__predict_std(np.concatenate([x0, u0])[None, :], None, 'ME', False, True)[3][0]
        return J[:, :self.__Ny].copy(), J[:, self.__Ny:].copy()

    def jacobian(self, x0, u0, cov0):
        """ Jacobian of posterior mean J = dmu/dx  (reference gp_class.py:664-672; no
        standardisation there either) """
        z = np.concatenate([np.asarray(x0, dtype=np.float64).reshape(-1),
                            np.asarray(u0, dtype=np.float64).reshape(-1)])
        J = self.__predict_std(z[None, :], None, 'ME', False, True)[3][0]
        return J[:, :self.__Ny].copy()

    def noise_variance(self):
        """ Get the noise variance  (gp_class.py:675-678) """
        return self.__hyper_noise_variance

    def sparse(self, M):
        """ Sparse Gaussian Process -- an empty stub in the reference too (gp_class.py:682-689) """

    # ------------------------------------------------------------------ factors / model I/O
    def __gather_factor(self, what):
        eng = self.__engine
        mine = [(a, eng.get(what, a)) for a in eng.local_outputs]
        if self.__comm.world > 1 and self.__mode == 'outputs':
            mine = [p for blk in self.__comm.allgather_object(mine) for p in blk]
        return np.stack([m for _, m in sorted(mine, key=lambda t: t[0])], 0)

    def get_chol(self):
        return self.__gather_factor(_lib.GET_CHOL)

    def get_alpha(self):
        return self.__gather_factor(_lib.GET_ALPHA)

    def get_invK(self):
        if self.__invK is None:
            self.__invK = self.__gather_factor(_lib.GET_INVK)
        return self.__invK

    def _GP__to_dict(self):
        """ Store model data in a dictionary  (reference gp_class.py:693-726, same schema) """
        gp_dict = {}
        gp_dict['X'] = self.__X.tolist()
        gp_dict['Y'] = self.__Y.tolist()
        gp_dict['hyper'] = dict(
            hyper=self.__hyper.tolist(),
            invK=self.get_invK().tolist(),
            alpha=self.get_alpha().tolist(),
            chol=self.get_chol().tolist(),
            length_scale=self.__hyper_length_scales.tolist(),
            signal_var=self.__hyper_signal_variance.tolist(),
            noise_var=self.__hyper_noise_variance.tolist(),
            mean=self.__hyper_mean.tolist())
        gp_dict['mean_func'] = self.__mean_func
        gp_dict['normalize'] = self.__normalize
        if self.__normalize:
            gp_dict['xlb'] = np.asarray(self.__xlb).tolist()
            gp_dict['xub'] = np.asarray(self.__xub).tolist()
            gp_dict['ulb'] = np.asarray(self.__ulb).tolist()
            gp_dict['uub'] = np.asarray(self.__uub).tolist()
            gp_dict['meta'] = dict(
                meanY=self.__meanY.tolist(), stdY=self.__stdY.tolist(),
                meanZ=self.__meanZ.tolist(), stdZ=self.__stdZ.tolist(),
                meanX=self.__meanX.tolist(), stdX=self.__stdX.tolist(),
                meanU=self.__meanU.tolist(), stdU=self.__stdU.tolist())
        return gp_dict

    def save_model(self, filename):
        """ Save model to a json file  (reference gp_class.py:729-734) """
        output_dict = self._GP__to_dict()
        with open(filename + ".json", "w") as outfile:
            json.dump(output_dict, outfile)

    def save_model_npz(self, filename):
        """ Binary side-car of save_model for large N (a 16384^2 factor is ~5 GB as JSON text):
        same fields, one compressed .npz; chol / invK are NOT stored (they are recomputed on the
        GPU at load time, as load_model does anyway). """
        d = dict(X=self.__X, Y=self.__Y, hyper=self.__hyper, mean_func=np.array(self.__mean_func),
                 normalize=np.array(bool(self.__normalize)))
        if self.__normalize:
            d.update(xlb=np.asarray(self.__xlb, dtype=np.float64), xub=np.asarray(self.__xub, dtype=np.float64),
                     ulb=np.asarray(self.__ulb, dtype=np.float64), uub=np.asarray(self.__uub, dtype=np.float64),
                     meanY=self.__meanY, stdY=self.__stdY, meanZ=self.__meanZ, stdZ=self.__stdZ,
                     meanX=self.__meanX, stdX=self.__stdX, meanU=self.__meanU, stdU=self.__stdU)
        np.savez_compressed(filename + '.npz', **d)

    @classmethod
    def load_model_npz(cls, filename, **kwargs):
        z = np.load(filename + '.npz')
        kw = dict(X=z['X'], Y=z['Y'], hyper=dict(hyper=z['hyper']), mean_func=str(z['mean_func']),
                  normalize=bool(z['normalize']))
        if kw['normalize']:
            kw.update(xlb=z['xlb'], xub=z['xub'], ulb=z['ulb'], uub=z['uub'],
                      meta={k: z[k] for k in ('meanY', 'stdY', 'meanZ', 'stdZ', 'meanX', 'stdX', 'meanU', 'stdU')})
        kw.update(kwargs)
        return cls(**kw)

    @classmethod
    def load_model(cls, filename, **kwargs):
        """ Create a new model from file  (reference gp_class.py:737-743) """
        with open(filename + ".json") as json_data:
            input_dict = json.load(json_data)
        input_dict.update(kwargs)
        return cls(**input_dict)

    def close(self):
        if self.__engine is not None:
            self.__engine.close()
            self.__engine = None
