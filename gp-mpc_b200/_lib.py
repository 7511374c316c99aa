"""ctypes binding of libgpmpc.so (the C ABI in include/gpmpc.h).

There is deliberately NO fallback: if the CUDA library has not been built
(``python -c "import __graft_entry__ as g; g.build()"``) importing the engine
fails loudly, and ``gpmpc_create`` fails when no sm_90 (H100) device is present.
"""
from __future__ import annotations

import ctypes as C
import threading
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('GPMPC_LIB', os.path.join(_HERE, 'lib', 'libgpmpc.so'))

OK, ERR_ARG, ERR_CUDA, ERR_STATE, ERR_NCCL, ERR_NOTPD = 0, -1, -2, -3, -4, -5
METHOD_ME, METHOD_TA, METHOD_EM, METHOD_UT = 0, 1, 2, 3
GET_CHOL, GET_ALPHA, GET_INVK, GET_K, GET_LOGDET, GET_LINV, GET_ALPHA_NLML = range(7)
PROF_KBUILD_FULL, PROF_KBUILD_LOWER, PROF_SYRK, PROF_FACTORIZE, PROF_TRIGEMM, PROF_KS, PROF_PREDICT_TAIL, PROF_PANEL = range(8)

# every symbol include/gpmpc.h declares: (name, restype, argtypes)
_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int)
_H = C.c_void_p
SYMBOLS = [
    ('gpmpc_version', C.c_int, []),
    ('gpmpc_create', C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(_H)]),
    ('gpmpc_create_reserve', C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(_H)]),
    ('gpmpc_destroy', C.c_int, [_H]),
    ('gpmpc_last_error', C.c_char_p, [_H]),
    ('gpmpc_set_data', C.c_int, [_H, _dp, _dp]),
    ('gpmpc_set_hyper', C.c_int, [_H, _dp, C.c_int]),
    ('gpmpc_set_y', C.c_int, [_H, C.c_int, _dp]),
    ('gpmpc_build_K', C.c_int, [_H, C.c_int, _dp]),
    ('gpmpc_factorize', C.c_int, [_H, C.c_double, _ip]),
    ('gpmpc_nlml', C.c_int, [_H, C.c_int, _dp, _dp, _dp]),
    ('gpmpc_nlml_batch', C.c_int, [_H, C.c_int, C.c_int, _dp, _dp, _dp, _ip]),
    ('gpmpc_loo', C.c_int, [_H, _dp, _dp, _dp]),
    ('gpmpc_loo_nlpp', C.c_int, [_H, C.c_int, _dp, _dp, _dp]),
    ('gpmpc_predict', C.c_int, [_H, C.c_int, C.c_int, _dp, _dp, C.c_int, _dp, _dp, _dp, _dp]),
    ('gpmpc_predict_grad', C.c_int, [_H, C.c_int, C.c_int, _dp, _dp, C.c_int, _dp, _dp, _dp, _dp, _dp, _dp, _dp]),
    ('gpmpc_predict_hess', C.c_int, [_H, C.c_int, C.c_int, _dp, _dp, C.c_int, _dp, _dp, _dp, _dp, _dp, _dp, _dp,
                                     _dp, _dp, _dp]),
    ('gpmpc_predict_em_grad', C.c_int, [_H, C.c_int, _dp, _dp, C.c_int, _dp, _dp, _dp, _dp, _dp, _dp, _dp]),
    ('gpmpc_predict_em_hess', C.c_int, [_H, C.c_int, _dp, _dp, C.c_int] + [_dp] * 13),
    ('gpmpc_get_size', C.c_int, [_H, _ip, _ip, _ip]),
    ('gpmpc_append', C.c_int, [_H, _dp, _dp]),
    ('gpmpc_append_greedy', C.c_int, [_H, C.c_int, _dp, _dp, C.c_int, _ip, _dp, _ip]),
    ('gpmpc_remove', C.c_int, [_H, C.c_int, _ip]),
    ('gpmpc_posterior_cov', C.c_int, [_H, C.c_int, _dp, _dp]),
    ('gpmpc_rollout', C.c_int, [_H, C.c_int, C.c_int, _dp, _dp, _dp, _dp, _dp, _dp, _dp]),
    ('gpmpc_rollout_batch', C.c_int, [_H, C.c_int, C.c_int, C.c_int] + [_dp] * 10),
    ('gpmpc_rollout_batch_grad', C.c_int, [_H, C.c_int, C.c_int, C.c_int] + [_dp] * 12),
    ('gpmpc_rollout_batch_em', C.c_int, [_H, C.c_int, C.c_int] + [_dp] * 10),
    ('gpmpc_rollout_batch_em_grad', C.c_int, [_H, C.c_int, C.c_int] + [_dp] * 12),
    ('gpmpc_rollout_sample', C.c_int, [_H, C.c_int, C.c_int] + [_dp] * 10 + [_ip]),
    ('gpmpc_rollout_sample_grad', C.c_int, [_H, C.c_int, C.c_int] + [_dp] * 10 + [_ip, _dp]),
    ('gpmpc_predict_device', C.c_int, [_H, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]),
    ('gpmpc_get', C.c_int, [_H, C.c_int, C.c_int, _dp]),
    ('gpmpc_set_option', C.c_int, [_H, C.c_char_p, C.c_double]),
    ('gpmpc_comm_unique_id', C.c_int, [C.c_void_p]),
    ('gpmpc_comm_init', C.c_int, [_H, C.c_void_p, C.c_int, C.c_int]),
    ('gpmpc_peer_export', C.c_int, [_H, C.c_int, C.c_void_p]),
    ('gpmpc_peer_attach', C.c_int, [_H, C.c_void_p]),
    ('gpmpc_stream', C.c_void_p, [_H]),
    ('gpmpc_synchronize', C.c_int, [_H]),
    ('gpmpc_profile', C.c_int, [_H, C.c_int, C.c_int, C.c_int, _dp]),
    ('gpmpc_profile_balance', C.c_int, [_H, C.c_int, _dp]),
    ('gpmpc_profile_leaf', C.c_int, [_H, _dp]),
    ('gpmpc_profile_tail', C.c_int, [_H, C.c_int, _dp]),
]

_ll = C.c_longlong
_llp = C.POINTER(C.c_longlong)
_dpp = C.POINTER(_dp)
# include/gpmpc_casadi.h: the CasADi `external` family (function + its Jacobian)
for _f in ('gp_b200', 'jac_gp_b200'):
    SYMBOLS += [
        (_f + '_n_in', _ll, []), (_f + '_n_out', _ll, []),
        (_f + '_name_in', C.c_char_p, [_ll]), (_f + '_name_out', C.c_char_p, [_ll]),
        (_f + '_sparsity_in', _llp, [_ll]), (_f + '_sparsity_out', _llp, [_ll]),
        (_f + '_work', C.c_int, [_llp, _llp, _llp, _llp]),
        (_f, C.c_int, [_dpp, _dpp, _llp, _dp, C.c_int]),
    ]
SYMBOLS += [('gp_b200_bind', C.c_int, [_H, C.c_int, C.c_int]), ('gp_b200_bind_em_hess', C.c_int, [_H, C.c_int]),
            ('gp_b200_unbind', None, []),
            ('gp_b200_incref', None, []), ('gp_b200_decref', None, [])]
# the Jacobian of jac_gp_b200 (second derivatives, include/gpmpc_casadi.h), bound by load() next to SYMBOLS
SYMBOLS_JAC_JAC = [
    ('jac_jac_gp_b200_n_in', _ll, []), ('jac_jac_gp_b200_n_out', _ll, []),
    ('jac_jac_gp_b200_name_in', C.c_char_p, [_ll]), ('jac_jac_gp_b200_name_out', C.c_char_p, [_ll]),
    ('jac_jac_gp_b200_sparsity_in', _llp, [_ll]), ('jac_jac_gp_b200_sparsity_out', _llp, [_ll]),
    ('jac_jac_gp_b200_work', C.c_int, [_llp, _llp, _llp, _llp]),
    ('jac_jac_gp_b200_incref', None, []), ('jac_jac_gp_b200_decref', None, []),
    ('jac_jac_gp_b200', C.c_int, [_dpp, _dpp, _llp, _dp, C.c_int]),
]

_lib = None


class GpmpcError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__('gpmpc error %d: %s' % (code, msg))
        self.code = code


def load():
    """Load libgpmpc.so once; raises ImportError when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            'libgpmpc.so not found at %s -- build it with `python -c "import __graft_entry__ as g; '
            'g.build()"` (nvcc, sm_90a).  This engine has no CPU fallback.' % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, res, args in SYMBOLS + SYMBOLS_JAC_JAC:
        fn = getattr(lib, name)      # AttributeError if the symbol is missing
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def _ptr(a):
    return None if a is None else a.ctypes.data_as(_dp)


def _f64(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.float64)
    if shape is not None:
        a = a.reshape(shape)
    return a


class Engine:
    """One handle = one GPU.  Thin, typed veneer over the C ABI; all heavy work is CUDA."""

    def __init__(self, N, Nx, Ny, out_begin=0, out_count=None, device=0, capacity=None):
        """capacity: training points to reserve room for (gpmpc_create_reserve), so appends up to it need no refit."""
        self.lib = load()
        N, self.Nx, self.Ny = int(N), int(Nx), int(Ny)
        self._stage, self._stage_lock = {}, threading.Lock()     # predict(): per-shape host staging arrays + their pointers
        self.out_begin = int(out_begin)
        self.out_count = int(Ny - out_begin if out_count is None else out_count)
        self.device = int(device)
        # the padded size the library allocates: appends succeed while N stays within it
        self.capacity = -(-max(N, int(capacity or 0)) // 128) * 128
        self.h = _H()
        if capacity is None:
            rc = self.lib.gpmpc_create(N, self.Nx, self.Ny, self.out_begin, self.out_count, self.device,
                                       C.byref(self.h))
        else:
            rc = self.lib.gpmpc_create_reserve(N, int(capacity), self.Nx, self.Ny, self.out_begin, self.out_count,
                                               self.device, C.byref(self.h))
        if rc != OK:
            msg = self.lib.gpmpc_last_error(None).decode()
            self.h = None
            raise GpmpcError(rc, msg)

    # -- plumbing ---------------------------------------------------------------------
    def _check(self, rc):
        if rc == ERR_NOTPD:          # factorize / nlml / loo_nlpp: K not positive definite even with jitter
            raise np.linalg.LinAlgError(self.lib.gpmpc_last_error(self.h).decode())
        if rc != OK:
            raise GpmpcError(rc, self.lib.gpmpc_last_error(self.h).decode())

    def close(self):
        if getattr(self, 'h', None):
            self.lib.gpmpc_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def local_outputs(self):
        return range(self.out_begin, self.out_begin + self.out_count)

    @property
    def N(self):                     # the handle's count: appends and removals change it
        n = C.c_int(0)
        self._check(self.lib.gpmpc_get_size(self.h, C.byref(n), None, None))
        return n.value

    # -- model ------------------------------------------------------------------------
    def set_data(self, X, Y):
        X = _f64(X, (self.N, self.Nx)); Y = _f64(Y, (self.N, self.Ny))
        self._check(self.lib.gpmpc_set_data(self.h, _ptr(X), _ptr(Y)))

    def set_hyper(self, hyper):
        hyper = _f64(hyper)
        assert hyper.ndim == 2 and hyper.shape[0] == self.Ny and hyper.shape[1] >= self.Nx + 2
        self._check(self.lib.gpmpc_set_hyper(self.h, _ptr(hyper), hyper.shape[1]))

    def set_y(self, a, y):
        y = _f64(y, (self.N,))
        self._check(self.lib.gpmpc_set_y(self.h, int(a), _ptr(y)))

    def build_K(self, a):
        K = np.empty((self.N, self.N))
        self._check(self.lib.gpmpc_build_K(self.h, int(a), _ptr(K)))
        return K

    def factorize(self, jitter=1e-8):
        info = np.zeros(self.out_count, dtype=np.int32)
        self._check(self.lib.gpmpc_factorize(self.h, float(jitter), info.ctypes.data_as(_ip)))
        return info

    def nlml(self, a, theta, grad=True):
        theta = _f64(theta, (self.Nx + 2,))
        nll = C.c_double(0.0)
        g = np.empty(self.Nx + 2) if grad else None
        self._check(self.lib.gpmpc_nlml(self.h, int(a), _ptr(theta), C.byref(nll), _ptr(g)))
        return (nll.value, g) if grad else nll.value

    def nlml_batch(self, a, thetas, grad=True):
        """gpmpc_nlml_batch: nlml at the S rows of thetas:(S,Nx+2) in one pass -> nll (S,), grad (S,Nx+2) or None,
        status (S,) int32 (0 ok, 1 ok after the jitter retry, ERR_NOTPD: that row's nll and grad are NaN).  Row s has the
        bits of nlml(a, thetas[s]); the factorisation stays valid."""
        thetas = _f64(thetas).reshape(-1, self.Nx + 2)
        S = thetas.shape[0]
        nll = np.empty(S)
        g = np.empty((S, self.Nx + 2)) if grad else None
        status = np.empty(S, dtype=np.int32)
        self._check(self.lib.gpmpc_nlml_batch(self.h, int(a), S, _ptr(thetas), _ptr(nll), _ptr(g),
                                              status.ctypes.data_as(_ip)))
        return nll, g, status

    def loo(self):
        """gpmpc_loo: leave-one-out predictions of the training points on the current factorisation of every owned
        output -> mean (out_count, N), var (out_count, N) (of the noisy targets), nlpp (out_count,)."""
        mean = np.empty((self.out_count, self.N)); var = np.empty((self.out_count, self.N))
        nlpp = np.empty(self.out_count)
        self._check(self.lib.gpmpc_loo(self.h, _ptr(mean), _ptr(var), _ptr(nlpp)))
        return mean, var, nlpp

    def loo_nlpp(self, a, theta, grad=True):
        """gpmpc_loo_nlpp: the negative LOO log predictive probability of output a at theta (and its gradient)."""
        theta = _f64(theta, (self.Nx + 2,))
        val = C.c_double(0.0)
        g = np.empty(self.Nx + 2) if grad else None
        self._check(self.lib.gpmpc_loo_nlpp(self.h, int(a), _ptr(theta), C.byref(val), _ptr(g)))
        return (val.value, g) if grad else val.value

    def get(self, what, a):
        N = self.N
        shape = {GET_CHOL: (N, N), GET_LINV: (N, N), GET_INVK: (N, N), GET_K: (N, N),
                 GET_ALPHA: (N,), GET_ALPHA_NLML: (N,), GET_LOGDET: (1,)}[what]
        out = np.empty(shape)
        self._check(self.lib.gpmpc_get(self.h, int(what), int(a), _ptr(out)))
        return out

    def set_option(self, name, value):
        self._check(self.lib.gpmpc_set_option(self.h, name.encode(), float(value)))

    def set_ut_params(self, alpha=1.0, beta=0.0, kappa=0.0):
        """The unscented transform's (alpha, beta, kappa) for METHOD_UT (options "ut_alpha", "ut_beta", "ut_kappa"; the
        defaults are the engine's).  Raises GpmpcError for alpha <= 0 or kappa <= -Nx."""
        for name, v in (('ut_alpha', alpha), ('ut_beta', beta), ('ut_kappa', kappa)):
            self.set_option(name, v)

    # -- predict ----------------------------------------------------------------------
    def _points(self, Z, Sigma):
        """Z -> (H,Nx); Sigma: None, one (Nx,Nx) for every point or one per point (H,Nx,Nx) -> (Z, Sigma, H, spp)."""
        Z = _f64(Z).reshape(-1, self.Nx)
        H = Z.shape[0]
        spp = 0
        if Sigma is not None:
            Sigma = _f64(Sigma)
            spp = 1 if Sigma.ndim == 3 else 0
            assert Sigma.shape == ((H, self.Nx, self.Nx) if spp else (self.Nx, self.Nx))
        return Z, Sigma, H, spp

    def predict(self, Z, Sigma=None, method=METHOD_TA, want_cov=True, want_jac=True):
        """Z:(H,Nx) -> mean:(H,Ny), var:(H,Ny), cov:(H,Ny,Ny)|None, jac:(H,Ny,Nx)|None (host arrays).  METHOD_UT needs
        Sigma; its jac is the 'ME' Jacobian at Z.
        Building the six ctypes pointer objects was a visible share of a small call, so the call
        goes through per-shape staging arrays whose pointers are built once; the results are returned as fresh copies."""
        Z, Sigma, H, spp = self._points(Z, Sigma)
        key = (H, spp, Sigma is None, bool(want_cov), bool(want_jac))
        with self._stage_lock:
            st = self._stage.get(key)
            if st is None:
                if len(self._stage) >= 16:
                    self._stage.clear()
                arrs = dict(Z=np.empty((H, self.Nx)),
                            S=None if Sigma is None else np.empty(Sigma.shape),
                            mean=np.empty((H, self.Ny)), var=np.empty((H, self.Ny)),
                            cov=np.empty((H, self.Ny, self.Ny)) if want_cov else None,
                            jac=np.empty((H, self.Ny, self.Nx)) if want_jac else None)
                st = self._stage[key] = (arrs, {k: _ptr(v) for k, v in arrs.items()})
            arrs, ptrs = st
            np.copyto(arrs['Z'], Z)
            if Sigma is not None:
                np.copyto(arrs['S'], Sigma)
            self._check(self.lib.gpmpc_predict(self.h, int(method), H, ptrs['Z'], ptrs['S'], spp,
                                               ptrs['mean'], ptrs['var'], ptrs['cov'], ptrs['jac']))
            return (arrs['mean'].copy(), arrs['var'].copy(),
                    arrs['cov'].copy() if want_cov else None, arrs['jac'].copy() if want_jac else None)

    def rollout(self, z0, U, Sigma0, method=METHOD_TA, scale=None):
        """gpmpc_rollout: Nt open-loop steps with the state kept on the device.  z0:(Nx,), U:(Nt,Nu) (GP input units),
        Sigma0:(Nx,Nx), scale:(4,Ny)|None -> means (Nt,Ny), vars (Nt,Ny), cov_last (Ny,Ny) in GP output units."""
        Nu = self.Nx - self.Ny
        z0 = _f64(z0, (self.Nx,)); Sigma0 = _f64(Sigma0, (self.Nx, self.Nx))
        U = _f64(U).reshape(-1, Nu) if Nu > 0 else np.zeros((int(np.shape(U)[0]), 0))
        Nt = U.shape[0]
        if scale is not None:
            scale = _f64(scale, (4, self.Ny))
        means = np.empty((Nt, self.Ny)); var = np.empty((Nt, self.Ny)); cov = np.empty((self.Ny, self.Ny))
        self._check(self.lib.gpmpc_rollout(self.h, int(method), Nt, _ptr(z0), _ptr(U) if Nu > 0 else None, _ptr(Sigma0),
                                           _ptr(scale), _ptr(means), _ptr(var), _ptr(cov)))
        return means, var, cov

    def _policy(self, B, Nt, U, scale, K, x_ref, uscale):
        """The batched roll-outs' policy as their C entries take it: U (B,Nt,Nu), None under K or without inputs; scale
        (4,Ny); K (Nu,Ny) and, with K only, x_ref (Ny,) and uscale (2,Nu)."""
        Nu = self.Nx - self.Ny
        U = _f64(U, (B, Nt, Nu)) if (Nu > 0 and K is None) else None
        if scale is not None:
            scale = _f64(scale, (4, self.Ny))
        if K is None:                                    # x_ref and uscale are read only with K
            return U, scale, None, None, None
        return (U, scale, _f64(K, (Nu, self.Ny)), None if x_ref is None else _f64(x_ref, (self.Ny,)),
                None if uscale is None else _f64(uscale, (2, Nu)))

    def _params(self, Nt, K):
        """P, the parameter columns of a differentiated roll-out: [z0 | U rows 1 .. Nt-1] open loop, [z0 | K] with K."""
        Nu = self.Nx - self.Ny
        return self.Nx + (Nu * self.Ny if K is not None else (Nt - 1) * Nu)

    def _rollout_batch(self, entry, method, tangents, z0, U, Sigma0, scale, K, x_ref, uscale):
        """The body of the batched roll-out wrappers: entry is the C function, method None for the 'EM' entries (which
        take none), tangents whether dmeans and dvars are returned."""
        z0 = _f64(z0).reshape(-1, self.Nx)
        B = z0.shape[0]
        Sigma0 = _f64(Sigma0, (B, self.Nx, self.Nx))
        Nt = int(np.shape(U)[1])
        U, scale, K, x_ref, uscale = self._policy(B, Nt, U, scale, K, x_ref, uscale)
        out = [np.empty((B, Nt, self.Ny)), np.empty((B, Nt, self.Ny)), np.empty((B, self.Ny, self.Ny))]
        if tangents:
            P = self._params(Nt, K)
            out += [np.empty((B, Nt, self.Ny, P)), np.empty((B, Nt, self.Ny, P))]
        head = (self.h,) if method is None else (self.h, int(method))
        self._check(entry(*head, B, Nt, _ptr(z0), _ptr(U), _ptr(Sigma0), _ptr(scale), _ptr(K), _ptr(x_ref), _ptr(uscale),
                          *[_ptr(a) for a in out]))
        return tuple(out)

    def rollout_batch(self, z0, U, Sigma0, method=METHOD_TA, scale=None, K=None, x_ref=None, uscale=None):
        """gpmpc_rollout_batch: B trajectories of Nt steps in one pass, open loop or with the feedback u = K (x - x_ref).
        z0:(B,Nx), U:(B,Nt,Nu) (GP input units; with K only its shape is used), Sigma0:(B,Nx,Nx), scale:(4,Ny)|None,
        K:(Nu,Ny)|None, x_ref:(Ny,)|None, uscale:(2,Nu)|None -> means (B,Nt,Ny), vars (B,Nt,Ny), cov_last (B,Ny,Ny)."""
        return self._rollout_batch(self.lib.gpmpc_rollout_batch, method, False, z0, U, Sigma0, scale, K, x_ref, uscale)

    def rollout_batch_em(self, z0, U, Sigma0, scale=None, K=None, x_ref=None, uscale=None):
        """gpmpc_rollout_batch_em: rollout_batch with exact moment matching ('EM'), same arguments (no method) and outputs;
        each trajectory's results are those of the host loop of predict(EM) calls, bit for bit."""
        return self._rollout_batch(self.lib.gpmpc_rollout_batch_em, None, False, z0, U, Sigma0, scale, K, x_ref, uscale)

    def rollout_batch_grad(self, z0, U, Sigma0, method=METHOD_TA, scale=None, K=None, x_ref=None, uscale=None):
        """gpmpc_rollout_batch_grad: rollout_batch's arguments and outputs (bit for bit) plus dmeans, dvars (B,Nt,Ny,P), the
        derivatives of every step's mean and variance (GP output units) w.r.t. P = Nx + (Nt-1) Nu parameters [z0[b] |
        U[b,1:] row-major] open loop, or P = Nx + Nu Ny parameters [z0[b] | K row-major] with K."""
        return self._rollout_batch(self.lib.gpmpc_rollout_batch_grad, method, True, z0, U, Sigma0, scale, K, x_ref, uscale)

    def rollout_batch_em_grad(self, z0, U, Sigma0, scale=None, K=None, x_ref=None, uscale=None):
        """gpmpc_rollout_batch_em_grad: rollout_batch_em's arguments and outputs (bit for bit) plus dmeans, dvars
        (B,Nt,Ny,P) with rollout_batch_grad's parameter columns, for exact moment matching ('EM')."""
        return self._rollout_batch(self.lib.gpmpc_rollout_batch_em_grad, None, True, z0, U, Sigma0, scale, K, x_ref,
                                   uscale)

    def _rollout_sample(self, entry, tangents, z0, U, eps, xi, scale, K, x_ref, uscale):
        """The body of the sampled roll-out wrappers: entry is the C function, tangents whether dsamples is returned."""
        z0 = _f64(z0).reshape(-1, self.Nx)
        B = z0.shape[0]
        eps = _f64(eps)
        Nt = int(eps.shape[1])
        eps = eps.reshape(B, Nt, self.Ny)
        xi = None if xi is None else _f64(xi, (B, Nt, self.Ny))
        U, scale, K, x_ref, uscale = self._policy(B, Nt, U, scale, K, x_ref, uscale)
        samples = np.empty((B, Nt, self.Ny)); z_out = np.empty((B, Nt, self.Nx))
        kept = np.empty((B, Nt, self.Ny), dtype=np.int32)
        out = [samples, z_out, kept] + ([np.empty((B, Nt, self.Ny, self._params(Nt, K)))] if tangents else [])
        self._check(entry(self.h, B, Nt, _ptr(z0), _ptr(U), _ptr(eps), _ptr(xi), _ptr(scale), _ptr(K), _ptr(x_ref),
                          _ptr(uscale), _ptr(samples), _ptr(z_out), kept.ctypes.data_as(_ip), *[_ptr(a) for a in out[3:]]))
        return tuple(out)

    def rollout_sample(self, z0, U, eps, xi=None, scale=None, K=None, x_ref=None, uscale=None):
        """gpmpc_rollout_sample: B trajectories of Nt steps, each one consistent draw of the GP posterior along the inputs
        it visits.  z0:(B,Nx) (drawn first inputs, GP input units), U:(B,Nt,Nu) (with K only its shape is used),
        eps:(B,Nt,Ny) standard normals of the draws, xi:(B,Nt,Ny)|None process-noise normals, scale / K / x_ref / uscale
        as rollout_batch -> samples (B,Nt,Ny) GP output units, z_out (B,Nt,Nx) inputs used, kept (B,Nt,Ny) int32 (1 where
        the point entered the conditioning set)."""
        return self._rollout_sample(self.lib.gpmpc_rollout_sample, False, z0, U, eps, xi, scale, K, x_ref, uscale)

    def rollout_sample_grad(self, z0, U, eps, xi=None, scale=None, K=None, x_ref=None, uscale=None):
        """gpmpc_rollout_sample_grad: rollout_sample's arguments and outputs (bit for bit) plus dsamples (B,Nt,Ny,P), the
        derivatives of every draw (GP output units) with eps and xi held fixed, w.r.t. rollout_batch_grad's P parameters
        [z0[b] | U[b,1:] row-major] open loop or [z0[b] | K row-major] with K."""
        return self._rollout_sample(self.lib.gpmpc_rollout_sample_grad, True, z0, U, eps, xi, scale, K, x_ref, uscale)

    def predict_grad(self, Z, Sigma=None, method=METHOD_TA, want_hess=False):
        """Predict + first derivatives w.r.t. the test inputs (gpmpc_predict_grad).
        Returns dict(mean (H,Ny), var, cov (H,Ny,Ny), jac = dmean_dz (H,Ny,Nx), dvar_dz (H,Ny,Nx),
        dcov_dz (H,Ny,Ny,Nx)[, hess (H,Ny,Nx,Nx)])."""
        Z, Sigma, H, spp = self._points(Z, Sigma)
        out = dict(mean=np.empty((H, self.Ny)), var=np.empty((H, self.Ny)), cov=np.empty((H, self.Ny, self.Ny)),
                   jac=np.empty((H, self.Ny, self.Nx)), dvar_dz=np.empty((H, self.Ny, self.Nx)),
                   dcov_dz=np.empty((H, self.Ny, self.Ny, self.Nx)))
        if want_hess:
            out['hess'] = np.empty((H, self.Ny, self.Nx, self.Nx))
        self._check(self.lib.gpmpc_predict_grad(self.h, int(method), H, _ptr(Z), _ptr(Sigma), spp, _ptr(out['mean']),
                                                _ptr(out['var']), _ptr(out['cov']), _ptr(out['jac']), _ptr(out['dvar_dz']),
                                                _ptr(out['dcov_dz']), _ptr(out.get('hess'))))
        return out

    def predict_hess(self, Z, Sigma=None, method=METHOD_TA):
        """predict_grad(..., want_hess=True) plus the second derivatives w.r.t. the test inputs (gpmpc_predict_hess):
        d2var_dz2 (H,Ny,Nx,Nx), d3mean_dz3 (H,Ny,Nx,Nx,Nx), d2cov_dz2 (H,Ny,Ny,Nx,Nx)."""
        Z, Sigma, H, spp = self._points(Z, Sigma)
        Ny, Nx = self.Ny, self.Nx
        out = dict(mean=np.empty((H, Ny)), var=np.empty((H, Ny)), cov=np.empty((H, Ny, Ny)), jac=np.empty((H, Ny, Nx)),
                   dvar_dz=np.empty((H, Ny, Nx)), dcov_dz=np.empty((H, Ny, Ny, Nx)), hess=np.empty((H, Ny, Nx, Nx)),
                   d2var_dz2=np.empty((H, Ny, Nx, Nx)), d3mean_dz3=np.empty((H, Ny, Nx, Nx, Nx)),
                   d2cov_dz2=np.empty((H, Ny, Ny, Nx, Nx)))
        self._check(self.lib.gpmpc_predict_hess(
            self.h, int(method), H, _ptr(Z), _ptr(Sigma), spp,
            *[_ptr(out[k]) for k in ('mean', 'var', 'cov', 'jac', 'dvar_dz', 'dcov_dz', 'hess', 'd2var_dz2', 'd3mean_dz3',
                                     'd2cov_dz2')]))
        return out

    def predict_em_grad(self, Z, Sigma):
        """'EM' prediction + first derivatives w.r.t. the test input mean and the input covariance
        (gpmpc_predict_em_grad).  Sigma: (Nx,Nx) shared or (H,Nx,Nx).  Returns dict(mean (H,Ny), var, cov (H,Ny,Ny),
        dmean_dz (H,Ny,Nx), dmean_dSigma (H,Ny,Nx,Nx), dcov_dz (H,Ny,Ny,Nx), dcov_dSigma (H,Ny,Ny,Nx,Nx))."""
        Z, Sigma, H, spp = self._points(Z, Sigma)
        Ny, Nx = self.Ny, self.Nx
        out = dict(mean=np.empty((H, Ny)), var=np.empty((H, Ny)), cov=np.empty((H, Ny, Ny)),
                   dmean_dz=np.empty((H, Ny, Nx)), dmean_dSigma=np.empty((H, Ny, Nx, Nx)),
                   dcov_dz=np.empty((H, Ny, Ny, Nx)), dcov_dSigma=np.empty((H, Ny, Ny, Nx, Nx)))
        self._check(self.lib.gpmpc_predict_em_grad(
            self.h, H, _ptr(Z), _ptr(Sigma), spp,
            *[_ptr(out[k]) for k in ('mean', 'var', 'cov', 'dmean_dz', 'dmean_dSigma', 'dcov_dz', 'dcov_dSigma')]))
        return out

    EM_HESS_KEYS = ('d2mean_dz2', 'd2mean_dSigma_dz', 'd2mean_dSigma2', 'd2cov_dz2', 'd2cov_dSigma_dz', 'd2cov_dSigma2')

    def predict_em_hess(self, Z, Sigma):
        """'EM' prediction + first and second derivatives w.r.t. the test input mean and the input covariance
        (gpmpc_predict_em_hess).  Returns predict_em_grad's dict (same bits) plus d2mean_dz2 (H,Ny,Nx,Nx),
        d2mean_dSigma_dz (H,Ny,Nx,Nx,Nx), d2mean_dSigma2 (H,Ny,Nx,Nx,Nx,Nx), d2cov_dz2 (H,Ny,Ny,Nx,Nx),
        d2cov_dSigma_dz (H,Ny,Ny,Nx,Nx,Nx), d2cov_dSigma2 (H,Ny,Ny,Nx,Nx,Nx,Nx); the differentiated index is the last."""
        Z, Sigma, H, spp = self._points(Z, Sigma)
        Ny, Nx = self.Ny, self.Nx
        out = dict(mean=np.empty((H, Ny)), var=np.empty((H, Ny)), cov=np.empty((H, Ny, Ny)),
                   dmean_dz=np.empty((H, Ny, Nx)), dmean_dSigma=np.empty((H, Ny, Nx, Nx)),
                   dcov_dz=np.empty((H, Ny, Ny, Nx)), dcov_dSigma=np.empty((H, Ny, Ny, Nx, Nx)),
                   d2mean_dz2=np.empty((H, Ny, Nx, Nx)), d2mean_dSigma_dz=np.empty((H, Ny, Nx, Nx, Nx)),
                   d2mean_dSigma2=np.empty((H, Ny, Nx, Nx, Nx, Nx)), d2cov_dz2=np.empty((H, Ny, Ny, Nx, Nx)),
                   d2cov_dSigma_dz=np.empty((H, Ny, Ny, Nx, Nx, Nx)), d2cov_dSigma2=np.empty((H, Ny, Ny, Nx, Nx, Nx, Nx)))
        self._check(self.lib.gpmpc_predict_em_hess(
            self.h, H, _ptr(Z), _ptr(Sigma), spp,
            *[_ptr(out[k]) for k in ('mean', 'var', 'cov', 'dmean_dz', 'dmean_dSigma', 'dcov_dz', 'dcov_dSigma')
              + self.EM_HESS_KEYS]))
        return out

    def append(self, x_new, y_new):
        """Rank-1 append of one training point; returns False when the padded capacity is full
        or positive definiteness is lost (caller refits), True on success.  After a lost positive
        definiteness the point is in the model (N counts it) and the handle needs factorize()."""
        x = _f64(x_new, (self.Nx,)); y = _f64(y_new, (self.Ny,))
        rc = self.lib.gpmpc_append(self.h, _ptr(x), _ptr(y))
        if rc in (ERR_STATE, ERR_NOTPD):
            return False
        self._check(rc)
        return True

    def append_greedy(self, Xc, Yc, n_new):
        """gpmpc_append_greedy: append n_new points of the pool Xc:(n,Nx), Yc:(n,Ny) (GP units), each the one of largest
        combined posterior variance after the previous appends.  Returns (picked (k,) pool indices in order, score (k,)
        combined variance at pick time, ok); ok False means positive definiteness was lost at the last pick, as for
        append (the k points are in, the handle needs a refactorisation)."""
        Xc = _f64(Xc).reshape(-1, self.Nx)
        n = Xc.shape[0]
        Yc = _f64(Yc, (n, self.Ny))
        n_new = int(n_new)
        picked = np.zeros(max(n_new, 1), dtype=np.int32)
        score = np.zeros(max(n_new, 1))
        added = C.c_int(0)
        rc = self.lib.gpmpc_append_greedy(self.h, n, _ptr(Xc), _ptr(Yc), n_new, picked.ctypes.data_as(_ip), _ptr(score),
                                          C.byref(added))
        if rc not in (OK, ERR_NOTPD):
            self._check(rc)
        k = added.value
        return picked[:k].astype(np.int64), score[:k].copy(), rc == OK

    def remove(self, idx):
        """gpmpc_remove: drop the training points idx (distinct indices into the current model, any order) by rank-1
        updates of L and L^-1; raises GpmpcError on a bad index or an unfactorised model (which is then untouched)."""
        idx = np.ascontiguousarray(np.asarray(idx, dtype=np.int64).reshape(-1), dtype=np.int32)
        self._check(self.lib.gpmpc_remove(self.h, idx.size, idx.ctypes.data_as(_ip) if idx.size else None))

    def posterior_cov(self, Z):
        """(out_count, H, H): sf2 - V^T V per owned output (GP.covar)."""
        Z = _f64(Z).reshape(-1, self.Nx)
        out = np.empty((self.out_count, Z.shape[0], Z.shape[0]))
        self._check(self.lib.gpmpc_posterior_cov(self.h, Z.shape[0], _ptr(Z), _ptr(out)))
        return out

    def predict_device(self, method, H, dZ, dSigma, spp, d_mean, d_var, d_cov, d_jac, sync=False):
        """Raw device-pointer variant (ints); enqueues on the handle's stream."""
        self._check(self.lib.gpmpc_predict_device(self.h, int(method), int(H), dZ, dSigma, int(spp),
                                                  d_mean, d_var, d_cov, d_jac, 1 if sync else 0))

    # -- multi-GPU --------------------------------------------------------------------
    @staticmethod
    def comm_unique_id():
        lib = load()
        buf = C.create_string_buffer(128)
        rc = lib.gpmpc_comm_unique_id(buf)
        if rc != OK:
            raise GpmpcError(rc, lib.gpmpc_last_error(None).decode())
        return bytes(buf.raw)

    def comm_init(self, uid, rank, world):
        buf = C.create_string_buffer(bytes(uid), 128)
        self._check(self.lib.gpmpc_comm_init(self.h, buf, int(rank), int(world)))

    def peer_export(self, Hcap=256):
        buf = C.create_string_buffer(64)
        self._check(self.lib.gpmpc_peer_export(self.h, int(Hcap), buf))
        return bytes(buf.raw)

    def peer_attach(self, handles):
        blob = b''.join(bytes(x) for x in handles)
        buf = C.create_string_buffer(blob, len(blob))
        self._check(self.lib.gpmpc_peer_attach(self.h, buf))

    def stream(self):
        return self.lib.gpmpc_stream(self.h)

    def synchronize(self):
        self._check(self.lib.gpmpc_synchronize(self.h))

    def profile_leaf(self):
        out = np.zeros(15)
        self._check(self.lib.gpmpc_profile_leaf(self.h, _ptr(out)))
        return out

    def profile_tail(self, H):
        out = np.zeros(8)
        self._check(self.lib.gpmpc_profile_tail(self.h, int(H), _ptr(out)))
        return dict(zip(('output_done', 'records', 'step_counter', 'staged', 'jsigma', 'written', 'kernel_span', 'tail_cta_span'), out))

    def profile_balance(self, H):
        out = np.zeros(4)
        self._check(self.lib.gpmpc_profile_balance(self.h, int(H), _ptr(out)))
        return dict(zip(('min_us', 'max_us', 'mean_us', 'span_us'), out))

    def profile(self, what, n=0, reps=5):
        ms = C.c_double(0.0)
        self._check(self.lib.gpmpc_profile(self.h, int(what), int(n), int(reps), C.byref(ms)))
        return ms.value
