/* gpmpc.h -- C ABI of the H100-native GP regression engine (libgpmpc.so).
 *
 * This is the drop-in boundary for the dense Gaussian-process hot path of
 * helgeanl/GP-MPC.  The reference has no FFI layer of its own (it is pure Python on
 * numpy/CasADi); the entry points below are what a ctypes binding inside the
 * reference's gp_mpc/gp_class.py would call instead of numpy/CasADi.  Each entry
 * point cites the reference code it replaces (file:line relative to the reference
 * checkout).  See INTEGRATION.md for the binding a maintainer would add.
 *
 * Conventions
 *   - all matrices are fp64, row-major, caller-owned;  "host" pointers are ordinary
 *     CPU memory, "device" pointers are CUDA device memory on the handle's GPU
 *   - hyper rows are [ell_1..ell_Nx, sf, sn] with sf, sn STANDARD DEVIATIONS
 *     (gp_class.py:139-142);  prior mean is zero (the only mean the reference's
 *     prediction graph ever uses, gp_class.py:69-71)
 *   - return value: 0 ok, <0 error (gpmpc_last_error(h) has the text),
 *     GPMPC_ERR_NOTPD when the Cholesky failed even after the jitter retry
 *   - a handle owns one CUDA stream and is not thread-safe; calls are synchronous
 *     unless stated otherwise
 *   - the library has NO CPU fallback: without a CUDA device gpmpc_create fails
 */
#ifndef GPMPC_H
#define GPMPC_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct gpmpc_handle_s* gpmpc_handle_t;

enum {
    GPMPC_OK = 0,
    GPMPC_ERR_ARG = -1,
    GPMPC_ERR_CUDA = -2,
    GPMPC_ERR_STATE = -3,
    GPMPC_ERR_NCCL = -4,
    GPMPC_ERR_NOTPD = -5
};

/* propagation method of GP.set_method / GP.predict (gp_class.py:193-237) */
enum { GPMPC_METHOD_ME = 0, GPMPC_METHOD_TA = 1, GPMPC_METHOD_EM = 2 /* gp_exact_moment, gp_functions.py:344-418; host API only */,
       GPMPC_METHOD_UT = 3 /* unscented transform, below */ };

/* 'UT', the unscented transform of the input distribution N(z, Sigma) through the 'ME' prediction.  With n = Nx and the
 * options "ut_alpha", "ut_beta", "ut_kappa" (alpha, beta, kappa; defaults 1, 0, 0), lambda = alpha^2 (n + kappa) - n and
 * c = sqrt(n + lambda):
 *   sigma points, in this order:  z_0 = z,  z_{2j-1} = z + c S_j,  z_{2j} = z - c S_j  (j = 1..n)
 *   S = the lower Cholesky factor of Sigma (S S^T = Sigma, S_j its column j), semidefinite input accepted: a pivot
 *       <= 1e-14 max(diag Sigma), or <= 0, makes its column exactly zero without error (a zero u-block, a rank-Ny
 *       feedback covariance).  That column's two points fall on z_0; the rule stays of degree 3 (the second moment
 *       along every column of S is matched).
 *   weights:  W0m = lambda / (n + lambda),  W0c = W0m + 1 - alpha^2 + beta,  Wi = 1 / (2 (n + lambda)) for i >= 1
 *   with m_i, v_i the 'ME' mean and variance of every output at z_i:
 *     mean = sum_i Wim m_i,  cov = sum_i Wic (m_i - mean)(m_i - mean)^T + diag(sum_i Wim v_i),  var = diag(cov)
 *     jac  = the 'ME' Jacobian at z_0: the linearisation at the mean, not a UT quantity
 * The defaults give lambda = 0, W0 = 0 and spread sqrt(n): the symmetric cubature rule, all weights non-negative.  The
 * mean is exact for mean functions up to cubic.  W0c < 0 (for example kappa < 0 or a small alpha) can make cov indefinite.
 * Every sum runs in point order: a point's results do not depend on H or its row.  One 'UT' point costs the predict work
 * of 2 Nx + 1 'ME' points, evaluated in one pass over H (2 Nx + 1) points; the handle's capacity grows to that count.
 * Taken by gpmpc_predict, gpmpc_predict_device (Sigma required), gpmpc_rollout and gpmpc_rollout_batch, on a handle
 * that owns every output (GPMPC_ERR_STATE otherwise); every other entry returns GPMPC_ERR_ARG for it. */

/* selector of gpmpc_get */
enum {
    GPMPC_GET_CHOL = 0,    /* (N,N) lower factor, exact zeros above the diagonal (optimize.py:491) */
    GPMPC_GET_ALPHA = 1,   /* (N,)  K^-1 y                                      (optimize.py:494) */
    GPMPC_GET_INVK = 2,    /* (N,N) K^-1, symmetric                             (optimize.py:489-490) */
    GPMPC_GET_K = 3,       /* (N,N) K + sn2 I                                   (optimize.py:480-482) */
    GPMPC_GET_LOGDET = 4,  /* (1,)  2 sum log L_ii                              (optimize.py:352) */
    GPMPC_GET_LINV = 5,    /* (N,N) L^-1 lower                                  (optimize.py:489 invL) */
    GPMPC_GET_ALPHA_NLML = 6 /* (N,) alpha of the last gpmpc_nlml evaluation for that output (mean-parameter gradient) */
};

/* selector of gpmpc_profile */
enum {
    GPMPC_PROF_KBUILD_FULL = 0,   /* covSEard K build, full square                     */
    GPMPC_PROF_KBUILD_LOWER = 1,  /* covSEard K build, lower triangle only            */
    GPMPC_PROF_SYRK = 2,          /* Cholesky trailing update C -= P P^T (DMMA GEMM)  */
    GPMPC_PROF_FACTORIZE = 3,     /* potrf + trtri of one output (K prebuilt each rep) */
    GPMPC_PROF_TRIGEMM = 4,       /* predict v = Linv ks product, all local outputs    */
    GPMPC_PROF_KS = 5,            /* ks / partial mean / partial Jacobian kernel alone (after a predict call) */
    GPMPC_PROF_PREDICT_TAIL = 6,  /* product + finalize + assembly in one launch, no ks kernel in front (after a predict call) */
    GPMPC_PROF_PANEL = 7          /* full repack of every local output's L^-1 panel (the predict product's B operand) */
};

int gpmpc_version(void);

/* Create an engine for N training points, Nx inputs, Ny outputs of which this handle
 * owns the contiguous block [out_begin, out_begin+out_count) (one block per GPU rank;
 * independent per-output GPs, optimize.py:433 / gp_functions.py:128).  device = CUDA
 * ordinal.  Replaces the array allocations of train_gp_numpy, optimize.py:424-427. */
int gpmpc_create(int N, int Nx, int Ny, int out_begin, int out_count, int device, gpmpc_handle_t* out);
/* gpmpc_create with room reserved for appends: the padded size is ceil(max(N, N_cap)/128)*128 instead of
 * ceil(N/128)*128, so gpmpc_append and gpmpc_append_greedy can grow the model up to it without a refit.  The padded
 * tail is an identity block of K; every entry point gives the results of an unreserved handle.  N_cap <= N is
 * gpmpc_create. */
int gpmpc_create_reserve(int N, int N_cap, int Nx, int Ny, int out_begin, int out_count, int device, gpmpc_handle_t* out);
int gpmpc_destroy(gpmpc_handle_t h);
const char* gpmpc_last_error(gpmpc_handle_t h);   /* h may be NULL: last create error */

/* Training data already in the GP's input space (standardised by the caller when
 * normalize=True, gp_class.py:101-117).  X:(N,Nx) Y:(N,Ny) host. */
int gpmpc_set_data(gpmpc_handle_t h, const double* X, const double* Y);

/* hyper:(Ny,ld) host, ld >= Nx+2; only the owned rows are used (gp_class.py:134-142). */
int gpmpc_set_hyper(gpmpc_handle_t h, const double* hyper, int ld);

/* Replace the target vector of global output a with y (N doubles, host): the GP class passes the
 * residual y - m(X) of a prior mean function (alpha = K^-1 (y - m(X)), optimize.py:492-494;
 * get_mean_function, gp_functions.py:25-69).  Invalidates the factorisation. */
int gpmpc_set_y(gpmpc_handle_t h, int a, const double* y);

/* K = covSEard(X,X) + sn2 I for global output a into K_out:(N,N) host (may be NULL:
 * build only).  Replaces calc_cov_matrix + noise + symmetrise, optimize.py:303-319,
 * :480-482 and GP.covSEard gp_class.py:314-350. */
int gpmpc_build_K(gpmpc_handle_t h, int a, double* K_out);

/* Post-fit block for every owned output: K -> L (blocked Cholesky on fp64 tensor
 * cores) -> L^-1 -> alpha, logdet.  On a non-positive pivot adds `jitter` (reference:
 * 1e-8) to that output's diagonal ONCE and retries; a second failure returns
 * GPMPC_ERR_NOTPD.  info:(out_count,) host, may be NULL: 0 ok, 1 = ok after jitter,
 * >1 = 1 + failing pivot index.  Replaces optimize.py:479-494 (= :267-285,
 * gp_class.py:516-537). */
int gpmpc_factorize(gpmpc_handle_t h, double jitter, int* info);

/* Negative log marginal likelihood of global output a at theta:(Nx+2,) host and
 * (grad != NULL) its analytic gradient:  NLL = 1/2 y^T alpha + 1/2 logdet K (no
 * N/2 log 2pi term), with the same jitter retry.  Replaces calc_NLL_numpy,
 * optimize.py:322-356; the gradient replaces SLSQP's finite differences
 * (optimize.py:466-467).  Invalidates the factorisation of output a: the evaluation,
 * gradient included, works in that output's factor slabs and needs no other Npad^2 scratch. */
int gpmpc_nlml(gpmpc_handle_t h, int a, const double* theta, double* nll, double* grad);

/* gpmpc_nlml at S hyper-parameter points of global output a in one pass.
 *   theta  (S, Nx+2)  host, rows as gpmpc_nlml's theta
 *   nll    (S)        host
 *   grad   (S, Nx+2)  host or NULL
 *   status (S)        host: 0 ok, 1 ok after the 1e-8 jitter retry, GPMPC_ERR_NOTPD (nll and grad rows NaN)
 * Entry s is bit-identical to gpmpc_nlml(h, a, theta_s, ...) on the same handle, whatever S, the order of the rows and
 * the pass size.  Entries are independent: a NOTPD entry does not change the others, and the call returns GPMPC_OK.
 * Unlike gpmpc_nlml it leaves the factorisation valid: its slabs are its own scratch.  A pass covers
 * min(S, option "nlml_batch_max") entries (0: all S) and holds, per entry, two Npad^2 slabs, the recursion's two
 * workspaces (about Npad^2 / 3 each) and O(Npad) vectors, kept with the handle; a pass that cannot be allocated is
 * halved, down to one entry.
 *   GPMPC_ERR_ARG: S < 1, a NULL theta, nll or status, a zero length scale in any row, an output the handle does not
 *   own.  GPMPC_ERR_STATE: no data.  Every check runs before any work. */
int gpmpc_nlml_batch(gpmpc_handle_t h, int a, int S, const double* theta, double* nll, double* grad, int* status);

/* Leave-one-out cross-validation on the current factorisation of every OWNED output (Rasmussen & Williams
 * eqs. 5.10-5.12): each training point predicted from the other N-1.  With C = K^-1, alpha = C y (y the target the
 * handle factorised, the residual y - m(X) under a prior mean) and c_i = C_ii, the column norms of L^-1:
 *   mean[a][i] = y_i - alpha_i / c_i,  var[a][i] = 1 / c_i (the variance of the noisy y_i),
 *   nlpp[a] = sum_i [ 1/2 log 2pi - 1/2 log c_i + alpha_i^2 / (2 c_i) ]  (the negative LOO log predictive probability).
 * mean, var:(out_count,N), nlpp:(out_count) host buffers, each may be NULL.  O(N^2) per output, no solve; works after
 * gpmpc_append, gpmpc_append_greedy and gpmpc_remove and on any handle, sharded or reserved.  Every sum runs in a
 * fixed order: repeated calls give identical bits.
 *   GPMPC_ERR_STATE: not factorised.  GPMPC_ERR_ARG: N < 2.  Every check runs before any work. */
int gpmpc_loo(gpmpc_handle_t h, double* mean, double* var, double* nlpp);

/* The LOO counterpart of gpmpc_nlml, as a hyper-parameter fit objective: factorises global output a at theta:(Nx+2,)
 * with the same single 1e-8 jitter retry, returns the NLPP of gpmpc_loo and (grad != NULL) its analytic gradient
 * (R&W eq. 5.13 as a trace: dNLPP/dtheta_j = tr(W dK/dtheta_j), W = C diag(w) C - sym(b alpha^T),
 * w_i = (1 + alpha_i^2/c_i) / (2 c_i), b = C (alpha / c)).  The NLPP has the same bits with and without grad.
 * Same argument checks as gpmpc_nlml, and GPMPC_ERR_ARG for N < 2.  Scratch: the two Npad^2 slabs of
 * gpmpc_get(GPMPC_GET_INVK).
 * Invalidates the factorisation of output a. */
int gpmpc_loo_nlpp(gpmpc_handle_t h, int a, const double* theta, double* nlpp, double* grad);

/* Batched prediction at H test points (host buffers; copies are part of the call).
 * Z:(H,Nx) in the GP's input space; Sigma:(Nx,Nx) or (H,Nx,Nx) when sigma_per_point
 * (ignored for ME, may be NULL; required for UT); outputs (any may be NULL): mean:(H,Ny) var:(H,Ny)
 * cov:(H,Ny,Ny) jac:(H,Ny,Nx).  With a communicator attached every rank passes the
 * same Z/Sigma and receives all Ny outputs (one all-gather of H*(2+Nx) doubles per
 * output).  Replaces build_gp / build_TA_cov evaluation gp_functions.py:111-147,
 * :167-171 and GP.covar gp_class.py:353-381. */
int gpmpc_predict(gpmpc_handle_t h, int method, int H, const double* Z, const double* Sigma,
                  int sigma_per_point, double* mean, double* var, double* cov, double* jac);

/* Append ONE training point (x_new:(Nx,), y_new:(Ny,) host, GP input space) to a factorised
 * model in O(N^2): new rows of L and L^-1, alpha refreshed.  Capacity is the padded size
 * ceil(N/128)*128, or the one reserved by gpmpc_create_reserve (GPMPC_ERR_STATE beyond it: refit on
 * a new handle).  GPMPC_ERR_NOTPD if the Schur complement is not positive: the point is in the model
 * (N counts it) and the handle needs gpmpc_factorize (the jitter policy applies there).  Appends every
 * point given, in order; gpmpc_append_greedy chooses.  Jitter: when gpmpc_factorize needed its jitter retry
 * for an output, the factor is that of K + jitter I, and every later append (and greedy pick) puts the same
 * jitter on its new diagonal entry, so the model stays the factor of K_aug + jitter I, as a refit of the
 * grown data that needed the retry would be.  The jitter is the one recorded by the last gpmpc_factorize;
 * gpmpc_nlml and gpmpc_loo_nlpp invalidate the factor, so no append can follow them without one. */
int gpmpc_append(gpmpc_handle_t h, const double* x_new, const double* y_new);

/* Greedy selection from a pool: n_new times, append the pool point with the largest sum over outputs of the
 * posterior variance sf2_a - |L_a^-1 k_a(X, c)|^2 (noise-free, q3), ties to the lowest index.  Each choice is made
 * after the previous point has been absorbed by the rank-1 update of gpmpc_append.  This is what GP.update_data
 * (gp_class.py:384-471) set out to do, with SURVEY q14 fixed (it takes argmin and sqrt(k - |l|)).
 *   Xc (n, Nx), Yc (n, Ny) host, GP input / output space (Yc = the residual y - m(x) under a prior mean)
 *   picked (n_new) pool indices in selection order; score (n_new) or NULL: combined variance at pick time
 *   n_added: points appended (== n_new on success)
 * Hyper-parameters kept; alpha and logdet refreshed once at the end.  Handle must own all outputs on one rank
 * (GPMPC_ERR_STATE); N + n_new > capacity -> GPMPC_ERR_STATE before any work (model untouched); n >= 1 and
 * 0 <= n_new <= n, non-null Xc, Yc, picked, n_added (GPMPC_ERR_ARG).  Pool memory: 8 Ny n Npad bytes on the device.
 * GPMPC_ERR_NOTPD as gpmpc_append: *n_added includes the failing point, the handle needs gpmpc_factorize. */
int gpmpc_append_greedy(gpmpc_handle_t h, int n, const double* Xc, const double* Yc, int n_new,
                        int* picked, double* score, int* n_added);

/* Remove the n distinct training points idx (indices into the model before the call, any order) from a factorised
 * model in O(N^2) per point: rank-1 updates of the trailing blocks of L and L^-1 (never a refit, and they cannot lose
 * positive definiteness), rows and columns past each point moved up, the freed row the identity tail again (the
 * capacity is unchanged, so a later gpmpc_append reuses it).  Points go in descending index order; the point leaves
 * X and every owned output's y.  Hyper-parameters kept; alpha and logdet refreshed once at the end.  Any handle,
 * sharded or not: it updates the outputs it owns.  With gpmpc_append this keeps a sliding window of the newest
 * measurements at a constant N, where the reference refits (replace_data_all, gp_class.py:553-626) or appends with
 * its broken update_data (gp_class.py:384-471).
 *   n = 0: no-op.  GPMPC_ERR_STATE: not factorised.  GPMPC_ERR_ARG: n < 0, idx NULL with n > 0, an index outside
 *   [0, N), a duplicate, or n >= N (one point must remain).  Every check runs before any work: an error leaves the
 *   model bit-identical.  Scratch: the two Npad^2 slabs of gpmpc_get(GPMPC_GET_INVK) (allocated once, if not yet). */
int gpmpc_remove(gpmpc_handle_t h, int n, const int* idx);

/* Full posterior covariance between H test points for every OWNED output:
 * out:(out_count,H,H) host, out[a] = sf2_a - V_a^T V_a with V_a = L_a \ k(X, Z)  (the scalar
 * kss = sf2 is broadcast over the whole matrix exactly as the reference does).  Replaces
 * GP.covar, gp_class.py:353-381. */
int gpmpc_posterior_cov(gpmpc_handle_t h, int H, const double* Z, double* out);

/* Prediction plus its first derivatives w.r.t. the test inputs -- what CasADi's AD extracts from
 * the symbolic build_gp / build_TA_cov graphs (gp_functions.py:111-173) when nlpsol differentiates
 * the MPC's NLP (mpc_class.py:390-412, :496-513).  Same arguments and outputs as gpmpc_predict
 * (methods ME and TA; jac = d mean / d z), plus, each optional (NULL to skip):
 *   dvar_dz (H,Ny,Nx)     d var_a / d z_e    = -2 (K^-1 ks)^T d ks/d z_e   (one extra L^-T product)
 *   dcov_dz (H,Ny,Ny,Nx)  d cov[a][b] / d z_e of diag(var) + J Sigma J^T  (needs the mean Hessian)
 *   hess    (H,Ny,Nx,Nx)  d^2 mean_a / d z_d d z_e
 * d cov[a][b] / d Sigma[d][e] = J_a[d] J_b[e] ('TA') is formed by the caller from jac.
 * The handle must own all outputs (single process, or a replicated handle). */
int gpmpc_predict_grad(gpmpc_handle_t h, int method, int H, const double* Z, const double* Sigma,
                       int sigma_per_point, double* mean, double* var, double* cov, double* jac,
                       double* dvar_dz, double* dcov_dz, double* hess);

/* gpmpc_predict_grad plus the second derivatives w.r.t. the test inputs: what CasADi's AD extracts from the
 * same graphs (gp_functions.py:111-173) when IPOPT runs with its default exact Hessian
 * (hessian_approximation 'exact'; nlpsol, mpc_class.py:496-513, over the shooting nodes of :390-412).  The
 * first seven outputs equal gpmpc_predict_grad's bit for bit; further outputs, each optional (NULL to skip):
 *   d2var_dz2  (H,Ny,Nx,Nx)        d^2 var_a / d z_d d z_e
 *   d3mean_dz3 (H,Ny,Nx,Nx,Nx)     d^3 mean_a / d z_d d z_e d z_f  (the derivative of hess)
 *   d2cov_dz2  (H,Ny,Ny,Nx,Nx)     d^2 cov[a][b] / d z_f d z_g of diag(var) ('ME') or diag(var) + J Sigma J^T ('TA')
 * Symmetric tensors are exactly symmetric.  The mixed and Sigma-only second derivatives of 'TA' need no new
 * quantities and are formed by the caller:  d^2 cov[a][b] / d z_f d Sigma[d][e] = hess_a[d][f] J_b[e] + J_a[d] hess_b[e][f],
 * d^2 cov / d Sigma^2 = 0.  Methods ME and TA (EM: GPMPC_ERR_ARG); the handle must own all outputs (GPMPC_ERR_STATE). */
int gpmpc_predict_hess(gpmpc_handle_t h, int method, int H, const double* Z, const double* Sigma,
                       int sigma_per_point, double* mean, double* var, double* cov, double* jac,
                       double* dvar_dz, double* dcov_dz, double* hess,
                       double* d2var_dz2, double* d3mean_dz3, double* d2cov_dz2);

/* 'EM' prediction plus its first derivatives w.r.t. the test input mean z and the input covariance Sigma: what CasADi's AD
 * extracts from gp_exact_moment (gp_functions.py:344-418) when nlpsol differentiates the MPC's NLP with gp_method 'EM'.
 * Same inputs as gpmpc_predict (Sigma required).  Outputs, each optional (NULL to skip):
 *   mean (H,Ny)  var (H,Ny)  cov (H,Ny,Ny)   -- bit-identical to gpmpc_predict(GPMPC_METHOD_EM)
 *   dmean_dz (H,Ny,Nx)   dmean_dSigma (H,Ny,Nx,Nx)   dcov_dz (H,Ny,Ny,Nx)   dcov_dSigma (H,Ny,Ny,Nx,Nx)
 * d/dSigma[d][e] holds every other entry fixed (the convention jac_gp_b200 already uses for 'TA'); at a symmetric Sigma
 * that gradient is symmetric in (d,e), and it is returned exactly symmetric.  The handle must own all outputs
 * (GPMPC_ERR_STATE); Ny <= 44 as for EM.  gpmpc_predict_grad keeps rejecting 'EM'. */
int gpmpc_predict_em_grad(gpmpc_handle_t h, int H, const double* Z, const double* Sigma, int sigma_per_point,
                          double* mean, double* var, double* cov,
                          double* dmean_dz, double* dmean_dSigma, double* dcov_dz, double* dcov_dSigma);

/* 'EM' prediction plus its first and second derivatives w.r.t. z and Sigma: the exact Hessian IPOPT asks for when nlpsol
 * runs the MPC with gp_method 'EM'.  Inputs as gpmpc_predict_em_grad; the first seven outputs are bit-identical to its.
 * Every output is optional (NULL to skip).  The differentiated index is always the last one:
 *   d2mean_dz2        (H,Ny,Nx,Nx)            d dmean_dz[a][d]          / d z_e
 *   d2mean_dSigma_dz  (H,Ny,Nx,Nx,Nx)         d dmean_dSigma[a][d][e]   / d z_f
 *   d2mean_dSigma2    (H,Ny,Nx,Nx,Nx,Nx)      d dmean_dSigma[a][d][e]   / d Sigma[f][g]
 *   d2cov_dz2         (H,Ny,Ny,Nx,Nx)         d dcov_dz[a][b][d]        / d z_e
 *   d2cov_dSigma_dz   (H,Ny,Ny,Nx,Nx,Nx)      d dcov_dSigma[a][b][d][e] / d z_f
 *   d2cov_dSigma2     (H,Ny,Ny,Nx,Nx,Nx,Nx)   d dcov_dSigma[a][b][d][e] / d Sigma[f][g]
 * The mixed block d dmean_dz[a][f] / d Sigma[d][e] is d2mean_dSigma_dz[a][d][e][f] (and likewise for cov): it is not
 * returned twice.  Sigma entries vary one at a time as in gpmpc_predict_em_grad, whose symmetric gradient is differentiated
 * w.r.t. the single entry Sigma[f][g]; at a symmetric Sigma the Sigma-Sigma blocks are exactly symmetric under d <-> e,
 * f <-> g and (d,e) <-> (f,g), the mean blocks fully symmetric (d mean/dSigma = 1/2 d^2 mean/dz^2), and every block
 * exactly symmetric in (a,b).  Every sum runs in a fixed order: a point's results do not depend on H or its row.
 * GPMPC_ERR_ARG: Z or Sigma NULL, H < 1, Ny > 44 or Nx > 16; GPMPC_ERR_STATE: not factorised, or the handle does not own
 * every output; all checked before any work.  Device scratch beyond gpmpc_predict_em_grad's (which includes a full
 * symmetric K^-1 per output, 8 B Ny Npad^2, kept until the next factor change): 8 B R (3 Ny + Ny (Ny+1)) (ceil(N/64) + H)
 * + 24 B Npad F, with F = (Nx+1)(Nx+2)/2 and R = the number of (monomial of degree <= 4, monomial of degree <= 2) pairs
 * of total degree <= 4 (3435 at Nx = 8, 41157 at Nx = 16); for the derivative tensors 8 B H (2 Ny T + Ny(Ny+1)/2 (9 Nx^2 + 1))
 * with T = 1 + Nx + ... + Nx^4, the outputs 8 B H (Ny + Ny^2)(Nx^2 + Nx^3 + Nx^4), and at most 512 MB of per-CTA scratch. */
int gpmpc_predict_em_hess(gpmpc_handle_t h, int H, const double* Z, const double* Sigma, int sigma_per_point,
                          double* mean, double* var, double* cov,
                          double* dmean_dz, double* dmean_dSigma, double* dcov_dz, double* dcov_dSigma,
                          double* d2mean_dz2, double* d2mean_dSigma_dz, double* d2mean_dSigma2,
                          double* d2cov_dz2, double* d2cov_dSigma_dz, double* d2cov_dSigma2);

/* Open-loop multi-step prediction with the state kept on the device: the numeric loop of GP.predict_compare
 * (gp_class.py:746-804, :779-792: mean_t, covar_x = predict(mean_t, u_t, covar); covar[:Ny,:Ny] = covar_x) for a
 * model whose inputs are z = [x, u] (Nx = Ny + Nu).  All Nt steps are enqueued back to back, one synchronisation.
 *   z0      (Nx)        first input [x_0, u_0], already in the GP's input units (standardised when the GP normalises)
 *   U       (Nt, Nu)    inputs u_0 .. u_{Nt-1}, GP input units (row 0 repeats z0's tail); may be NULL when Nu = 0
 *   Sigma0  (Nx, Nx)    covariance of z0; afterwards only its top-left Ny x Ny block is replaced by cov_t
 *   scale   (4, Ny)     [stdY | meanY | meanX | stdX] or NULL: next x = ((mean * stdY + meanY) - meanX) / stdX, the
 *                       inverse_mean / standardize pair of gp_class.py:629-638 in the same operation order
 *   means, vars (Nt, Ny) predicted means / diag(cov_t) (the propagated variance the reference records, gp_class.py:793)
 *                       in the GP's output units, cov_last (Ny, Ny) or NULL
 * method GPMPC_METHOD_ME, _TA or _UT; the handle must own all outputs.  Same as gpmpc_rollout_batch with B = 1, K = NULL. */
int gpmpc_rollout(gpmpc_handle_t h, int method, int Nt, const double* z0, const double* U, const double* Sigma0,
                  const double* scale, double* means, double* vars, double* cov_last);

/* gpmpc_rollout for B trajectories in one pass, optionally closed-loop: the feedback branch of GP.predict_compare
 * (gp_class.py:770-804) with a gain K from the reference's lqr (mpc_class.py:956-976: DARE, K = -(R + B^T P B)^-1 B^T P A).
 * Each step is one predict pass over the B current inputs (H = B, one Sigma per trajectory); a kernel then forms every
 * trajectory's next input and covariance.  With K, after step t (x = mean_t * stdY + meanY, or mean_t without scale):
 *   u = K (x - x_ref), then (u - meanU) / stdU when uscale is given  (the caller's units, as GP.predict standardises u)
 *   Sigma_uu = K cov_t K^T,  Sigma_xu = cov_t K^T,  Sigma_ux = Sigma_xu^T,  then cov_t into the top-left block
 * with cov_t in the GP's output units, as the reference does (q4).  Without K the inputs come from U as in gpmpc_rollout and
 * the u blocks of Sigma are kept.
 *   z0      (B, Nx)       first inputs [x_0, u_0] in the GP's input units (with K: u_0 = K (x_0 - x_ref), standardised)
 *   U       (B, Nt, Nu)   open-loop inputs, GP input units; NULL when Nu = 0 or K is given
 *   Sigma0  (B, Nx, Nx)   input covariance of each trajectory's first step
 *   scale   (4, Ny)       [stdY | meanY | meanX | stdX] or NULL, as gpmpc_rollout
 *   K       (Nu, Ny)      feedback gain in the caller's units, or NULL (open loop); needs Nu > 0
 *   x_ref   (Ny)          caller units, NULL = 0 (read only with K)
 *   uscale  (2, Nu)       [meanU | stdU] or NULL (read only with K)
 *   means, vars (B, Nt, Ny) as gpmpc_rollout per trajectory;  cov_last (B, Ny, Ny) or NULL
 * Methods ME, TA and UT (EM: GPMPC_ERR_ARG); B, Nt >= 1; the handle must own all outputs (GPMPC_ERR_STATE).  With UT each
 * step is one 'ME' pass over the B (2 Nx + 1) sigma points of the B current (z_t, Sigma_t), formed on the device, and the
 * recombination; the next input and covariance follow the same rules as ME and TA. */
int gpmpc_rollout_batch(gpmpc_handle_t h, int method, int B, int Nt, const double* z0, const double* U,
                        const double* Sigma0, const double* scale, const double* K, const double* x_ref,
                        const double* uscale, double* means, double* vars, double* cov_last);

/* gpmpc_rollout_batch with exact moment matching ('EM'): same arguments (no method) and outputs, the same slab layout,
 * policy and feedback update; only each step's predict differs.  Step t copies the B current Sigma to the host (one copy,
 * one synchronisation), prepares each point's Nx x Nx quantities there as gpmpc_predict(EM) does, copies them back and
 * runs the batched 'EM' forward over the B points (chunks of at most gpmpc_set_option("em_points") points, else a scratch
 * budget).  The preparation stays on the host on purpose: it takes logarithms of determinants, and a device port (CUDA's
 * log is not glibc's) would break bit-identity with gpmpc_predict(EM); the synchronisation costs microseconds against
 * about a millisecond of EM device work per point at N = 1000.  Each trajectory's means, vars and cov_last are those of
 * the host loop of gpmpc_predict(EM, H = 1) calls with the same inputs, bit for bit, whatever B and its row.
 * GPMPC_ERR_ARG: every argument error of gpmpc_rollout_batch, checked before any work (Nx = Ny + Nu with Nu >= 0 keeps
 * Ny <= Nx <= 32 inside gpmpc_predict(EM)'s Ny <= 44, so a model with more outputs fails there); Sigma + Lambda not
 * positive definite at step t (gpmpc_last_error names t and the trajectory; the outputs are then undefined and the handle
 * stays usable).  GPMPC_ERR_STATE: not factorised, or the handle does not own every output. */
int gpmpc_rollout_batch_em(gpmpc_handle_t h, int B, int Nt, const double* z0, const double* U, const double* Sigma0,
                           const double* scale, const double* K, const double* x_ref, const double* uscale,
                           double* means, double* vars, double* cov_last);

/* gpmpc_rollout_batch plus the exact derivatives of every step's mean and variance w.r.t. what produced the trajectory,
 * by forward-mode tangents carried on the device beside the roll-out (one derivative chain of gpmpc_predict_grad per step
 * on the same points, then one tangent kernel).  Same arguments; means, vars, cov_last are bit-identical to
 * gpmpc_rollout_batch's.  Further outputs, both required:
 *   dmeans, dvars (B, Nt, Ny, P)  d means[b,t,a] / d theta_p and d vars[b,t,a] / d theta_p, GP output units
 * with the P parameters of trajectory b, in this column order:
 *   z0[b] (Nx), then open loop the rows U[b,1..Nt-1] ((Nt-1) Nu; row 0 is unused, z0 carries u_0), or with K the
 *   entries of K row-major (Nu Ny):  P = Nx + (Nt-1) Nu open loop, Nx + Nu Ny with feedback, Nx when Nu = 0.
 * Sigma0, scale, x_ref and uscale are held fixed.  Per parameter, step t (J_t, dcov_dz_t, dvar_dz_t of gpmpc_predict_grad):
 *   dm = J dz,  dC = sum_e dcov_dz[.,.,e] dz_e + J dSigma J^T ('TA')  or  diag(dvar_dz dz) ('ME'),  dvars = diag(dC)
 *   next dz[:Ny] = dm stdY / stdX (dm without scale);  open loop: dz[Ny:] the unit tangent of U[t+1], dSigma x block = dC,
 *   u blocks kept;  with K, x = mean stdY + meanY:  du = (K dx + dK (x - x_ref)) / stdU,  dSigma_xu = dC K^T + C dK^T,
 *   dSigma_uu = dK C K^T + K dC K^T + K C dK^T  (the derivatives of the feedback update of gpmpc_rollout_batch).
 * Every sum runs in a fixed order: trajectory b's results do not depend on B or its row.  Methods ME and TA (EM:
 * GPMPC_ERR_ARG); GPMPC_ERR_STATE: not factorised, or the handle does not own every output; GPMPC_ERR_ARG: every argument
 * error of gpmpc_rollout_batch, or dmeans / dvars NULL.  Every check runs before any work.  Device memory: 8 B P (Nx + Nx^2)
 * bytes of tangents ('TA'; 8 B P Nx for 'ME') plus 16 Nt B Ny P bytes of outputs. */
int gpmpc_rollout_batch_grad(gpmpc_handle_t h, int method, int B, int Nt, const double* z0, const double* U,
                             const double* Sigma0, const double* scale, const double* K, const double* x_ref,
                             const double* uscale, double* means, double* vars, double* cov_last,
                             double* dmeans, double* dvars);

/* gpmpc_rollout_batch_em plus the exact derivatives of every step's mean and variance: the 'EM' counterpart of
 * gpmpc_rollout_batch_grad.  Arguments as gpmpc_rollout_batch_em; means, vars, cov_last are bit-identical to its.  dmeans,
 * dvars (B, Nt, Ny, P), both required, have gpmpc_rollout_batch_grad's shapes, parameter columns (z0[b], then U rows
 * 1..Nt-1 open loop or K row-major with feedback), units and next-tangent rules.  Sigma0, scale, x_ref and uscale are held
 * fixed.  Per parameter, step t takes the four blocks of gpmpc_predict_em_grad at (z_t, Sigma_t), bit-identical to that
 * entry's at the same inputs, and forms
 *   dm = dmean_dz dz + sum_{d,e} dmean_dSigma[., d, e] dSigma[d, e],  dC = dcov_dz dz + sum_{d,e} dcov_dSigma[., ., d, e] dSigma[d, e]
 * summed over all Nx^2 entries of the symmetric dSigma (the blocks hold every other entry fixed, so this is the directional
 * derivative); dvars = diag(dC).  Unlike 'TA' the mean depends on Sigma, so Sigma tangents are carried in open loop too.
 * Each step synchronises twice: once to bring Sigma_t to the host (as gpmpc_rollout_batch_em) and once to bring the
 * step's derivative records and means there, where the derivatives are finished as gpmpc_predict_em_grad finishes them.
 * Every sum runs in a fixed order: trajectory b's results do not depend on B, its row or gpmpc_set_option("em_points").
 * GPMPC_ERR_ARG: every argument error of gpmpc_rollout_batch_em, or dmeans / dvars NULL, checked before any work; Sigma +
 * Lambda not positive definite at step t (gpmpc_last_error names t and the trajectory; the outputs are then undefined and
 * the handle stays usable).  GPMPC_ERR_STATE: not factorised, or the handle does not own every output.  Device memory
 * beyond gpmpc_rollout_batch_em's: the full symmetric K^-1 per output of gpmpc_predict_em_grad (8 B Ny Npad^2, kept until
 * the next factor change; 17 GB at N = 16384, Ny = 8), that entry's D = 2 records of B points, 8 B P (Nx + Nx^2) bytes of
 * tangents, 8 B (Ny Nx + Ny Nx^2 + Ny^2 Nx + Ny^2 Nx^2) bytes of derivative blocks and 16 Nt B Ny P bytes of outputs. */
int gpmpc_rollout_batch_em_grad(gpmpc_handle_t h, int B, int Nt, const double* z0, const double* U,
                                const double* Sigma0, const double* scale, const double* K, const double* x_ref,
                                const double* uscale, double* means, double* vars, double* cov_last,
                                double* dmeans, double* dvars);

/* Sample trajectories of the learned dynamics: each of the B trajectories is one draw f of the GP posterior, evaluated along
 * the inputs that draw visits.  Per output a and step t, f_t(z_t) is drawn conditioned on the values the same draw took
 * at the earlier points z_0 .. z_{t-1} of the trajectory, so the whole trajectory satisfies f - m = R eps with R the
 * Cholesky factor of the joint posterior covariance of its points (a consistent function sample, not fresh noise per
 * step).  A point whose conditional variance is at the rounding level (<= 1e-12 sf2: the trajectory returns to a point
 * it visited) is determined by the earlier ones: f_t is the conditional mean and its eps is unused.  The next input is
 * formed from the sampled state exactly as gpmpc_rollout_batch forms it from the mean (scale, K, x_ref, uscale).
 *   z0      (B, Nx)       first inputs, already drawn, GP input units
 *   U       (B, Nt, Nu)   open-loop inputs; NULL when Nu = 0 or K is given (as gpmpc_rollout_batch)
 *   eps     (B, Nt, Ny)   standard normals of the function draws
 *   xi      (B, Nt, Ny)   process-noise standard normals, or NULL: the state is f_t + sn_a xi (the noise does not enter
 *                         the conditioning, which is on the latent f)
 *   scale, K, x_ref, uscale  as gpmpc_rollout_batch
 *   samples (B, Nt, Ny)   the next states, GP output units (like gpmpc_rollout_batch's means)
 *   z_out   (B, Nt, Nx)   or NULL: the input used at each step
 *   kept    (B, Nt, Ny)   or NULL: 1 where the point entered the conditioning set
 * GPMPC_ERR_ARG: B < 1, Nt < 1, z0 / eps / samples NULL, Nu > 0 with neither U nor K, K with Nu = 0, Nt too large for
 * the per-trajectory factor's shared memory (Nt <= 4095).  GPMPC_ERR_STATE: not factorised, or the handle does not own
 * every output.  Every check runs before any work.  Device memory: 8 Ny Nt B Npad bytes of solved rows (8 GB at
 * Ny = 8, Npad = 16384, B = 256, Nt = 30) plus 8 (Ny B Nt^2 + B Nt (Nx + 4 Ny)) bytes. */
int gpmpc_rollout_sample(gpmpc_handle_t h, int B, int Nt, const double* z0, const double* U, const double* eps,
                         const double* xi, const double* scale, const double* K, const double* x_ref,
                         const double* uscale, double* samples, double* z_out, int* kept);

/* gpmpc_rollout_sample plus the pathwise derivatives of every draw with its normals eps (and xi) held fixed: what a
 * sample-average objective over fixed draws (scenario MPC, reparameterised policy search) needs.  Arguments as
 * gpmpc_rollout_sample; samples, z_out and kept are bit-identical to its.  dsamples (B, Nt, Ny, P), required, GP output
 * units, with gpmpc_rollout_batch_grad's parameter columns: z0[b] (Nx), then U rows 1..Nt-1 open loop or K row-major with
 * feedback (P = Nx + (Nt-1) Nu, Nx + Nu Ny, or Nx when Nu = 0); scale, x_ref and uscale are held fixed.  Per output a and
 * step t, with beta_s = K_a^-1 k_a(X, z_s), w = R^-1 c and d = c_tt - |w|^2 of the draw:
 *   dm = J dz_t,  dc_tt = dvar_dz . dz_t,  dc_s = g(t,s) . dz_t + g(s,t) . dz_s  (s kept before t),
 *   g(t,s)_e = -(z_t,e - z_s,e) / ell_e^2 k(z_t, z_s) + sum_i (z_t,e - x_i,e) / ell_e^2 k(x_i, z_t) beta_s[i],
 *   dw = R^-1 (dc - dR w),  dd = dc_tt - 2 w . dw,  df = dm + dw . eps_S (+ dd / (2 sqrt d) eps_t when kept),
 * where J, dvar_dz are gpmpc_predict_grad's at z_t and dR carries the tangent of R's rows.  The kept decision is the
 * draw's and is not differentiated: the result is the derivative of the branch taken.  The next tangent is
 * gpmpc_rollout_batch_grad's with dm replaced by df and the mean by the sample.  Every sum runs in a fixed order:
 * trajectory b's results do not depend on B or its row.  GPMPC_ERR_ARG: every argument error of gpmpc_rollout_sample,
 * dsamples NULL, or Nt > 64 (the tangent kernel keeps each trajectory's R in shared memory); GPMPC_ERR_STATE: not
 * factorised, or the handle does not own every output.  Every check runs before any work.  Device memory beyond
 * gpmpc_rollout_sample's: the beta store 8 Ny Nt B Npad bytes (as large as its V store), U = L^-1^T of the derivative
 * chain 8 Ny Npad^2 bytes (17 GB at Ny = 8, Npad = 16384), the tangents of R 8 Ny B P Nt^2 bytes, the tangent history
 * 8 Nt B P Nx bytes, 16 Ny B Nt Nx bytes of cross terms and 8 Nt B Ny P bytes of outputs.  At Ny = 8, Npad = 16384 with
 * B = 256, Nt = 30 the two stores alone are 16 GB beside the 55 GB of the factor and its copies: that does not fit on
 * an 80 GB card; B = 64 does. */
int gpmpc_rollout_sample_grad(gpmpc_handle_t h, int B, int Nt, const double* z0, const double* U, const double* eps,
                              const double* xi, const double* scale, const double* K, const double* x_ref,
                              const double* uscale, double* samples, double* z_out, int* kept, double* dsamples);

/* Problem sizes of a handle (GP.get_size, gp_class.py:266-274: N, and Nx, Ny). */
int gpmpc_get_size(gpmpc_handle_t h, int* N, int* Nx, int* Ny);

/* Same with DEVICE pointers, enqueued on the handle's stream; returns without
 * synchronising unless sync != 0. */
int gpmpc_predict_device(gpmpc_handle_t h, int method, int H, const double* dZ, const double* dSigma,
                         int sigma_per_point, double* d_mean, double* d_var, double* d_cov,
                         double* d_jac, int sync);

/* Copy a result of the last factorisation for global output a into dst (host). */
int gpmpc_get(gpmpc_handle_t h, int what, int a, double* dst);

/* Engine options: "refine" (0/1: one step of iterative refinement of v = L\ks through
 * the stored factor), "predict_ctas" (persistent grid of the stream-K predict product,
 * 0 = two CTAs per SM), "peer" (0/1), "peer_timeout_s" (consumer wait for a peer's flag),
 * "small_tiles" (batched 128x64 tile count of a factorisation GEMM below which it runs on
 * 64x32 tiles; default 4 per SM), "nlml_batch_max" (entries per gpmpc_nlml_batch pass, a cap
 * on its scratch; 0 = all, the default), "em_points" (points per batched 'EM' forward, a cap
 * on its scratch of two Npad^2 slabs per point; 0 = a 1 GiB budget decides, the default; the
 * results do not depend on it), "ut_alpha", "ut_beta", "ut_kappa" (the 'UT' parameters, see GPMPC_METHOD_UT;
 * GPMPC_ERR_ARG and no change for a non-finite value, alpha <= 0 or n + lambda <= 0, i.e. kappa <= -Nx).  Any other
 * name returns GPMPC_ERR_ARG. */
int gpmpc_set_option(gpmpc_handle_t h, const char* name, double value);

/* Multi-GPU: one process per GPU.  Rank 0 calls gpmpc_comm_unique_id and ships the
 * 128 bytes to the other ranks (any transport); every rank then calls
 * gpmpc_comm_init.  NCCL is loaded with dlopen("libnccl.so.2"). */
int gpmpc_comm_unique_id(void* id128);
int gpmpc_comm_init(gpmpc_handle_t h, const void* id128, int rank, int world);

/* Fused epilogue + all-gather over NVLink peer memory (optional, after gpmpc_comm_init):
 * every rank exports one exchange block (gpmpc_peer_export -> 64-byte CUDA IPC handle, room
 * for Hcap test points), the handles of ALL ranks (world x 64 bytes, rank order) are passed
 * to gpmpc_peer_attach.  gpmpc_predict* then stores each rank's results directly into every
 * peer's buffer from the predict epilogue and synchronises with flags; ncclAllGather remains
 * the fallback (H > Hcap, option "peer" = 0, or no attach). */
int gpmpc_peer_export(gpmpc_handle_t h, int Hcap, void* handle64);
int gpmpc_peer_attach(gpmpc_handle_t h, const void* handles);

/* The handle's CUDA stream (cudaStream_t) so a caller can record events on it. */
void* gpmpc_stream(gpmpc_handle_t h);
int gpmpc_synchronize(gpmpc_handle_t h);

/* Time one kernel of the path with CUDA events on the handle's stream: `reps` launches
 * after one warm-up, average milliseconds in ms_out[0]; n = problem size override
 * (0 = the handle's N).  flops/bytes are derived by the caller (DESIGN.md). */
int gpmpc_profile(gpmpc_handle_t h, int what, int n, int reps, double* ms_out);

/* Load balance of the persistent predict product for an H-point batch: per-CTA busy time
 * out4 = {shortest, longest, mean, first start -> last end} in microseconds (%globaltimer). */
int gpmpc_profile_balance(gpmpc_handle_t h, int H, double* out4);

/* Serial tail of the fused predict kernel (the CTA that completes the step), H-point batch, after a predict call:
 * out8 = microseconds relative to the latest end of every other CTA of {last output complete, records built,
 * step counter passed, records staged, J Sigma done, outputs written}, kernel span, tail CTA span. */
int gpmpc_profile_tail(gpmpc_handle_t h, int H, double* out8);

/* Phase clock stamps (SM cycles since kernel start) of one 128x128 potrf+trtri leaf: out15 =
 * {start, block loaded, first panel, block steps 1..7, L stored, inverse levels 16/32/64, L^-1 stored}. */
int gpmpc_profile_leaf(gpmpc_handle_t h, double* out15);

#ifdef __cplusplus
}
#endif
#endif /* GPMPC_H */
