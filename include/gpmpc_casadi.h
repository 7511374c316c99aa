/* CasADi `external` entry points of libgpmpc.so -- the C side of the adapter that lets
 * mpc_class.py keep its CasADi/IPOPT NLP while the GP inside it runs on the GPU
 * (SURVEY.md 8f row 1; reference call sites mpc_class.py:361-423, :496-513,
 * gp_class.py:207-263).  Usage from Python, once CasADi is installed:
 *
 *     lib.gp_b200_bind(engine_handle, GPMPC_METHOD_TA, Nt)
 *     F = casadi.external('gp_b200', '.../libgpmpc.so')    # F(z, sigma) -> (mean, cov)
 *
 * CasADi resolves `gp_b200`, `gp_b200_n_in/_n_out/_name_in/_name_out/_sparsity_in/_sparsity_out/
 * _work/_incref/_decref` and, for derivatives, the Jacobian function `jac_gp_b200` with the same
 * family of helpers.  Conventions: casadi_int = long long, casadi_real = double, dense blocks are
 * column-major, sparsity patterns are compressed-column {nrow, ncol, colind[ncol+1], row[nnz]}
 * ({nrow, ncol, 1} = dense).  Shapes for Nt shooting nodes (all in the GP's standardised space;
 * the scaling of gp_class.py:253-262 is two elementwise CasADi expressions around F):
 *   z (Nx x Nt), sigma (Nx x Nx*Nt)  ->  mean (Ny x Nt), cov (Ny x Ny*Nt)
 *   jac_gp_b200(z, sigma, mean, cov) -> jac_mean_z, jac_mean_sigma, jac_cov_z, jac_cov_sigma
 *   (block-diagonal: node t only depends on node t's inputs).  jac_mean_sigma is empty for 'ME' / 'TA' and
 *   Ny x Nx^2 per node for 'EM'; jac_cov_sigma is Ny^2 x Nx^2 per node for 'TA' and 'EM' (empty for 'ME');
 *   column d + Nx*e holds d / d Sigma[d][e] with every other entry fixed.  'EM' values come from
 *   gpmpc_predict_em_grad.
 *   jac_jac_gp_b200(z, sigma, mean, cov, jac_mean_z, jac_mean_sigma, jac_cov_z, jac_cov_sigma) -> 16 blocks of
 *   second derivatives (IPOPT's default exact Hessian; see below).
 */
#ifndef GPMPC_CASADI_H
#define GPMPC_CASADI_H
#include "gpmpc.h"
#ifdef __cplusplus
extern "C" {
#endif

/* method GPMPC_METHOD_ME, _TA or _EM; Nt shooting nodes per call.  GPMPC_ERR_ARG otherwise. */
int gp_b200_bind(gpmpc_handle_t h, int method, int Nt);
/* As gp_b200_bind(h, GPMPC_METHOD_EM, Nt) -- the same gp_b200 and jac_gp_b200 values and patterns -- with
 * jac_jac_gp_b200 served from gpmpc_predict_em_hess: the blocks of the four Jacobians w.r.t. z and sigma (output-major
 * numbering o*4 + i: 0, 1, 4, 5, 8, 9, 12, 13) are block-diagonal over the nodes, rows the column-major vec of the
 * differentiated Jacobian, column d + Nx*e <-> Sigma[d][e]; the blocks w.r.t. mean and cov stay empty.
 * GPMPC_ERR_ARG as gp_b200_bind, or Nx > 16. */
int gp_b200_bind_em_hess(gpmpc_handle_t h, int Nt);
void gp_b200_unbind(void);

long long gp_b200_n_in(void);
long long gp_b200_n_out(void);
const char* gp_b200_name_in(long long i);
const char* gp_b200_name_out(long long i);
const long long* gp_b200_sparsity_in(long long i);
const long long* gp_b200_sparsity_out(long long i);
int gp_b200_work(long long* sz_arg, long long* sz_res, long long* sz_iw, long long* sz_w);
void gp_b200_incref(void);
void gp_b200_decref(void);
int gp_b200(const double** arg, double** res, long long* iw, double* w, int mem);

long long jac_gp_b200_n_in(void);
long long jac_gp_b200_n_out(void);
const char* jac_gp_b200_name_in(long long i);
const char* jac_gp_b200_name_out(long long i);
const long long* jac_gp_b200_sparsity_in(long long i);
const long long* jac_gp_b200_sparsity_out(long long i);
int jac_gp_b200_work(long long* sz_arg, long long* sz_res, long long* sz_iw, long long* sz_w);
int jac_gp_b200(const double** arg, double** res, long long* iw, double* w, int mem);

/* Second derivatives for IPOPT's exact Hessian: the Jacobian function CasADi looks up by name when it
 * differentiates jac_gp_b200.  Inputs (z, sigma, out_mean, out_cov, out_jac_mean_z, out_jac_mean_sigma,
 * out_jac_cov_z, out_jac_cov_sigma); outputs jac_jac_<o>_<i> for o in jac_gp_b200's outputs x i in its inputs
 * (output-major, 16).  Rows index the column-major dense vec of the differentiated Jacobian, columns the
 * dense vec of the input.  Nonzero: jac_mean_z/z, jac_cov_z/z and, for 'TA', jac_cov_z/sigma and
 * jac_cov_sigma/z (block-diagonal over the nodes); all other outputs are structurally empty.  With 'EM' bound there
 * are no second derivatives and jac_jac_gp_b200 returns failure (IPOPT: hessian_approximation 'limited-memory'). */
long long jac_jac_gp_b200_n_in(void);
long long jac_jac_gp_b200_n_out(void);
const char* jac_jac_gp_b200_name_in(long long i);
const char* jac_jac_gp_b200_name_out(long long i);
const long long* jac_jac_gp_b200_sparsity_in(long long i);
const long long* jac_jac_gp_b200_sparsity_out(long long i);
int jac_jac_gp_b200_work(long long* sz_arg, long long* sz_res, long long* sz_iw, long long* sz_w);
void jac_jac_gp_b200_incref(void);
void jac_jac_gp_b200_decref(void);
int jac_jac_gp_b200(const double** arg, double** res, long long* iw, double* w, int mem);

#ifdef __cplusplus
}
#endif
#endif /* GPMPC_CASADI_H */
