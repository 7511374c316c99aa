// CasADi `external`-shaped entry points around gpmpc_predict_grad / gpmpc_predict_hess / gpmpc_predict_em_grad
// (SURVEY 8f row 1).
//
// mpc_class.py:361-423 calls gp.predict(mean_t, u_t, covar_t) once per shooting node with MX
// symbols and nlpsol (:496-513) differentiates the resulting graph.  With
//     F = casadi.external('gp_b200', 'libgpmpc.so')
// the GP becomes ONE opaque call for all Nt nodes per NLP iterate, evaluated on the GPU, with the
// analytic Jacobian function `jac_gp_b200` CasADi looks up by name.  The signatures follow
// CasADi's C API for external functions (casadi_int = long long, casadi_real = double; dense
// matrices are column-major, sparsity patterns are compressed-column: {nrow, ncol, colind[ncol+1],
// row[nnz]}, with the 3-entry form {nrow, ncol, 1} meaning dense).  Nothing here needs CasADi to
// compile or to be tested: tests drive these entry points through ctypes.
//
//   inputs : i0 = Z     (Nx  x Nt)     test inputs of all shooting nodes, standardised space
//            i1 = Sigma (Nx  x Nx*Nt)  input covariance of every node (Nt blocks side by side)
//   outputs: o0 = mean  (Ny  x Nt)
//            o1 = cov   (Ny  x Ny*Nt)  'TA' / 'ME' / 'EM' covariance blocks
//   jac_gp_b200: inputs (i0, i1, o0, o1), outputs block-diagonal sparse
//            jac_o0_i0 (Ny*Nt x Nx*Nt), jac_o0_i1 (empty; 'EM': Ny x Nx*Nx per node, d mean_a / d Sigma[d][e]),
//            jac_o1_i0 (Ny*Ny*Nt x Nx*Nt),
//            jac_o1_i1 (Ny*Ny*Nt x Nx*Nx*Nt;  d cov[a][b] / d Sigma[d][e] = J_a[d] J_b[e] for 'TA', the exact
//            gradient of gpmpc_predict_em_grad for 'EM'; column d + Nx*e <-> Sigma[d][e]; empty for 'ME')
//   jac_jac_gp_b200: inputs (i0, i1, o0, o1, and the four outputs of jac_gp_b200), outputs the Jacobians of
//            jac_gp_b200's four outputs w.r.t. its four inputs (output-major), what IPOPT's exact Hessian
//            needs.  Rows index the column-major dense vec of the differentiated Jacobian, columns the dense
//            vec of the input (the convention of jac_gp_b200).  Nonzero blocks per node:
//              jac_mean_z  / z      Ny*Nx*Nx         d^2 mean_a / d z_d d z_e        (hess)
//              jac_cov_z   / z      Ny*Ny*Nx*Nx      d^2 cov[a][b] / d z_e d z_f     (d2cov_dz2)
//              jac_cov_z   / sigma  Ny*Ny*Nx*Nx*Nx   hess_a[d][e] J_b[e'] + J_a[d] hess_b[e'][e]   ('TA')
//              jac_cov_sigma / z    Ny*Ny*Nx*Nx*Nx   the same values, w.r.t. z_f of d cov / d Sigma[d][e]  ('TA')
//            everything else is structurally zero.  'EM' bound by gp_b200_bind: jac_jac_gp_b200 returns failure.
//            'EM' bound by gp_b200_bind_em_hess: gpmpc_predict_em_hess serves the blocks of the four Jacobians w.r.t.
//            z and sigma (0, 1, 4, 5, 8, 9, 12, 13), block-diagonal over the nodes; those w.r.t. mean and cov stay empty.
#include "../../include/gpmpc.h"

#include <functional>
#include <mutex>
#include <vector>

typedef long long casadi_int;
typedef double casadi_real;

namespace {
struct Bound {
    gpmpc_handle_t h = nullptr;
    int method = GPMPC_METHOD_TA, Nt = 0, Nx = 0, Ny = 0;
    std::vector<casadi_int> sp_in[2], sp_out[2], sp_jac[4], sp_jj[16];
    std::vector<double> sig, mean, var, cov, jac, dvar, dcov, hess, d2cov, dmS, dcS;   // dmS / dcS: 'EM' d / d Sigma
    bool em_hess = false;                               // 'EM' bound by gp_b200_bind_em_hess: second derivatives served
    std::vector<double> mSz, mSS, cSz, cSS;             // 'EM' d2mean_dSigma_dz, d2mean_dSigma2, d2cov_dSigma_dz, d2cov_dSigma2
    int refs = 0;
};
Bound g_b;
std::mutex g_mtx;

std::vector<casadi_int> dense_sp(casadi_int r, casadi_int c) { return {r, c, 1}; }

// block-diagonal CCS pattern: Nt dense blocks of R rows x Cc columns
std::vector<casadi_int> blockdiag_sp(casadi_int R, casadi_int Cc, casadi_int Nt)
{
    std::vector<casadi_int> sp;
    sp.reserve(2 + Cc * Nt + 1 + R * Cc * Nt);
    sp.push_back(R * Nt); sp.push_back(Cc * Nt);
    for (casadi_int c = 0; c <= Cc * Nt; ++c) sp.push_back(c * R);
    for (casadi_int t = 0; t < Nt; ++t)
        for (casadi_int c = 0; c < Cc; ++c)
            for (casadi_int r = 0; r < R; ++r) sp.push_back(t * R + r);
    return sp;
}
std::vector<casadi_int> empty_sp(casadi_int r, casadi_int c)
{
    std::vector<casadi_int> sp(2 + c + 1, 0);
    sp[0] = r; sp[1] = c;
    return sp;
}

// CCS pattern of Nt diagonal blocks: node t owns the C columns [t*C, (t+1)*C), each holding the rows rows(t)
// (ascending)
std::vector<casadi_int> nodes_sp(casadi_int nrow, casadi_int C, casadi_int Nt,
                                 const std::function<std::vector<casadi_int>(casadi_int)>& rows)
{
    std::vector<casadi_int> sp = {nrow, C * Nt};
    std::vector<casadi_int> ri;
    casadi_int nnz = 0;
    sp.push_back(0);
    for (casadi_int t = 0; t < Nt; ++t) {
        const std::vector<casadi_int> r = rows(t);
        for (casadi_int c = 0; c < C; ++c) {
            ri.insert(ri.end(), r.begin(), r.end());
            nnz += (casadi_int)r.size();
            sp.push_back(nnz);
        }
    }
    sp.insert(sp.end(), ri.begin(), ri.end());
    return sp;
}

enum { EVAL_VALUE = 0, EVAL_GRAD = 1, EVAL_HESS = 2 };

// evaluate mean/cov (+ derivatives for EVAL_GRAD / EVAL_HESS) for the bound handle; Sigma blocks are
// transposed to the engine's row-major convention (a symmetric Sigma is unchanged)
int eval(const casadi_real* Z, const casadi_real* Sigma, int mode)
{
    Bound& b = g_b;
    if (!b.h || !Z) return 1;
    const int Nt = b.Nt, Nx = b.Nx;
    const bool ta = b.method == GPMPC_METHOD_TA, em = b.method == GPMPC_METHOD_EM;
    if (ta || em) {
        if (!Sigma) return 1;
        for (int t = 0; t < Nt; ++t)
            for (int d = 0; d < Nx; ++d)
                for (int e = 0; e < Nx; ++e)
                    b.sig[((size_t)t * Nx + d) * Nx + e] = Sigma[((size_t)t * Nx + e) * Nx + d];
    }
    if (em) {
        if (mode == EVAL_VALUE)
            return gpmpc_predict(b.h, b.method, Nt, Z, b.sig.data(), 1, b.mean.data(), b.var.data(), b.cov.data(), nullptr) == GPMPC_OK ? 0 : 1;
        if (mode == EVAL_GRAD)
            return gpmpc_predict_em_grad(b.h, Nt, Z, b.sig.data(), 1, b.mean.data(), b.var.data(), b.cov.data(), b.jac.data(),
                                         b.dmS.data(), b.dcov.data(), b.dcS.data()) == GPMPC_OK ? 0 : 1;
        if (!b.em_hess) return 1;       // bound by gp_b200_bind: no second derivatives of 'EM'
        return gpmpc_predict_em_hess(b.h, Nt, Z, b.sig.data(), 1, b.mean.data(), b.var.data(), b.cov.data(), b.jac.data(),
                                     b.dmS.data(), b.dcov.data(), b.dcS.data(), b.hess.data(), b.mSz.data(), b.mSS.data(),
                                     b.d2cov.data(), b.cSz.data(), b.cSS.data()) == GPMPC_OK ? 0 : 1;
    }
    if (mode == EVAL_HESS)
        return gpmpc_predict_hess(b.h, b.method, Nt, Z, ta ? b.sig.data() : nullptr, 1, b.mean.data(), b.var.data(),
                                  b.cov.data(), b.jac.data(), b.dvar.data(), b.dcov.data(), b.hess.data(), nullptr, nullptr,
                                  b.d2cov.data()) == GPMPC_OK ? 0 : 1;
    if (mode == EVAL_VALUE)
        return gpmpc_predict(b.h, b.method, Nt, Z, ta ? b.sig.data() : nullptr, 1, b.mean.data(), b.var.data(),
                             b.cov.data(), b.jac.data()) == GPMPC_OK ? 0 : 1;
    return gpmpc_predict_grad(b.h, b.method, Nt, Z, ta ? b.sig.data() : nullptr, 1, b.mean.data(), b.var.data(),
                              b.cov.data(), b.jac.data(), b.dvar.data(), b.dcov.data(), nullptr) == GPMPC_OK ? 0 : 1;
}
}  // namespace

namespace {
int bind(gpmpc_handle_t h, int method, int Nt, bool em_hess)
{
    std::lock_guard<std::mutex> lock(g_mtx);
    int N = 0, Nx = 0, Ny = 0;
    if (!h || Nt < 1 || (method != GPMPC_METHOD_ME && method != GPMPC_METHOD_TA && method != GPMPC_METHOD_EM)) return GPMPC_ERR_ARG;
    if (gpmpc_get_size(h, &N, &Nx, &Ny) != GPMPC_OK) return GPMPC_ERR_ARG;
    if (em_hess && Nx > 16) return GPMPC_ERR_ARG;
    Bound& b = g_b;
    b.h = h; b.method = method; b.Nt = Nt; b.Nx = Nx; b.Ny = Ny; b.em_hess = em_hess;
    b.sp_in[0] = dense_sp(Nx, Nt); b.sp_in[1] = dense_sp(Nx, (casadi_int)Nx * Nt);
    b.sp_out[0] = dense_sp(Ny, Nt); b.sp_out[1] = dense_sp(Ny, (casadi_int)Ny * Nt);
    b.sp_jac[0] = blockdiag_sp(Ny, Nx, Nt);
    b.sp_jac[1] = (method == GPMPC_METHOD_EM) ? blockdiag_sp(Ny, (casadi_int)Nx * Nx, Nt)
                                              : empty_sp((casadi_int)Ny * Nt, (casadi_int)Nx * Nx * Nt);
    b.sp_jac[2] = blockdiag_sp((casadi_int)Ny * Ny, Nx, Nt);
    b.sp_jac[3] = (method != GPMPC_METHOD_ME) ? blockdiag_sp((casadi_int)Ny * Ny, (casadi_int)Nx * Nx, Nt)
                                              : empty_sp((casadi_int)Ny * Ny * Nt, (casadi_int)Nx * Nx * Nt);
    b.sig.assign((size_t)Nt * Nx * Nx, 0.0);
    b.mean.assign((size_t)Nt * Ny, 0.0); b.var.assign((size_t)Nt * Ny, 0.0);
    b.cov.assign((size_t)Nt * Ny * Ny, 0.0); b.jac.assign((size_t)Nt * Ny * Nx, 0.0);
    b.dvar.assign((size_t)Nt * Ny * Nx, 0.0); b.dcov.assign((size_t)Nt * Ny * Ny * Nx, 0.0);
    b.hess.assign((size_t)Nt * Ny * Nx * Nx, 0.0); b.d2cov.assign((size_t)Nt * Ny * Ny * Nx * Nx, 0.0);
    if (method == GPMPC_METHOD_EM) { b.dmS.assign((size_t)Nt * Ny * Nx * Nx, 0.0); b.dcS.assign((size_t)Nt * Ny * Ny * Nx * Nx, 0.0); }
    else { b.dmS.clear(); b.dcS.clear(); }
    // jac_jac_gp_b200: numel of jac_gp_b200's outputs (rows) and inputs (columns)
    const casadi_int T = Nt, X = Nx, Y = Ny;
    const casadi_int n_out[4] = {Y * T * X * T, Y * T * X * X * T, Y * Y * T * X * T, Y * Y * T * X * X * T};
    const casadi_int n_in[4] = {X * T, X * X * T, Y * T, Y * Y * T};
    for (int o = 0; o < 4; ++o)
        for (int i = 0; i < 4; ++i) b.sp_jj[o * 4 + i] = empty_sp(n_out[o], n_in[i]);
    auto mean_z_rows = [&](casadi_int t) {                            // jac_mean_z (a + Y t, d + X t)
        std::vector<casadi_int> r;
        for (casadi_int d = 0; d < X; ++d)
            for (casadi_int a = 0; a < Y; ++a) r.push_back((a + Y * t) + Y * T * (d + X * t));
        return r;
    };
    auto cov_s_rows = [&](casadi_int t) {                             // jac_cov_sigma (a + Y b + Y^2 t, d + X e + X^2 t)
        std::vector<casadi_int> r;
        for (casadi_int e = 0; e < X; ++e)
            for (casadi_int d = 0; d < X; ++d)
                for (casadi_int bb = 0; bb < Y; ++bb)
                    for (casadi_int a = 0; a < Y; ++a) r.push_back((a + Y * bb + Y * Y * t) + Y * Y * T * (d + X * e + X * X * t));
        return r;
    };
    b.sp_jj[0] = nodes_sp(n_out[0], X, T, mean_z_rows);
    auto cov_z_rows = [&](casadi_int t) {                             // jac_cov_z (a + Y b + Y^2 t, e + X t)
        std::vector<casadi_int> r;
        for (casadi_int e = 0; e < X; ++e)
            for (casadi_int bb = 0; bb < Y; ++bb)
                for (casadi_int a = 0; a < Y; ++a) r.push_back((a + Y * bb + Y * Y * t) + Y * Y * T * (e + X * t));
        return r;
    };
    b.sp_jj[8] = nodes_sp(n_out[2], X, T, cov_z_rows);
    if (method == GPMPC_METHOD_TA) {
        b.sp_jj[9] = nodes_sp(n_out[2], X * X, T, cov_z_rows);
        b.sp_jj[12] = nodes_sp(n_out[3], X, T, cov_s_rows);
    }
    b.mSz.clear(); b.mSS.clear(); b.cSz.clear(); b.cSS.clear();
    if (em_hess) {
        const size_t t = Nt, x = Nx, y = Ny;
        b.mSz.assign(t * y * x * x * x, 0.0); b.mSS.assign(t * y * x * x * x * x, 0.0);
        b.cSz.assign(t * y * y * x * x * x, 0.0); b.cSS.assign(t * y * y * x * x * x * x, 0.0);
        auto mean_s_rows = [&](casadi_int t) {                        // jac_mean_sigma (a + Y t, d + X e + X^2 t)
            std::vector<casadi_int> r;
            for (casadi_int e = 0; e < X; ++e)
                for (casadi_int d = 0; d < X; ++d)
                    for (casadi_int a = 0; a < Y; ++a) r.push_back((a + Y * t) + Y * T * (d + X * e + X * X * t));
            return r;
        };
        b.sp_jj[1] = nodes_sp(n_out[0], X * X, T, mean_z_rows);
        b.sp_jj[4] = nodes_sp(n_out[1], X, T, mean_s_rows);
        b.sp_jj[5] = nodes_sp(n_out[1], X * X, T, mean_s_rows);
        b.sp_jj[9] = nodes_sp(n_out[2], X * X, T, cov_z_rows);
        b.sp_jj[12] = nodes_sp(n_out[3], X, T, cov_s_rows);
        b.sp_jj[13] = nodes_sp(n_out[3], X * X, T, cov_s_rows);
    }
    return GPMPC_OK;
}
}  // namespace

// Bind the (process-global) external to a factorised engine handle: method GPMPC_METHOD_ME / _TA / _EM,
// Nt shooting nodes per call.  Call again to re-bind (e.g. after a refit or another horizon).
extern "C" int gp_b200_bind(gpmpc_handle_t h, int method, int Nt) { return bind(h, method, Nt, false); }

// As gp_b200_bind(h, GPMPC_METHOD_EM, Nt), with jac_jac_gp_b200 served from gpmpc_predict_em_hess (Nx <= 16)
extern "C" int gp_b200_bind_em_hess(gpmpc_handle_t h, int Nt) { return bind(h, GPMPC_METHOD_EM, Nt, true); }

extern "C" void gp_b200_unbind(void)
{
    std::lock_guard<std::mutex> lock(g_mtx);
    g_b = Bound();
}

// ---- the function itself
extern "C" casadi_int gp_b200_n_in(void) { return 2; }
extern "C" casadi_int gp_b200_n_out(void) { return 2; }
extern "C" const char* gp_b200_name_in(casadi_int i) { return i == 0 ? "z" : (i == 1 ? "sigma" : nullptr); }
extern "C" const char* gp_b200_name_out(casadi_int i) { return i == 0 ? "mean" : (i == 1 ? "cov" : nullptr); }
extern "C" const casadi_int* gp_b200_sparsity_in(casadi_int i) { return (i >= 0 && i < 2 && g_b.h) ? g_b.sp_in[i].data() : nullptr; }
extern "C" const casadi_int* gp_b200_sparsity_out(casadi_int i) { return (i >= 0 && i < 2 && g_b.h) ? g_b.sp_out[i].data() : nullptr; }
extern "C" int gp_b200_work(casadi_int* sz_arg, casadi_int* sz_res, casadi_int* sz_iw, casadi_int* sz_w)
{
    if (sz_arg) *sz_arg = 2;
    if (sz_res) *sz_res = 2;
    if (sz_iw) *sz_iw = 0;
    if (sz_w) *sz_w = 0;
    return 0;
}
extern "C" void gp_b200_incref(void) { std::lock_guard<std::mutex> lock(g_mtx); ++g_b.refs; }
extern "C" void gp_b200_decref(void) { std::lock_guard<std::mutex> lock(g_mtx); --g_b.refs; }

extern "C" int gp_b200(const casadi_real** arg, casadi_real** res, casadi_int* iw, casadi_real* w, int mem)
{
    (void)iw; (void)w; (void)mem;
    std::lock_guard<std::mutex> lock(g_mtx);
    if (!arg || !res) return 1;
    if (eval(arg[0], arg[1], EVAL_VALUE)) return 1;
    const Bound& b = g_b;
    // (Nt,Ny) row-major == Ny x Nt column-major; each Ny x Ny block is written column-major
    // (element (a,b) at a + Ny*b) -- the blocks are symmetric only up to rounding
    if (res[0]) std::copy(b.mean.begin(), b.mean.end(), res[0]);
    if (res[1])
        for (int t = 0; t < b.Nt; ++t)
            for (int bb = 0; bb < b.Ny; ++bb)
                for (int a = 0; a < b.Ny; ++a)
                    res[1][((size_t)t * b.Ny + bb) * b.Ny + a] = b.cov[((size_t)t * b.Ny + a) * b.Ny + bb];
    return 0;
}

// ---- its Jacobian: inputs (z, sigma, mean, cov), outputs the four blocks in CCS nonzero order
extern "C" casadi_int jac_gp_b200_n_in(void) { return 4; }
extern "C" casadi_int jac_gp_b200_n_out(void) { return 4; }
extern "C" const char* jac_gp_b200_name_in(casadi_int i)
{
    static const char* n[] = {"z", "sigma", "out_mean", "out_cov"};
    return (i >= 0 && i < 4) ? n[i] : nullptr;
}
extern "C" const char* jac_gp_b200_name_out(casadi_int i)
{
    static const char* n[] = {"jac_mean_z", "jac_mean_sigma", "jac_cov_z", "jac_cov_sigma"};
    return (i >= 0 && i < 4) ? n[i] : nullptr;
}
extern "C" const casadi_int* jac_gp_b200_sparsity_in(casadi_int i)
{
    if (!g_b.h || i < 0 || i > 3) return nullptr;
    return i < 2 ? g_b.sp_in[i].data() : g_b.sp_out[i - 2].data();
}
extern "C" const casadi_int* jac_gp_b200_sparsity_out(casadi_int i) { return (i >= 0 && i < 4 && g_b.h) ? g_b.sp_jac[i].data() : nullptr; }
extern "C" int jac_gp_b200_work(casadi_int* sz_arg, casadi_int* sz_res, casadi_int* sz_iw, casadi_int* sz_w)
{
    if (sz_arg) *sz_arg = 4;
    if (sz_res) *sz_res = 4;
    if (sz_iw) *sz_iw = 0;
    if (sz_w) *sz_w = 0;
    return 0;
}

extern "C" int jac_gp_b200(const casadi_real** arg, casadi_real** res, casadi_int* iw, casadi_real* w, int mem)
{
    (void)iw; (void)w; (void)mem;
    std::lock_guard<std::mutex> lock(g_mtx);
    if (!arg || !res) return 1;
    if (eval(arg[0], arg[1], EVAL_GRAD)) return 1;
    const Bound& b = g_b;
    const int Nt = b.Nt, Nx = b.Nx, Ny = b.Ny;
    if (res[0])          // block t, column d, row a:  d mean_a / d z_d
        for (int t = 0; t < Nt; ++t)
            for (int d = 0; d < Nx; ++d)
                for (int a = 0; a < Ny; ++a) res[0][((size_t)t * Nx + d) * Ny + a] = b.jac[((size_t)t * Ny + a) * Nx + d];
    if (res[2])          // block t, column e, row a + Ny*b (column-major vec of the Ny x Ny block)
        for (int t = 0; t < Nt; ++t)
            for (int e = 0; e < Nx; ++e)
                for (int bb = 0; bb < Ny; ++bb)
                    for (int a = 0; a < Ny; ++a)
                        res[2][(((size_t)t * Nx + e) * Ny + bb) * Ny + a] = b.dcov[(((size_t)t * Ny + a) * Ny + bb) * Nx + e];
    if (b.method == GPMPC_METHOD_EM) {
        if (res[1])      // block t, column d + Nx*e (vec of Sigma), row a:  d mean_a / d Sigma[d][e]
            for (int t = 0; t < Nt; ++t)
                for (int e = 0; e < Nx; ++e)
                    for (int d = 0; d < Nx; ++d)
                        for (int a = 0; a < Ny; ++a)
                            res[1][(((size_t)t * Nx + e) * Nx + d) * Ny + a] = b.dmS[(((size_t)t * Ny + a) * Nx + d) * Nx + e];
        if (res[3])      // column d + Nx*e, row a + Ny*b:  d cov[a][b] / d Sigma[d][e]
            for (int t = 0; t < Nt; ++t)
                for (int e = 0; e < Nx; ++e)
                    for (int d = 0; d < Nx; ++d)
                        for (int bb = 0; bb < Ny; ++bb)
                            for (int a = 0; a < Ny; ++a)
                                res[3][((((size_t)t * Nx + e) * Nx + d) * Ny + bb) * Ny + a] =
                                    b.dcS[((((size_t)t * Ny + a) * Ny + bb) * Nx + d) * Nx + e];
        return 0;
    }
    if (res[3] && b.method == GPMPC_METHOD_TA)   // column d + Nx*e (vec of Sigma), row a + Ny*b:  J_a[d] J_b[e]
        for (int t = 0; t < Nt; ++t)
            for (int e = 0; e < Nx; ++e)
                for (int d = 0; d < Nx; ++d)
                    for (int bb = 0; bb < Ny; ++bb)
                        for (int a = 0; a < Ny; ++a)
                            res[3][((((size_t)t * Nx + e) * Nx + d) * Ny + bb) * Ny + a] =
                                b.jac[((size_t)t * Ny + a) * Nx + d] * b.jac[((size_t)t * Ny + bb) * Nx + e];
    return 0;
}

// ---- the Jacobian of jac_gp_b200 (second derivatives): inputs (z, sigma, mean, cov, and jac_gp_b200's four outputs),
// outputs jac_jac_<o>_<i> in CCS nonzero order
extern "C" casadi_int jac_jac_gp_b200_n_in(void) { return 8; }
extern "C" casadi_int jac_jac_gp_b200_n_out(void) { return 16; }
extern "C" const char* jac_jac_gp_b200_name_in(casadi_int i)
{
    static const char* n[] = {"z", "sigma", "out_mean", "out_cov", "out_jac_mean_z", "out_jac_mean_sigma", "out_jac_cov_z",
                              "out_jac_cov_sigma"};
    return (i >= 0 && i < 8) ? n[i] : nullptr;
}
extern "C" const char* jac_jac_gp_b200_name_out(casadi_int i)
{
    static const char* n[] = {
        "jac_jac_mean_z_z", "jac_jac_mean_z_sigma", "jac_jac_mean_z_out_mean", "jac_jac_mean_z_out_cov",
        "jac_jac_mean_sigma_z", "jac_jac_mean_sigma_sigma", "jac_jac_mean_sigma_out_mean", "jac_jac_mean_sigma_out_cov",
        "jac_jac_cov_z_z", "jac_jac_cov_z_sigma", "jac_jac_cov_z_out_mean", "jac_jac_cov_z_out_cov",
        "jac_jac_cov_sigma_z", "jac_jac_cov_sigma_sigma", "jac_jac_cov_sigma_out_mean", "jac_jac_cov_sigma_out_cov"};
    return (i >= 0 && i < 16) ? n[i] : nullptr;
}
extern "C" const casadi_int* jac_jac_gp_b200_sparsity_in(casadi_int i)
{
    if (!g_b.h || i < 0 || i > 7) return nullptr;
    return i < 2 ? g_b.sp_in[i].data() : i < 4 ? g_b.sp_out[i - 2].data() : g_b.sp_jac[i - 4].data();
}
extern "C" const casadi_int* jac_jac_gp_b200_sparsity_out(casadi_int i)
{
    return (i >= 0 && i < 16 && g_b.h) ? g_b.sp_jj[i].data() : nullptr;
}
extern "C" int jac_jac_gp_b200_work(casadi_int* sz_arg, casadi_int* sz_res, casadi_int* sz_iw, casadi_int* sz_w)
{
    if (sz_arg) *sz_arg = 8;
    if (sz_res) *sz_res = 16;
    if (sz_iw) *sz_iw = 0;
    if (sz_w) *sz_w = 0;
    return 0;
}
extern "C" void jac_jac_gp_b200_incref(void) { std::lock_guard<std::mutex> lock(g_mtx); ++g_b.refs; }
extern "C" void jac_jac_gp_b200_decref(void) { std::lock_guard<std::mutex> lock(g_mtx); --g_b.refs; }

extern "C" int jac_jac_gp_b200(const casadi_real** arg, casadi_real** res, casadi_int* iw, casadi_real* w, int mem)
{
    (void)iw; (void)w; (void)mem;
    std::lock_guard<std::mutex> lock(g_mtx);
    if (!arg || !res) return 1;
    if (eval(arg[0], arg[1], EVAL_HESS)) return 1;
    const Bound& b = g_b;
    const size_t Nt = b.Nt, Nx = b.Nx, Ny = b.Ny;
    const double* Hs = b.hess.data();
    const double* J = b.jac.data();
    auto H = [&](size_t t, size_t a, size_t d, size_t e) { return Hs[((t * Ny + a) * Nx + d) * Nx + e]; };
    auto Jv = [&](size_t t, size_t a, size_t d) { return J[(t * Ny + a) * Nx + d]; };
    // nonzeros in the order of the patterns built by gp_b200_bind: node, column, then rows ascending
    if (res[0]) {        // column e, rows (d, a):  d^2 mean_a / d z_d d z_e
        size_t k = 0;
        for (size_t t = 0; t < Nt; ++t)
            for (size_t e = 0; e < Nx; ++e)
                for (size_t d = 0; d < Nx; ++d)
                    for (size_t a = 0; a < Ny; ++a) res[0][k++] = H(t, a, d, e);
    }
    if (res[8]) {        // column f, rows (e, b, a):  d^2 cov[a][b] / d z_e d z_f
        size_t k = 0;
        for (size_t t = 0; t < Nt; ++t)
            for (size_t f = 0; f < Nx; ++f)
                for (size_t e = 0; e < Nx; ++e)
                    for (size_t bb = 0; bb < Ny; ++bb)
                        for (size_t a = 0; a < Ny; ++a) res[8][k++] = b.d2cov[((((t * Ny + a) * Ny + bb) * Nx + e) * Nx + f)];
    }
    if (b.method == GPMPC_METHOD_EM) {
        // column f (z_f) or f + Nx g (Sigma[f][g]); rows as the vec of the differentiated jac_gp_b200 output
        const size_t X = Nx, Y = Ny;
        auto mz = [&](size_t t, size_t a, size_t d, size_t e, size_t f) { return b.mSz[(((t * Y + a) * X + d) * X + e) * X + f]; };
        auto cz = [&](size_t t, size_t a, size_t bb, size_t d, size_t e, size_t f) { return b.cSz[((((t * Y + a) * Y + bb) * X + d) * X + e) * X + f]; };
        size_t k;
        if (res[1]) {    // d dmean_dz[a][d] / d Sigma[f][g] = d2mean_dSigma_dz[a][f][g][d]; rows (d, a)
            k = 0;
            for (size_t t = 0; t < Nt; ++t)
                for (size_t g = 0; g < X; ++g)
                    for (size_t f = 0; f < X; ++f)
                        for (size_t d = 0; d < X; ++d)
                            for (size_t a = 0; a < Y; ++a) res[1][k++] = mz(t, a, f, g, d);
        }
        if (res[4]) {    // d dmean_dSigma[a][d][e] / d z_f; rows (e, d, a)
            k = 0;
            for (size_t t = 0; t < Nt; ++t)
                for (size_t f = 0; f < X; ++f)
                    for (size_t e = 0; e < X; ++e)
                        for (size_t d = 0; d < X; ++d)
                            for (size_t a = 0; a < Y; ++a) res[4][k++] = mz(t, a, d, e, f);
        }
        if (res[5]) {    // d dmean_dSigma[a][d][e] / d Sigma[f][g]; rows (e, d, a)
            k = 0;
            for (size_t t = 0; t < Nt; ++t)
                for (size_t g = 0; g < X; ++g)
                    for (size_t f = 0; f < X; ++f)
                        for (size_t e = 0; e < X; ++e)
                            for (size_t d = 0; d < X; ++d)
                                for (size_t a = 0; a < Y; ++a) res[5][k++] = b.mSS[((((t * Y + a) * X + d) * X + e) * X + f) * X + g];
        }
        if (res[9]) {    // d dcov_dz[a][b][e] / d Sigma[f][g] = d2cov_dSigma_dz[a][b][f][g][e]; rows (e, b, a)
            k = 0;
            for (size_t t = 0; t < Nt; ++t)
                for (size_t g = 0; g < X; ++g)
                    for (size_t f = 0; f < X; ++f)
                        for (size_t e = 0; e < X; ++e)
                            for (size_t bb = 0; bb < Y; ++bb)
                                for (size_t a = 0; a < Y; ++a) res[9][k++] = cz(t, a, bb, f, g, e);
        }
        if (res[12]) {   // d dcov_dSigma[a][b][d][e] / d z_f; rows (e, d, b, a)
            k = 0;
            for (size_t t = 0; t < Nt; ++t)
                for (size_t f = 0; f < X; ++f)
                    for (size_t e = 0; e < X; ++e)
                        for (size_t d = 0; d < X; ++d)
                            for (size_t bb = 0; bb < Y; ++bb)
                                for (size_t a = 0; a < Y; ++a) res[12][k++] = cz(t, a, bb, d, e, f);
        }
        if (res[13]) {   // d dcov_dSigma[a][b][d][e] / d Sigma[f][g]; rows (e, d, b, a)
            k = 0;
            for (size_t t = 0; t < Nt; ++t)
                for (size_t g = 0; g < X; ++g)
                    for (size_t f = 0; f < X; ++f)
                        for (size_t e = 0; e < X; ++e)
                            for (size_t d = 0; d < X; ++d)
                                for (size_t bb = 0; bb < Y; ++bb)
                                    for (size_t a = 0; a < Y; ++a)
                                        res[13][k++] = b.cSS[(((((t * Y + a) * Y + bb) * X + d) * X + e) * X + f) * X + g];
        }
        return 0;
    }
    if (b.method != GPMPC_METHOD_TA) return 0;
    if (res[9]) {        // column d' + Nx e' (vec of Sigma), rows (e, b, a):  d^2 cov[a][b] / d z_e d Sigma[d'][e']
        size_t k = 0;
        for (size_t t = 0; t < Nt; ++t)
            for (size_t ep = 0; ep < Nx; ++ep)
                for (size_t dp = 0; dp < Nx; ++dp)
                    for (size_t e = 0; e < Nx; ++e)
                        for (size_t bb = 0; bb < Ny; ++bb)
                            for (size_t a = 0; a < Ny; ++a)
                                res[9][k++] = H(t, a, dp, e) * Jv(t, bb, ep) + Jv(t, a, dp) * H(t, bb, ep, e);
    }
    if (res[12]) {       // column f, rows (e, d, b, a) of d cov[a][b] / d Sigma[d][e]:  its derivative by z_f
        size_t k = 0;
        for (size_t t = 0; t < Nt; ++t)
            for (size_t f = 0; f < Nx; ++f)
                for (size_t e = 0; e < Nx; ++e)
                    for (size_t d = 0; d < Nx; ++d)
                        for (size_t bb = 0; bb < Ny; ++bb)
                            for (size_t a = 0; a < Ny; ++a)
                                res[12][k++] = H(t, a, d, f) * Jv(t, bb, e) + Jv(t, a, d) * H(t, bb, e, f);
    }
    return 0;
}
