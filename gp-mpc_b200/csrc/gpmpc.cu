// libgpmpc.so -- host side of the C ABI declared in include/gpmpc.h.
// One handle = one GPU = one CUDA stream.  No CPU fallback exists in this library.
#include "../../include/gpmpc.h"

#include <dlfcn.h>
#include <limits.h>
#include <math.h>
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <array>
#include <cmath>
#include <functional>
#include <map>
#include <memory>
#include <type_traits>
#include <vector>

#include <nvtx3/nvToolsExt.h>

#include "common.cuh"
#include "gemm_dmma.cuh"
#include "predict_streamk.cuh"
#include "kernels.cuh"

#define GPMPC_VERSION 100
#define HB 64                 // test points per predict pass (rows of the KS^T operand)
#define NX_MAX 32
#define PSK_MAX_CTAS 2048
#define MAX_DEPTH 12           // recursion depth bound: 128 * 2^12 rows
#define LOOKAHEAD_MIN_ROWS 1024   // potrf_inv_rec defers part of a trailing update only on blocks at least this tall

// ------------------------------------------------------------------------------------
// minimal NCCL surface, bound at run time with dlopen (no link-time dependency)
// ------------------------------------------------------------------------------------
typedef struct { char internal[128]; } nccl_uid_t;
typedef void* nccl_comm_t;
struct NcclApi {
    void* lib = nullptr;
    int (*GetUniqueId)(nccl_uid_t*) = nullptr;
    int (*CommInitRank)(nccl_comm_t*, int, nccl_uid_t, int) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, nccl_comm_t, cudaStream_t) = nullptr;
    int (*CommDestroy)(nccl_comm_t) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
};
static NcclApi g_nccl;
static char g_create_err[512] = "";

static bool nccl_load(char* err, size_t errn)
{
    if (g_nccl.lib) return true;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
        g_nccl.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
        if (g_nccl.lib) break;
    }
    if (!g_nccl.lib) { snprintf(err, errn, "dlopen(libnccl.so.2) failed: %s", dlerror()); return false; }
    g_nccl.GetUniqueId = (int (*)(nccl_uid_t*))dlsym(g_nccl.lib, "ncclGetUniqueId");
    g_nccl.CommInitRank = (int (*)(nccl_comm_t*, int, nccl_uid_t, int))dlsym(g_nccl.lib, "ncclCommInitRank");
    g_nccl.AllGather = (int (*)(const void*, void*, size_t, int, nccl_comm_t, cudaStream_t))dlsym(g_nccl.lib, "ncclAllGather");
    g_nccl.CommDestroy = (int (*)(nccl_comm_t))dlsym(g_nccl.lib, "ncclCommDestroy");
    g_nccl.GetErrorString = (const char* (*)(int))dlsym(g_nccl.lib, "ncclGetErrorString");
    if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.AllGather || !g_nccl.CommDestroy) {
        snprintf(err, errn, "libnccl is missing required symbols");
        g_nccl.lib = nullptr;
        return false;
    }
    return true;
}

// ------------------------------------------------------------------------------------
// One device allocation of `cap` elements, freed with its owner.  It converts to its pointer, so kernels and copies take
// it as they take a raw pointer.
template <typename T>
struct DevBuf {
    T* p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { cudaFree(p); }
    operator T*() const { return p; }
    int ensure(gpmpc_handle_t h, long long count, const char* name);
    void release() { cudaFree(p); p = nullptr; cap = 0; }     // the caller has drained the streams that use it
};

// 'EM' derivative records of total degree D (2: gpmpc_predict_em_grad, 4: gpmpc_predict_em_hess): the unique monomials of
// degree <= D in Nx variables (by degree, then lexicographic over sorted index tuples), the index of every (unsorted)
// k-tuple (mid, k <= D), and the record entries (owner monomial, feature of degree <= D/2) with total degree <= D
struct EmTables {
    int Nx = 0, D = 0, nf = 0, nent = 0;
    std::vector<int> mono, ent, entpos, deg;
    std::vector<int> mid[5];
    std::vector<int> dev;                  // the device copy's layout: [mono | ent | mid (orders 0..D back to back) | entpos]
    const int* uploaded_to = nullptr;      // the device buffer dev was copied to
    EmTables(int nx, int d) : Nx(nx), D(d)
    {
        std::map<std::array<int, 4>, int> idx;
        for (int k = 0; k <= D; ++k) {
            std::array<int, 4> t = {-1, -1, -1, -1};
            std::function<void(int, int)> rec = [&](int s, int lo) {
                if (s == k) {
                    idx[t] = (int)deg.size();
                    for (int q = 0; q < 4; ++q) mono.push_back(t[q]);
                    deg.push_back(k);
                    return;
                }
                for (int d = lo; d < Nx; ++d) { t[s] = d; rec(s + 1, d); }
                t[s] = -1;
            };
            rec(0, 0);
            if (k == D / 2) nf = (int)deg.size();
            long long nk = 1;
            for (int q = 0; q < k; ++q) nk *= Nx;
            mid[k].resize(nk);
            for (long long f = 0; f < nk; ++f) {
                std::array<int, 4> u = {-1, -1, -1, -1};
                long long r = f;
                for (int q = k - 1; q >= 0; --q) { u[q] = (int)(r % Nx); r /= Nx; }
                std::sort(u.begin(), u.begin() + k);
                mid[k][f] = idx[u];
            }
        }
        const int nm = (int)deg.size();
        entpos.assign((size_t)nm * nf, -1);
        for (int m = 0; m < nm; ++m)
            for (int f = 0; f < nf; ++f)
                if (deg[m] + deg[f] <= D) { entpos[(size_t)m * nf + f] = nent++; ent.push_back(m); ent.push_back(f); }
        dev = mono;
        dev.insert(dev.end(), ent.begin(), ent.end());
        for (int k = 0; k <= D; ++k) dev.insert(dev.end(), mid[k].begin(), mid[k].end());
        dev.insert(dev.end(), entpos.begin(), entpos.end());
    }
    const int* d_mid(const int* base) const { return base + mono.size() + ent.size(); }
    const int* d_entpos(const int* base) const { return d_mid(base) + mid[0].size() + mid[1].size() + mid[2].size() + mid[3].size() + mid[4].size(); }
    // records per point: [mean a | cross pair p, owner rows / columns | trace remainder a | trace backbone a | (D = 2) backbone Gram a]
    int nrec(int Ny) const { return (D == 2 ? 4 : 3) * Ny + Ny * (Ny + 1); }
};

// One 'EM' record set per D: its tables (built once, they depend on Nx only, and uploaded to idx once), the block
// partials, the summed records of every point and the backbone rows [e o features | their L^-1 | K^-1 products]
struct EmRecords {
    std::unique_ptr<EmTables> tb;
    DevBuf<double> part, rec, bb;
    DevBuf<int> idx;
};

struct gpmpc_handle_s {
    int N = 0, Nx = 0, Ny = 0, a0 = 0, nloc = 0, Npad = 0, device = 0;
    int nloc_max = 0;                 // ceil(Ny / world): slots per rank in the gather buffer
    cudaStream_t st = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    // factorisation overlap: step 5a of every recursion depth runs on its own side stream
    cudaStream_t sideSt[MAX_DEPTH] = {nullptr}; cudaEvent_t evA[MAX_DEPTH] = {nullptr}, evB[MAX_DEPTH] = {nullptr}, evT[MAX_DEPTH] = {nullptr}, evS[MAX_DEPTH] = {nullptr};
    long long w2off[MAX_DEPTH + 1] = {0};
    // model
    DevBuf<double> dXT, dMu, dY, dHyp, dJit, dHypTmp;   // dJit: the jitter of each K build (scratch)
    DevBuf<double> dFacJit;           // the jitter on the diagonal of the K each output's current factor factorises
    DevBuf<double> dL, dLi, dW1, dW2;
    DevBuf<double> dAlpha, dTmp, dRes;
    DevBuf<int> dInfo;
    // predict
    DevBuf<double> dKST, dPart, dPMJ, dSQ, dV, dR, dR2;
    // L^-1 of every output in the product's k-step order (panel_pack_kernel, lazy) and, per output, the first L^-1 row
    // whose panel copy may be stale (Npad: current).  Every writer of dLi lowers it; panel_refresh repacks from there.
    DevBuf<double> dLiP; std::vector<int> panel_row;
    DevBuf<unsigned int> dCnt;        // stream-K counters: [nloc*nt tile | nloc output | 1 done], self-cleaning
    int psk_ctas = 0, opt_predict_ctas = 0;   // persistent grid of the predict product (PSK_CTAS_PER_SM per SM)
    DevBuf<double> dCovV, dCovOut;    // GP.covar scratch pool; dCovV also holds the greedy selection's pool V
    DevBuf<double> dGrD;              // gpmpc_append_greedy: [var (nloc, n) | Xc (n, Nx) | Yc (n, Ny) | score (n_new)]
    DevBuf<int> dGrI;                 //                      [active (n) | picked (n_new) | stop]
    DevBuf<double> dRm;               // gpmpc_remove: [p | d | g] (Npad each) per owned output
    // predict_grad: U = Linv^T per output (lazy), beta rows, partial sums, per-batch derivative slabs
    DevBuf<double> dUall, dBeta, dPDV, dPH, dGradOut; bool u_valid = false;
    // predict_hess: derivative rows d ks / dz and their L^-1 products (lazy), block partials, per-batch second-derivative slabs
    DevBuf<double> dDR, dVD, dPG, dPB2, dPM3, dHessOut;
    DevBuf<double> dG;
    double *dZ = nullptr, *dSigma = nullptr, *dMean = nullptr, *dVar = nullptr, *dJ = nullptr, *dCov = nullptr;   // in dIn / dOut
    DevBuf<double> dRoll;             // gpmpc_rollout_batch: [Z | Sigma | U | scale | K | x_ref | uscale | means | vars | cov]
    DevBuf<double> dRollTg;           // gpmpc_rollout_batch_grad, _em_grad: [dZ | dSigma ('TA', 'EM') | dmeans | dvars | 'EM' blocks]
    DevBuf<double> dSmV;              // gpmpc_rollout_sample: V rows of every step (nloc, Nt, B, Npad)
    DevBuf<double> dSmp;              //   [eps | xi | U | scale | K | x_ref | uscale | Z (Nt,B,Nx) | samples | kept | m | R]
    DevBuf<double> dSmB;              // gpmpc_rollout_sample_grad: beta rows of every step (nloc, Nt, B, Npad)
    DevBuf<double> dSmTg;             //   [G (nloc,B,Nt,2,Nx) | dR (nloc,B,P,Nt,Nt) | dz (Nt,B,P,Nx) | dsamples (Nt,B,Ny,P)]
    DevBuf<double> dIn, dOut;         // [Z | Sigma] and [mean | var | J | cov] slabs: one H2D + one D2H per host call
    int Hcap = 0;                     // test points the slab layout behind dZ .. dCov holds (0: not laid out)
    double* hPinned = nullptr; double* dPinnedAlias = nullptr; size_t hPinnedBytes = 0;
    // K^-1 and gradient scratch (ensure_kinv_scratch; dGrad: the gradient of one output)
    DevBuf<double> dU, dKinv, dGradPart, dGrad;
    DevBuf<double> dLoo;              // gpmpc_loo / gpmpc_loo_nlpp: [mean | var | nlpp | c partials | sw | u | b | tmp | 0]
    // gpmpc_nlml_batch: per entry of a pass its own L, Li slabs and recursion workspaces (nlml_batch_scratch)
    DevBuf<double> dNbL, dNbLi, dNbW1, dNbW2, dNbV; DevBuf<int> dNbInfo;
    int opt_nlml_batch_max = 0;       // entries per gpmpc_nlml_batch pass (0: all)
    bool has_data = false, has_hyper = false, factorized = false;
    // EM scratch
    DevBuf<double> dEmTr, dEMP, dEmE, dEmF, dEmW, dEmIJ;
    DevBuf<double> dEmMeanPart, dEmPart, dEmLQ, dEmVec, dEmE2, dEmF2;
    // EM derivatives: full symmetric K^-1 per output (lazy, one per factorisation), the records of D = 2 and D = 4
    DevBuf<double> dEmKinv; bool em_kinv_valid = false;
    EmRecords em_rec[2];
    // EM second derivatives: per-pair matrices, v-moments, mean derivatives, finish scratch and output slabs
    DevBuf<double> dEmHEHP, dEmHMU, dEmHD, dEmHScr, dEmHOut;
    std::vector<double> hyper;        // (nloc, Nx+2)
    // host copy of X (N, Nx) row-major, kept by set_data, append, append_greedy and remove: the K build's centre dMu is
    // recomputed from it (mu_stale) before the next K build, so appends and removals never leave K centred on an old mean
    std::vector<double> hX; bool mu_stale = false;
    std::vector<double> logdet, yalpha;
    std::vector<int> jitter_used;
    int sms = 132;                    // multiprocessors of the device (queried in create)
    int opt_refine = 0, opt_small_tiles = 528;   // 128x64-tile count below which 64x32 tiles are used (4 per SM)
    int opt_em_points = 0;            // points per batched 'EM' forward (0: the scratch budget EM_CHUNK_BYTES decides)
    double ut_alpha = 1.0, ut_beta = 0.0, ut_kappa = 0.0;   // 'UT' parameters (options "ut_alpha", "ut_beta", "ut_kappa")
    DevBuf<double> dUt;               // 'UT' pass: [sigma points (Hs,Nx) | 'ME' means (Hs,Ny) | variances (Hs,Ny) | J (Hs,Ny,Nx)]
    // comm
    nccl_comm_t comm = nullptr; int rank = 0, world = 1;
    // peer (CUDA IPC) exchange: [flags: 2*MAXW u64][gather buffer parity 0][parity 1]
    DevBuf<double> dPeerBlock; long long peerGsz = 0; int peerHcap = 0; bool peer_ready = false;
    double* peerBase[GPMPC_MAXW] = {nullptr}; bool peerOpened[GPMPC_MAXW] = {false};
    int* dPeerStatus = nullptr; int* hPeerStatus = nullptr;
    unsigned long long peer_step = 0; int opt_peer = 1; double opt_peer_timeout_s = 60.0; int clock_khz = 1980000;
    char err[512] = "";
};

static void set_error(gpmpc_handle_t h, const char* fmt, ...)
{
    va_list ap; va_start(ap, fmt);
    vsnprintf(h ? h->err : g_create_err, 512, fmt, ap);
    va_end(ap);
}

// Grow to at least `count` elements, zero-filled on the handle's stream (the stream-K counters, the zero upper tiles of
// Li and the zero rows of dDR rely on it).  The old buffer is freed only once the stream has drained.  On failure the
// buffer is left empty and the error names it.
template <typename T>
int DevBuf<T>::ensure(gpmpc_handle_t h, long long count, const char* name)
{
    if ((size_t)count <= cap) return GPMPC_OK;
    if (p) {
        CUDA_TRY(cudaStreamSynchronize(h->st));
        cudaFree(p);
        p = nullptr; cap = 0;
    }
    const size_t bytes = (size_t)count * sizeof(T);
    cudaError_t e = cudaMalloc((void**)&p, bytes);
    if (e != cudaSuccess) {
        p = nullptr;
        set_error(h, "cudaMalloc(%s, %zu bytes) failed: %s", name, bytes, cudaGetErrorString(e));
        return GPMPC_ERR_CUDA;
    }
    e = cudaMemsetAsync(p, 0, bytes, h->st);
    if (e != cudaSuccess) { cudaFree(p); p = nullptr; }
    CUDA_TRY(e);
    cap = (size_t)count;
    return GPMPC_OK;
}

// buf.ensure(count), returning its error code; the message names the buffer as written at the call
#define ENSURE(buf, count)                                          \
    do {                                                            \
        const int _rc = (buf).ensure(h, (long long)(count), #buf);  \
        if (_rc) return _rc;                                        \
    } while (0)

// NVTX range per phase (header-only nvtx3: a no-op unless a profiler injects the library)
struct NvtxRange {
    explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
};

static inline long long slab(gpmpc_handle_t h) { return (long long)h->Npad * h->Npad; }
static inline long long w2slab(gpmpc_handle_t h) { return h->w2off[MAX_DEPTH]; }   // all depths, one batch entry

// L^-1 rows from `row` on of local output al (every output: al < 0) were written: their panel copy is stale
static void panel_stale(gpmpc_handle_t h, int al, int row)
{
    for (int a = 0; a < h->nloc; ++a)
        if (al < 0 || a == al) h->panel_row[a] = std::min(h->panel_row[a], std::max(row, 0));
}

// f(std::integral_constant<int, NXP>) with NXP = 8, 16 or 32 >= Nx: the register-array extent of the kernels that keep
// one Nx-vector per thread (nlml gradient, EM, predict derivatives)
template <typename F>
static cudaError_t nxp_dispatch(int Nx, F&& f)
{
    if (Nx <= 8) return f(std::integral_constant<int, 8>());
    if (Nx <= 16) return f(std::integral_constant<int, 16>());
    return f(std::integral_constant<int, 32>());
}

// ------------------------------------------------------------------------------------
// GEMM helpers (all operands live in slabs with leading dimension ld)
// ------------------------------------------------------------------------------------
// Callers describe the problem in 128x128 tiles (mt, nt); the launch re-tiles it.  Tile-granular TMA
// (tensor maps, 128B swizzle) serves the NT products that fill the GPU for at least two waves; everything
// else (NN products, small launches) takes the cp.async kernel.  The feed is chosen from the tiles of `sel_batch` slabs
// while the launch covers `batch`: the feeds round differently, so a caller whose slabs must get the bits of a lone slab
// passes sel_batch = 1.
static cudaError_t gemm128(gpmpc_handle_t h, cudaStream_t st, bool bt, const GemmParams& p, int batch, int sel_batch)
{
    const long long tiles = (long long)sel_batch * (p.lower ? (long long)p.mt * (p.mt + 1) : 2LL * p.mt * p.nt);
    GemmParams q = p;
    if (tiles < h->opt_small_tiles) {
        // deep recursion levels: a handful of 128x64 tiles cannot occupy 132 SMs; 64x32 tiles
        // (8x more CTAs, 4 CTAs/SM) cut the latency of these critical-path launches
        q.mt = p.mt * 2; q.nt = p.nt * 4;
        return bt ? gemm_launch<64, 32, 2, 2, true, 3, 4>(q, batch, st)
                  : gemm_launch<64, 32, 2, 2, false, 3, 4>(q, batch, st);
    }
    q.nt = p.nt * 2;
    if (bt && tiles >= 4LL * h->sms) {
        if (p.sA != 0 || batch == 1) return gemm_tmap_launch<128, 64, 2, 2, 4, 2>(q, batch, st);
        // a tensor map cannot step a zero batch stride: one launch per slab (each already fills four waves)
        for (int z = 0; z < batch; ++z) {
            GemmParams r = q;
            r.B += z * p.sB; r.C += z * p.sC;
            if (r.Cin) r.Cin += z * p.sCin;
            const cudaError_t e = gemm_tmap_launch<128, 64, 2, 2, 4, 2>(r, 1, st);
            if (e != cudaSuccess) return e;
        }
        return cudaSuccess;
    }
    return bt ? gemm_launch<128, 64, 2, 2, true, 3, 2>(q, batch, st)
              : gemm_launch<128, 64, 2, 2, false, 3, 2>(q, batch, st);
}

// Recursive blocked Cholesky + triangular inverse on the diagonal block
// [off, off+n) of every slab in the batch:  A -> L (in place, lower), Li -> L^-1.
//   1. (L11, Li11) = rec(A11)
//   2. L21 = A21 Li11^T                 (explicit-inverse panel solve, DMMA GEMM NT)
//   3. A22 -= L21 L21^T                 (trailing SYRK update, DMMA GEMM NT, lower tiles)
//   4. (L22, Li22) = rec(A22)
//   5. Li21 = -Li22 (L21 Li11)          (two DMMA GEMMs NN)
// All flops except the 128x128 leaves run on the fp64 tensor pipe.  Workspace: W1b, W2b (w2slab per batch entry); every
// GEMM picks its feed as for sel_batch slabs (gemm128).
static int potrf_inv_rec(gpmpc_handle_t h, double* A, double* Li, long long sA, long long sLi,
                         int* dInfo, int off, int n, int batch, int sel_batch, double* W1b, double* W2b, int depth = 0,
                         cudaEvent_t pend = nullptr)
{
    const int ld = h->Npad;
    if (n <= LEAF_N) {
        if (pend) CUDA_TRY(cudaStreamWaitEvent(h->st, pend, 0));
        CUDA_TRY(smem_opt_in<leaf_potrf_trtri_kernel>(LEAF_SMEM_DOUBLES * 8));
        leaf_potrf_trtri_kernel<<<batch, 256, LEAF_SMEM_DOUBLES * 8, h->st>>>(A + (long long)off * ld + off, ld, sA,
                                                                           Li + (long long)off * ld + off, ld, sLi, dInfo, off);
        CUDA_TRY(cudaGetLastError());
        return GPMPC_OK;
    }
    const int nb = n / GPMPC_TILE;
    const int n1 = (nb / 2) * GPMPC_TILE, n2 = n - n1;
    int rc = potrf_inv_rec(h, A, Li, sA, sLi, dInfo, off, n1, batch, sel_batch, W1b, W2b, depth + 1, nullptr);
    if (rc) return rc;
    // the caller deferred part of its trailing update to its side stream (look-ahead, see below): everything outside this
    // sub-problem's leading n1 x n1 block is only valid once that work has finished
    if (pend) CUDA_TRY(cudaStreamWaitEvent(h->st, pend, 0));
    double* A21 = A + (long long)(off + n1) * ld + off;
    double* A22 = A + (long long)(off + n1) * ld + off + n1;
    double* Li11 = Li + (long long)off * ld + off;
    double* Li21 = Li + (long long)(off + n1) * ld + off;
    double* Li22 = Li + (long long)(off + n1) * ld + off + n1;
    double* W1 = W1b + h->w2off[depth];                    // one region per depth (deferred work of different depths is in flight together)
    double* W2 = W2b + h->w2off[depth];
    const long long sW = w2slab(h), sW2 = w2slab(h);
    const bool ovl = depth < MAX_DEPTH;
    cudaStream_t side = ovl ? h->sideSt[depth] : h->st;
    // LOOK-AHEAD.  rec(A22) starts with the leading h2 x h2 block of A22 (its own first half) and does not touch the rest
    // before its panel step.  So only the top h2 rows of the panel and the (1,1) block of the trailing update stay on the
    // critical stream; the bottom panel rows, the (2,1) and (2,2) blocks of the update and W2 run on this depth's
    // low-priority side stream beside the latency-bound recursion into A22_11 (leaves, small products) and are joined by
    // the child right before its panel step (`pend`).  On-chain share of a level's flops: 0.44 instead of 0.75.
    const int h2 = ((n2 / GPMPC_TILE) / 2) * GPMPC_TILE;
    const bool split = ovl && h2 >= GPMPC_TILE && n >= LOOKAHEAD_MIN_ROWS;
    GemmParams p;
    auto panel = [&](cudaStream_t st, int r0, int rows) -> cudaError_t {     // W1[r0:r0+rows] = A21[r0:..] Li11^T ; L21 rows <- W1 rows
        GemmParams q;
        memset(&q, 0, sizeof(q));
        q.A = A21 + (long long)r0 * ld; q.lda = ld; q.sA = sA;
        q.B = Li11; q.ldb = ld; q.sB = sLi;                                   // B[j][k] = Li11[j][k] != 0 only for k <= j
        q.C = W1 + (long long)r0 * n1; q.ldc = n1; q.sC = sW;
        q.mt = rows / 128; q.nt = n1 / 128; q.K = n1; q.alpha = 1.0; q.beta = 0.0; q.kflags = GEMM_KJ_LE;
        cudaError_t e = gemm128(h, st, true, q, batch, sel_batch);
        if (e != cudaSuccess) return e;
        dim3 g(std::max(1, std::min(64, n1 / 2 / 128)), std::min(rows, 4096), batch);
        copy2d_kernel<<<g, 128, 0, st>>>(W1 + (long long)r0 * n1, n1, sW, A21 + (long long)r0 * ld, ld, sA, rows, n1);
        return cudaGetLastError();
    };
    auto update = [&](cudaStream_t st, int r0, int rows, int c0, int cols, int lower) -> cudaError_t {   // A22[r0.., c0..] -= W1[r0..] W1[c0..]^T
        GemmParams q;
        memset(&q, 0, sizeof(q));
        q.A = W1 + (long long)r0 * n1; q.lda = n1; q.sA = sW;
        q.B = W1 + (long long)c0 * n1; q.ldb = n1; q.sB = sW;
        q.C = A22 + (long long)r0 * ld + c0; q.ldc = ld; q.sC = sA; q.Cin = q.C; q.ldcin = ld; q.sCin = sA;
        q.mt = rows / 128; q.nt = cols / 128; q.K = n1; q.alpha = -1.0; q.beta = 1.0; q.lower = lower;
        return gemm128(h, st, true, q, batch, sel_batch);
    };
    if (ovl) {
        CUDA_TRY(cudaEventRecord(h->evA[depth], h->st));
        CUDA_TRY(cudaStreamWaitEvent(side, h->evA[depth], 0));
    }
    if (split) {
        CUDA_TRY(panel(h->st, 0, h2));                                        // 2. top rows (critical)
        CUDA_TRY(cudaEventRecord(h->evT[depth], h->st));
        CUDA_TRY(update(h->st, 0, h2, 0, h2, 1));                             // 3. (1,1) block (critical)
        CUDA_TRY(panel(side, h2, n2 - h2));                                   // 2. bottom rows (side)
        CUDA_TRY(cudaStreamWaitEvent(side, h->evT[depth], 0));                //    needs W1's top rows
        CUDA_TRY(update(side, h2, n2 - h2, 0, h2, 0));                        // 3. (2,1) block
        CUDA_TRY(update(side, h2, n2 - h2, h2, n2 - h2, 1));                  // 3. (2,2) block
        CUDA_TRY(cudaEventRecord(h->evS[depth], side));
    } else {
        CUDA_TRY(panel(h->st, 0, n2));                                        // 2. W1 = A21 Li11^T, L21 <- W1
        CUDA_TRY(update(h->st, 0, n2, 0, n2, 1));                             // 3. A22 -= W1 W1^T (lower tiles)
        if (ovl) {       // the side stream must not start 5a before L21 is in place
            CUDA_TRY(cudaEventRecord(h->evT[depth], h->st));
            CUDA_TRY(cudaStreamWaitEvent(side, h->evT[depth], 0));
        }
    }
    // 5a. W2 = L21 * Li11     Bop[k][j] = Li11[k][j] != 0 only for k >= j.  Independent of step 4: on the side stream it
    //     fills the SMs the recursion into A22 leaves idle.  L21 is read from the matrix; W2 has one region per depth.
    memset(&p, 0, sizeof(p));
    p.A = A21; p.lda = ld; p.sA = sA;
    p.B = Li11; p.ldb = ld; p.sB = sLi;
    p.C = W2; p.ldc = n1; p.sC = sW2;
    p.mt = n2 / 128; p.nt = n1 / 128; p.K = n1; p.alpha = 1.0; p.beta = 0.0; p.kflags = GEMM_KJ_GE;
    if (ovl) {
        CUDA_TRY(gemm128(h, side, false, p, batch, sel_batch));
        CUDA_TRY(cudaEventRecord(h->evB[depth], side));
    }
    // 4.
    rc = potrf_inv_rec(h, A, Li, sA, sLi, dInfo, off + n1, n2, batch, sel_batch, W1b, W2b, depth + 1,
                       split ? h->evS[depth] : nullptr);
    if (rc) return rc;
    if (ovl) CUDA_TRY(cudaStreamWaitEvent(h->st, h->evB[depth], 0));
    else CUDA_TRY(gemm128(h, h->st, false, p, batch, sel_batch));
    // 5b. Li21 = -Li22 * W2   A[i][k] = Li22[i][k] != 0 only for k <= i
    memset(&p, 0, sizeof(p));
    p.A = Li22; p.lda = ld; p.sA = sLi;
    p.B = W2; p.ldb = n1; p.sB = sW2;
    p.C = Li21; p.ldc = ld; p.sC = sLi;
    p.mt = n2 / 128; p.nt = n1 / 128; p.K = n2; p.alpha = -1.0; p.beta = 0.0; p.kflags = GEMM_KI_LE;
    CUDA_TRY(gemm128(h, h->st, false, p, batch, sel_batch));
    return GPMPC_OK;
}

// K(theta) for `batch` consecutive outputs: hyper rows at dHyp (stride Nx+2), jitter at dJit,
// output slabs at K (stride slab).  full = 1 writes the whole square, 0 the lower triangle.
static int launch_kbuild(gpmpc_handle_t h, const double* dHyp, const double* dJit, double* K, int batch, int full)
{
    if (h->mu_stale) {
        // column means of the current X: the K build centres its inputs (translation invariant), and its cancellation
        // error grows with |u|^2 measured from that centre.  Same order as every earlier value, so a handle given its
        // X by set_data and one that reached the same X by appends and removals build the same K bit for bit.
        const int N = h->N, Nx = h->Nx;
        double mu[NX_MAX] = {0.0};
        for (int d = 0; d < Nx; ++d) {
            double sacc = 0.0;
            for (int i = 0; i < N; ++i) sacc += h->hX[(size_t)i * Nx + d];
            mu[d] = sacc / N;
        }
        CUDA_TRY(cudaMemcpyAsync(h->dMu, mu, NX_MAX * 8, cudaMemcpyHostToDevice, h->st));
        h->mu_stale = false;
    }
    const int KD = (h->Nx + 3) & ~3, S = ((KD >> 2) & 1) ? KD : KD + 4;
    const int smem = (2 * KB2_TILE * S + 2 * KB2_TILE + 256) * 8;
    const int smem_max = (2 * KB2_TILE * 36 + 2 * KB2_TILE + 256) * 8;   // S at NX_MAX
    CUDA_TRY(smem_opt_in<kbuild_dmma_kernel<true>>(smem_max));
    CUDA_TRY(smem_opt_in<kbuild_dmma_kernel<false>>(smem_max));
    const int T = h->Npad / KB2_TILE;
    dim3 grid(T * (T + 1) / 2, 1, batch);
    if (full)
        kbuild_dmma_kernel<true><<<grid, 256, smem, h->st>>>(h->dXT, h->Npad, h->N, h->Nx, h->dMu, dHyp, h->Nx + 2, dJit, K, h->Npad, slab(h));
    else
        kbuild_dmma_kernel<false><<<grid, 256, smem, h->st>>>(h->dXT, h->Npad, h->N, h->Nx, h->dMu, dHyp, h->Nx + 2, dJit, K, h->Npad, slab(h));
    CUDA_TRY(cudaGetLastError());
    return GPMPC_OK;
}

// c factor entries, entry s at: the hyper row hyp + s (Nx+2), the jitter jit[s] and the pivot info info[s] of its K build
// and recursion; its L and L^-1 slabs L, Li + s slab and recursion workspaces W1, W2 + s w2slab (W1 also takes the alpha
// partials); its target y + s sy; tmp, alpha + s Npad and res + 2 s (log det, y . alpha)
struct FactorSet {
    int c;
    double *hyp, *jit; int* info;
    double *L, *Li, *W1, *W2;
    const double* y; long long sy;
    double *tmp, *alpha, *res;
};

// the owned outputs al .. al + c - 1 in the model's own slots
static FactorSet model_entries(gpmpc_handle_t h, int al, int c)
{
    const long long np = h->Npad;
    return {c, h->dHyp + al * (h->Nx + 2LL), h->dJit + al, h->dInfo + al, h->dL + al * slab(h), h->dLi + al * slab(h),
            h->dW1 + al * w2slab(h), h->dW2 + al * w2slab(h), h->dY + al * np, np, h->dTmp + al * np,
            h->dAlpha + al * np, h->dRes + 2LL * al};
}

// alpha = Li^T (Li y), log det K and y . alpha of the entries, from their factor slabs
static int alpha_pass(gpmpc_handle_t h, const FactorSet& e)
{
    const int n = h->Npad;
    dim3 g1((n + 7) / 8, 1, e.c);
    trmv_lower_kernel<<<g1, 256, 0, h->st>>>(e.Li, n, slab(h), e.y, e.sy, e.tmp, n, n);
    CUDA_TRY(cudaGetLastError());
    // alpha = Li^T tmp in row chunks (partials in a W1 workspace, free outside the recursion), then
    // one pass that sums the partials, takes log det and y . alpha
    const int nch = (n + TRT_ROWS - 1) / TRT_ROWS;
    dim3 g2(n / 32, nch, e.c);
    trmv_lower_T_part_kernel<<<g2, 256, 0, h->st>>>(e.Li, n, slab(h), e.tmp, n, e.W1, w2slab(h), n);
    CUDA_TRY(cudaGetLastError());
    alpha_logdet_kernel<<<e.c, 1024, 0, h->st>>>(e.W1, w2slab(h), nch, e.L, n, slab(h), e.y, e.sy, e.alpha, n, n, e.res);
    CUDA_TRY(cudaGetLastError());
    return GPMPC_OK;
}

// K(theta) -> L, Li of the entries with the reference's single jitter retry (optimize.py:483-488): one K build at zero
// jitter and one recursion for all c (GEMM feeds chosen as for sel_batch slabs), then each entry whose pivot failed alone:
// first at zero jitter when sel_batch > 1 (a lone slab's feeds round differently from the batch's), then with `jitter`.
// used[s] (host): 0 ok, 1 ok with the jitter, > 1: 1 + the failing pivot.
static int factor_entries(gpmpc_handle_t h, const FactorSet& e, int sel_batch, double jitter, int* used)
{
    const int c = e.c, np = h->Npad;
    CUDA_TRY(cudaMemsetAsync(e.jit, 0, (size_t)c * sizeof(double), h->st));
    CUDA_TRY(cudaMemsetAsync(e.info, 0, (size_t)c * sizeof(int), h->st));
    int rc = launch_kbuild(h, e.hyp, e.jit, e.L, c, 0);
    if (rc) return rc;
    rc = potrf_inv_rec(h, e.L, e.Li, slab(h), slab(h), e.info, 0, np, c, sel_batch, e.W1, e.W2);
    if (rc) return rc;
    std::vector<int> info(c);
    CUDA_TRY(cudaMemcpyAsync(info.data(), e.info, (size_t)c * sizeof(int), cudaMemcpyDeviceToHost, h->st));
    CUDA_TRY(cudaStreamSynchronize(h->st));
    bool jittered = false;
    for (int s = 0; s < c; ++s) {
        used[s] = 0;
        for (int attempt = sel_batch > 1 ? 0 : 1; info[s] && attempt < 2; ++attempt) {
            const double jit = attempt ? jitter : 0.0;
            double* L = e.L + s * slab(h);
            CUDA_TRY(cudaMemcpyAsync(e.jit + s, &jit, sizeof(double), cudaMemcpyHostToDevice, h->st));
            CUDA_TRY(cudaMemsetAsync(e.info + s, 0, sizeof(int), h->st));
            rc = launch_kbuild(h, e.hyp + s * (h->Nx + 2LL), e.jit + s, L, 1, 0);
            if (rc) return rc;
            rc = potrf_inv_rec(h, L, e.Li + s * slab(h), slab(h), slab(h), e.info + s, 0, np, 1, 1, e.W1 + s * w2slab(h),
                               e.W2 + s * w2slab(h));
            if (rc) return rc;
            if (attempt) { used[s] = 1; jittered = true; break; }
            CUDA_TRY(cudaMemcpyAsync(&info[s], e.info + s, sizeof(int), cudaMemcpyDeviceToHost, h->st));
            CUDA_TRY(cudaStreamSynchronize(h->st));
        }
    }
    if (jittered) {         // the jittered recursions of every entry, read back together
        CUDA_TRY(cudaMemcpyAsync(info.data(), e.info, (size_t)c * sizeof(int), cudaMemcpyDeviceToHost, h->st));
        CUDA_TRY(cudaStreamSynchronize(h->st));
        for (int s = 0; s < c; ++s) if (used[s]) used[s] += info[s];
    }
    return GPMPC_OK;
}

// ------------------------------------------------------------------------------------
extern "C" int gpmpc_version(void) { return GPMPC_VERSION; }

extern "C" const char* gpmpc_last_error(gpmpc_handle_t h) { return h ? h->err : g_create_err; }

extern "C" int gpmpc_destroy(gpmpc_handle_t h);

// N_cap: training points the padded slabs must hold (appends up to it need no refit); the tail past N is identity in K
static int create_fill(gpmpc_handle_t h, int N, int N_cap, int Nx, int Ny, int out_begin, int out_count, int device)
{
    h->N = N; h->Nx = Nx; h->Ny = Ny; h->a0 = out_begin; h->nloc = out_count; h->device = device;
    h->nloc_max = out_count; h->world = 1; h->rank = 0;
    h->Npad = (std::max(N, N_cap) + GPMPC_TILE - 1) / GPMPC_TILE * GPMPC_TILE;
    h->panel_row.assign(out_count, 0);
    CUDA_TRY(cudaSetDevice(device));
    CUDA_TRY(cudaDeviceGetAttribute(&h->sms, cudaDevAttrMultiProcessorCount, device));
    h->opt_small_tiles = 4 * h->sms;      // two waves of 2 CTAs per SM
    h->psk_ctas = PSK_CTAS_PER_SM * h->sms;
    cudaDeviceGetAttribute(&h->clock_khz, cudaDevAttrClockRate, device);
    {
        int lo = 0, hi = 0;
        cudaDeviceGetStreamPriorityRange(&lo, &hi);
        CUDA_TRY(cudaStreamCreateWithPriority(&h->st, cudaStreamNonBlocking, hi));   // critical path first
    }
    CUDA_TRY(cudaEventCreate(&h->ev0));
    CUDA_TRY(cudaEventCreate(&h->ev1));
    const long long np = h->Npad;
    ENSURE(h->dXT, (long long)Nx * np);
    ENSURE(h->dMu, NX_MAX);
    ENSURE(h->dY, (long long)out_count * np);
    ENSURE(h->dHyp, (long long)out_count * (Nx + 2));
    ENSURE(h->dHypTmp, Nx + 2);
    ENSURE(h->dJit, out_count);
    ENSURE(h->dFacJit, out_count);
    ENSURE(h->dL, out_count * slab(h));
    ENSURE(h->dLi, out_count * slab(h));
    {   // W2 workspace: one region per recursion depth (n_d = ceil(nb / 2^d) * 128 rows at depth d)
        const int nb = h->Npad / 128;
        long long off = 0;
        for (int d = 0; d < MAX_DEPTH; ++d) {
            h->w2off[d] = off;
            const long long nd = (long long)((nb + (1 << d) - 1) >> d) * 128;
            off += nd * nd / 4 + 128;
        }
        h->w2off[MAX_DEPTH] = off;
        int lo = 0, hi = 0;
        cudaDeviceGetStreamPriorityRange(&lo, &hi);
        for (int d = 0; d < MAX_DEPTH; ++d) {
            CUDA_TRY(cudaStreamCreateWithPriority(&h->sideSt[d], cudaStreamNonBlocking, lo));
            CUDA_TRY(cudaEventCreateWithFlags(&h->evA[d], cudaEventDisableTiming));
            CUDA_TRY(cudaEventCreateWithFlags(&h->evB[d], cudaEventDisableTiming));
            CUDA_TRY(cudaEventCreateWithFlags(&h->evT[d], cudaEventDisableTiming));
            CUDA_TRY(cudaEventCreateWithFlags(&h->evS[d], cudaEventDisableTiming));
        }
    }
    ENSURE(h->dW1, out_count * w2slab(h));      // same per-depth layout as W2
    ENSURE(h->dW2, out_count * w2slab(h));
    ENSURE(h->dAlpha, (long long)out_count * np);
    ENSURE(h->dTmp, (long long)out_count * np);
    ENSURE(h->dRes, 2 * out_count);
    ENSURE(h->dInfo, out_count);
    ENSURE(h->dGrad, Nx + 2);
    h->hyper.assign((size_t)out_count * (Nx + 2), 0.0);
    h->logdet.assign(out_count, 0.0); h->yalpha.assign(out_count, 0.0); h->jitter_used.assign(out_count, 0);
    CUDA_TRY(cudaStreamSynchronize(h->st));
    return GPMPC_OK;
}


extern "C" int gpmpc_create(int N, int Nx, int Ny, int out_begin, int out_count, int device, gpmpc_handle_t* out)
{
    return gpmpc_create_reserve(N, N, Nx, Ny, out_begin, out_count, device, out);
}

extern "C" int gpmpc_create_reserve(int N, int N_cap, int Nx, int Ny, int out_begin, int out_count, int device,
                                    gpmpc_handle_t* out)
{
    gpmpc_handle_t h = nullptr;
    if (!out) return GPMPC_ERR_ARG;
    *out = nullptr;
    if (N < 1 || Nx < 1 || Nx > NX_MAX || Ny < 1 || out_begin < 0 || out_count < 1 || out_begin + out_count > Ny) {
        set_error(nullptr, "gpmpc_create: bad sizes N=%d (capacity %d) Nx=%d (max %d) Ny=%d outputs [%d,%d)", N, N_cap, Nx,
                  NX_MAX, Ny, out_begin, out_begin + out_count);
        return GPMPC_ERR_ARG;
    }
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev < 1 || device < 0 || device >= ndev) {
        set_error(nullptr, "gpmpc_create: no usable CUDA device %d (count %d, %s) -- this engine has no CPU path",
                  device, ndev, cudaGetErrorString(e));
        return GPMPC_ERR_CUDA;
    }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess || prop.major != 9 || prop.minor != 0) {
        set_error(nullptr, "gpmpc_create: device %d is sm_%d%d; this library is built for sm_90a (H100) only", device,
                  prop.major, prop.minor);
        return GPMPC_ERR_CUDA;
    }
    h = new gpmpc_handle_s();
    const int rc = create_fill(h, N, N_cap, Nx, Ny, out_begin, out_count, device);
    if (rc != GPMPC_OK) {            // no partially built handle survives: message to the create slot, everything freed
        snprintf(g_create_err, sizeof(g_create_err), "gpmpc_create: %s", h->err);
        gpmpc_destroy(h);
        return rc;
    }
    *out = h;
    return GPMPC_OK;
}

extern "C" int gpmpc_destroy(gpmpc_handle_t h)
{
    if (!h) return GPMPC_OK;
    cudaSetDevice(h->device);
    if (h->st) cudaStreamSynchronize(h->st);
    if (h->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(h->comm);
    for (int r = 0; r < GPMPC_MAXW; ++r) if (h->peerOpened[r]) cudaIpcCloseMemHandle(h->peerBase[r]);
    if (h->hPeerStatus) cudaFreeHost(h->hPeerStatus);
    if (h->hPinned) cudaFreeHost(h->hPinned);
    for (int d = 0; d < MAX_DEPTH; ++d) {
        if (h->sideSt[d]) { cudaStreamSynchronize(h->sideSt[d]); cudaStreamDestroy(h->sideSt[d]); }
        if (h->evA[d]) cudaEventDestroy(h->evA[d]);
        if (h->evB[d]) cudaEventDestroy(h->evB[d]);
        if (h->evT[d]) cudaEventDestroy(h->evT[d]);
        if (h->evS[d]) cudaEventDestroy(h->evS[d]);
    }
    if (h->ev0) cudaEventDestroy(h->ev0);
    if (h->ev1) cudaEventDestroy(h->ev1);
    if (h->st) cudaStreamDestroy(h->st);
    delete h;                        // frees the device buffers
    return GPMPC_OK;
}

static int ensure_pinned(gpmpc_handle_t h, size_t bytes)
{
    if (h->hPinnedBytes >= bytes) return GPMPC_OK;
    if (h->hPinned) cudaFreeHost(h->hPinned);
    h->hPinned = nullptr; h->hPinnedBytes = 0;
    // mapped: small batches are read / written by the kernels directly (zero copy), see gpmpc_predict
    CUDA_TRY(cudaHostAlloc((void**)&h->hPinned, bytes, cudaHostAllocMapped));
    CUDA_TRY(cudaHostGetDevicePointer((void**)&h->dPinnedAlias, h->hPinned, 0));
    h->hPinnedBytes = bytes;
    return GPMPC_OK;
}

// the caches derived from the factor (Li^T for predict_grad, K^-1 for the EM derivatives) no longer match it
static void factor_caches_stale(gpmpc_handle_t h) { h->u_valid = false; h->em_kinv_valid = false; }
// the factor no longer matches the data or hyper-parameters, or its slabs were used as scratch: gpmpc_factorize first
static void factor_stale(gpmpc_handle_t h) { h->factorized = false; factor_caches_stale(h); panel_stale(h, -1, 0); }

enum ModelNeed { NEED_DATA, NEED_HYPER, NEED_FACTOR };     // data; data and hyper-parameters; a factorised model

// State check of the model entry `fn` (the name its errors carry), then the handle's device is selected
static int model_guard(gpmpc_handle_t h, const char* fn, ModelNeed need)
{
    if (!h) return GPMPC_ERR_ARG;
    if (need == NEED_DATA && !h->has_data) { set_error(h, "%s: set_data first", fn); return GPMPC_ERR_STATE; }
    if (need == NEED_HYPER && (!h->has_data || !h->has_hyper)) { set_error(h, "%s: set_data and set_hyper first", fn); return GPMPC_ERR_STATE; }
    if (need == NEED_FACTOR && !h->factorized) { set_error(h, "%s: call gpmpc_factorize first", fn); return GPMPC_ERR_STATE; }
    CUDA_TRY(cudaSetDevice(h->device));
    return GPMPC_OK;
}

// alpha, log det K and y^T alpha of every owned output from the factor, after the factor changed
static int refresh_alpha(gpmpc_handle_t h)
{
    const int nl = h->nloc;
    factor_caches_stale(h);
    int rc = alpha_pass(h, model_entries(h, 0, nl));
    if (rc) return rc;
    std::vector<double> res(2 * nl);
    CUDA_TRY(cudaMemcpyAsync(res.data(), h->dRes, 2 * nl * 8, cudaMemcpyDeviceToHost, h->st));
    CUDA_TRY(cudaStreamSynchronize(h->st));
    for (int a = 0; a < nl; ++a) { h->logdet[a] = res[2 * a]; h->yalpha[a] = res[2 * a + 1]; }
    return GPMPC_OK;
}

extern "C" int gpmpc_set_data(gpmpc_handle_t h, const double* X, const double* Y)
{
    if (!h || !X || !Y) return GPMPC_ERR_ARG;
    CUDA_TRY(cudaSetDevice(h->device));
    const int N = h->N, Nx = h->Nx, np = h->Npad;
    std::vector<double> xt((size_t)Nx * np, 0.0), yl((size_t)h->nloc * np, 0.0);
    for (int i = 0; i < N; ++i)
        for (int d = 0; d < Nx; ++d) xt[(size_t)d * np + i] = X[(size_t)i * Nx + d];
    for (int a = 0; a < h->nloc; ++a)
        for (int i = 0; i < N; ++i) yl[(size_t)a * np + i] = Y[(size_t)i * h->Ny + h->a0 + a];
    h->hX.assign(X, X + (size_t)N * Nx);
    h->mu_stale = true;                     // launch_kbuild centres on the column means of hX
    CUDA_TRY(cudaMemcpyAsync(h->dXT, xt.data(), xt.size() * 8, cudaMemcpyHostToDevice, h->st));
    CUDA_TRY(cudaMemcpyAsync(h->dY, yl.data(), yl.size() * 8, cudaMemcpyHostToDevice, h->st));
    CUDA_TRY(cudaStreamSynchronize(h->st));
    h->has_data = true; factor_stale(h);
    return GPMPC_OK;
}

static int local_index(gpmpc_handle_t h, int a);

// Replace the target vector of global output a (N doubles): GP passes the residual y - m(X) when a
// prior mean function is in use (alpha = K^-1 (y - m(X)), optimize.py:492-494).
extern "C" int gpmpc_set_y(gpmpc_handle_t h, int a, const double* y)
{
    if (!h || !y) return GPMPC_ERR_ARG;
    { int rc = model_guard(h, __func__, NEED_DATA); if (rc) return rc; }
    const int al = local_index(h, a);
    if (al < 0) return GPMPC_ERR_ARG;
    CUDA_TRY(cudaMemcpyAsync(h->dY + (long long)al * h->Npad, y, (size_t)h->N * 8, cudaMemcpyHostToDevice, h->st));
    CUDA_TRY(cudaStreamSynchronize(h->st));
    factor_stale(h);
    return GPMPC_OK;
}

extern "C" int gpmpc_set_hyper(gpmpc_handle_t h, const double* hyper, int ld)
{
    if (!h || !hyper || ld < h->Nx + 2) { if (h) set_error(h, "gpmpc_set_hyper: ld < Nx+2"); return GPMPC_ERR_ARG; }
    CUDA_TRY(cudaSetDevice(h->device));
    const int m = h->Nx + 2;
    for (int a = 0; a < h->nloc; ++a)
        for (int q = 0; q < m; ++q) {
            const double v = hyper[(size_t)(h->a0 + a) * ld + q];
            if (q < h->Nx && v == 0.0) { set_error(h, "gpmpc_set_hyper: zero length scale"); return GPMPC_ERR_ARG; }
            h->hyper[(size_t)a * m + q] = v;
        }
    CUDA_TRY(cudaMemcpyAsync(h->dHyp, h->hyper.data(), h->hyper.size() * 8, cudaMemcpyHostToDevice, h->st));
    CUDA_TRY(cudaStreamSynchronize(h->st));
    h->has_hyper = true; factor_stale(h);
    return GPMPC_OK;
}

static int local_index(gpmpc_handle_t h, int a)
{
    if (a < h->a0 || a >= h->a0 + h->nloc) { set_error(h, "output %d is not owned by this handle [%d,%d)", a, h->a0, h->a0 + h->nloc); return -1; }
    return a - h->a0;
}

// T(T+1)/2 tiles of the gradient's trace pass
static inline int grad_tiles(gpmpc_handle_t h) { const int T = h->Npad / KB_TILE; return T * (T + 1) / 2; }

// dU, dKinv: the work slabs of compute_kinv, the host extracts, gpmpc_loo_nlpp's gradient, gpmpc_remove and EM;
// dGradPart: the trace pass's tile partials of the gradients of one output
static int ensure_kinv_scratch(gpmpc_handle_t h)
{
    ENSURE(h->dU, slab(h));
    ENSURE(h->dKinv, slab(h));
    ENSURE(h->dGradPart, (long long)grad_tiles(h) * (h->Nx + 2));
    return GPMPC_OK;
}

static int extract_to_host(gpmpc_handle_t h, const double* src, double* dst, int mode)
{
    const int N = h->N;
    { int rc = ensure_kinv_scratch(h); if (rc) return rc; }
    // stage through dU (N*N fits: Npad >= N)
    dim3 g((N + 127) / 128, N);
    extract_kernel<<<g, 128, 0, h->st>>>(src, h->Npad, h->dU, N, mode);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(dst, h->dU, (size_t)N * N * 8, cudaMemcpyDeviceToHost, h->st));
    CUDA_TRY(cudaStreamSynchronize(h->st));
    return GPMPC_OK;
}

extern "C" int gpmpc_build_K(gpmpc_handle_t h, int a, double* K_out)
{
    int rc = model_guard(h, __func__, NEED_HYPER);
    if (rc) return rc;
    const int al = local_index(h, a);
    if (al < 0) return GPMPC_ERR_ARG;
    rc = ensure_kinv_scratch(h);
    if (rc) return rc;
    const double zero = 0.0;
    CUDA_TRY(cudaMemcpyAsync(h->dJit + al, &zero, 8, cudaMemcpyHostToDevice, h->st));
    rc = launch_kbuild(h, h->dHyp + (long long)al * (h->Nx + 2), h->dJit + al, h->dKinv, 1, 1);
    if (rc) return rc;
    if (K_out) return extract_to_host(h, h->dKinv, K_out, 0);
    CUDA_TRY(cudaStreamSynchronize(h->st));
    return GPMPC_OK;
}

extern "C" int gpmpc_factorize(gpmpc_handle_t h, double jitter, int* info)
{
    int rc = model_guard(h, __func__, NEED_HYPER);
    if (rc) return rc;
    NvtxRange nvtx_r("gpmpc.factorize");
    const int nl = h->nloc;
    panel_stale(h, -1, 0);
    rc = factor_entries(h, model_entries(h, 0, nl), nl, jitter, h->jitter_used.data());
    if (rc) return rc;
    int worst = GPMPC_OK;
    for (int a = 0; a < nl; ++a) {
        const int used = h->jitter_used[a];
        if (used > 1) { worst = GPMPC_ERR_NOTPD; set_error(h, "output %d: K not positive definite even with jitter %g (pivot %d)", h->a0 + a, jitter, used - 1); }
        if (info) info[a] = used;
    }
    if (worst) return worst;
    // dJit now holds each output's jitter (0 or the retry's); the appends extend K + that jitter, and dJit itself is
    // scratch for later K builds (gpmpc_build_K, gpmpc_profile)
    CUDA_TRY(cudaMemcpyAsync(h->dFacJit, h->dJit, nl * sizeof(double), cudaMemcpyDeviceToDevice, h->st));
    rc = refresh_alpha(h);
    if (rc) return rc;
    h->factorized = true;
    return GPMPC_OK;
}

// K^-1 (lower) of `batch` factors, slabs at stride slab:  U = Li^T,  K^-1 = U U^T.  The product's feed is the one of a
// single slab, so every entry gets the bits compute_kinv gives it alone.
static int kinv_at(gpmpc_handle_t h, const double* Li, double* U, double* Kinv, int batch)
{
    const int np = h->Npad;
    dim3 g(np / 32, np / 32, batch), b(32, 8);
    transpose_lower_kernel<<<g, b, 0, h->st>>>(Li, slab(h), U, slab(h), np, np / 32);
    CUDA_TRY(cudaGetLastError());
    GemmParams p;
    memset(&p, 0, sizeof(p));
    p.A = U; p.lda = np; p.sA = slab(h); p.B = U; p.ldb = np; p.sB = slab(h); p.C = Kinv; p.ldc = np; p.sC = slab(h);
    p.mt = np / 128; p.nt = np / 128; p.K = np; p.alpha = 1.0; p.beta = 0.0;
    p.kflags = GEMM_KI_GE | GEMM_KJ_GE; p.lower = 1;
    CUDA_TRY(gemm128(h, h->st, true, p, batch, 1));
    return GPMPC_OK;
}

// K^-1 (lower) of local output al into dKinv
static int compute_kinv(gpmpc_handle_t h, int al)
{
    int rc = ensure_kinv_scratch(h);
    if (rc) return rc;
    return kinv_at(h, h->dLi + (long long)al * slab(h), h->dU, h->dKinv, 1);
}

// 1/2 tr((W - alpha alpha^T) dK/dtheta) for every hyper-parameter of `batch` entries: hyper rows at dHyp (stride Nx+2),
// W = the lower triangle of the Kinv slabs (stride slab), alpha at stride Npad, tile partials in part (grad_tiles rows of
// Nx+2 per entry), gradients into grad (stride Nx+2)
static int launch_grad_at(gpmpc_handle_t h, const double* dHyp, const double* Kinv, const double* alpha, double* part,
                          double* grad, int batch)
{
    const int nt = grad_tiles(h), m = h->Nx + 2;
    const int smem = 2 * h->Nx * KB_TILE * 8;
    CUDA_TRY(nxp_dispatch(h->Nx, [&](auto nxp) {
        nlml_grad_kernel<decltype(nxp)::value><<<dim3(nt, batch), 256, smem, h->st>>>(
            h->dXT, h->Npad, h->N, h->Nx, dHyp, m, Kinv, h->Npad, slab(h), alpha, h->Npad, part, (long long)nt * m);
        return cudaGetLastError();
    }));
    nlml_grad_final_kernel<<<dim3(m, batch), 256, 0, h->st>>>(part, (long long)nt * m, nt, h->Nx, dHyp, m, grad);
    CUDA_TRY(cudaGetLastError());
    return GPMPC_OK;
}

// Argument check of the objectives gpmpc_nlml, gpmpc_nlml_batch and gpmpc_loo_nlpp (fn) at the S hyper rows theta
// (stride Nx+2), in this order: the NULL pointers and S (args_ok; a batch's message names them), the model state, the
// output (its local index into *al), zero length scales (a batch's message names the row)
static int objective_check(gpmpc_handle_t h, const char* fn, bool batch, bool args_ok, int a, const double* theta, int S,
                           int* al)
{
    if (!h) return GPMPC_ERR_ARG;
    if (!args_ok) { if (batch) set_error(h, "%s: NULL pointer or S < 1", fn); return GPMPC_ERR_ARG; }
    const int rc = model_guard(h, fn, NEED_DATA);
    if (rc) return rc;
    if ((*al = local_index(h, a)) < 0) return GPMPC_ERR_ARG;
    for (int s = 0; s < S; ++s)
        for (int d = 0; d < h->Nx; ++d)
            if (theta[(size_t)s * (h->Nx + 2) + d] == 0.0) {
                if (batch) set_error(h, "%s: zero length scale in row %d", fn, s);
                else set_error(h, "%s: zero length scale", fn);
                return GPMPC_ERR_ARG;
            }
    return GPMPC_OK;
}

// The objective pass of gpmpc_nlml and gpmpc_nlml_batch at the entries' hyper rows theta (host): the factor step with the
// 1e-8 jitter retry of optimize.py:345-350, every GEMM on the feed of a single slab, so no entry depends on c; the alpha
// pass; log det and y . alpha; with grad the gradient in place: U = Li^T into the L slab (log det has been read from it),
// K^-1 = U U^T into the Li slab (alpha is done), tile partials in part and gradients in g (c rows each); then the NLL.
// status (host, c): 0, 1 (jitter) or GPMPC_ERR_NOTPD, whose entry runs on with its slabs as they are (every pass is per
// entry, so it touches no other) and gets NaN.  Without status a failed entry is an error of fn, before the alpha pass.
static int objective_pass(gpmpc_handle_t h, const char* fn, const FactorSet& e, const double* theta, double* part,
                          double* g, double* nll, double* grad, int* status)
{
    const int c = e.c, m = h->Nx + 2;
    CUDA_TRY(cudaMemcpyAsync(e.hyp, theta, (size_t)c * m * 8, cudaMemcpyHostToDevice, h->st));
    std::vector<int> used(c);
    int rc = factor_entries(h, e, 1, 1e-8, used.data());
    if (rc) return rc;
    for (int s = 0; s < c; ++s) {
        if (status) status[s] = used[s] > 1 ? GPMPC_ERR_NOTPD : used[s];
        else if (used[s] > 1) { set_error(h, "%s: K not positive definite even with jitter", fn); return GPMPC_ERR_NOTPD; }
    }
    rc = alpha_pass(h, e);
    if (rc) return rc;
    std::vector<double> res(2 * c);
    CUDA_TRY(cudaMemcpyAsync(res.data(), e.res, (size_t)c * 16, cudaMemcpyDeviceToHost, h->st));
    if (grad) {
        rc = kinv_at(h, e.Li, e.L, e.Li, c);
        if (rc) return rc;
        rc = launch_grad_at(h, e.hyp, e.Li, e.alpha, part, g, c);
        if (rc) return rc;
        CUDA_TRY(cudaMemcpyAsync(grad, g, (size_t)c * m * 8, cudaMemcpyDeviceToHost, h->st));
    }
    CUDA_TRY(cudaStreamSynchronize(h->st));
    for (int s = 0; s < c; ++s) {
        if (used[s] > 1) {
            nll[s] = NAN;
            if (grad) for (int q = 0; q < m; ++q) grad[(size_t)s * m + q] = NAN;
        } else {
            nll[s] = 0.5 * res[2 * s + 1] + 0.5 * res[2 * s];      // optimize.py:355
        }
    }
    return GPMPC_OK;
}

extern "C" int gpmpc_nlml(gpmpc_handle_t h, int a, const double* theta, double* nll, double* grad)
{
    int al = 0;
    int rc = objective_check(h, __func__, false, theta && nll, a, theta, 1, &al);
    if (rc) return rc;
    NvtxRange nvtx_r("gpmpc.nlml");
    if (grad) ENSURE(h->dGradPart, (long long)grad_tiles(h) * (h->Nx + 2));
    // a one-entry pass in output al's own slots, the hyper row in dHypTmp: the model needs gpmpc_factorize afterwards
    factor_stale(h);
    FactorSet e = model_entries(h, al, 1);
    e.hyp = h->dHypTmp;
    return objective_pass(h, __func__, e, theta, h->dGradPart, h->dGrad, nll, grad, nullptr);
}

// gpmpc_nlml_batch scratch for a pass of c entries of local output al: the factor slabs dNbL, dNbLi, the recursion
// workspaces dNbW1, dNbW2, the pivot infos dNbInfo and dNbV = [hyper rows (c, Nx+2) | jitter (c) | tmp (c, Npad) |
// alpha (c, Npad) | res (c, 2) | gradient partials (c, grad_tiles, Nx+2) | gradients (c, Nx+2)]; every entry's target is
// al's y.  The entries go to *e, the gradient partials and gradients to *part and *g.
static int nlml_batch_scratch(gpmpc_handle_t h, int al, int c, FactorSet* e, double** part, double** g)
{
    const long long m = h->Nx + 2, np = h->Npad;
    ENSURE(h->dNbL, c * slab(h));
    ENSURE(h->dNbLi, c * slab(h));
    ENSURE(h->dNbW1, c * w2slab(h));
    ENSURE(h->dNbW2, c * w2slab(h));
    ENSURE(h->dNbV, c * (m + 1 + 2 * np + 2 + grad_tiles(h) * m + m));
    ENSURE(h->dNbInfo, c);
    double* jit = h->dNbV + c * m;
    double* tmp = jit + c;
    double* alpha = tmp + c * np;
    double* res = alpha + c * np;
    *e = {c, h->dNbV, jit, h->dNbInfo, h->dNbL, h->dNbLi, h->dNbW1, h->dNbW2, h->dY + al * np, 0, tmp, alpha, res};
    *part = res + 2 * c;
    *g = *part + c * grad_tiles(h) * m;
    return GPMPC_OK;
}

static void nlml_batch_release(gpmpc_handle_t h)
{
    cudaStreamSynchronize(h->st);
    h->dNbL.release(); h->dNbLi.release(); h->dNbW1.release(); h->dNbW2.release(); h->dNbV.release(); h->dNbInfo.release();
}

extern "C" int gpmpc_nlml_batch(gpmpc_handle_t h, int a, int S, const double* theta, double* nll, double* grad,
                                int* status)
{
    int al = 0;
    int rc = objective_check(h, __func__, true, theta && nll && status && S >= 1, a, theta, S, &al);
    if (rc) return rc;
    const int m = h->Nx + 2;
    NvtxRange nvtx_r("gpmpc.nlml_batch");
    // results do not depend on the pass size, so a pass that does not fit is halved
    int pass = h->opt_nlml_batch_max > 0 ? std::min(S, h->opt_nlml_batch_max) : S;
    for (int s0 = 0; s0 < S;) {
        const int c = std::min(pass, S - s0);
        FactorSet e;
        double *part, *g;
        rc = nlml_batch_scratch(h, al, c, &e, &part, &g);
        if (rc) {
            const bool oom = cudaGetLastError() == cudaErrorMemoryAllocation;
            nlml_batch_release(h);
            if (!oom || c == 1) return rc;
            pass = c / 2;
            continue;
        }
        rc = objective_pass(h, __func__, e, theta + (size_t)s0 * m, part, g, nll + s0,
                            grad ? grad + (size_t)s0 * m : nullptr, status + s0);
        if (rc) return rc;
        s0 += c;
    }
    return GPMPC_OK;
}

// ------------------------------------------------------------------------------------
// leave-one-out cross-validation (kernels.cuh, loo_*)
// ------------------------------------------------------------------------------------
// dLoo for `batch` outputs at the current N: [mean (batch*N) | var (batch*N) | nlpp (batch) | c partials
// (batch*nch*N) | sw | u | b | tmp | zero (Npad each)]
struct LooLayout {
    int nch; double *mean, *var, *nlpp, *P, *sw, *u, *b, *tmp, *zero;
};

static int loo_layout(gpmpc_handle_t h, int batch, LooLayout* o)
{
    const long long N = h->N, np = h->Npad;
    o->nch = (int)((N + TRT_ROWS - 1) / TRT_ROWS);
    ENSURE(h->dLoo, 2 * batch * N + batch + (long long)batch * o->nch * N + 5 * np);
    o->mean = h->dLoo; o->var = o->mean + batch * N; o->nlpp = o->var + batch * N; o->P = o->nlpp + batch;
    o->sw = o->P + (long long)batch * o->nch * N; o->u = o->sw + np; o->b = o->u + np; o->tmp = o->b + np;
    o->zero = o->tmp + np;
    return GPMPC_OK;
}

// LOO mean, variance and NLPP of `batch` consecutive local outputs from al on the current factors (O(N^2) each);
// with_w: also sqrt(w) and u of the (single) output
static int loo_launch(gpmpc_handle_t h, int al, int batch, const LooLayout& o, bool with_w)
{
    const int N = h->N, np = h->Npad;
    const long long nN = (long long)o.nch * N;
    loo_colnorm_part_kernel<<<dim3((N + 31) / 32, o.nch, batch), 256, 0, h->st>>>(h->dLi + (long long)al * slab(h), np,
                                                                                 slab(h), o.P, nN, N);
    CUDA_TRY(cudaGetLastError());
    loo_point_kernel<<<batch, 1024, 0, h->st>>>(o.P, nN, o.nch, h->dAlpha + (long long)al * np, h->dY + (long long)al * np,
                                                np, N, o.mean, o.var, o.nlpp, with_w ? o.sw : nullptr,
                                                with_w ? o.u : nullptr, np);
    CUDA_TRY(cudaGetLastError());
    return GPMPC_OK;
}

extern "C" int gpmpc_loo(gpmpc_handle_t h, double* mean, double* var, double* nlpp)
{
    int rc = model_guard(h, __func__, NEED_FACTOR);
    if (rc) return rc;
    if (h->N < 2) { set_error(h, "gpmpc_loo: needs N >= 2 training points (N = %d)", h->N); return GPMPC_ERR_ARG; }
    NvtxRange nvtx_r("gpmpc.loo");
    const int nl = h->nloc;
    LooLayout o;
    rc = loo_layout(h, nl, &o);
    if (rc) return rc;
    rc = loo_launch(h, 0, nl, o, false);
    if (rc) return rc;
    const size_t bytes = (size_t)nl * h->N * 8;
    if (mean) CUDA_TRY(cudaMemcpyAsync(mean, o.mean, bytes, cudaMemcpyDeviceToHost, h->st));
    if (var) CUDA_TRY(cudaMemcpyAsync(var, o.var, bytes, cudaMemcpyDeviceToHost, h->st));
    if (nlpp) CUDA_TRY(cudaMemcpyAsync(nlpp, o.nlpp, nl * 8, cudaMemcpyDeviceToHost, h->st));
    CUDA_TRY(cudaStreamSynchronize(h->st));
    return GPMPC_OK;
}

extern "C" int gpmpc_loo_nlpp(gpmpc_handle_t h, int a, const double* theta, double* nlpp, double* grad)
{
    int al = 0;
    int rc = objective_check(h, __func__, false, theta && nlpp, a, theta, 1, &al);
    if (rc) return rc;
    const int m = h->Nx + 2, N = h->N, np = h->Npad;
    if (N < 2) { set_error(h, "gpmpc_loo_nlpp: needs N >= 2 training points (N = %d)", N); return GPMPC_ERR_ARG; }
    NvtxRange nvtx_r("gpmpc.loo_nlpp");
    // gpmpc_nlml's factor step and alpha pass in output al's own slots: the model needs gpmpc_factorize afterwards
    factor_stale(h);
    FactorSet e = model_entries(h, al, 1);
    e.hyp = h->dHypTmp;
    CUDA_TRY(cudaMemcpyAsync(e.hyp, theta, m * 8, cudaMemcpyHostToDevice, h->st));
    int used = 0;
    rc = factor_entries(h, e, 1, 1e-8, &used);
    if (rc) return rc;
    if (used > 1) { set_error(h, "gpmpc_loo_nlpp: K not positive definite even with jitter"); return GPMPC_ERR_NOTPD; }
    rc = alpha_pass(h, e);
    if (rc) return rc;
    LooLayout o;
    rc = loo_layout(h, 1, &o);
    if (rc) return rc;
    rc = loo_launch(h, al, 1, o, grad != nullptr);        // c always from the column norms: the same NLPP bits either way
    if (rc) return rc;
    double val = 0.0;
    CUDA_TRY(cudaMemcpyAsync(&val, o.nlpp, 8, cudaMemcpyDeviceToHost, h->st));
    if (grad) {
        rc = compute_kinv(h, al);                          // C (lower) in dKinv
        if (rc) return rc;
        // b = C u = Li^T (Li u)
        trmv_lower_kernel<<<(N + 7) / 8, 256, 0, h->st>>>(e.Li, np, 0, o.u, 0, o.tmp, 0, N);
        CUDA_TRY(cudaGetLastError());
        trmv_lower_T_kernel<<<(N + 31) / 32, 256, 0, h->st>>>(e.Li, np, 0, o.tmp, 0, o.b, 0, N);
        CUDA_TRY(cudaGetLastError());
        // G = (C diag(sqrt w)) (C diag(sqrt w))^T = C diag(w) C: lower tiles into dKinv, over C diag(sqrt w) in dU
        loo_mirror_scale_kernel<<<dim3(np / 32, np / 32), dim3(32, 8), 0, h->st>>>(h->dKinv, np, o.sw, h->dU, N);
        CUDA_TRY(cudaGetLastError());
        GemmParams p;
        memset(&p, 0, sizeof(p));
        p.A = h->dU; p.lda = np; p.B = h->dU; p.ldb = np; p.C = h->dKinv; p.ldc = np;
        p.mt = np / 128; p.nt = np / 128; p.K = np; p.alpha = 1.0; p.beta = 0.0; p.lower = 1;
        CUDA_TRY(gemm128(h, h->st, true, p, 1, 1));
        loo_w_kernel<<<dim3((N + 255) / 256, N), 256, 0, h->st>>>(h->dKinv, np, o.b, e.alpha, N);
        CUDA_TRY(cudaGetLastError());
        // the trace pass with W in place of K^-1 and alpha = 0: 1/2 tr(W dK/dtheta), doubled on the host (exact)
        CUDA_TRY(cudaMemsetAsync(o.zero, 0, (size_t)np * 8, h->st));
        rc = launch_grad_at(h, e.hyp, h->dKinv, o.zero, h->dGradPart, h->dGrad, 1);
        if (rc) return rc;
        CUDA_TRY(cudaMemcpyAsync(grad, h->dGrad, m * 8, cudaMemcpyDeviceToHost, h->st));
    }
    CUDA_TRY(cudaStreamSynchronize(h->st));
    if (grad)
        for (int q = 0; q < m; ++q) grad[q] *= 2.0;
    *nlpp = val;
    return GPMPC_OK;
}

extern "C" int gpmpc_get(gpmpc_handle_t h, int what, int a, double* dst)
{
    if (!h || !dst) return GPMPC_ERR_ARG;
    CUDA_TRY(cudaSetDevice(h->device));
    const int al = local_index(h, a);
    if (al < 0) return GPMPC_ERR_ARG;
    if (what == GPMPC_GET_K) return gpmpc_build_K(h, a, dst);
    if (what != GPMPC_GET_ALPHA_NLML) {       // that one: alpha of the last gpmpc_nlml(a, theta) evaluation
        const int rc = model_guard(h, __func__, NEED_FACTOR);
        if (rc) return rc;
    }
    switch (what) {
    case GPMPC_GET_CHOL: return extract_to_host(h, h->dL + (long long)al * slab(h), dst, 1);
    case GPMPC_GET_LINV: return extract_to_host(h, h->dLi + (long long)al * slab(h), dst, 1);
    case GPMPC_GET_ALPHA:
    case GPMPC_GET_ALPHA_NLML:
        CUDA_TRY(cudaMemcpyAsync(dst, h->dAlpha + (long long)al * h->Npad, h->N * 8, cudaMemcpyDeviceToHost, h->st));
        CUDA_TRY(cudaStreamSynchronize(h->st));
        return GPMPC_OK;
    case GPMPC_GET_LOGDET: dst[0] = h->logdet[al]; return GPMPC_OK;
    case GPMPC_GET_INVK: {
        int rc = compute_kinv(h, al);
        if (rc) return rc;
        // dKinv -> host through dU is not possible (dU is an input of compute_kinv but free now)
        return extract_to_host(h, h->dKinv, dst, 2);
    }
    default: set_error(h, "gpmpc_get: unknown selector %d", what); return GPMPC_ERR_ARG;
    }
}

extern "C" int gpmpc_set_option(gpmpc_handle_t h, const char* name, double value)
{
    if (!h || !name) return GPMPC_ERR_ARG;
    if (!strcmp(name, "refine")) { h->opt_refine = value != 0.0; return GPMPC_OK; }
    if (!strcmp(name, "predict_ctas")) {       // persistent grid of the predict product (0 = PSK_CTAS_PER_SM per SM)
        const int v = (int)value;
        if (v < 0 || v > PSK_MAX_CTAS) { set_error(h, "predict_ctas must be in [0, %d]", PSK_MAX_CTAS); return GPMPC_ERR_ARG; }
        h->opt_predict_ctas = v; return GPMPC_OK;
    }
    if (!strcmp(name, "peer_timeout_s")) { h->opt_peer_timeout_s = value > 0.0 ? value : 60.0; return GPMPC_OK; }
    if (!strcmp(name, "small_tiles")) { h->opt_small_tiles = (int)value; return GPMPC_OK; }
    if (!strcmp(name, "peer")) { h->opt_peer = value != 0.0; return GPMPC_OK; }
    if (!strcmp(name, "em_points")) {          // points per batched 'EM' forward (0 = the scratch budget decides)
        if (!(value >= 0.0 && value <= 1e9)) { set_error(h, "em_points must be >= 0"); return GPMPC_ERR_ARG; }
        h->opt_em_points = (int)value; return GPMPC_OK;
    }
    if (!strcmp(name, "nlml_batch_max")) {     // entries per gpmpc_nlml_batch pass (0 = all): a cap on its scratch
        if (!(value >= 0.0 && value <= 1e9)) { set_error(h, "nlml_batch_max must be >= 0"); return GPMPC_ERR_ARG; }
        h->opt_nlml_batch_max = (int)value; return GPMPC_OK;
    }
    if (!strcmp(name, "ut_alpha") || !strcmp(name, "ut_beta") || !strcmp(name, "ut_kappa")) {
        double a = h->ut_alpha, b = h->ut_beta, k = h->ut_kappa;
        (name[3] == 'a' ? a : name[3] == 'b' ? b : k) = value;
        const double n = h->Nx, lam = a * a * (n + k) - n;
        if (!std::isfinite(value) || !(a > 0.0) || !(n + lam > 0.0)) {
            set_error(h, "%s = %g: 'UT' needs a finite value, alpha > 0 and n + lambda > 0 (kappa > -Nx)", name, value);
            return GPMPC_ERR_ARG;
        }
        h->ut_alpha = a; h->ut_beta = b; h->ut_kappa = k;
        return GPMPC_OK;
    }
    set_error(h, "unknown option %s", name);
    return GPMPC_ERR_ARG;
}

// ------------------------------------------------------------------------------------
// predict
// ------------------------------------------------------------------------------------
// training points per CTA of the ks kernel (ks_tile_kernel): 128-point chunks below N = 8192 so small problems still fill
// the machine; 512 at large N (few partial blocks for the record sums); 1024 when a rank also holds several outputs --
// the per-CTA prologue / epilogue (a large share of a CTA's time at 512) is then amortised over twice the evaluations, and the
// 16 chunks x 7 row groups x outputs still cover the SMs.  (Nx <= 12: the chunk of X^T must leave room for 2 CTAs per SM.)
static inline int ks_chunk(gpmpc_handle_t h)
{
    if (h->Npad < 8192) return 128;
    return (h->nloc >= 2 && h->Nx <= 12) ? 1024 : 512;
}

// blocks of the ks kernel along the training points (one partial record each)
static inline int ks_blocks(gpmpc_handle_t h) { return (h->Npad + ks_chunk(h) - 1) / ks_chunk(h); }

// rows of the A-side tile (BM) of the predict product for n <= HB solved rows, and of the ks kernel's grid
static inline int round8(int n) { return (n + 7) / 8 * 8; }

// the solved rows v (and r, for refinement and append) of one 64-point chunk, every output
static int ensure_rows(gpmpc_handle_t h)
{
    ENSURE(h->dV, (long long)h->nloc * HB * h->Npad);
    ENSURE(h->dR, (long long)h->nloc * HB * h->Npad);
    return GPMPC_OK;
}

static int ensure_predict_bufs(gpmpc_handle_t h, int H)
{
    const long long np = h->Npad, nt = np / 128;      // nt >= the product's tiles per output (tile_cnt below)
    ENSURE(h->dKST, (long long)h->nloc * HB * np);
    ENSURE(h->dPMJ, (long long)h->nloc * HB * ks_blocks(h) * (h->Nx + 1));
    ENSURE(h->dSQ, (long long)h->nloc * HB * nt);
    ENSURE(h->dCnt, (long long)h->nloc * nt + h->nloc + 1);
    // parked stream-K partials: two BM x PSK_BN slots per persistent CTA
    ENSURE(h->dPart, (long long)std::max(h->psk_ctas, h->opt_predict_ctas) * 2 * HB * PSK_BN);
    if (h->opt_refine) {
        int rc = ensure_rows(h);
        if (rc) return rc;
        ENSURE(h->dR2, (long long)h->nloc * HB * np);
    }
    if (H > h->Hcap) {
        // dZ .. dCov point into dIn / dOut: they are laid out again once both hold the new capacity
        h->Hcap = 0;
        h->dZ = h->dSigma = h->dMean = h->dVar = h->dJ = h->dCov = nullptr;
        const long long cap = std::max(H, HB);
        const int nyp = h->nloc_max * h->world;
        const long long Nx = h->Nx, Ny = h->Ny;
        ENSURE(h->dG, (long long)nyp * cap * (Nx + 2));
        ENSURE(h->dIn, cap * Nx + cap * Nx * Nx);
        ENSURE(h->dOut, cap * (2 * Ny + Ny * Nx + Ny * Ny));
        h->dZ = h->dIn; h->dSigma = h->dIn + cap * Nx;
        h->dMean = h->dOut; h->dVar = h->dOut + cap * Ny; h->dJ = h->dOut + 2 * cap * Ny;
        h->dCov = h->dOut + 2 * cap * Ny + cap * Ny * Nx;
        h->Hcap = (int)cap;
    }
    return GPMPC_OK;
}

// Persistent stream-K launch of the fused predict product (predict_streamk.cuh)
template <int BM>
static cudaError_t psk_launch_bm(const PredictParams& p, const double* A, long long sA, const double* B, long long sB,
                                 int np, int grid, cudaStream_t st)
{
    constexpr int BYTES = psk_pipe_doubles(BM) * 8 + 2 * PSK_STAGES * 8 + 1024;
    const cudaError_t e = smem_opt_in<predict_streamk_kernel<BM>>(BYTES);
    if (e != cudaSuccess) return e;
    CUtensorMap tmA, tmB;
    if (!tmap_make(&tmA, A, np, BM, np, sA, p.nloc, BM)) return cudaErrorInvalidValue;
    if (!tmap_make(&tmB, B, np, np, np, sB, p.nloc, PSK_BN)) return cudaErrorInvalidValue;
    // programmatic dependent launch after the ks kernel (the kernel's griddepcontrol.wait guards its inputs)
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(PSK_THREADS); cfg.dynamicSmemBytes = BYTES; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, predict_streamk_kernel<BM>, p, tmA, tmB);
}

// persistent grid: PSK_CTAS_PER_SM CTAs per SM, but never fewer than 4 k-steps per CTA (at small N, more CTAs with fewer steps each beat
// fewer with more -- the fixed cost per CTA overlaps across SMs, the steps do not)
static int psk_grid(gpmpc_handle_t h, long long G)
{
    int ctas = h->opt_predict_ctas > 0 ? h->opt_predict_ctas : h->psk_ctas;
    ctas = std::min(ctas, PSK_MAX_CTAS);
    const long long by_work = std::max(1LL, G / 4);
    return (int)std::min<long long>(ctas, h->opt_predict_ctas > 0 ? G : by_work);
}

// The schedule of the predict product p of the slab B; returns its grid.  A lower-mode product of L^-1 streams it from the
// panel, on the paired schedule when its tile pairs fill the grid (psk_pair_units: the same choice for every such product
// at one (nloc, ntb) and grid), on psk_pair_grid's CTAs unless predict_ctas sets the grid.
static int psk_schedule(gpmpc_handle_t h, PredictParams& p, const double* B)
{
    int grid = psk_grid(h, p.G);
    if (B == h->dLi.p && !p.upper) {
        p.Lp = h->dLiP;
        p.upo = psk_pair_units(p.nloc, p.ntb, grid);
        if (p.upo && h->opt_predict_ctas == 0) grid = psk_pair_grid((long long)p.nloc * p.upo, grid);
    }
    return grid;
}

// the predict product p (psk_base) of A (h-major rows, HB * Npad per output) and the slab B of each output: BM = round8(p.Hc).
// A product of L^-1 reads its panel, which panel_refresh must have brought up to date.
static cudaError_t psk_launch(gpmpc_handle_t h, const PredictParams& p0, const double* A, const double* B)
{
    const long long sA = (long long)HB * h->Npad, sB = slab(h);
    const int np = h->Npad;
    PredictParams p = p0;
    const int grid = psk_schedule(h, p, B);
    if (p.Lp)
        for (int a = 0; a < h->nloc; ++a)
            if (h->panel_row[a] < np) return cudaErrorIllegalState;
    switch (round8(p.Hc)) {
    case 8: return psk_launch_bm<8>(p, A, sA, B, sB, np, grid, h->st);
    case 16: return psk_launch_bm<16>(p, A, sA, B, sB, np, grid, h->st);
    case 24: return psk_launch_bm<24>(p, A, sA, B, sB, np, grid, h->st);
    case 32: return psk_launch_bm<32>(p, A, sA, B, sB, np, grid, h->st);
    case 40: return psk_launch_bm<40>(p, A, sA, B, sB, np, grid, h->st);
    case 48: return psk_launch_bm<48>(p, A, sA, B, sB, np, grid, h->st);
    case 56: return psk_launch_bm<56>(p, A, sA, B, sB, np, grid, h->st);
    default: return psk_launch_bm<64>(p, A, sA, B, sB, np, grid, h->st);
    }
}

// upper: the L-side operand is upper triangular (its k-step list is shorter when Npad / 128 is odd)
static void psk_base(gpmpc_handle_t h, PredictParams& p, int Hc, int upper = 0)
{
    memset(&p, 0, sizeof(p));
    const long long nt = h->Npad / 128;
    p.nloc = h->nloc; p.nt = (int)nt; p.Hc = Hc; p.upper = upper;
    p.ntb = (int)((h->Npad + PSK_BN - 1) / PSK_BN); p.nk = h->Npad / GEMM_BK;
    p.T = psk_steps_per_output(p.ntb, p.nk, upper); p.G = p.T * h->nloc;
    p.part = h->dPart;
    p.tile_cnt = h->dCnt; p.out_cnt = h->dCnt + (long long)h->nloc * nt; p.done_cnt = p.out_cnt + h->nloc;
    p.SQ = h->dSQ;
    p.hyp = h->dHyp; p.hyp_ld = h->Nx + 2; p.Nx = h->Nx;
}

// Brings the L^-1 panel up to date: output a is repacked from the tile of its first stale row, so an append costs one tile
// band and a factorisation everything.  Runs before any product of L^-1 (predict_prepare, gpmpc_profile).
static int panel_refresh(gpmpc_handle_t h)
{
    PredictParams p;
    psk_base(h, p, HB);
    const long long blk = PSK_BN * GEMM_BK;
    const double* old = h->dLiP;
    ENSURE(h->dLiP, p.G * blk);
    if (h->dLiP.p != old) panel_stale(h, -1, 0);
    for (int a = 0; a < h->nloc; ++a) {
        if (h->panel_row[a] >= h->Npad) continue;
        const int jt0 = h->panel_row[a] / PSK_BN;
        panel_pack_kernel<<<dim3(p.nk, p.ntb - jt0), 256, 0, h->st>>>(h->dLi + a * slab(h), h->Npad, h->dLiP + a * p.T * blk,
                                                                      p.ntb, jt0);
        CUDA_TRY(cudaGetLastError());
        h->panel_row[a] = h->Npad;
    }
    return GPMPC_OK;
}

// after psk_base: the product also finalises chunk [h0, h0 + Hc) of an H-point step (records from the ks partials into dG)
static void psk_finalize(gpmpc_handle_t h, PredictParams& p, int H, int h0)
{
    p.finalize = 1; p.PMJ = h->dPMJ; p.nblk_mj = ks_blocks(h);
    p.Gloc = h->dG; p.slot0 = h->a0; p.Htot = H; p.h0 = h0;
}

// assembly of a single-rank step of H points (predict_core adds the multi-rank fields).  stage_g: the gather records fit
// next to J Sigma in the product kernel's stage buffers (psk_pipe_doubles), read by the fused assembly only
static AssembleArgs assemble_args(gpmpc_handle_t h, int H, int method, const double* Sigma, int spp,
                                  double* mean, double* var, double* J, double* cov)
{
    AssembleArgs as;
    memset(&as, 0, sizeof(as));
    as.G = h->dG; as.Ny = h->Ny; as.Nx = h->Nx; as.H = H; as.method_ta = (method == GPMPC_METHOD_TA);
    as.Sigma = Sigma; as.sigma_per_point = spp;
    as.mean = mean; as.var = var; as.J = J; as.cov = cov;
    as.world = 1;
    as.stage_g = (assemble_rows_doubles(H, h->Ny, h->Nx) <= psk_pipe_doubles(round8(std::min(H, HB)))) ? 1 : 0;
    return as;
}

// ks rows of the Hc points at dZc into dKST (round8(Hc) rows per output), their mean / Jacobian partials into dPMJ
template <int NXP, int CH>
static cudaError_t launch_ks(gpmpc_handle_t h, const double* dZc, int Hc)
{
    const int smem = (NXP + 1) * CH * 8, nblk = ks_blocks(h);
    const cudaError_t e = smem_opt_in<ks_tile_kernel<NXP, CH>>(smem);      // static + dynamic may pass 48 KB
    if (e != cudaSuccess) return e;
    dim3 g(nblk, round8(Hc) / 8, h->nloc);
    ks_tile_kernel<NXP, CH><<<g, 256, smem, h->st>>>(h->dXT, h->Npad, h->N, h->Nx, h->dHyp, h->Nx + 2, h->dAlpha, h->Npad,
                                                     dZc, Hc, h->dKST, h->Npad, (long long)HB * h->Npad, h->dPMJ, nblk);
    return cudaGetLastError();
}

template <int CH>
static cudaError_t launch_ks_nx(gpmpc_handle_t h, const double* dZc, int Hc)
{
    const int Nx = h->Nx;       // register-array extent NXP: the next even count up to 12, then 16 / 24 / 32
    if (Nx <= 4) return launch_ks<4, CH>(h, dZc, Hc);
    if (Nx <= 6) return launch_ks<6, CH>(h, dZc, Hc);
    if (Nx <= 8) return launch_ks<8, CH>(h, dZc, Hc);
    if (Nx <= 10) return launch_ks<10, CH>(h, dZc, Hc);
    if (Nx <= 12) return launch_ks<12, CH>(h, dZc, Hc);
    if (CH <= 512) {
        if (Nx <= 16) return launch_ks<16, (CH <= 512 ? CH : 512)>(h, dZc, Hc);
        if (Nx <= 24) return launch_ks<24, (CH <= 512 ? CH : 512)>(h, dZc, Hc);
        return launch_ks<32, (CH <= 512 ? CH : 512)>(h, dZc, Hc);
    }
    return cudaErrorInvalidValue;                              // ks_chunk never picks 1024 above Nx = 12
}

static cudaError_t launch_ks(gpmpc_handle_t h, const double* dZc, int Hc)
{
    switch (ks_chunk(h)) {
    case 1024: return launch_ks_nx<1024>(h, dZc, Hc);
    case 512: return launch_ks_nx<512>(h, dZc, Hc);
    default: return launch_ks_nx<128>(h, dZc, Hc);
    }
}

// rows of Amat (h-major, stride HB*np per output) times T^T with T = Li or L (lower triangular):
// the solved rows go to Vout (may be null), their per-tile squared norms to dSQ
static int tri_product(gpmpc_handle_t h, const double* Amat, const double* T, int Hc, double* Vout)
{
    PredictParams p;
    psk_base(h, p, Hc);
    p.Vout = Vout; p.sV = (long long)HB * h->Npad; p.ldv = h->Npad;
    CUDA_TRY(psk_launch(h, p, Amat, T));
    return GPMPC_OK;
}

// r = ks - L v   (elementwise epilogue of the refinement residual) and v += dv
__global__ void axpby_rows_kernel(const double* __restrict__ x, const double* __restrict__ y, double a, double b,
                                  double* __restrict__ out, long long rowlen, long long srow, int rows)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int r = blockIdx.y, bz = blockIdx.z;
    if (i >= rowlen || r >= rows) return;
    const long long o = (long long)bz * srow + (long long)r * rowlen + i;
    out[o] = a * x[o] + b * y[o];
}

static int predict_core(gpmpc_handle_t h, int method, int H, const double* dZ, const double* dSigma, int spp,
                        double* d_mean, double* d_var, double* d_cov, double* d_jac)
{
    const int np = h->Npad, Nx = h->Nx;
    NvtxRange nvtx_r("gpmpc.predict");
    // fused epilogue + all-gather over peer memory when the exchange block is attached
    const int use_peers = (h->world > 1 && h->peer_ready && h->opt_peer && H <= h->peerHcap) ? 1 : 0;
    const int nccl_gather = (h->world > 1 && !use_peers) ? 1 : 0;
    const long long timeout_clocks = (long long)(h->opt_peer_timeout_s * 1e3 * (double)h->clock_khz);
    PeerArgs pa;
    memset(&pa, 0, sizeof(pa));
    if (use_peers) {
        h->peer_step += 1;
        for (int r = 0; r < h->world; ++r) pa.base[r] = h->peerBase[r];
        pa.world = h->world; pa.rank = h->rank;
        pa.goff = 2 * GPMPC_MAXW + (long long)(h->peer_step & 1) * h->peerGsz;
        pa.flag_idx = (int)(h->peer_step & 1) * GPMPC_MAXW + h->rank;
        pa.step = h->peer_step;
        pa.timeout_clocks = timeout_clocks;
    }
    AssembleArgs as = assemble_args(h, H, method, dSigma, spp, d_mean, d_var, d_jac, d_cov);
    if (use_peers) as.G = h->dPeerBlock + pa.goff;
    as.flags = use_peers ? reinterpret_cast<const unsigned long long*>(h->dPeerBlock.p) + (h->peer_step & 1) * GPMPC_MAXW : nullptr;
    as.world = h->world; as.step = h->peer_step; as.status = h->dPeerStatus; as.timeout_clocks = timeout_clocks;
    // one chunk and no NCCL call in between: the product kernel's last CTA assembles too (2 launches per step)
    // (it keeps J Sigma for all H points in the pipeline's shared memory: H Ny Nx doubles, >= 68 KB available)
    const bool fused_assemble = (H <= HB) && !nccl_gather && ((long long)H * h->Ny * Nx * 8 <= 64 * 1024);
    for (int h0 = 0; h0 < H; h0 += HB) {
        const int Hc = std::min(HB, H - h0);
        const bool last_chunk = (h0 + HB >= H);
        const double* dZc = dZ + (long long)h0 * Nx;
        CUDA_TRY(launch_ks(h, dZc, Hc));
        PredictParams p;
        psk_base(h, p, Hc);
        psk_finalize(h, p, H, h0);
        p.pa = pa; p.use_peers = use_peers; p.publish = last_chunk ? 1 : 0;
        p.as = as; p.do_assemble = (fused_assemble && !h->opt_refine) ? 1 : 0;
        if (!h->opt_refine) {
            CUDA_TRY(psk_launch(h, p, h->dKST, h->dLi));
        } else {
            // v1 = Li ks ; r = ks - L v1 ; v = v1 + Li r   (one step of iterative refinement)
            int rc = tri_product(h, h->dKST, h->dLi, Hc, h->dV);
            if (rc) return rc;
            rc = tri_product(h, h->dV, h->dL, Hc, h->dR);                      // dR = L v1
            if (rc) return rc;
            const int bm = round8(Hc);
            dim3 g((np + 255) / 256, bm, h->nloc);
            axpby_rows_kernel<<<g, 256, 0, h->st>>>(h->dKST, h->dR, 1.0, -1.0, h->dR, np, (long long)HB * np, bm);
            CUDA_TRY(cudaGetLastError());
            rc = tri_product(h, h->dR, h->dLi, Hc, h->dR2);                    // dR2 = Li r
            if (rc) return rc;
            axpby_rows_kernel<<<g, 256, 0, h->st>>>(h->dV, h->dR2, 1.0, 1.0, h->dV, np, (long long)HB * np, bm);
            CUDA_TRY(cudaGetLastError());
            sq_rows_kernel<<<dim3(np / 128, Hc, h->nloc), 128, 0, h->st>>>(h->dV, np, (long long)HB * np, h->dSQ, np / 128);
            CUDA_TRY(cudaGetLastError());
            finalize_kernel<<<h->nloc, PSK_THREADS, 0, h->st>>>(p);
            CUDA_TRY(cudaGetLastError());
        }
    }
    if (nccl_gather) {
        const size_t cnt = (size_t)h->nloc_max * H * (Nx + 2);
        int r = g_nccl.AllGather(h->dG + (size_t)h->rank * cnt, h->dG, cnt, 8 /* ncclFloat64 */, h->comm, h->st);
        if (r) { set_error(h, "ncclAllGather failed: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?"); return GPMPC_ERR_NCCL; }
    }
    if (!fused_assemble || h->opt_refine) {
        const int smem = (2 * h->Ny * Nx + h->Ny) * 8;
        assemble_kernel<<<std::min(H, 2048), 128, smem, h->st>>>(as);
        CUDA_TRY(cudaGetLastError());
    }
    return GPMPC_OK;
}

// ------------------------------------------------------------------------------------
// 'UT': the unscented transform around the unchanged 'ME' pass.  With n = Nx, lambda = alpha^2 (n + kappa) - n and
// c = sqrt(n + lambda), the 2n+1 sigma points of (z, Sigma) are z, then z + c S_j, z - c S_j for j = 1..n (S_j column j
// of the semidefinite lower Cholesky factor S of Sigma); the weights are W0m = lambda / (n + lambda),
// W0c = W0m + 1 - alpha^2 + beta, Wi = 1 / (2 (n + lambda)).  ut_sigma_kernel writes the points, predict_core evaluates
// 'ME' at all of them in one pass, ut_combine_kernel recombines: every sum runs in point order with separate multiplies
// and adds, so a point's results depend on its own inputs only.
// ------------------------------------------------------------------------------------
struct UtWeights { double c, wm0, wc0, wi; };

static UtWeights ut_weights(gpmpc_handle_t h)
{
    const double n = h->Nx, a2 = h->ut_alpha * h->ut_alpha, lam = a2 * (n + h->ut_kappa) - n;
    return {std::sqrt(n + lam), lam / (n + lam), lam / (n + lam) + 1.0 - a2 + h->ut_beta, 1.0 / (2.0 * (n + lam))};
}

// points of the pass behind H 'UT' points
static inline long long ut_points(gpmpc_handle_t h, long long H) { return H * (2LL * h->Nx + 1); }

// One warp per point p: S = the lower Cholesky factor of Sigma_p (Sigma or Sigma + p Nx^2) in shared memory, left-looking
// column by column.  A pivot <= 1e-14 max(diag Sigma), or <= 0, makes its column exactly zero (a semidefinite Sigma: a zero
// u-block, a rank-Ny feedback covariance).  Lane i owns row i.  Then the 2 Nx + 1 rows of point p into Zs.
__global__ void __launch_bounds__(32)
ut_sigma_kernel(const double* __restrict__ Z, const double* __restrict__ Sigma, int spp, int Nx, double c,
                double* __restrict__ Zs)
{
    __shared__ double L[NX_MAX * (NX_MAX + 1)];
    constexpr int LD = NX_MAX + 1;
    const int p = blockIdx.x, i = threadIdx.x;
    const double* S = Sigma + (spp ? (size_t)p * Nx * Nx : 0);
    for (int idx = i; idx < Nx * Nx; idx += 32) {
        const int r = idx / Nx, k = idx - r * Nx;
        L[r * LD + k] = k <= r ? S[idx] : 0.0;
    }
    __syncwarp();
    double dmax = 0.0;
    for (int k = 0; k < Nx; ++k) dmax = fmax(dmax, L[k * LD + k]);
    const double tol = 1e-14 * dmax;
    for (int j = 0; j < Nx; ++j) {
        double d = L[j * LD + j];                            // every lane forms the same pivot in the same order
        for (int k = 0; k < j; ++k) d = __dsub_rn(d, __dmul_rn(L[j * LD + k], L[j * LD + k]));
        const bool keep = d > tol;
        const double piv = keep ? sqrt(d) : 0.0;
        double s = 0.0;
        if (i > j && i < Nx) {
            s = L[i * LD + j];
            for (int k = 0; k < j; ++k) s = __dsub_rn(s, __dmul_rn(L[i * LD + k], L[j * LD + k]));
        }
        __syncwarp();
        if (i == j) L[j * LD + j] = piv;
        if (i > j && i < Nx) L[i * LD + j] = keep ? __ddiv_rn(s, piv) : 0.0;
        __syncwarp();
    }
    const double* z = Z + (size_t)p * Nx;
    double* out = Zs + (size_t)p * (2 * Nx + 1) * Nx;
    if (i < Nx) {
        const double ze = z[i];
        out[i] = ze;
        for (int j = 0; j < Nx; ++j) {
            const double s = __dmul_rn(c, L[i * LD + j]);
            out[(2 * j + 1) * Nx + i] = __dadd_rn(ze, s);
            out[(2 * j + 2) * Nx + i] = __dsub_rn(ze, s);
        }
    }
}

// One CTA per point p: the 2 Nx + 1 'ME' means m and variances v of its sigma points (rows p (2 Nx + 1) .. of the pass) ->
//   mean = sum_i Wim m_i,  cov = sum_i Wic (m_i - mean)(m_i - mean)^T + diag(sum_i Wim v_i),  var = diag(cov),
// each sum from i = 0 in point order; jac = the 'ME' Jacobian at z (row 0).  Every output may be null.
__global__ void __launch_bounds__(128)
ut_combine_kernel(const double* __restrict__ m, const double* __restrict__ v, const double* __restrict__ J, int Nx, int Ny,
                  double wm0, double wc0, double wi, double* __restrict__ mean, double* __restrict__ var,
                  double* __restrict__ cov, double* __restrict__ jac)
{
    extern __shared__ double ut_sh[];                        // mean (Ny) | sum_i Wim v_i (Ny)
    const int p = blockIdx.x, tid = threadIdx.x, np = 2 * Nx + 1;
    m += (size_t)p * np * Ny; v += (size_t)p * np * Ny;
    for (int a = tid; a < Ny; a += blockDim.x) {
        double s = 0.0, sv = 0.0;
        for (int k = 0; k < np; ++k) {
            const double w = k ? wi : wm0;
            s = __dadd_rn(s, __dmul_rn(w, m[k * Ny + a]));
            sv = __dadd_rn(sv, __dmul_rn(w, v[k * Ny + a]));
        }
        ut_sh[a] = s; ut_sh[Ny + a] = sv;
        if (mean) mean[(size_t)p * Ny + a] = s;
    }
    __syncthreads();
    const int n_out = cov ? Ny * Ny : (var ? Ny : 0);        // without cov only the diagonal is formed
    for (int idx = tid; idx < n_out; idx += blockDim.x) {
        const int a = cov ? idx / Ny : idx, b = cov ? idx - a * Ny : idx;
        const double ma = ut_sh[a], mb = ut_sh[b];
        double s = 0.0;
        for (int k = 0; k < np; ++k)
            s = __dadd_rn(s, __dmul_rn(k ? wi : wc0, __dmul_rn(__dsub_rn(m[k * Ny + a], ma), __dsub_rn(m[k * Ny + b], mb))));
        if (a == b) {
            s = __dadd_rn(s, ut_sh[Ny + a]);
            if (var) var[(size_t)p * Ny + a] = s;
        }
        if (cov) cov[(size_t)p * Ny * Ny + idx] = s;
    }
    if (jac)
        for (int idx = tid; idx < Ny * Nx; idx += blockDim.x)
            jac[(size_t)p * Ny * Nx + idx] = J[(size_t)p * np * Ny * Nx + idx];
}

// 'UT' at the H points dZ (H,Nx) with covariances dSigma (one, or one per point), device pointers: the sigma points into
// dUt, one 'ME' pass of predict_core over the H (2 Nx + 1) points (the caller's predict_prepare has laid out the
// buffers for that many), the recombination into the outputs (any may be null).
static int ut_pass(gpmpc_handle_t h, int H, const double* dZ, const double* dSigma, int spp, double* mean, double* var,
                   double* cov, double* jac)
{
    const int Nx = h->Nx, Ny = h->Ny;
    const long long Hs = ut_points(h, H);
    ENSURE(h->dUt, Hs * (Nx + 2 * Ny + (jac ? (long long)Ny * Nx : 0)));
    double* Zs = h->dUt;
    double* m = Zs + Hs * Nx;
    double* v = m + Hs * Ny;
    double* J = jac ? v + Hs * Ny : nullptr;
    const UtWeights w = ut_weights(h);
    ut_sigma_kernel<<<H, 32, 0, h->st>>>(dZ, dSigma, spp, Nx, w.c, Zs);
    CUDA_TRY(cudaGetLastError());
    const int rc = predict_core(h, GPMPC_METHOD_ME, (int)Hs, Zs, nullptr, 0, m, v, nullptr, J);
    if (rc) return rc;
    ut_combine_kernel<<<H, 128, 2 * Ny * 8, h->st>>>(m, v, J, Nx, Ny, w.wm0, w.wc0, w.wi, mean, var, cov, jac);
    CUDA_TRY(cudaGetLastError());
    return GPMPC_OK;
}

// ------------------------------------------------------------------------------------
// 'EM' exact moment matching (gp_functions.py:344-418): small dense helpers on the host
// (Nx <= 32), everything O(N), O(N^2) on the GPU
// ------------------------------------------------------------------------------------
static bool lu_factor(int n, double* A, int* piv, double* det)
{
    double d = 1.0;
    for (int k = 0; k < n; ++k) {
        int p = k; double mx = fabs(A[k * n + k]);
        for (int i = k + 1; i < n; ++i) if (fabs(A[i * n + k]) > mx) { mx = fabs(A[i * n + k]); p = i; }
        piv[k] = p;
        if (mx == 0.0) { *det = 0.0; return false; }
        if (p != k) { for (int j = 0; j < n; ++j) std::swap(A[k * n + j], A[p * n + j]); d = -d; }
        d *= A[k * n + k];
        for (int i = k + 1; i < n; ++i) {
            const double f = A[i * n + k] / A[k * n + k];
            A[i * n + k] = f;
            for (int j = k + 1; j < n; ++j) A[i * n + j] -= f * A[k * n + j];
        }
    }
    *det = d;
    return true;
}

static void lu_solve(int n, const double* LU, const int* piv, double* B, int m)
{
    for (int k = 0; k < n; ++k) if (piv[k] != k) for (int j = 0; j < m; ++j) std::swap(B[k * m + j], B[piv[k] * m + j]);
    for (int k = 0; k < n; ++k)
        for (int i = k + 1; i < n; ++i) { const double f = LU[i * n + k]; for (int j = 0; j < m; ++j) B[i * m + j] -= f * B[k * m + j]; }
    for (int k = n - 1; k >= 0; --k) {
        for (int j = 0; j < m; ++j) B[k * m + j] /= LU[k * n + k];
        for (int i = 0; i < k; ++i) { const double f = LU[i * n + k]; for (int j = 0; j < m; ++j) B[i * m + j] -= f * B[k * m + j]; }
    }
}

// pack the per-output / per-pair Nx x Nx quantities of one test point (layout: kernels.cuh)
static int em_prepare_point(gpmpc_handle_t h, const double* S, double* out)
{
    const int Nx = h->Nx, Ny = h->Ny, nn = Nx * Nx, m = Nx + 2;
    std::vector<double> R(nn), B(nn), lc(Ny);
    std::vector<int> piv(Nx);
    double det = 0.0;
    for (int a = 0; a < Ny; ++a) {
        const double* hp = &h->hyper[(size_t)a * m];
        for (int i = 0; i < Nx; ++i) for (int j = 0; j < Nx; ++j) R[i * Nx + j] = S[i * Nx + j] + (i == j ? hp[i] * hp[i] : 0.0);
        if (!lu_factor(Nx, R.data(), piv.data(), &det) || !(det > 0.0)) { set_error(h, "EM: Sigma + Lambda is not positive definite"); return GPMPC_ERR_ARG; }
        for (int i = 0; i < nn; ++i) B[i] = 0.0;
        for (int i = 0; i < Nx; ++i) B[i * Nx + i] = 1.0;
        lu_solve(Nx, R.data(), piv.data(), B.data(), Nx);                 // iR = (Sigma + Lambda)^-1   (:383-385)
        double* o = out + (size_t)a * (2 * nn + 2);
        memcpy(o, B.data(), nn * 8);
        double pe = 1.0;
        for (int d = 0; d < Nx; ++d) pe *= hp[d];
        o[nn] = hp[Nx] * hp[Nx] / sqrt(det) * pe;                         // c (:386-387)
        // G_a = Lambda^-1 Sigma (Sigma + Lambda)^-1  (= Lambda^-1 - (Sigma+Lambda)^-1, formed without the subtraction)
        for (int i = 0; i < Nx; ++i)
            for (int j = 0; j < Nx; ++j) {
                double sacc = 0.0;
                for (int k = 0; k < Nx; ++k) sacc += S[i * Nx + k] * B[k * Nx + j];
                o[nn + 1 + i * Nx + j] = sacc / (hp[i] * hp[i]);
            }
        // lc_a = log sf2_a - log c_a = 1/2 log det(I + Sigma Lambda^-1): determinant of I + small, not a difference of logs
        for (int i = 0; i < Nx; ++i) for (int j = 0; j < Nx; ++j) R[i * Nx + j] = S[i * Nx + j] / (hp[j] * hp[j]) + (i == j ? 1.0 : 0.0);
        if (!lu_factor(Nx, R.data(), piv.data(), &det) || !(det > 0.0)) { set_error(h, "EM: det(I + Sigma Lambda^-1) <= 0"); return GPMPC_ERR_ARG; }
        lc[a] = 0.5 * log(det);
        o[2 * nn + 1] = lc[a];
    }
    int p = 0;
    for (int a = 0; a < Ny; ++a)
        for (int b = 0; b <= a; ++b, ++p) {
            const double* ha = &h->hyper[(size_t)a * m];
            const double* hb = &h->hyper[(size_t)b * m];
            for (int i = 0; i < Nx; ++i)
                for (int j = 0; j < Nx; ++j)
                    R[i * Nx + j] = S[i * Nx + j] * (1.0 / (ha[j] * ha[j]) + 1.0 / (hb[j] * hb[j])) + (i == j ? 1.0 : 0.0);   // :396-397
            if (!lu_factor(Nx, R.data(), piv.data(), &det) || !(det > 0.0)) { set_error(h, "EM: det(R_ab) <= 0"); return GPMPC_ERR_ARG; }
            for (int i = 0; i < nn; ++i) B[i] = 0.5 * S[i];
            lu_solve(Nx, R.data(), piv.data(), B.data(), Nx);             // solve(R, Sigma/2)  (:402)
            double* o = out + (size_t)Ny * (2 * nn + 2) + (size_t)p * (nn + 4);
            memcpy(o, B.data(), nn * 8);
            o[nn] = 1.0 / sqrt(det); o[nn + 1] = a; o[nn + 2] = b;        // t (:398)
            o[nn + 3] = -0.5 * log(det) + lc[a] + lc[b];                  // log t + (log sf2_a - log c_a) + (log sf2_b - log c_b)
        }
    return GPMPC_OK;
}

// ------------------------------------------------------------------------------------
// The batched 'EM' forward (DESIGN 4.8): one launch set per chunk of points, each point in its own slice of the scratch
// (EmStrides).  The chunk is bounded by a byte budget, dominated by the two Npad^2 slabs per point (Q~ in dKinv, L^-1 Q~ in
// dU): 20 MB a point in all at Npad 1024, one point from Npad ~ 5800 on.
// ------------------------------------------------------------------------------------
#define EM_CHUNK_BYTES (1LL << 30)

static inline int em_npairs(gpmpc_handle_t h) { return h->Ny * (h->Ny + 1) / 2; }
static inline size_t em_per(gpmpc_handle_t h)     // doubles of one point's em_prepare_point block
{
    const size_t nn = (size_t)h->Nx * h->Nx;
    return (size_t)h->Ny * (2 * nn + 2) + (size_t)em_npairs(h) * (nn + 4);
}

static EmStrides em_strides(gpmpc_handle_t h)
{
    const long long np = h->Npad, Ny = h->Ny, npairs = em_npairs(h), T = (h->N + 63) / 64, Tq = np / 64;
    EmStrides s;
    s.z = h->Nx; s.emp = (long long)em_per(h);
    s.mpart = Ny * ((np + 255) / 256); s.pair = npairs * np; s.w = npairs * h->Nx * np;
    s.lq = Ny * np; s.part = npairs * T * T; s.q = slab(h);
    s.tr = Ny * (Tq * (Tq + 1) / 2); s.vec = 2 * np + Ny;
    return s;
}

// points per forward for H points: the byte budget, the grid's z extent of the pair sums (points x pairs) and em_points
static int em_chunk(gpmpc_handle_t h, int H)
{
    const EmStrides s = em_strides(h);
    const long long bytes = 8 * (2 * s.q + s.mpart + 4 * s.pair + 2 * s.w + s.lq + s.part + s.tr + s.vec);
    long long n = std::min<long long>({(long long)H, EM_CHUNK_BYTES / bytes, 65535 / em_npairs(h)});
    if (h->opt_em_points > 0) n = std::min<long long>(n, h->opt_em_points);
    return (int)std::max(1LL, n);
}

// scratch of one em_chunk of H points and the em_prepare_point blocks of all H
static int em_scratch(gpmpc_handle_t h, int H)
{
    const EmStrides s = em_strides(h);
    const int n = em_chunk(h, H);
    ENSURE(h->dEmTr, n * s.tr);
    ENSURE(h->dEmLQ, n * s.lq);
    ENSURE(h->dEmVec, n * s.vec);
    ENSURE(h->dEmE, n * s.pair); ENSURE(h->dEmF, n * s.pair);
    ENSURE(h->dEmE2, n * s.pair); ENSURE(h->dEmF2, n * s.pair);
    ENSURE(h->dEmW, n * s.w); ENSURE(h->dEmIJ, n * s.w);
    ENSURE(h->dEmMeanPart, n * s.mpart); ENSURE(h->dEmPart, n * s.part);
    { int rcs = ensure_kinv_scratch(h); if (rcs) return rcs; }
    ENSURE(h->dKinv, n * s.q); ENSURE(h->dU, n * s.q);
    ENSURE(h->dEMP, (long long)H * s.emp);
    return GPMPC_OK;
}

template <int NXP>
static cudaError_t launch_em_prep(gpmpc_handle_t h, int n, int npairs, const double* dz, const double* dEMP, int nblk, const EmStrides& s)
{
    dim3 g(nblk, h->Ny + npairs, n);
    em_prep_kernel<NXP><<<g, 256, 0, h->st>>>(h->dXT, h->Npad, h->N, h->Nx, h->Ny, npairs, h->dHyp, h->Nx + 2, h->dAlpha, h->Npad,
                                              dz, dEMP, h->dEmMeanPart, nblk, h->dEmE, h->dEmF, h->dEmW, h->dEmIJ, h->Npad, h->dEmLQ, h->dEmE2, h->dEmF2, s);
    return cudaGetLastError();
}

// The forward of n <= em_chunk points: z at dz (stride Nx, device), their em_prepare_point blocks at dP (stride em_per, device),
// mean / var / cov out at strides Ny / Ny / Ny^2 (device).  Point k's scratch stays in slot k for the derivative records.
static int em_forward(gpmpc_handle_t h, int n, const double* dz, const double* dP, double* mean, double* var, double* cov)
{
    const int Nx = h->Nx, Ny = h->Ny, np = h->Npad, npairs = em_npairs(h);
    const int nblk = (np + 255) / 256, T = (h->N + 63) / 64, Tq = np / 64, ntr = Tq * (Tq + 1) / 2;
    const EmStrides s = em_strides(h);
    CUDA_TRY(nxp_dispatch(Nx, [&](auto nxp) { return launch_em_prep<decltype(nxp)::value>(h, n, npairs, dz, dP, nblk, s); }));
    em_pair_kernel<<<dim3(T, T, n * npairs), 256, 2 * Nx * 64 * 8, h->st>>>(h->N, Nx, Ny, dP, h->dAlpha, np,
                                                                          h->dEmE, h->dEmF, h->dEmW, h->dEmIJ, np, h->dEmLQ, h->dEmE2, h->dEmF2, h->dEmPart, 0, 0, nullptr, 0, s);
    CUDA_TRY(cudaGetLastError());
    // E[var] term of the diagonal pairs, Cholesky-based: t tr(K^-1 Q_aa) = t tr(L^-1 Q_aa L^-T)
    for (int a = 0; a < Ny; ++a) {
        const int paa = a * (a + 1) / 2 + a;
        const double* Li = h->dLi + (long long)a * slab(h);
        em_pair_kernel<<<dim3(Tq, Tq, n), 256, 2 * Nx * 64 * 8, h->st>>>(h->N, Nx, Ny, dP, h->dAlpha, np,
                                                                      h->dEmE, h->dEmF, h->dEmW, h->dEmIJ, np, h->dEmLQ, h->dEmE2, h->dEmF2, nullptr, 1, paa, h->dKinv, np, s);
        CUDA_TRY(cudaGetLastError());
        // rank-one backbone: |L^-1 e^E|^2 (same kernels as alpha's first half)
        em_qvec_kernel<<<dim3((np + 255) / 256, 1, n), 256, 0, h->st>>>(h->dEmE + (long long)paa * np, h->N, np, h->dEmVec, s);
        CUDA_TRY(cudaGetLastError());
        trmv_lower_kernel<<<dim3((np + 7) / 8, 1, n), 256, 0, h->st>>>(Li, np, 0, h->dEmVec, s.vec, h->dEmVec + np, s.vec, np);
        CUDA_TRY(cudaGetLastError());
        sumsq_kernel<<<n, 256, 0, h->st>>>(h->dEmVec + np, s.vec, np, h->dEmVec + 2LL * np + a, s.vec);
        CUDA_TRY(cudaGetLastError());
        // L^-1 Q~ of every point: the same L^-1 (sA = 0), the feed of one slab so each point keeps its lone bits
        GemmParams gp;
        memset(&gp, 0, sizeof(gp));
        gp.A = Li; gp.lda = np;
        gp.B = h->dKinv; gp.ldb = np; gp.sB = s.q;    // Q symmetric: row-major (j,k) storage is the NT operand
        gp.C = h->dU; gp.ldc = np; gp.sC = s.q;
        gp.mt = np / 128; gp.nt = np / 128; gp.K = np; gp.alpha = 1.0; gp.beta = 0.0;
        gp.kflags = GEMM_KI_LE; gp.lower = 1;
        CUDA_TRY(gemm128(h, h->st, true, gp, n, 1));
        em_trdot_kernel<<<dim3(ntr, n), 256, 0, h->st>>>(h->dU, Li, np, h->dEmTr + (long long)a * ntr, s);
        CUDA_TRY(cudaGetLastError());
    }
    em_finalize_kernel<<<n, 1024, 0, h->st>>>(Nx, Ny, npairs, dP, h->dHyp, Nx + 2, h->dEmMeanPart, nblk, h->dEmPart, T * T,
                                              h->dEmTr, ntr, h->dEmVec + 2LL * np, mean, var, cov, s);
    CUDA_TRY(cudaGetLastError());
    return GPMPC_OK;
}

// ------------------------------------------------------------------------------------
// 'EM' derivatives w.r.t. z and Sigma (DESIGN 4.8).  Per point, after the forward chain, the O(N) / O(N^2) sums go into
// records of total degree D (kernels.cuh, em_owner_rec_kernel / em_pair_rec_kernel; EmTables):
//   D = 2 (gpmpc_predict_em_grad): the host forms the Nx x Nx first derivatives from them (em_grad_finish).
//   D = 4 (gpmpc_predict_em_hess): every term of mean and cov is a Gaussian expectation, Gaussian in z, so its
//     z-derivatives are Hermite polynomials of (y, S): He_1 = y, He_2 = y y - S, He_3 = y y y - 3 sym(S y),
//     He_4 = y^4 - 6 sym(S y y) + 3 sym(S S); and d/dSigma = 1/2 d^2/dz^2 (heat equation).  The device forms
//     d^k mean_a / dz^k (k <= 4) and d^k cov_ab / dz^k (k = 2..4) from the records and assembles the Sigma blocks.
// ------------------------------------------------------------------------------------
struct EmGradOutputs {
    double *dmean_dz, *dmean_dSigma, *dcov_dz, *dcov_dSigma;
};

struct EmHessOutputs {
    double *d2mean_dz2, *d2mean_dSigma_dz, *d2mean_dSigma2, *d2cov_dz2, *d2cov_dSigma_dz, *d2cov_dSigma2;
};

// the records of one point (EmTables::nrec order) into rec_out, through R's partials and backbone rows
template <int NXP, int D>
static cudaError_t launch_em_records(gpmpc_handle_t h, const EmRecords& R, const double* dz, const double* dP, int npairs,
                                     int nb, int slot, double* rec_out)
{
    const EmStrides s = em_strides(h);
    const double *E = h->dEmE + slot * s.pair, *F = h->dEmF + slot * s.pair, *E2 = h->dEmE2 + slot * s.pair;
    const double *F2 = h->dEmF2 + slot * s.pair, *W = h->dEmW + slot * s.w, *IJ = h->dEmIJ + slot * s.w;
    const double* LQ = h->dEmLQ + slot * s.lq;
    const EmTables& tb = *R.tb;
    const int N = h->N, Nx = h->Nx, Ny = h->Ny, np = h->Npad, nf = tb.nf, RL = tb.nent;
    constexpr int NFP = em_nmono(NXP, D / 2);
    const int r_cross = Ny, r_tr = Ny + 2 * npairs, r_bb = r_tr + Ny, r_gram = r_bb + Ny;
    const int* MONO = R.idx;
    const int* ENT = MONO + tb.mono.size();
    double* part = R.part;
    const long long srec = (long long)nb * RL;
    const int smem_pair = (3 * NXP * 64 + 64 * 65 + NFP * 64) * 8, smem_own = (NXP * 64 + 64 * NFP) * 8;
    cudaError_t e = smem_opt_in<em_pair_rec_kernel<NXP, D>>(smem_pair);
    if (e == cudaSuccess) e = smem_opt_in<em_owner_rec_kernel<NXP, D>>(smem_own);
    if (e != cudaSuccess) return e;
    em_owner_rec_kernel<NXP, D><<<dim3(nb, Ny), 256, smem_own, h->st>>>(h->dXT, np, N, Nx, dz, h->dAlpha, LQ, np, nullptr, 0, 0, 1,
                                                                         MONO, ENT, RL, part, srec);
    em_pair_rec_kernel<NXP, D><<<dim3(nb, npairs, 2), 256, smem_pair, h->st>>>(N, Nx, Ny, dP, h->dAlpha, np, h->dXT, np, dz, E,
                                                                               F, W, IJ, np, LQ, E2, F2,
                                                                               nullptr, 0, r_cross, MONO, ENT, RL, part, nb);
    em_pair_rec_kernel<NXP, D><<<dim3(nb, Ny, 1), 256, smem_pair, h->st>>>(N, Nx, Ny, dP, h->dAlpha, np, h->dXT, np, dz, E,
                                                                           F, W, IJ, np, LQ, E2, F2,
                                                                           h->dEmKinv, 1, r_tr, MONO, ENT, RL, part, nb);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    // rank-one backbone e e^T of Q_aa: rows e o mono_f for the nf features through L^-1 in one batched trmv.
    // D = 2: K^-1 e = L^-T (L^-1 e), owner records of e_i (K^-1 e)_i, and the Gram Y^T Y of Y_d = L^-1 (e o v_d).
    // D = 4: Z_f = K^-1 (e o mono_f) = L^-T L^-1 (e o mono_f) for every feature, owner records with features e_i Z_f,i.
    const int nkz = D == 2 ? 1 : nf;
    double* rows = R.bb;
    double* prod = rows + (long long)nf * np;
    double* kz = prod + (long long)nf * np;
    for (int a = 0; a < Ny; ++a) {
        const int paa = a * (a + 1) / 2 + a;
        const double* Li = h->dLi + (long long)a * slab(h);
        em_backbone_rows_kernel<<<(np + 255) / 256, 256, 0, h->st>>>(h->dXT, np, N, Nx, dz, E + (long long)paa * np, np, MONO, nf, rows);
        trmv_lower_kernel<<<dim3((np + 7) / 8, 1, nf), 256, 0, h->st>>>(Li, np, 0, rows, np, prod, np, np);
        trmv_lower_T_kernel<<<dim3(np / 32, 1, nkz), 256, 0, h->st>>>(Li, np, 0, prod, np, kz, np, np);
        em_owner_rec_kernel<NXP, D><<<dim3(nb, 1), 256, smem_own, h->st>>>(h->dXT, np, N, Nx, dz, nullptr, E + (long long)paa * np, 0,
                                                                            kz, 0, np, nkz, MONO, ENT, RL, part + (long long)(r_bb + a) * srec, 0);
        if (D == 2)
            em_owner_rec_kernel<NXP, D><<<dim3(nb, 1), 256, smem_own, h->st>>>(prod + np, np, N, Nx, nullptr, nullptr, nullptr, 0, nullptr, 0, 0, 1,
                                                                                MONO, ENT, RL, part + (long long)(r_gram + a) * srec, 0);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
    }
    em_sum_parts_kernel<<<tb.nrec(Ny), 256, 0, h->st>>>(part, nb, RL, rec_out);
    return cudaGetLastError();
}

// n x n helpers for the host side of the EM derivatives
static void mat_mul(int n, const double* A, const double* B, double* C, bool bt = false)
{
    for (int i = 0; i < n; ++i)
        for (int j = 0; j < n; ++j) {
            double s = 0.0;
            for (int k = 0; k < n; ++k) s += A[i * n + k] * (bt ? B[j * n + k] : B[k * n + j]);
            C[i * n + j] = s;
        }
}

static bool mat_inv(int n, const double* A, double* Ai)
{
    std::vector<double> LU(A, A + n * n);
    std::vector<int> piv(n);
    double det = 0.0;
    if (!lu_factor(n, LU.data(), piv.data(), &det)) return false;
    for (int i = 0; i < n * n; ++i) Ai[i] = 0.0;
    for (int i = 0; i < n; ++i) Ai[i * n + i] = 1.0;
    lu_solve(n, LU.data(), piv.data(), Ai, n);
    return true;
}

// The per-pair matrices of the 'EM' derivatives (O(Nx^3), host): ila, ilb = diag of La^-1, Lb^-1 (inverse squared
// lengthscales of outputs a and b), C = (I + P Sigma)^-1, Fa = C La^-1, Fb = C Lb^-1, CP = C P,
// A = -C Lb^-1 Sigma iR_a = C La^-1 - iR_a and B = -C La^-1 Sigma iR_b (formed as products, without the subtraction)
struct EmPairMats {
    int Nx;
    std::vector<double> ila, ilb, C, Fa, Fb, CP, A, B, t;
    explicit EmPairMats(int nx)
        : Nx(nx), ila(nx), ilb(nx), C(nx * nx), Fa(nx * nx), Fb(nx * nx), CP(nx * nx), A(nx * nx), B(nx * nx), t(nx * nx) {}
    int form(gpmpc_handle_t h, const double* S, int a, int b, const double* iRa, const double* iRb)
    {
        const int nn = Nx * Nx, m = Nx + 2;
        const double* la = &h->hyper[(size_t)a * m];
        const double* lb = &h->hyper[(size_t)b * m];
        for (int d = 0; d < Nx; ++d) { ila[d] = 1.0 / (la[d] * la[d]); ilb[d] = 1.0 / (lb[d] * lb[d]); }
        for (int i = 0; i < Nx; ++i)
            for (int j = 0; j < Nx; ++j) t[i * Nx + j] = (i == j ? 1.0 : 0.0) + (ila[i] + ilb[i]) * S[i * Nx + j];
        if (!mat_inv(Nx, t.data(), C.data())) { set_error(h, "EM: I + P Sigma is singular"); return GPMPC_ERR_ARG; }
        for (int i = 0; i < Nx; ++i)
            for (int j = 0; j < Nx; ++j) {
                Fa[i * Nx + j] = C[i * Nx + j] * ila[j]; Fb[i * Nx + j] = C[i * Nx + j] * ilb[j];
                CP[i * Nx + j] = C[i * Nx + j] * (ila[j] + ilb[j]);
            }
        mat_mul(Nx, Fb.data(), S, t.data()); mat_mul(Nx, t.data(), iRa, A.data());
        mat_mul(Nx, Fa.data(), S, t.data()); mat_mul(Nx, t.data(), iRb, B.data());
        for (int q = 0; q < nn; ++q) { A[q] = -A[q]; B[q] = -B[q]; }
        return GPMPC_OK;
    }
};

// first derivatives of one point from its D = 2 records (DESIGN 4.8).  emp: the point's em_prepare_point block (iR_a, t_ab),
// rec: its records, mean: its Ny means.  d/dSigma is symmetrised (the gradient at a symmetric Sigma is symmetric).
static int em_grad_finish(gpmpc_handle_t h, const EmTables& tb, const double* S, const double* emp, const double* rec,
                          const double* mean, double* dmz, double* dmS, double* dcz, double* dcS)
{
    const int Nx = h->Nx, Ny = h->Ny, nn = Nx * Nx, npairs = Ny * (Ny + 1) / 2;
    const int r_cross = Ny, r_tr = Ny + 2 * npairs, r_bb = r_tr + Ny, r_gram = r_bb + Ny;
    const int *M1 = tb.mid[1].data(), *M2 = tb.mid[2].data();
    // entry (owner monomial mo, feature f) of record r: at(r, 0, 0) = sum m, at(r, M1[d], 0) = sum m v_d,
    // at(r, M2[d Nx + e], 0) = sum m v_d v_e, at(r, 0, M1[e]) = sum m v'_e and at(r, M1[d], M1[e]) = sum m v_d v'_e
    // (v' the other index's v)
    auto at = [&](int r, int mo, int f) { return rec[(size_t)r * tb.nent + tb.entpos[(size_t)mo * tb.nf + f]]; };
    auto sym_store = [&](const double* G, double* o1, double* o2) {
        for (int d = 0; d < Nx; ++d)
            for (int e = 0; e <= d; ++e) {
                const double v = 0.5 * (G[d * Nx + e] + G[e * Nx + d]);
                o1[d * Nx + e] = o1[e * Nx + d] = v;
                if (o2) o2[d * Nx + e] = o2[e * Nx + d] = v;
            }
    };
    std::vector<double> t1(nn), t2(nn), t3(nn), G(nn), Z1(nn), dz(Nx), ga(Nx), gb(Nx);
    std::vector<double> s1((size_t)Ny * Nx), s2((size_t)Ny * nn), u1(Nx), u2(Nx), Mii(nn), Mij(nn), Mjj(nn);
    for (int a = 0; a < Ny; ++a) {
        const double* iR = emp + (size_t)a * (2 * nn + 2);
        double* sa = &s1[(size_t)a * Nx];
        double* Sa = &s2[(size_t)a * nn];
        for (int d = 0; d < Nx; ++d) {
            sa[d] = at(a, M1[d], 0);
            for (int e = 0; e < Nx; ++e) Sa[d * Nx + e] = at(a, M2[d * Nx + e], 0);
        }
        for (int d = 0; d < Nx; ++d) {
            double s = 0.0;
            for (int k = 0; k < Nx; ++k) s += iR[d * Nx + k] * sa[k];
            if (dmz) dmz[(size_t)a * Nx + d] = s;
        }
        mat_mul(Nx, iR, Sa, t1.data());
        mat_mul(Nx, t1.data(), iR, G.data());
        for (int q = 0; q < nn; ++q) G[q] = 0.5 * G[q] - 0.5 * mean[a] * iR[q];
        if (dmS) sym_store(G.data(), dmS + (size_t)a * nn, nullptr);
    }
    EmPairMats pm(Nx);
    const double *ila = pm.ila.data(), *ilb = pm.ilb.data(), *C = pm.C.data(), *Fa = pm.Fa.data(), *Fb = pm.Fb.data();
    const double *CP = pm.CP.data(), *A = pm.A.data(), *B = pm.B.data();
    int p = 0;
    for (int a = 0; a < Ny; ++a)
        for (int b = 0; b <= a; ++b, ++p) {
            const double* iRa = emp + (size_t)a * (2 * nn + 2);
            const double* iRb = emp + (size_t)b * (2 * nn + 2);
            const double t = emp[(size_t)Ny * (2 * nn + 2) + (size_t)p * (nn + 4) + nn];
            const double Ma = mean[a], Mb = mean[b];
            const double *sa = &s1[(size_t)a * Nx], *Sa = &s2[(size_t)a * nn], *sb = &s1[(size_t)b * Nx], *Sb = &s2[(size_t)b * nn];
            const int rc = pm.form(h, S, a, b, iRa, iRb);
            if (rc) return rc;
            // cross records: owner rows r0 (u1 = sum m v_i, Mii, Mij = sum m v_i v_j^T, u2 = sum m v_j), owner columns r1 (Mjj)
            const int r0 = r_cross + 2 * p, r1 = r0 + 1;
            for (int d = 0; d < Nx; ++d) {
                u1[d] = at(r0, M1[d], 0); u2[d] = at(r0, 0, M1[d]);
                for (int e = 0; e < Nx; ++e) {
                    Mii[d * Nx + e] = at(r0, M2[d * Nx + e], 0); Mjj[d * Nx + e] = at(r1, M2[d * Nx + e], 0);
                    Mij[d * Nx + e] = at(r0, M1[d], M1[e]);
                }
            }
            // d/dz: iR_a u1 + iR_b u2 + A (u1 + s_a Mb) + B (u2 + Ma s_b)
            for (int d = 0; d < Nx; ++d) {
                double s = 0.0;
                for (int k = 0; k < Nx; ++k)
                    s += iRa[d * Nx + k] * u1[k] + iRb[d * Nx + k] * u2[k] + A[d * Nx + k] * (u1[k] + sa[k] * Mb) + B[d * Nx + k] * (u2[k] + Ma * sb[k]);
                dz[d] = s;
            }
            // d/dSigma: 1/2 C Z1 C^T - 1/2 (sum m) C P  (the expm1 part), Z1 = sum m zeta zeta^T
            for (int d = 0; d < Nx; ++d)
                for (int e = 0; e < Nx; ++e)
                    Z1[d * Nx + e] = Mii[d * Nx + e] * ila[d] * ila[e] + Mij[d * Nx + e] * ila[d] * ilb[e]
                                   + Mij[e * Nx + d] * ilb[d] * ila[e] + Mjj[d * Nx + e] * ilb[d] * ilb[e];
            mat_mul(Nx, C, Z1.data(), t1.data()); mat_mul(Nx, t1.data(), C, G.data(), true);
            const double m0 = at(r0, 0, 0);
            for (int q = 0; q < nn; ++q) G[q] = 0.5 * G[q] - 0.5 * m0 * CP[q];
            // + sum_ij w_ij d delta_ij: w is rank one, so these are products of the per-output moments
            auto add_side = [&](const double* X, const double* S_, const double* iR, double scale) {   // scale (X S iR + iR S X^T + X S X^T) / 2
                mat_mul(Nx, X, S_, t1.data());
                mat_mul(Nx, t1.data(), iR, t2.data());
                mat_mul(Nx, t1.data(), X, t3.data(), true);
                for (int d = 0; d < Nx; ++d)
                    for (int e = 0; e < Nx; ++e) G[d * Nx + e] += 0.5 * scale * (t2[d * Nx + e] + t2[e * Nx + d] + t3[d * Nx + e]);
            };
            add_side(A, Sa, iRa, Mb);
            add_side(B, Sb, iRb, Ma);
            for (int d = 0; d < Nx; ++d) {
                ga[d] = 0.0; gb[d] = 0.0;
                for (int k = 0; k < Nx; ++k) { ga[d] += Fa[d * Nx + k] * sa[k]; gb[d] += Fb[d * Nx + k] * sb[k]; }
            }
            for (int d = 0; d < Nx; ++d)
                for (int e = 0; e < Nx; ++e)
                    G[d * Nx + e] += 0.5 * (ga[d] * gb[e] + gb[d] * ga[e]) - 0.5 * (A[d * Nx + e] + B[d * Nx + e]) * Ma * Mb;
            if (a == b) {       // - d T_a, T_a = t tr(K^-1 Q_aa): backbone records plus the remainder's
                const int rt = r_tr + a, rb = r_bb + a, rg = r_gram + a;
                const double T = t * (at(rb, 0, 0) + at(rt, 0, 0));
                for (int d = 0; d < Nx; ++d) {
                    double s = 0.0;
                    for (int k = 0; k < Nx; ++k) s += Fa[d * Nx + k] * t * (at(rb, M1[k], 0) + at(rt, M1[k], 0));
                    dz[d] -= 2.0 * s;
                }
                for (int d = 0; d < Nx; ++d)
                    for (int e = 0; e < Nx; ++e) {
                        const int m2 = M2[d * Nx + e];
                        Z1[d * Nx + e] = t * (at(rb, m2, 0) + at(rt, m2, 0) + at(rg, m2, 0) + at(rt, M1[d], M1[e]));
                    }
                mat_mul(Nx, Fa, Z1.data(), t1.data()); mat_mul(Nx, t1.data(), Fa, t2.data(), true);
                for (int q = 0; q < nn; ++q) G[q] -= t2[q] - 0.5 * T * CP[q];
            }
            if (dcz)
                for (int d = 0; d < Nx; ++d) dcz[((size_t)a * Ny + b) * Nx + d] = dcz[((size_t)b * Ny + a) * Nx + d] = dz[d];
            if (dcS) sym_store(G.data(), dcS + ((size_t)a * Ny + b) * nn, dcS + ((size_t)b * Ny + a) * nn);
        }
    return GPMPC_OK;
}

// per (point, pair) inputs of em_hess_pair_finish_kernel (EmPairMats): [Fa Fb CP At Bt sAt sBt sFa sFb] (Nx^2 each), t;
// CP as its symmetric part, At = A = Fa - iR_a and Bt = B = Fb - iR_b, sX = symmetric part of X
static int em_hess_pair_params(gpmpc_handle_t h, const double* S, const double* emp, double* out)
{
    const int Nx = h->Nx, Ny = h->Ny, nn = Nx * Nx;
    EmPairMats pm(Nx);
    int p = 0;
    for (int a = 0; a < Ny; ++a)
        for (int b = 0; b <= a; ++b, ++p) {
            const double* iRa = emp + (size_t)a * (2 * nn + 2);
            const double* iRb = emp + (size_t)b * (2 * nn + 2);
            const int rc = pm.form(h, S, a, b, iRa, iRb);
            if (rc) return rc;
            double* o = out + (size_t)p * (9 * nn + 1);
            double *Fa = o, *Fb = o + nn, *CP = o + 2 * nn, *At = o + 3 * nn, *Bt = o + 4 * nn, *sAt = o + 5 * nn;
            double *sBt = o + 6 * nn, *sFa = o + 7 * nn, *sFb = o + 8 * nn;
            std::copy(pm.Fa.begin(), pm.Fa.end(), Fa); std::copy(pm.Fb.begin(), pm.Fb.end(), Fb);
            std::copy(pm.CP.begin(), pm.CP.end(), CP);
            std::copy(pm.A.begin(), pm.A.end(), At); std::copy(pm.B.begin(), pm.B.end(), Bt);
            for (int i = 0; i < Nx; ++i)        // CP = (P^-1 + Sigma)^-1 is symmetric: use the symmetric part
                for (int j = 0; j < i; ++j) CP[i * Nx + j] = CP[j * Nx + i] = 0.5 * (CP[i * Nx + j] + CP[j * Nx + i]);
            for (int i = 0; i < Nx; ++i)
                for (int j = 0; j < Nx; ++j) {
                    sAt[i * Nx + j] = 0.5 * (At[i * Nx + j] + At[j * Nx + i]); sBt[i * Nx + j] = 0.5 * (Bt[i * Nx + j] + Bt[j * Nx + i]);
                    sFa[i * Nx + j] = iRa[i * Nx + j] + sAt[i * Nx + j]; sFb[i * Nx + j] = iRb[i * Nx + j] + sBt[i * Nx + j];
                }
            o[9 * nn] = emp[(size_t)Ny * (2 * nn + 2) + (size_t)p * (nn + 4) + nn];
        }
    return GPMPC_OK;
}

// The record set of degree D for H points: its tables built and uploaded once, the block partials, the records of H points
// and the backbone rows
static int em_records_prepare(gpmpc_handle_t h, int D, int H)
{
    const int Ny = h->Ny, T = (h->N + 63) / 64;
    EmRecords& R = h->em_rec[D / 2 - 1];
    if (!R.tb) R.tb.reset(new EmTables(h->Nx, D));
    EmTables& tb = *R.tb;
    ENSURE(R.part, (long long)tb.nrec(Ny) * T * tb.nent);
    ENSURE(R.rec, (long long)H * tb.nrec(Ny) * tb.nent);
    ENSURE(R.bb, 3LL * tb.nf * h->Npad);
    ENSURE(R.idx, (long long)tb.dev.size());
    if (tb.uploaded_to != R.idx.p) {
        CUDA_TRY(cudaMemcpyAsync(R.idx, tb.dev.data(), tb.dev.size() * 4, cudaMemcpyHostToDevice, h->st));
        tb.uploaded_to = R.idx.p;
    }
    return GPMPC_OK;
}

// The full symmetric K^-1 of every output that the records' trace terms read (dEmKinv, 8 B Ny Npad^2, kept until the next
// factor change)
static int em_kinv_prepare(gpmpc_handle_t h)
{
    const int np = h->Npad;
    ENSURE(h->dEmKinv, (long long)h->Ny * slab(h));
    if (!h->em_kinv_valid) {        // K^-1 = U U^T per output (compute_kinv, lower), stored full and symmetric
        for (int a = 0; a < h->Ny; ++a) {
            int rck = compute_kinv(h, a);
            if (rck) return rck;
            sym_from_lower_kernel<<<dim3(np / 32, np / 32), dim3(32, 8), 0, h->st>>>(h->dKinv, h->dEmKinv + (long long)a * slab(h), np);
            CUDA_TRY(cudaGetLastError());
        }
        h->em_kinv_valid = true;
    }
    return GPMPC_OK;
}

// The 'EM' pass over H points, shared by predict_em and the 'EM' roll-out step: z at dz (device, stride Nx), Sigma on the
// host (one per point with spp, else shared).  Every point's em_prepare_point block goes to emp (host, em_per doubles a
// point; the caller keeps it for the derivative finishes) and then up to dEMP.  Per em_chunk of points em_forward writes
// mean / var / cov (device, strides Ny / Ny / Ny^2); then, from the scratch slots that forward left (the next chunk
// overwrites them), each point's records of degree 2 go to em_rec[0].rec when rec2 and of degree 4 to em_rec[1].rec when
// rec4.  When em_prepare_point rejects a point, its error code returns and *bad (if given) is that point.
static int em_pass(gpmpc_handle_t h, int H, const double* dz, const double* Sigma, int spp, double* emp, double* mean,
                   double* var, double* cov, bool rec2, bool rec4, int* bad = nullptr)
{
    const int Nx = h->Nx, Ny = h->Ny, nn = Nx * Nx, npairs = em_npairs(h), T = (h->N + 63) / 64, nc = em_chunk(h, H);
    const size_t per = em_per(h);
    const EmRecords& R2 = h->em_rec[0];
    const EmRecords& R4 = h->em_rec[1];
    for (int p = 0; p < H; ++p) {
        const int rc = em_prepare_point(h, Sigma + (spp ? (size_t)p * nn : 0), emp + (size_t)p * per);
        if (rc) {
            if (bad) *bad = p;
            return rc;
        }
    }
    CUDA_TRY(cudaMemcpyAsync(h->dEMP, emp, (size_t)H * per * 8, cudaMemcpyHostToDevice, h->st));
    for (int c0 = 0; c0 < H; c0 += nc) {
        const int n = std::min(nc, H - c0);
        const double* zc = dz + (size_t)c0 * Nx;
        const double* Pc = h->dEMP + (size_t)c0 * per;
        const int rc = em_forward(h, n, zc, Pc, mean + (size_t)c0 * Ny, var + (size_t)c0 * Ny, cov + (size_t)c0 * Ny * Ny);
        if (rc) return rc;
        for (int k = 0; k < n && (rec2 || rec4); ++k) {
            const size_t p = (size_t)c0 + k;
            const double* z = zc + (size_t)k * Nx;
            const double* P = Pc + (size_t)k * per;
            if (rec2) {
                double* rec = R2.rec + p * R2.tb->nrec(Ny) * R2.tb->nent;
                CUDA_TRY(nxp_dispatch(Nx, [&](auto nxp) { return launch_em_records<decltype(nxp)::value, 2>(h, R2, z, P, npairs, T, k, rec); }));
            }
            if (rec4) {
                double* rec = R4.rec + p * R4.tb->nrec(Ny) * R4.tb->nent;
                CUDA_TRY((Nx <= 8 ? launch_em_records<8, 4>(h, R4, z, P, npairs, T, k, rec)
                                  : launch_em_records<16, 4>(h, R4, z, P, npairs, T, k, rec)));   // Nx <= 16
            }
        }
    }
    return GPMPC_OK;
}

// The first-derivative finish of H points after em_pass with rec2: the D = 2 records and the means (dmean, device) to the
// host, one synchronisation, then em_grad_finish per point with Sigma (one per point with spp, else shared) and em_pass's
// blocks emp; point p's outputs at p times their block in go (null members skipped).  On failure *bad (if given) is the
// failing point.
static int em_grad_finish_points(gpmpc_handle_t h, int H, const double* Sigma, int spp, const double* emp,
                                 const double* dmean, const EmGradOutputs& go, int* bad = nullptr)
{
    const int Nx = h->Nx, Ny = h->Ny, nn = Nx * Nx;
    const EmRecords& R2 = h->em_rec[0];
    const EmTables& tb = *R2.tb;
    const size_t per = em_per(h), rl = (size_t)tb.nrec(Ny) * tb.nent;
    std::vector<double> recs((size_t)H * rl), mh((size_t)H * Ny);
    CUDA_TRY(cudaMemcpyAsync(recs.data(), R2.rec, recs.size() * 8, cudaMemcpyDeviceToHost, h->st));
    CUDA_TRY(cudaMemcpyAsync(mh.data(), dmean, mh.size() * 8, cudaMemcpyDeviceToHost, h->st));
    CUDA_TRY(cudaStreamSynchronize(h->st));
    for (int p = 0; p < H; ++p) {
        const int rc = em_grad_finish(h, tb, Sigma + (spp ? (size_t)p * nn : 0), emp + (size_t)p * per, recs.data() + (size_t)p * rl,
                                      mh.data() + (size_t)p * Ny,
                                      go.dmean_dz ? go.dmean_dz + (size_t)p * Ny * Nx : nullptr,
                                      go.dmean_dSigma ? go.dmean_dSigma + (size_t)p * Ny * nn : nullptr,
                                      go.dcov_dz ? go.dcov_dz + (size_t)p * Ny * Ny * Nx : nullptr,
                                      go.dcov_dSigma ? go.dcov_dSigma + (size_t)p * Ny * Ny * nn : nullptr);
        if (rc) {
            if (bad) *bad = p;
            return rc;
        }
    }
    return GPMPC_OK;
}

static int predict_em(gpmpc_handle_t h, int H, const double* Z, const double* Sigma, int spp,
                      double* mean, double* var, double* cov, const EmGradOutputs* go = nullptr,
                      const EmHessOutputs* ho = nullptr)
{
    const int Nx = h->Nx, Ny = h->Ny, nn = Nx * Nx;
    NvtxRange nvtx_r("gpmpc.predict_em");
    if (!Sigma) { set_error(h, "EM needs an input covariance"); return GPMPC_ERR_ARG; }
    const int npairs = em_npairs(h);
    if (npairs > 1024) { set_error(h, "EM supports Ny <= 44"); return GPMPC_ERR_ARG; }
    const size_t per = em_per(h);
    { const int rcs = em_scratch(h, H); if (rcs) return rcs; }
    if (go) { const int rc = em_records_prepare(h, 2, H); if (rc) return rc; }
    const long long TS = 1 + Nx + nn + (long long)nn * Nx + (long long)nn * nn, Q = (long long)nn * nn;
    const long long per_pair = 6 * TS + 8 * Q, nout = (long long)nn + nn * Nx + nn * nn;    // finish scratch per CTA; one output slab
    const int Hc = (int)std::max(1LL, std::min((long long)H, (64LL << 20) / ((long long)npairs * per_pair)));   // points per finish launch
    if (ho) {
        const int rc = em_records_prepare(h, 4, H);
        if (rc) return rc;
        ENSURE(h->dEmHEHP, (long long)H * npairs * (9 * nn + 1));
        ENSURE(h->dEmHMU, (long long)H * Ny * TS);
        ENSURE(h->dEmHD, (long long)H * Ny * TS);
        ENSURE(h->dEmHScr, std::max((long long)H * Ny * Q, (long long)Hc * npairs * per_pair));
        ENSURE(h->dEmHOut, (long long)H * (Ny + Ny * Ny) * nout);
    }
    if (go || ho) { const int rc = em_kinv_prepare(h); if (rc) return rc; }
    CUDA_TRY(cudaMemcpyAsync(h->dZ, Z, (size_t)H * Nx * 8, cudaMemcpyHostToDevice, h->st));
    std::vector<double> emp((size_t)H * per);
    const int rc = em_pass(h, H, h->dZ, Sigma, spp, emp.data(), h->dMean, h->dVar, h->dCov, go != nullptr, ho != nullptr);
    if (rc) return rc;
    if (mean) CUDA_TRY(cudaMemcpyAsync(mean, h->dMean, (size_t)H * Ny * 8, cudaMemcpyDeviceToHost, h->st));
    if (var) CUDA_TRY(cudaMemcpyAsync(var, h->dVar, (size_t)H * Ny * 8, cudaMemcpyDeviceToHost, h->st));
    if (cov) CUDA_TRY(cudaMemcpyAsync(cov, h->dCov, (size_t)H * Ny * Ny * 8, cudaMemcpyDeviceToHost, h->st));
    if (ho) {           // the derivatives from the records, on the device: mean part, then the pairs in chunks of points
        std::vector<double> ehp((size_t)H * npairs * (9 * nn + 1));
        for (int p = 0; p < H; ++p) {
            const int rc = em_hess_pair_params(h, Sigma + (spp ? (size_t)p * nn : 0), emp.data() + (size_t)p * per,
                                               ehp.data() + (size_t)p * npairs * (9 * nn + 1));
            if (rc) return rc;
        }
        CUDA_TRY(cudaMemcpyAsync(h->dEmHEHP, ehp.data(), ehp.size() * 8, cudaMemcpyHostToDevice, h->st));
        const EmRecords& R4 = h->em_rec[1];
        const EmTables& tb = *R4.tb;
        const int nrech = tb.nrec(Ny);
        const int* MID = tb.d_mid(R4.idx);
        const int* ENTPOS = tb.d_entpos(R4.idx);
        double* om = h->dEmHOut;
        double* oc = om + (long long)H * Ny * nout;
        double *m2 = om, *m3 = m2 + (long long)H * Ny * nn, *m4 = m3 + (long long)H * Ny * nn * Nx;
        double *c2 = oc, *c3 = c2 + (long long)H * Ny * Ny * nn, *c4 = c3 + (long long)H * Ny * Ny * nn * Nx;
        em_hess_mean_finish_kernel<<<dim3(Ny, H), 256, 0, h->st>>>(Nx, Ny, h->dEMP, (long long)per, R4.rec, nrech, tb.nent,
                                                                   MID, ENTPOS, tb.nf, h->dEmHMU, h->dEmHD, h->dEmHScr, m2, m3, m4);
        CUDA_TRY(cudaGetLastError());
        for (int h0 = 0; h0 < H; h0 += Hc) {
            em_hess_pair_finish_kernel<<<dim3(npairs, std::min(Hc, H - h0)), 256, 0, h->st>>>(
                Nx, Ny, h0, h->dEMP, (long long)per, h->dEmHEHP, R4.rec, nrech, tb.nent, MID, ENTPOS, tb.nf,
                h->dEmHMU, h->dEmHD, h->dEmHScr, c2, c3, c4);
            CUDA_TRY(cudaGetLastError());
        }
        const double* src[6] = {m2, m3, m4, c2, c3, c4};
        double* dst[6] = {ho->d2mean_dz2, ho->d2mean_dSigma_dz, ho->d2mean_dSigma2, ho->d2cov_dz2, ho->d2cov_dSigma_dz, ho->d2cov_dSigma2};
        const long long cnt[6] = {(long long)H * Ny * nn, (long long)H * Ny * nn * Nx, (long long)H * Ny * nn * nn,
                                  (long long)H * Ny * Ny * nn, (long long)H * Ny * Ny * nn * Nx, (long long)H * Ny * Ny * nn * nn};
        for (int q = 0; q < 6; ++q)
            if (dst[q]) CUDA_TRY(cudaMemcpyAsync(dst[q], src[q], cnt[q] * 8, cudaMemcpyDeviceToHost, h->st));
    }
    if (go) return em_grad_finish_points(h, H, Sigma, spp, emp.data(), h->dMean, *go);
    CUDA_TRY(cudaStreamSynchronize(h->st));
    return GPMPC_OK;
}

// after a stream sync: did a consumer give up waiting for a peer's flag?
static int peer_status_check(gpmpc_handle_t h)
{
    if (!h->peer_ready) return GPMPC_OK;
    const int st = h->hPeerStatus ? *(volatile int*)h->hPeerStatus : 0;
    if (st) {
        set_error(h, "peer exchange timed out waiting for rank %d (step %llu)", st - 1, h->peer_step);
        *h->hPeerStatus = 0;
        return GPMPC_ERR_NCCL;
    }
    return GPMPC_OK;
}

// The 'UT' pass of H points must be indexable by int
static int ut_size_check(gpmpc_handle_t h, const char* fn, int H)
{
    if (ut_points(h, H) > INT_MAX) { set_error(h, "%s: H (2 Nx + 1) = %lld 'UT' points exceed INT_MAX", fn, ut_points(h, H)); return GPMPC_ERR_ARG; }
    return GPMPC_OK;
}

// First check of every predict-family entry `fn` (the name its errors carry): a factorised model, H >= 1 and a known method;
// 'UT' only where the entry takes it (ut).
static int predict_guard(gpmpc_handle_t h, const char* fn, int method, int H, bool ut = false)
{
    const int rc = model_guard(h, fn, NEED_FACTOR);
    if (rc) return rc;
    if (H < 1) { set_error(h, "%s: H < 1", fn); return GPMPC_ERR_ARG; }
    if (method == GPMPC_METHOD_UT) {
        if (!ut) { set_error(h, "%s: method UT is taken by gpmpc_predict, gpmpc_predict_device, gpmpc_rollout and gpmpc_rollout_batch only", fn); return GPMPC_ERR_ARG; }
        return ut_size_check(h, fn, H);
    }
    if (method != GPMPC_METHOD_ME && method != GPMPC_METHOD_TA && method != GPMPC_METHOD_EM) { set_error(h, "%s: unknown method %d", fn, method); return GPMPC_ERR_ARG; }
    return GPMPC_OK;
}

// after the guard (device selected) and the entry's own checks: all outputs on one handle and rank if all_outputs; buffers
static int predict_prepare(gpmpc_handle_t h, const char* fn, int H, bool all_outputs)
{
    if (all_outputs && (h->nloc != h->Ny || h->world != 1)) { set_error(h, "%s needs all outputs on one handle (replicate the model, shard the points)", fn); return GPMPC_ERR_STATE; }
    const int rc = ensure_predict_bufs(h, H);
    return rc ? rc : panel_refresh(h);
}

extern "C" int gpmpc_predict_device(gpmpc_handle_t h, int method, int H, const double* dZ, const double* dSigma,
                                    int spp, double* d_mean, double* d_var, double* d_cov, double* d_jac, int sync)
{
    int rc = predict_guard(h, __func__, method, H, true);
    if (rc) return rc;
    const bool ut = method == GPMPC_METHOD_UT;
    if (method == GPMPC_METHOD_EM) { set_error(h, "gpmpc_predict_device: EM needs host inputs (use gpmpc_predict)"); return GPMPC_ERR_ARG; }
    if (!dZ || (method == GPMPC_METHOD_TA && d_cov && !dSigma) || (ut && !dSigma)) { set_error(h, "gpmpc_predict_device: null Z / Sigma"); return GPMPC_ERR_ARG; }
    rc = predict_prepare(h, __func__, ut ? (int)ut_points(h, H) : H, ut);
    if (rc) return rc;
    rc = ut ? ut_pass(h, H, dZ, dSigma, spp, d_mean, d_var, d_cov, d_jac)
            : predict_core(h, method, H, dZ, dSigma, spp, d_mean, d_var, d_cov, d_jac);
    if (rc) return rc;
    if (sync) CUDA_TRY(cudaStreamSynchronize(h->st));
    return GPMPC_OK;
}

// ------------------------------------------------------------------------------------
// Multi-step prediction of B trajectories with the state kept on the device (GP.rollout = the numeric loop of
// predict_compare, gp_class.py:746-804).  The host loop pays a call (launches + sync + copies + Python) per step
// although a step's device work at MPC sizes is tens of microseconds; here all Nt steps are enqueued back to back, each one
// predict pass over the B current inputs (H = B, one Sigma per point):
//   open loop:  z_t = [ (mean_{t-1} sY + mY - mX) / sX , u_{t-1} ],  Sigma_t = [cov_{t-1} Sigma_xu; Sigma_ux Sigma_uu] (u blocks kept)
//   feedback:   x = mean_{t-1} sY + mY,  u = K (x - x_ref) [then (u - mU) / sU],  Sigma_uu = K cov K^T,  Sigma_xu = cov K^T
//               (gp_class.py:770-804 with the LQR gain of mpc_class.py:956-976; cov stays in the GP's units, q4)
// with the reference's operation order (gp_class.py:629-638), so the trajectory is the host loop's bit for bit in open loop.
// ------------------------------------------------------------------------------------
// One CTA per trajectory b.  Null cov_t and Sigma: only the next input is formed (gpmpc_rollout_sample).  The roll-out
// kernels' dynamic shared memory is laid out once for kernel and launch, as kernels.cuh's SampleCondSmem; per-warp
// offsets count from the warp's slice.  rollout_feedback_kernel, with K: x (Ny) | K cov (Nu Ny), with cov only.
struct FeedbackSmem { long long KC; int bytes; };
__host__ __device__ __forceinline__ FeedbackSmem rollout_feedback_smem(int Ny, int Nu, bool with_K, bool with_cov)
{
    return {Ny, with_K ? (Ny + (with_cov ? Nu * Ny : 0)) * 8 : 0};
}

__global__ void __launch_bounds__(256)
rollout_feedback_kernel(const double* __restrict__ mean_t, const double* __restrict__ cov_t, const double* __restrict__ u_t,
                        long long u_stride, const double* __restrict__ scale, const double* __restrict__ K,
                        const double* __restrict__ x_ref, const double* __restrict__ uscale, int Ny, int Nu,
                        double* __restrict__ Z, double* __restrict__ Sigma)
{
    extern __shared__ double fb_sh[];
    const int Nx = Ny + Nu, tid = threadIdx.x, b = blockIdx.x;
    const bool with_cov = Sigma != nullptr;                  // before the offsets below
    mean_t += (size_t)b * Ny; cov_t += (size_t)b * Ny * Ny;
    Z += (size_t)b * Nx; Sigma += (size_t)b * Nx * Nx;
    for (int j = tid; j < Nx; j += 256) {
        if (j < Ny) {
            double z = mean_t[j], x = z;
            if (scale) {                                     // [sY | mY | mX | sX]; no fused multiply-add: numpy does not fuse
                x = __dadd_rn(__dmul_rn(z, scale[j]), scale[Ny + j]);
                z = __ddiv_rn(__dsub_rn(x, scale[2 * Ny + j]), scale[3 * Ny + j]);
            }
            Z[j] = z;
            if (K) fb_sh[j] = x;
        } else if (!K) {
            Z[j] = u_t[(size_t)b * u_stride + (j - Ny)];
        }
    }
    if (with_cov)
        for (int idx = tid; idx < Ny * Ny; idx += 256) {
            const int r = idx / Ny, c = idx - r * Ny;
            Sigma[r * Nx + c] = cov_t[idx];
        }
    if (!K) return;                                          // uniform over the CTA
    double* KC = fb_sh + rollout_feedback_smem(Ny, Nu, true, with_cov).KC;
    __syncthreads();
    // u = K (x - x_ref), standardised as GP.predict standardises its input
    for (int i = tid; i < Nu; i += 256) {
        double u = 0.0;
        for (int k = 0; k < Ny; ++k) u = __dadd_rn(u, __dmul_rn(K[i * Ny + k], x_ref ? __dsub_rn(fb_sh[k], x_ref[k]) : fb_sh[k]));
        if (uscale) u = __ddiv_rn(__dsub_rn(u, uscale[i]), uscale[Nu + i]);
        Z[Ny + i] = u;
    }
    if (!with_cov) return;                                   // a sampled roll-out carries no input covariance
    // K cov (kept for Sigma_uu = (K cov) K^T) and Sigma_xu = cov K^T, Sigma_ux = Sigma_xu^T
    for (int idx = tid; idx < Nu * Ny; idx += 256) {
        const int i = idx / Ny, c = idx - i * Ny;
        double s = 0.0;
        for (int k = 0; k < Ny; ++k) s = __dadd_rn(s, __dmul_rn(K[i * Ny + k], cov_t[k * Ny + c]));
        KC[idx] = s;
    }
    for (int idx = tid; idx < Ny * Nu; idx += 256) {
        const int r = idx / Nu, i = idx - r * Nu;
        double s = 0.0;
        for (int k = 0; k < Ny; ++k) s = __dadd_rn(s, __dmul_rn(cov_t[r * Ny + k], K[i * Ny + k]));
        Sigma[r * Nx + Ny + i] = s;
        Sigma[(Ny + i) * Nx + r] = s;
    }
    __syncthreads();
    for (int idx = tid; idx < Nu * Nu; idx += 256) {
        const int i = idx / Nu, j = idx - i * Nu;
        double s = 0.0;
        for (int k = 0; k < Ny; ++k) s = __dadd_rn(s, __dmul_rn(KC[i * Ny + k], K[j * Ny + k]));
        Sigma[(Ny + i) * Nx + Ny + j] = s;
    }
}

// Forward-mode tangents of one roll-out step, one CTA per trajectory b (gpmpc_rollout_batch_grad).  The P parameters of a
// trajectory are [z0 (Nx) | U rows 1 .. Nt-1 (Nu each)] open loop or [z0 | K row-major (Nu x Ny)] with feedback; the
// tangents are dZ (B, P, Nx) and, for 'TA', dS (B, P, Nx, Nx), each parameter's column contiguous.  Step t reads J_t, dcov_t
// ('TA') or dvar_t ('ME') of the derivative chain and writes, per parameter p,
//   dm = J dz,   dC = sum_e dcov[.,.,e] dz_e + J dS J^T ('TA')  or  diag(dvar dz) ('ME'),   dmeans_t = dm, dvars_t = diag(dC)
// and unless last the next tangents, the derivatives of what rollout_feedback_kernel forms:
//   dz[:Ny] = dm * stdY / stdX (dm without scale);  open loop: dz[Ny+i] = [p is U[t+1][i]], dS x block = dC, u blocks kept;
//   feedback, x~ = x - x_ref, dx = dm * stdY:  du = (K dx + dK x~) / stdU,  dS_xu = dC K^T + C dK^T,
//   dS_uu = dK C K^T + K dC K^T + K C dK^T  (dK = the unit matrix of p when p is an entry of K, else 0).
// At t = 0 the tangents are the unit columns of z0 and zero covariance (nothing is read).  Each of the ROLL_TG_WARPS warps
// owns one column at a time and rewrites it in place; every sum runs in index order in one thread, so a trajectory's bits
// do not depend on B.  Dynamic shared memory: rollout_tangent_smem(em = false).
//
// The dynamic shared memory of rollout_tangent_kernel (em = false) and rollout_tangent_em_kernel (em = true): J or dmz
// (Ny Nx) | x~ (Ny) | C K^T (Ny Nu) | K C (Nu Ny) | per warp [dz (Nx) | dm (Ny) | dC (Ny Ny) | T (Ny Nx)], or with em per
// warp [dz (Nx) | dm (Ny) | dC (Ny Ny) | K dC (Nu Ny) | dS (Nx Nx)].
struct TangentSmem { long long xt, CKt, KC, warps, wm, wC, wT, wS; int per_warp, bytes; };
__host__ __device__ __forceinline__ TangentSmem rollout_tangent_smem(int Ny, int Nu, bool em)
{
    const int Nx = Ny + Nu;
    TangentSmem L;
    L.xt = Ny * Nx; L.CKt = L.xt + Ny; L.KC = L.CKt + Ny * Nu; L.warps = L.KC + Nu * Ny;
    L.wm = Nx; L.wC = L.wm + Ny; L.wT = L.wC + Ny * Ny; L.wS = L.wT + (em ? Nu * Ny : Ny * Nx);
    L.per_warp = (int)(em ? L.wS + Nx * Nx : L.wS);
    L.bytes = (int)(L.warps + ROLL_TG_WARPS * L.per_warp) * 8;
    return L;
}

// The two stages every tangent kernel shares.  tangent_policy: per trajectory, before its columns, x~ = x - x_ref (feedback,
// unless last) and, with Sigma tangents (sig), C K^T and K C; cov_t is the trajectory's.
__device__ __forceinline__ void tangent_policy(int Ny, int Nu, int b, bool fb_next, bool sig, const double* __restrict__ mean_t,
                                               const double* __restrict__ cov_t, const double* __restrict__ scale,
                                               const double* __restrict__ K, const double* __restrict__ x_ref,
                                               double* xt, double* CKt, double* KC)
{
    const int tid = threadIdx.x;
    if (fb_next) {
        for (int k = tid; k < Ny; k += blockDim.x) {
            const double m = mean_t[(size_t)b * Ny + k];
            const double x = scale ? m * scale[k] + scale[Ny + k] : m;
            xt[k] = x_ref ? x - x_ref[k] : x;
        }
        if (sig)
            for (int idx = tid; idx < Ny * Nu; idx += blockDim.x) {
                const int r = idx / Nu, i = idx - r * Nu;
                double s1 = 0.0, s2 = 0.0;
                for (int k = 0; k < Ny; ++k) {
                    s1 = fma(cov_t[r * Ny + k], K[i * Ny + k], s1);      // (C K^T)[r][i]
                    s2 = fma(K[i * Ny + k], cov_t[k * Ny + r], s2);      // (K C)[i][r]
                }
                CKt[idx] = s1; KC[i * Ny + r] = s2;
            }
    }
}

// tangent_next_z: one warp's next input tangent z of column p from step t's output tangent wm (dm, or df of a draw) and,
// with K, x~ of tangent_policy: dz[:Ny] = wm stdY / stdX; open loop the unit tangent of U[t+1]; with K
// du = (K dx + dK x~) / stdU.
__device__ __forceinline__ void tangent_next_z(int Ny, int Nu, int t, int p, const double* wm, const double* xt,
                                               const double* __restrict__ scale, const double* __restrict__ K,
                                               const double* __restrict__ uscale, double* __restrict__ z)
{
    const int Nx = Ny + Nu, lane = threadIdx.x & 31;
    const bool fb = K != nullptr;
    // the entry of K this column stands for (ki, kk), or -1
    const int q = p - Nx, ki = (fb && q >= 0) ? q / Ny : -1, kk = (fb && q >= 0) ? q - ki * Ny : -1;
    for (int j = lane; j < Nx; j += 32) {
        double d;
        if (j < Ny) {
            d = wm[j];
            if (scale) d = d * scale[j] / scale[3 * Ny + j];
        } else if (!fb) {
            d = (p == Nx + t * Nu + (j - Ny)) ? 1.0 : 0.0;
        } else {
            const int i = j - Ny;
            d = 0.0;
            for (int k = 0; k < Ny; ++k) d = fma(K[i * Ny + k], scale ? wm[k] * scale[k] : wm[k], d);
            if (i == ki) d += xt[kk];
            if (uscale) d = d / uscale[Nu + i];
        }
        z[j] = d;
    }
}

// tangent_column: one warp's column p after dm (wm) and dC (wC) are formed: dmeans_t, dvars_t and, unless last, the next
// tangents dz into z and, with Sigma tangents (sig), dSigma into S, with wT (at least Nu Ny) as scratch for K dC.
__device__ __forceinline__ void tangent_column(int Ny, int Nu, int P, int t, int p, int b, int first, int last, bool sig,
                                               const double* wm, const double* wC, double* wT, const double* xt,
                                               const double* CKt, const double* KC, const double* __restrict__ cov_t,
                                               const double* __restrict__ scale, const double* __restrict__ K,
                                               const double* __restrict__ uscale, double* __restrict__ z,
                                               double* __restrict__ S, double* __restrict__ dmeans_t,
                                               double* __restrict__ dvars_t)
{
    const int Nx = Ny + Nu, lane = threadIdx.x & 31;
    const bool fb = K != nullptr;
    for (int a = lane; a < Ny; a += 32) {
        dmeans_t[((size_t)b * Ny + a) * P + p] = wm[a];
        dvars_t[((size_t)b * Ny + a) * P + p] = wC[a * Ny + a];
    }
    if (!last) {
        // the entry of K this column stands for (ki, kk), or -1
        const int q = p - Nx, ki = (fb && q >= 0) ? q / Ny : -1, kk = (fb && q >= 0) ? q - ki * Ny : -1;
        tangent_next_z(Ny, Nu, t, p, wm, xt, scale, K, uscale, z);
        if (sig) {
            if (fb)
                for (int idx = lane; idx < Nu * Ny; idx += 32) {     // K dC, into T (read only above this point)
                    const int i = idx / Ny, c = idx - i * Ny;
                    double s = 0.0;
                    for (int k = 0; k < Ny; ++k) s = fma(K[i * Ny + k], wC[k * Ny + c], s);
                    wT[idx] = s;
                }
            __syncwarp();
            for (int idx = lane; idx < Nx * Nx; idx += 32) {
                const int r = idx / Nx, c = idx - r * Nx;
                if (r < Ny && c < Ny) { S[idx] = wC[r * Ny + c]; continue; }
                if (!fb) {                                           // u blocks kept (zero at the start)
                    if (first) S[idx] = 0.0;
                    continue;
                }
                double s = 0.0;
                if (r < Ny || c < Ny) {                              // dS_xu[x][i] = (dC K^T + C dK^T)[x][i], dS_ux its transpose
                    const int x = r < Ny ? r : c, i = (r < Ny ? c : r) - Ny;
                    for (int k = 0; k < Ny; ++k) s = fma(wC[x * Ny + k], K[i * Ny + k], s);
                    if (i == ki) s += cov_t[x * Ny + kk];
                } else {                                             // dS_uu[i][j]
                    const int i = r - Ny, j = c - Ny;
                    for (int k = 0; k < Ny; ++k) s = fma(wT[i * Ny + k], K[j * Ny + k], s);
                    if (i == ki) s += CKt[kk * Nu + j];
                    if (j == ki) s += KC[i * Ny + kk];
                }
                S[idx] = s;
            }
        }
    }
}

__global__ void __launch_bounds__(ROLL_TG_WARPS * 32, 2)
rollout_tangent_kernel(int Ny, int Nu, int P, int t, int first, int last, int method_ta,
                       const double* __restrict__ J, const double* __restrict__ dvar, const double* __restrict__ dcov,
                       const double* __restrict__ mean_t, const double* __restrict__ cov_t, const double* __restrict__ scale,
                       const double* __restrict__ K, const double* __restrict__ x_ref, const double* __restrict__ uscale,
                       double* __restrict__ dZ, double* __restrict__ dS, double* __restrict__ dmeans_t, double* __restrict__ dvars_t)
{
    extern __shared__ double tg_sh[];
    const int Nx = Ny + Nu, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5, b = blockIdx.x;
    const bool fb = K != nullptr;
    const TangentSmem L = rollout_tangent_smem(Ny, Nu, false);
    double* sJ = tg_sh;
    double* xt = tg_sh + L.xt;
    double* CKt = tg_sh + L.CKt;
    double* KC = tg_sh + L.KC;
    double* wz = tg_sh + L.warps + warp * L.per_warp;
    double* wm = wz + L.wm;
    double* wC = wz + L.wC;
    double* wT = wz + L.wT;
    J += (size_t)b * Ny * Nx;
    cov_t += (size_t)b * Ny * Ny;
    for (int i = tid; i < Ny * Nx; i += blockDim.x) sJ[i] = J[i];
    tangent_policy(Ny, Nu, b, fb && !last, method_ta, mean_t, cov_t, scale, K, x_ref, xt, CKt, KC);
    __syncthreads();
    const double* dcv = dcov + (size_t)b * Ny * Ny * Nx;
    const double* dvr = dvar + (size_t)b * Ny * Nx;
    for (int p = warp; p < P; p += nwarps) {
        double* z = dZ + ((size_t)b * P + p) * Nx;
        double* S = method_ta ? dS + ((size_t)b * P + p) * Nx * Nx : nullptr;
        for (int e = lane; e < Nx; e += 32) wz[e] = first ? (e == p ? 1.0 : 0.0) : z[e];
        __syncwarp();
        for (int a = lane; a < Ny; a += 32) {
            double s = 0.0;
            for (int e = 0; e < Nx; ++e) s = fma(sJ[a * Nx + e], wz[e], s);
            wm[a] = s;
        }
        if (method_ta)
            for (int idx = lane; idx < Ny * Nx; idx += 32) {         // T = J dS
                const int a = idx / Nx, f = idx - a * Nx;
                double s = 0.0;
                if (!first)
                    for (int e = 0; e < Nx; ++e) s = fma(sJ[a * Nx + e], S[e * Nx + f], s);
                wT[idx] = s;
            }
        __syncwarp();
        for (int idx = lane; idx < Ny * Ny; idx += 32) {
            const int a = idx / Ny, c = idx - a * Ny;
            double s = 0.0;
            if (method_ta) {
                const double* dc = dcv + (size_t)idx * Nx;
                for (int e = 0; e < Nx; ++e) s = fma(dc[e], wz[e], s);
                double q = 0.0;
                for (int f = 0; f < Nx; ++f) q = fma(wT[a * Nx + f], sJ[c * Nx + f], q);
                s += q;
            } else if (a == c) {
                for (int e = 0; e < Nx; ++e) s = fma(dvr[a * Nx + e], wz[e], s);
            }
            wC[idx] = s;
        }
        __syncwarp();
        tangent_column(Ny, Nu, P, t, p, b, first, last, method_ta, wm, wC, wT, xt, CKt, KC, cov_t, scale, K, uscale, z, S,
                       dmeans_t, dvars_t);
        __syncwarp();
    }
}

// Forward-mode tangents of one 'EM' roll-out step (gpmpc_rollout_batch_em_grad), one CTA per trajectory b: the parameters,
// tangent slabs (dS always: the 'EM' mean depends on Sigma), outputs and next tangents of rollout_tangent_kernel.  Step t
// reads gpmpc_predict_em_grad's blocks at (z_t, Sigma_t), per trajectory dmz (Ny,Nx), dmS (Ny,Nx,Nx), dcz (Ny,Ny,Nx) and
// dcS (Ny,Ny,Nx,Nx), and forms per parameter
//   dm = dmz dz + sum_{d,e} dmS[., d, e] dS[d, e],   dC = dcz dz + sum_{d,e} dcS[., ., d, e] dS[d, e]
// over all Nx^2 entries of the symmetric dS: the blocks hold every other entry fixed, so this is the directional derivative.
// At t = 0 dS is zero and is not read.  dmz and the column's dS are staged in shared memory; dmS and dcS are read from global
// memory (Ny^2 Nx^2 doubles a trajectory do not fit at Nx = 32).  Every sum runs in index order in one thread.
// Dynamic shared memory: rollout_tangent_smem(em = true).
__global__ void __launch_bounds__(ROLL_TG_WARPS * 32, 2)
rollout_tangent_em_kernel(int Ny, int Nu, int P, int t, int first, int last,
                          const double* __restrict__ dmz, const double* __restrict__ dmS, const double* __restrict__ dcz,
                          const double* __restrict__ dcS, const double* __restrict__ mean_t, const double* __restrict__ cov_t,
                          const double* __restrict__ scale, const double* __restrict__ K, const double* __restrict__ x_ref,
                          const double* __restrict__ uscale, double* __restrict__ dZ, double* __restrict__ dS,
                          double* __restrict__ dmeans_t, double* __restrict__ dvars_t)
{
    extern __shared__ double tg_sh[];
    const int Nx = Ny + Nu, nn = Nx * Nx, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
    const int b = blockIdx.x;
    const TangentSmem L = rollout_tangent_smem(Ny, Nu, true);
    double* sG = tg_sh;
    double* xt = tg_sh + L.xt;
    double* CKt = tg_sh + L.CKt;
    double* KC = tg_sh + L.KC;
    double* wz = tg_sh + L.warps + warp * L.per_warp;
    double* wm = wz + L.wm;
    double* wC = wz + L.wC;
    double* wT = wz + L.wT;
    double* wS = wz + L.wS;
    dmz += (size_t)b * Ny * Nx;
    dmS += (size_t)b * Ny * nn;
    dcz += (size_t)b * Ny * Ny * Nx;
    dcS += (size_t)b * Ny * Ny * nn;
    cov_t += (size_t)b * Ny * Ny;
    for (int i = tid; i < Ny * Nx; i += blockDim.x) sG[i] = dmz[i];
    tangent_policy(Ny, Nu, b, K != nullptr && !last, true, mean_t, cov_t, scale, K, x_ref, xt, CKt, KC);
    __syncthreads();
    for (int p = warp; p < P; p += nwarps) {
        double* z = dZ + ((size_t)b * P + p) * Nx;
        double* S = dS + ((size_t)b * P + p) * nn;
        for (int e = lane; e < Nx; e += 32) wz[e] = first ? (e == p ? 1.0 : 0.0) : z[e];
        if (!first)
            for (int q = lane; q < nn; q += 32) wS[q] = S[q];
        __syncwarp();
        for (int a = lane; a < Ny; a += 32) {
            double s = 0.0;
            for (int e = 0; e < Nx; ++e) s = fma(sG[a * Nx + e], wz[e], s);
            if (!first) {
                const double* g = dmS + (size_t)a * nn;
                for (int q = 0; q < nn; ++q) s = fma(g[q], wS[q], s);
            }
            wm[a] = s;
        }
        for (int idx = lane; idx < Ny * Ny; idx += 32) {
            const double* gz = dcz + (size_t)idx * Nx;
            double s = 0.0;
            for (int e = 0; e < Nx; ++e) s = fma(gz[e], wz[e], s);
            if (!first) {
                const double* g = dcS + (size_t)idx * nn;
                for (int q = 0; q < nn; ++q) s = fma(g[q], wS[q], s);
            }
            wC[idx] = s;
        }
        __syncwarp();
        tangent_column(Ny, Nu, P, t, p, b, first, last, true, wm, wC, wT, xt, CKt, KC, cov_t, scale, K, uscale, z, S,
                       dmeans_t, dvars_t);
        __syncwarp();
    }
}

// The input tangents of step t of a sampled roll-out (gpmpc_rollout_sample_grad), one CTA per trajectory b, warps over
// the P columns: at t = 0 the unit columns of z0, else tangent_next_z of step t-1's draw tangents dsamp_prev (B, Ny, P)
// with x the draw samp_prev (B, Ny) in place of the mean, as rollout_feedback_kernel forms the next input from it.
// Writes dZt (B, P, Nx).  Dynamic shared memory: x~ (Ny) | per warp df (Ny).
struct SampleNextSmem { long long warps; int bytes; };
__host__ __device__ __forceinline__ SampleNextSmem sample_next_smem(int Ny)
{
    return {Ny, (Ny + ROLL_TG_WARPS * Ny) * 8};
}

__global__ void __launch_bounds__(ROLL_TG_WARPS * 32, 2)
sample_next_kernel(int Ny, int Nu, int P, int t, const double* __restrict__ samp_prev, const double* __restrict__ dsamp_prev,
                   const double* __restrict__ scale, const double* __restrict__ K, const double* __restrict__ x_ref,
                   const double* __restrict__ uscale, double* __restrict__ dZt)
{
    extern __shared__ double sn_sh[];
    const int Nx = Ny + Nu, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5, b = blockIdx.x;
    double* xt = sn_sh;
    double* wm = sn_sh + sample_next_smem(Ny).warps + warp * Ny;
    if (t > 0) tangent_policy(Ny, Nu, b, K != nullptr, false, samp_prev, nullptr, scale, K, x_ref, xt, nullptr, nullptr);
    __syncthreads();
    for (int p = warp; p < P; p += nwarps) {
        double* z = dZt + ((size_t)b * P + p) * Nx;
        if (t == 0) {
            for (int e = lane; e < Nx; e += 32) z[e] = e == p ? 1.0 : 0.0;
            continue;
        }
        for (int a = lane; a < Ny; a += 32) wm[a] = dsamp_prev[((size_t)b * Ny + a) * P + p];
        __syncwarp();
        tangent_next_z(Ny, Nu, t - 1, p, wm, xt, scale, K, uscale, z);
        __syncwarp();
    }
}

// Host outputs of the tangent stage of rollout_batch (gpmpc_rollout_batch_grad): (B, Nt, Ny, P) each
struct RolloutTangents {
    double *dmeans, *dvars;
};

// Device slabs of the derivative chain for H points: dvar (H,Ny,Nx) | dcov (H,Ny,Ny,Nx) | hess (H,Ny,Nx,Nx) in dGradOut,
// and with second derivatives d2var | SH scratch | d3mean | d2cov in dHessOut (null otherwise)
struct DerivSlabs {
    double *dvar, *dcov, *hess;
    double *d2var, *sh, *d3mean, *d2cov;
};

static int derivs_prepare(gpmpc_handle_t h, int H, bool second, DerivSlabs* s);
static int derivs_enqueue(gpmpc_handle_t h, int method, int H, const double* dZ, const double* dSigma, int spp,
                          const DerivSlabs& s, double* beta = nullptr, long long sbeta = 0);

// Device views of a roll-out's feedback policy, null where absent (x_ref and uscale only with K)
struct RolloutPolicy { const double *scale, *K, *x_ref, *uscale; };

// A roll-out's policy block [U (B,Nt,Nu), open loop only | scale (4,Ny) | K (Nu,Ny) | x_ref (Ny) | uscale (2,Nu)] at slab
// offset o: returns the offset past it.  Given the pinned mirror pin, also packs the block there and sets *pol to its
// views in the device slab d.
static size_t rollout_policy(int B, int Nt, int Ny, int Nu, const double* U, const double* scale, const double* K,
                             const double* x_ref, const double* uscale, size_t o, double* pin = nullptr,
                             const double* d = nullptr, RolloutPolicy* pol = nullptr)
{
    const size_t nU = U && !K ? (size_t)B * Nt * Nu : 0, o_sc = o + nU, o_k = o_sc + 4 * (size_t)Ny;
    const size_t o_xr = o_k + (size_t)Nu * Ny, o_us = o_xr + Ny, end = o_us + 2 * (size_t)Nu;
    if (!pin) return end;
    if (nU) memcpy(pin + o, U, nU * 8);
    if (scale) memcpy(pin + o_sc, scale, 4 * (size_t)Ny * 8);
    if (K) memcpy(pin + o_k, K, (size_t)Nu * Ny * 8);
    if (K && x_ref) memcpy(pin + o_xr, x_ref, (size_t)Ny * 8);
    if (K && uscale) memcpy(pin + o_us, uscale, 2 * (size_t)Nu * 8);
    *pol = {scale ? d + o_sc : nullptr, K ? d + o_k : nullptr, K && x_ref ? d + o_xr : nullptr, K && uscale ? d + o_us : nullptr};
    return end;
}

// The argument checks every roll-out entry shares; nulls is the entry's own null-pointer test
static int rollout_args(gpmpc_handle_t h, const char* fn, int B, int Nt, bool nulls, const double* U, const double* K)
{
    const int Nx = h->Nx, Ny = h->Ny, Nu = Nx - Ny;
    if (B < 1 || Nt < 1 || nulls || (Nu > 0 && !K && !U)) { set_error(h, "%s: null argument / B < 1 / Nt < 1", fn); return GPMPC_ERR_ARG; }
    if (Nu < 0) { set_error(h, "%s: needs Nx = Ny + Nu with Nu >= 0 (Nx=%d, Ny=%d)", fn, Nx, Ny); return GPMPC_ERR_ARG; }
    if (K && Nu == 0) { set_error(h, "%s: a feedback gain needs inputs (Nu = 0)", fn); return GPMPC_ERR_ARG; }
    return GPMPC_OK;
}

// P, the parameters of a differentiated roll-out: [z0 (Nx) | K row-major (Nu Ny)] with K, else [z0 | U rows 1 .. Nt-1]
static size_t rollout_params(int Nx, int Ny, int Nt, bool with_K) { return Nx + (size_t)(Nx - Ny) * (with_K ? Ny : Nt - 1); }

// (t, b) -> (b, t): row t B + b of the step-major src to row b Nt + t of dst, n doubles per row
static void rows_by_trajectory(double* dst, const double* src, int B, int Nt, size_t n)
{
    for (size_t b = 0; b < (size_t)B; ++b)
        for (int t = 0; t < Nt; ++t)
            memcpy(dst + (b * Nt + t) * n, src + ((size_t)t * B + b) * n, n * 8);
}

// gpmpc_rollout_batch, gpmpc_rollout, with tg gpmpc_rollout_batch_grad and with em_entry gpmpc_rollout_batch_em (the
// entries that take 'EM'; with tg gpmpc_rollout_batch_em_grad); fn names the entry in errors
static int rollout_batch(gpmpc_handle_t h, const char* fn, int method, int B, int Nt, const double* z0, const double* U,
                         const double* Sigma0, const double* scale, const double* K, const double* x_ref,
                         const double* uscale, double* means, double* vars, double* cov_last, const RolloutTangents* tg = nullptr,
                         bool em_entry = false)
{
    int rc = predict_guard(h, fn, method, 1, !tg && !em_entry);
    if (rc) return rc;
    const int Nx = h->Nx, Ny = h->Ny, Nu = Nx - Ny;
    const bool em = method == GPMPC_METHOD_EM, ut = method == GPMPC_METHOD_UT;
    if (em && !em_entry) { set_error(h, "%s: methods ME, TA and UT (EM: gpmpc_rollout_batch_em)", fn); return GPMPC_ERR_ARG; }
    rc = rollout_args(h, fn, B, Nt, !z0 || !Sigma0 || !means || !vars, U, K);
    if (!rc && ut) rc = ut_size_check(h, fn, B);
    if (rc) return rc;
    if (tg && (!tg->dmeans || !tg->dvars)) { set_error(h, "%s: null dmeans / dvars", fn); return GPMPC_ERR_ARG; }
    rc = predict_prepare(h, fn, ut ? (int)ut_points(h, B) : B, true);
    if (rc) return rc;
    NvtxRange nvtx_r(tg ? "gpmpc.rollout_grad" : "gpmpc.rollout");
    // device slab: [Z (B,Nx) | Sigma (B,Nx,Nx) | policy (rollout_policy) | means (Nt,B,Ny) | vars (Nt,B,Ny) |
    //               cov (Nt,B,Ny,Ny)], host mirror in the pinned buffer.  Step t reads and writes B consecutive points,
    //               so its outputs are one (B,...) block.
    const size_t Bs = (size_t)B, o_sig = Bs * Nx, o_u = o_sig + Bs * Nx * Nx;
    const size_t o_m = rollout_policy(B, Nt, Ny, Nu, U, scale, K, x_ref, uscale, o_u);
    const size_t o_v = o_m + (size_t)Nt * Bs * Ny, o_c = o_v + (size_t)Nt * Bs * Ny, tot = o_c + (size_t)Nt * Bs * Ny * Ny;
    ENSURE(h->dRoll, tot);
    // tangent slab: [dZ (B,P,Nx) | dS (B,P,Nx,Nx), 'TA' and 'EM' | dmeans (Nt,B,Ny,P) | dvars (Nt,B,Ny,P) | 'EM': the step's
    // gpmpc_predict_em_grad blocks dmz (B,Ny,Nx) | dmS (B,Ny,Nx,Nx) | dcz (B,Ny,Ny,Nx) | dcS (B,Ny,Ny,Nx,Nx)], dmeans and
    // dvars mirrored in the pinned buffer after the roll-out's outputs
    const size_t nn = (size_t)Nx * Nx;
    const size_t P = tg ? rollout_params(Nx, Ny, Nt, K != nullptr) : 0;
    const size_t o_ds = Bs * P * Nx, o_dm = o_ds + (method != GPMPC_METHOD_ME ? Bs * P * nn : 0);
    const size_t o_dv = o_dm + (size_t)Nt * Bs * Ny * P, o_g = o_dv + (size_t)Nt * Bs * Ny * P;
    const size_t n_mz = Bs * Ny * Nx, n_mS = Bs * Ny * nn, n_cz = Bs * Ny * Ny * Nx, n_g = em ? n_mz + n_mS + n_cz + n_cz * Nx : 0;
    DerivSlabs ds;
    if (tg) {
        if (!em) {
            rc = derivs_prepare(h, B, false, &ds);
            if (rc) return rc;
        }
        ENSURE(h->dRollTg, o_g + n_g);
    }
    rc = ensure_pinned(h, (tot + (tg ? o_g - o_dm : 0)) * 8);
    if (rc) return rc;
    double* pin = h->hPinned;
    memcpy(pin, z0, Bs * Nx * 8);
    memcpy(pin + o_sig, Sigma0, Bs * Nx * Nx * 8);
    double* d = h->dRoll;
    RolloutPolicy pol;
    rollout_policy(B, Nt, Ny, Nu, U, scale, K, x_ref, uscale, o_u, pin, d, &pol);
    CUDA_TRY(cudaMemcpyAsync(d, pin, o_m * 8, cudaMemcpyHostToDevice, h->st));
    // 'EM': the scratch of em_pass over the B points and, with tangents, the D = 2 records of a step's points and K^-1;
    // the em_prepare_point blocks and gpmpc_predict_em_grad's blocks staged on the host
    if (em) {
        rc = em_scratch(h, B);
        if (!rc && tg) rc = em_records_prepare(h, 2, B);
        if (!rc && tg) rc = em_kinv_prepare(h);
        if (rc) return rc;
    }
    std::vector<double> emp(em ? Bs * em_per(h) : 0), hg(n_g);
    const EmGradOutputs hgo = {hg.data(), hg.data() + n_mz, hg.data() + n_mz + n_mS, hg.data() + n_mz + n_mS + n_cz};
    const int fb_smem = rollout_feedback_smem(Ny, Nu, K != nullptr, true).bytes;
    for (int t = 0; t < Nt; ++t) {
        double* mean_t = d + o_m + (size_t)t * Bs * Ny;
        double* var_t = d + o_v + (size_t)t * Bs * Ny;
        double* cov_t = d + o_c + (size_t)t * Bs * Ny * Ny;
        if (!em) {
            rc = ut ? ut_pass(h, B, d, d + o_sig, 1, mean_t, var_t, cov_t, nullptr)
                    : predict_core(h, method, B, d, d + o_sig, 1, mean_t, var_t, cov_t, nullptr);
            if (rc) return rc;
        } else {
            // the step's Sigma back to the host (step 0: Sigma0, already in the pinned mirror), then predict_em's pass over
            // the B points (the em_prepare_point blocks from glibc's log and the host LU: the bits of gpmpc_predict(EM))
            if (t > 0) {
                CUDA_TRY(cudaMemcpyAsync(pin + o_sig, d + o_sig, Bs * Nx * Nx * 8, cudaMemcpyDeviceToHost, h->st));
                CUDA_TRY(cudaStreamSynchronize(h->st));
            }
            int bad = -1;
            rc = em_pass(h, B, d, pin + o_sig, 1, emp.data(), mean_t, var_t, cov_t, tg != nullptr, false, &bad);
            // gpmpc_predict_em_grad's finish at (z_t, Sigma_t), the step's second synchronisation; its blocks go back up below
            if (!rc && tg) rc = em_grad_finish_points(h, B, pin + o_sig, 1, emp.data(), mean_t, hgo, &bad);
            if (rc) {
                if (bad >= 0) {                   // a rejected point: name the step and the trajectory
                    char why[512];
                    snprintf(why, sizeof(why), "%s", h->err);
                    set_error(h, "%s: step %d, trajectory %d: %s", fn, t, bad, why);
                }
                return rc;
            }
            if (tg) CUDA_TRY(cudaMemcpyAsync(h->dRollTg + o_g, hg.data(), hg.size() * 8, cudaMemcpyHostToDevice, h->st));
        }
        if (tg) {                                 // the step's derivatives at the same points, then its tangents
            // the opt-in covers every shape: either layout grows with Nu at a fixed Ny and with Ny at Nx = NX_MAX
            const int smem_max = rollout_tangent_smem(NX_MAX, 0, em).bytes;
            const int tg_smem = rollout_tangent_smem(Ny, Nu, em).bytes;
            double* g = h->dRollTg;
            if (!em) {                            // J_t, dvar_t, dcov_t
                rc = derivs_enqueue(h, method, B, d, d + o_sig, 1, ds);
                if (rc) return rc;
                CUDA_TRY(smem_opt_in<rollout_tangent_kernel>(smem_max));
                rollout_tangent_kernel<<<B, ROLL_TG_WARPS * 32, tg_smem, h->st>>>(Ny, Nu, (int)P, t, t == 0, t + 1 == Nt, method == GPMPC_METHOD_TA,
                                                                      h->dJ, ds.dvar, ds.dcov, mean_t, cov_t,
                                                                      pol.scale, pol.K, pol.x_ref, pol.uscale, g, g + o_ds, g + o_dm + (size_t)t * Bs * Ny * P,
                                                                      g + o_dv + (size_t)t * Bs * Ny * P);
            } else {
                CUDA_TRY(smem_opt_in<rollout_tangent_em_kernel>(smem_max));
                const double* G = g + o_g;
                rollout_tangent_em_kernel<<<B, ROLL_TG_WARPS * 32, tg_smem, h->st>>>(Ny, Nu, (int)P, t, t == 0, t + 1 == Nt, G, G + n_mz,
                                                                         G + n_mz + n_mS, G + n_mz + n_mS + n_cz, mean_t, cov_t,
                                                                         pol.scale, pol.K, pol.x_ref, pol.uscale, g, g + o_ds,
                                                                         g + o_dm + (size_t)t * Bs * Ny * P,
                                                                         g + o_dv + (size_t)t * Bs * Ny * P);
            }
            CUDA_TRY(cudaGetLastError());
        }
        if (t + 1 < Nt) {
            rollout_feedback_kernel<<<B, 256, fb_smem, h->st>>>(mean_t, cov_t, d + o_u + (size_t)(t + 1) * Nu,
                                                                (long long)Nt * Nu, pol.scale, pol.K, pol.x_ref, pol.uscale,
                                                                Ny, Nu, d, d + o_sig);
            CUDA_TRY(cudaGetLastError());
        }
    }
    CUDA_TRY(cudaMemcpyAsync(pin + o_m, d + o_m, (tot - o_m) * 8, cudaMemcpyDeviceToHost, h->st));
    if (tg) CUDA_TRY(cudaMemcpyAsync(pin + tot, h->dRollTg + o_dm, (o_g - o_dm) * 8, cudaMemcpyDeviceToHost, h->st));
    CUDA_TRY(cudaStreamSynchronize(h->st));
    // (t, b) -> (b, t); the reference records diag(covar_x) of every step (gp_class.py:793): the propagated variance, J Sigma J^T included
    rows_by_trajectory(means, pin + o_m, B, Nt, Ny);
    for (size_t b = 0; b < Bs; ++b)
        for (int t = 0; t < Nt; ++t) {
            const size_t src = (size_t)t * Bs + b, dst = b * Nt + t;
            for (int a = 0; a < Ny; ++a) vars[dst * Ny + a] = pin[o_c + src * Ny * Ny + (size_t)a * Ny + a];
        }
    if (tg) {
        rows_by_trajectory(tg->dmeans, pin + tot, B, Nt, (size_t)Ny * P);
        rows_by_trajectory(tg->dvars, pin + tot + (o_dv - o_dm), B, Nt, (size_t)Ny * P);
    }
    if (cov_last) rows_by_trajectory(cov_last, pin + o_c + (size_t)(Nt - 1) * Bs * Ny * Ny, B, 1, (size_t)Ny * Ny);
    return GPMPC_OK;
}

extern "C" int gpmpc_rollout_batch(gpmpc_handle_t h, int method, int B, int Nt, const double* z0, const double* U,
                                   const double* Sigma0, const double* scale, const double* K, const double* x_ref,
                                   const double* uscale, double* means, double* vars, double* cov_last)
{
    return rollout_batch(h, __func__, method, B, Nt, z0, U, Sigma0, scale, K, x_ref, uscale, means, vars, cov_last);
}

// gpmpc_rollout_batch with 'EM': the same slab, policy and feedback, the step's predict the batched EM forward
extern "C" int gpmpc_rollout_batch_em(gpmpc_handle_t h, int B, int Nt, const double* z0, const double* U, const double* Sigma0,
                                      const double* scale, const double* K, const double* x_ref, const double* uscale,
                                      double* means, double* vars, double* cov_last)
{
    return rollout_batch(h, __func__, GPMPC_METHOD_EM, B, Nt, z0, U, Sigma0, scale, K, x_ref, uscale, means, vars, cov_last,
                         nullptr, true);
}

// gpmpc_rollout_batch plus the forward-mode derivatives of every step's mean and variance (see include/gpmpc.h)
extern "C" int gpmpc_rollout_batch_grad(gpmpc_handle_t h, int method, int B, int Nt, const double* z0, const double* U,
                                        const double* Sigma0, const double* scale, const double* K, const double* x_ref,
                                        const double* uscale, double* means, double* vars, double* cov_last,
                                        double* dmeans, double* dvars)
{
    const RolloutTangents tg = {dmeans, dvars};
    return rollout_batch(h, __func__, method, B, Nt, z0, U, Sigma0, scale, K, x_ref, uscale, means, vars, cov_last, &tg);
}

// gpmpc_rollout_batch_em plus the forward-mode derivatives of gpmpc_rollout_batch_grad (see include/gpmpc.h)
extern "C" int gpmpc_rollout_batch_em_grad(gpmpc_handle_t h, int B, int Nt, const double* z0, const double* U,
                                           const double* Sigma0, const double* scale, const double* K, const double* x_ref,
                                           const double* uscale, double* means, double* vars, double* cov_last,
                                           double* dmeans, double* dvars)
{
    const RolloutTangents tg = {dmeans, dvars};
    return rollout_batch(h, __func__, GPMPC_METHOD_EM, B, Nt, z0, U, Sigma0, scale, K, x_ref, uscale, means, vars, cov_last,
                         &tg, true);
}

// the single open-loop trajectory: B = 1 of the batched loop
extern "C" int gpmpc_rollout(gpmpc_handle_t h, int method, int Nt, const double* z0, const double* U, const double* Sigma0,
                             const double* scale, double* means, double* vars, double* cov_last)
{
    return rollout_batch(h, __func__, method, 1, Nt, z0, U, Sigma0, scale, nullptr, nullptr, nullptr, means, vars, cov_last);
}

extern "C" int gpmpc_predict(gpmpc_handle_t h, int method, int H, const double* Z, const double* Sigma,
                             int spp, double* mean, double* var, double* cov, double* jac)
{
    int rc = predict_guard(h, __func__, method, H, true);
    if (rc) return rc;
    const bool ut = method == GPMPC_METHOD_UT;
    if (!Z || (method == GPMPC_METHOD_TA && cov && !Sigma) || (ut && !Sigma)) { set_error(h, "gpmpc_predict: null Z / Sigma"); return GPMPC_ERR_ARG; }
    if (method == GPMPC_METHOD_EM && jac) { set_error(h, "gpmpc_predict: EM does not return a Jacobian"); return GPMPC_ERR_ARG; }
    rc = predict_prepare(h, __func__, ut ? (int)ut_points(h, H) : H, method == GPMPC_METHOD_EM || ut);
    if (rc) return rc;
    if (method == GPMPC_METHOD_EM) return predict_em(h, H, Z, Sigma, spp, mean, var, cov);
    const int Nx = h->Nx, Ny = h->Ny;
    const size_t nz = (size_t)H * Nx, ns = ((method == GPMPC_METHOD_TA && Sigma) || ut) ? (size_t)(spp ? H : 1) * Nx * Nx : 0;
    const size_t nm = (size_t)H * Ny, nj = (size_t)H * Ny * Nx, nc = (size_t)H * Ny * Ny;
    // device slabs: [Z | Sigma] and [mean | var | J | cov] at capacity-based offsets -> one copy each way
    const size_t cap = (size_t)h->Hcap;
    const size_t in_span = ns ? cap * Nx + ns : nz;
    const size_t off_var = cap * Ny, off_j = 2 * cap * Ny, off_c = 2 * cap * Ny + cap * Ny * Nx;
    size_t lo = (size_t)-1, hi = 0;
    if (mean) { lo = std::min(lo, (size_t)0); hi = std::max(hi, nm); }
    if (var) { lo = std::min(lo, off_var); hi = std::max(hi, off_var + nm); }
    if (jac) { lo = std::min(lo, off_j); hi = std::max(hi, off_j + nj); }
    if (cov) { lo = std::min(lo, off_c); hi = std::max(hi, off_c + nc); }
    const size_t out_span = (hi > lo) ? hi - lo : 0;
    rc = ensure_pinned(h, (in_span + out_span) * 8);
    if (rc) return rc;
    double* pin = h->hPinned;
    memcpy(pin, Z, nz * 8);
    if (ns) memcpy(pin + cap * Nx, Sigma, ns * 8);
    // Small batches skip both copy operations: the ks kernel reads Z / Sigma from the mapped pinned buffer
    // (each of its CTAs reads HG x Nx doubles once: only worthwhile while that re-read volume is small) and the
    // assembling CTA writes mean / var / J / cov straight into it (posted writes, visible after the stream sync).
    const long long ks_ctas = (long long)ks_blocks(h) * round8(std::min(H, HB)) * h->nloc;
    const bool zc_in = H <= HB && ks_ctas * Nx * 8 <= 256 * 1024 && in_span * 8 <= 64 * 1024;
    const bool zc_out = out_span * 8 <= 1024 * 1024;
    double* po = pin + in_span;
    const double* dZ_ = h->dZ; const double* dS_ = h->dSigma;
    if (zc_in) { dZ_ = h->dPinnedAlias; dS_ = h->dPinnedAlias + cap * Nx; }
    else CUDA_TRY(cudaMemcpyAsync(h->dIn, pin, in_span * 8, cudaMemcpyHostToDevice, h->st));
    auto fld = [&](size_t off) { return zc_out ? h->dPinnedAlias + in_span + (off - lo) : h->dOut + off; };
    double* o_mean = mean ? fld(0) : nullptr;
    double* o_var = var ? fld(off_var) : nullptr;
    double* o_cov = cov ? fld(off_c) : nullptr;
    double* o_jac = jac ? fld(off_j) : nullptr;
    rc = ut ? ut_pass(h, H, dZ_, dS_, spp, o_mean, o_var, o_cov, o_jac)
            : predict_core(h, method, H, dZ_, dS_, spp, o_mean, o_var, o_cov, o_jac);
    if (rc) return rc;
    if (out_span && !zc_out) CUDA_TRY(cudaMemcpyAsync(po, h->dOut + lo, out_span * 8, cudaMemcpyDeviceToHost, h->st));
    CUDA_TRY(cudaStreamSynchronize(h->st));
    { int prc = peer_status_check(h); if (prc) return prc; }
    if (mean) memcpy(mean, po + (0 - lo), nm * 8);
    if (var) memcpy(var, po + (off_var - lo), nm * 8);
    if (jac) memcpy(jac, po + (off_j - lo), nj * 8);
    if (cov) memcpy(cov, po + (off_c - lo), nc * 8);
    return GPMPC_OK;
}

// ------------------------------------------------------------------------------------
// predict + first derivatives w.r.t. the test inputs (SURVEY 8f row 1: the GPU half of the
// CasADi adapter).  Same outputs as gpmpc_predict plus
//   dvar_dz (H,Ny,Nx), dcov_dz (H,Ny,Ny,Nx), hess (H,Ny,Nx,Nx) = d^2 mean / dz^2   (each optional)
// (d mean / dz is `jac`.)  Needs all outputs on this handle.
// ------------------------------------------------------------------------------------
template <int NXP>
static cudaError_t launch_grad_reduce(gpmpc_handle_t h, const double* dZc, int Hc, int nblk)
{
    dim3 g(nblk, Hc, h->nloc);
    const int smem = (h->Nx * 257 + 256) * 8;
    const cudaError_t e = smem_opt_in<grad_reduce_kernel<NXP>>((NX_MAX * 257 + 256) * 8);   // static + dynamic may pass 48 KB
    if (e != cudaSuccess) return e;
    grad_reduce_kernel<NXP><<<g, 256, smem, h->st>>>(h->dXT, h->Npad, h->N, h->Nx, h->dHyp, h->Nx + 2, h->dAlpha, h->Npad, dZc,
                                                      h->dKST, h->dBeta, h->Npad, (long long)HB * h->Npad, h->dPDV, h->dPH, nblk, Hc);
    return cudaGetLastError();
}

template <int NXP>
static cudaError_t launch_hess_reduce(gpmpc_handle_t h, const double* dZc, int Hc, int p0, int Rc, int nblk)
{
    dim3 g(nblk, Rc, h->nloc);
    const int smem = (2 * h->Nx * 257 + 512) * 8;
    const cudaError_t e = smem_opt_in<hess_reduce_kernel<NXP>>((2 * NX_MAX * 257 + 512) * 8);   // static + dynamic may pass 48 KB
    if (e != cudaSuccess) return e;
    hess_reduce_kernel<NXP><<<g, 256, smem, h->st>>>(h->dXT, h->Npad, h->N, h->Nx, h->dHyp, h->Nx + 2, h->dAlpha, h->Npad, dZc,
                                                      h->dKST, h->dBeta, h->dVD, h->Npad, (long long)HB * h->Npad,
                                                      h->dPG, h->dPB2, h->dPM3, nblk, Hc, p0);
    return cudaGetLastError();
}

// Second derivatives of one chunk of Hc <= 64 points, after predict_grad's chain for it (ks, v, beta, records):
// R = 64/Nx points per pass, each pass = derivative rows -> V_d = L^-1 d_d ks on the predict product (lower
// mode, rows stored, no finalize) -> Gram / moment partials; one finalize per chunk.
static int hess_chunk(gpmpc_handle_t h, const double* dZc, int Hc, int H, int h0, double* d_d2var, double* d_d3mean)
{
    const int np = h->Npad, Nx = h->Nx, R = HB / Nx, nblk = (np + GR_CHUNK - 1) / GR_CHUNK;
    for (int p0 = 0; p0 < Hc; p0 += R) {
        const int Rc = std::min(R, Hc - p0), rows = Rc * Nx;
        hess_rows_kernel<<<dim3((np + 255) / 256, Rc, h->nloc), 256, 0, h->st>>>(h->dXT, np, h->N, Nx, h->dHyp, Nx + 2, dZc,
                                                                                h->dKST, np, (long long)HB * np, h->dDR, p0);
        CUDA_TRY(cudaGetLastError());
        int rc = tri_product(h, h->dDR, h->dLi, rows, h->dVD);
        if (rc) return rc;
        CUDA_TRY(nxp_dispatch(Nx, [&](auto nxp) { return launch_hess_reduce<decltype(nxp)::value>(h, dZc, Hc, p0, Rc, nblk); }));
    }
    hess_finalize_kernel<<<dim3(Hc, h->nloc), 128, 0, h->st>>>(h->dPG, h->dPB2, h->dPM3, nblk, Hc, h->dHyp, Nx + 2, Nx, h->Ny,
                                                               h->dG, H, h0, d_d2var, d_d3mean);
    CUDA_TRY(cudaGetLastError());
    return GPMPC_OK;
}

// Second-derivative outputs of predict_derivs (null: first derivatives only, gpmpc_predict_grad)
struct HessOutputs {
    double *d2var_dz2, *d3mean_dz3, *d2cov_dz2;
};

// Buffers of the derivative chain for H points (predict_prepare first) and U = Linv^T, built once per factorisation
static int derivs_prepare(gpmpc_handle_t h, int H, bool second, DerivSlabs* s)
{
    const int np = h->Npad, Nx = h->Nx, Ny = h->Ny, npairs = Nx * (Nx + 1) / 2;
    const int nblk_g = (np + GR_CHUNK - 1) / GR_CHUNK;
    ENSURE(h->dUall, (long long)h->nloc * slab(h));
    ENSURE(h->dBeta, (long long)h->nloc * HB * np);
    ENSURE(h->dPDV, (long long)h->nloc * HB * nblk_g * Nx);
    ENSURE(h->dPH, (long long)h->nloc * HB * nblk_g * npairs);
    const int rc = ensure_rows(h);
    if (rc) return rc;
    if (!h->u_valid) {                 // U = Linv^T (upper): the K-contiguous operand of beta = Linv^T v
        dim3 g(np / 32, np / 32), b(32, 8);
        for (int a = 0; a < h->nloc; ++a) {
            transpose_lower_kernel<<<g, b, 0, h->st>>>(h->dLi + (long long)a * slab(h), 0, h->dUall + (long long)a * slab(h), 0, np,
                                                       np / 32);
            CUDA_TRY(cudaGetLastError());
        }
        h->u_valid = true;
    }
    const long long per = (long long)Ny * Nx + (long long)Ny * Ny * Nx + (long long)Ny * Nx * Nx;   // dvar | dcov | hess per point
    ENSURE(h->dGradOut, (long long)std::max(H, HB) * per);
    s->dvar = h->dGradOut;
    s->dcov = s->dvar + (long long)H * Ny * Nx;
    s->hess = s->dcov + (long long)H * Ny * Ny * Nx;
    const long long nxx = (long long)Nx * Nx, ntri = (long long)Nx * (Nx + 1) * (Nx + 2) / 6;
    s->d2var = s->d3mean = s->d2cov = s->sh = nullptr;
    if (second) {
        ENSURE(h->dDR, (long long)h->nloc * HB * np);      // zero-filled: rows past a pass's last are never written
        ENSURE(h->dVD, (long long)h->nloc * HB * np);
        ENSURE(h->dPG, (long long)h->nloc * HB * nblk_g * npairs);
        ENSURE(h->dPB2, (long long)h->nloc * HB * nblk_g * npairs);
        ENSURE(h->dPM3, (long long)h->nloc * HB * nblk_g * ntri);
        const long long hper = 2 * Ny * nxx + Ny * nxx * Nx + (long long)Ny * Ny * nxx;      // d2var | SH scratch | d3mean | d2cov
        ENSURE(h->dHessOut, (long long)std::max(H, HB) * hper);
        s->d2var = h->dHessOut;
        s->sh = s->d2var + (long long)H * Ny * nxx;
        s->d3mean = s->sh + (long long)H * Ny * nxx;
        s->d2cov = s->d3mean + (long long)H * Ny * nxx * Nx;
    }
    return GPMPC_OK;
}

// The derivative chain of H device-resident points dZ (H,Nx), Sigma dSigma (per point if spp), after derivs_prepare:
// per 64-point chunk ks, v = Linv ks with the gather records, beta = Linv^T v, the block partials of dvar / mean Hessian
// and their finalisation (with s.d2var, the second-derivative passes); then the assembly of mean, var, J, cov into dOut
// and d cov / dz.  gpmpc_predict_grad / _hess run it on their uploaded points, gpmpc_rollout_batch_grad on every step's.
// beta (may be null): every chunk's beta rows are copied there, row h of output a at beta + a * sbeta + h * Npad
// (gpmpc_rollout_sample_grad's store).
static int derivs_enqueue(gpmpc_handle_t h, int method, int H, const double* dZ, const double* dSigma, int spp,
                          const DerivSlabs& s, double* beta, long long sbeta)
{
    const int np = h->Npad, Nx = h->Nx, Ny = h->Ny;
    const int nblk_g = (np + GR_CHUNK - 1) / GR_CHUNK;
    const AssembleArgs as = assemble_args(h, H, method, dSigma, spp, h->dMean, h->dVar, h->dJ, h->dCov);
    for (int h0 = 0; h0 < H; h0 += HB) {
        const int Hc = std::min(HB, H - h0);
        const double* dZc = dZ + (long long)h0 * Nx;
        CUDA_TRY(launch_ks(h, dZc, Hc));
        PredictParams p;
        psk_base(h, p, Hc);                                   // v = Linv ks: records + the rows themselves
        psk_finalize(h, p, H, h0);
        p.Vout = h->dV; p.sV = (long long)HB * np; p.ldv = np;
        CUDA_TRY(psk_launch(h, p, h->dKST, h->dLi));
        psk_base(h, p, Hc, 1);                                // beta = Linv^T v = K^-1 ks  (rows of V times U^T)
        p.Vout = h->dBeta; p.sV = (long long)HB * np; p.ldv = np;
        CUDA_TRY(psk_launch(h, p, h->dV, h->dUall));
        if (beta) {
            copy2d_kernel<<<dim3(16, std::min(Hc, 64), h->nloc), 128, 0, h->st>>>(h->dBeta, np, (long long)HB * np,
                                                                           beta + (long long)h0 * np, np, sbeta, Hc, np);
            CUDA_TRY(cudaGetLastError());
        }
        CUDA_TRY(nxp_dispatch(Nx, [&](auto nxp) { return launch_grad_reduce<decltype(nxp)::value>(h, dZc, Hc, nblk_g); }));
        grad_finalize_kernel<<<dim3(Hc, h->nloc), 128, 0, h->st>>>(h->dPDV, h->dPH, nblk_g, Hc, h->dHyp, Nx + 2, Nx, Ny,
                                                                   h->dG, H, h0, s.dvar, s.hess);
        CUDA_TRY(cudaGetLastError());
        if (s.d2var) {
            const int rc = hess_chunk(h, dZc, Hc, H, h0, s.d2var, s.d3mean);
            if (rc) return rc;
        }
    }
    const int smem = (2 * Ny * Nx + Ny) * 8;
    assemble_kernel<<<std::min(H, 2048), 128, smem, h->st>>>(as);
    CUDA_TRY(cudaGetLastError());
    grad_cov_kernel<<<H, 128, 2 * Ny * Nx * 8, h->st>>>(Ny, Nx, method == GPMPC_METHOD_TA, dSigma, spp, h->dJ, s.dvar, s.hess, s.dcov);
    CUDA_TRY(cudaGetLastError());
    if (s.d2var) {
        hess_cov_kernel<<<H, 128, 2 * Ny * Nx * 8, h->st>>>(Ny, Nx, method == GPMPC_METHOD_TA, dSigma, spp, h->dJ, s.hess,
                                                            s.d2var, s.d3mean, s.sh, s.d2cov);
        CUDA_TRY(cudaGetLastError());
    }
    return GPMPC_OK;
}

static int predict_derivs(gpmpc_handle_t h, const char* fn, int method, int H, const double* Z, const double* Sigma, int spp,
                          double* mean, double* var, double* cov, double* jac,
                          double* dvar_dz, double* dcov_dz, double* hess, const HessOutputs* ho)
{
    int rc = predict_guard(h, fn, method, H);
    if (rc) return rc;
    if (method == GPMPC_METHOD_EM) { set_error(h, "%s: derivatives are available for ME and TA", fn); return GPMPC_ERR_ARG; }
    if (!Z || (method == GPMPC_METHOD_TA && !Sigma)) { set_error(h, "%s: null Z / Sigma", fn); return GPMPC_ERR_ARG; }
    rc = predict_prepare(h, fn, H, true);
    if (rc) return rc;
    NvtxRange nvtx_r(ho ? "gpmpc.predict_hess" : "gpmpc.predict_grad");
    const int Nx = h->Nx, Ny = h->Ny;
    const long long nxx = (long long)Nx * Nx;
    DerivSlabs s;
    rc = derivs_prepare(h, H, ho != nullptr, &s);
    if (rc) return rc;
    const size_t nz = (size_t)H * Nx, ns = (method == GPMPC_METHOD_TA) ? (size_t)(spp ? H : 1) * Nx * Nx : 0;
    CUDA_TRY(cudaMemcpyAsync(h->dZ, Z, nz * 8, cudaMemcpyHostToDevice, h->st));
    if (ns) CUDA_TRY(cudaMemcpyAsync(h->dSigma, Sigma, ns * 8, cudaMemcpyHostToDevice, h->st));
    rc = derivs_enqueue(h, method, H, h->dZ, h->dSigma, spp, s);
    if (rc) return rc;
    const double *d_dvar = s.dvar, *d_dcov = s.dcov, *d_hess = s.hess, *d_d2var = s.d2var, *d_d3mean = s.d3mean, *d_d2cov = s.d2cov;
    if (mean) CUDA_TRY(cudaMemcpyAsync(mean, h->dMean, (size_t)H * Ny * 8, cudaMemcpyDeviceToHost, h->st));
    if (var) CUDA_TRY(cudaMemcpyAsync(var, h->dVar, (size_t)H * Ny * 8, cudaMemcpyDeviceToHost, h->st));
    if (cov) CUDA_TRY(cudaMemcpyAsync(cov, h->dCov, (size_t)H * Ny * Ny * 8, cudaMemcpyDeviceToHost, h->st));
    if (jac) CUDA_TRY(cudaMemcpyAsync(jac, h->dJ, (size_t)H * Ny * Nx * 8, cudaMemcpyDeviceToHost, h->st));
    if (dvar_dz) CUDA_TRY(cudaMemcpyAsync(dvar_dz, d_dvar, (size_t)H * Ny * Nx * 8, cudaMemcpyDeviceToHost, h->st));
    if (dcov_dz) CUDA_TRY(cudaMemcpyAsync(dcov_dz, d_dcov, (size_t)H * Ny * Ny * Nx * 8, cudaMemcpyDeviceToHost, h->st));
    if (hess) CUDA_TRY(cudaMemcpyAsync(hess, d_hess, (size_t)H * Ny * Nx * Nx * 8, cudaMemcpyDeviceToHost, h->st));
    if (ho && ho->d2var_dz2) CUDA_TRY(cudaMemcpyAsync(ho->d2var_dz2, d_d2var, (size_t)H * Ny * nxx * 8, cudaMemcpyDeviceToHost, h->st));
    if (ho && ho->d3mean_dz3) CUDA_TRY(cudaMemcpyAsync(ho->d3mean_dz3, d_d3mean, (size_t)H * Ny * nxx * Nx * 8, cudaMemcpyDeviceToHost, h->st));
    if (ho && ho->d2cov_dz2) CUDA_TRY(cudaMemcpyAsync(ho->d2cov_dz2, d_d2cov, (size_t)H * Ny * Ny * nxx * 8, cudaMemcpyDeviceToHost, h->st));
    CUDA_TRY(cudaStreamSynchronize(h->st));
    return GPMPC_OK;
}

extern "C" int gpmpc_predict_grad(gpmpc_handle_t h, int method, int H, const double* Z, const double* Sigma, int spp,
                                  double* mean, double* var, double* cov, double* jac,
                                  double* dvar_dz, double* dcov_dz, double* hess)
{
    return predict_derivs(h, "gpmpc_predict_grad", method, H, Z, Sigma, spp, mean, var, cov, jac, dvar_dz, dcov_dz, hess, nullptr);
}

// predict_grad plus the second derivatives IPOPT's exact Hessian needs (see include/gpmpc.h)
extern "C" int gpmpc_predict_hess(gpmpc_handle_t h, int method, int H, const double* Z, const double* Sigma, int spp,
                                  double* mean, double* var, double* cov, double* jac,
                                  double* dvar_dz, double* dcov_dz, double* hess,
                                  double* d2var_dz2, double* d3mean_dz3, double* d2cov_dz2)
{
    const HessOutputs ho = {d2var_dz2, d3mean_dz3, d2cov_dz2};
    return predict_derivs(h, "gpmpc_predict_hess", method, H, Z, Sigma, spp, mean, var, cov, jac, dvar_dz, dcov_dz, hess, &ho);
}

// The 'EM' derivative entry points (see include/gpmpc.h): first derivatives, and second ones when ho is given (Nx <= 16)
static int predict_em_derivs(gpmpc_handle_t h, const char* fn, int H, const double* Z, const double* Sigma, int spp,
                             double* mean, double* var, double* cov, const EmGradOutputs& go, const EmHessOutputs* ho)
{
    int rc = predict_guard(h, fn, GPMPC_METHOD_EM, H);
    if (rc) return rc;
    if (!Z || !Sigma) { set_error(h, "%s: null Z / Sigma", fn); return GPMPC_ERR_ARG; }
    if (ho && h->Nx > 16) { set_error(h, "%s supports Nx <= 16", fn); return GPMPC_ERR_ARG; }
    rc = predict_prepare(h, fn, H, true);
    if (rc) return rc;
    NvtxRange nvtx_r(ho ? "gpmpc.predict_em_hess" : "gpmpc.predict_em_grad");
    const bool any_g = go.dmean_dz || go.dmean_dSigma || go.dcov_dz || go.dcov_dSigma;   // none: no K^-1 cache for them
    const bool any_h = ho && (ho->d2mean_dz2 || ho->d2mean_dSigma_dz || ho->d2mean_dSigma2 || ho->d2cov_dz2 ||
                              ho->d2cov_dSigma_dz || ho->d2cov_dSigma2);
    return predict_em(h, H, Z, Sigma, spp, mean, var, cov, any_g ? &go : nullptr, any_h ? ho : nullptr);
}

extern "C" int gpmpc_predict_em_grad(gpmpc_handle_t h, int H, const double* Z, const double* Sigma, int spp,
                                     double* mean, double* var, double* cov,
                                     double* dmean_dz, double* dmean_dSigma, double* dcov_dz, double* dcov_dSigma)
{
    const EmGradOutputs go = {dmean_dz, dmean_dSigma, dcov_dz, dcov_dSigma};
    return predict_em_derivs(h, __func__, H, Z, Sigma, spp, mean, var, cov, go, nullptr);
}

extern "C" int gpmpc_predict_em_hess(gpmpc_handle_t h, int H, const double* Z, const double* Sigma, int spp,
                                     double* mean, double* var, double* cov,
                                     double* dmean_dz, double* dmean_dSigma, double* dcov_dz, double* dcov_dSigma,
                                     double* d2mean_dz2, double* d2mean_dSigma_dz, double* d2mean_dSigma2,
                                     double* d2cov_dz2, double* d2cov_dSigma_dz, double* d2cov_dSigma2)
{
    const EmGradOutputs go = {dmean_dz, dmean_dSigma, dcov_dz, dcov_dSigma};
    const EmHessOutputs ho = {d2mean_dz2, d2mean_dSigma_dz, d2mean_dSigma2, d2cov_dz2, d2cov_dSigma_dz, d2cov_dSigma2};
    return predict_em_derivs(h, __func__, H, Z, Sigma, spp, mean, var, cov, go, &ho);
}

// Row Nk of L and L^-1 of every owned output from l = L^-1 k (rows < Nk of dV): r = Li^T l over the Nk rows l occupies,
// then append_row_kernel.  stop (may be null): a greedy step after a failed pivot writes nothing.
static int append_rows(gpmpc_handle_t h, int Nk, const int* stop)
{
    const int np = h->Npad, Nx = h->Nx, nl = h->nloc;
    const long long sl = (long long)HB * np;
    panel_stale(h, -1, Nk);
    trmv_lower_T_kernel<<<dim3((Nk + 31) / 32, 1, nl), 256, 0, h->st>>>(h->dLi, np, slab(h), h->dV, sl, h->dR, sl, Nk);
    CUDA_TRY(cudaGetLastError());
    append_row_kernel<<<nl, 256, 0, h->st>>>(h->dL, h->dLi, np, slab(h), h->dV, h->dR, sl, h->dHyp, Nx + 2, Nx, h->dFacJit,
                                             Nk, h->dInfo, stop);
    CUDA_TRY(cudaGetLastError());
    return GPMPC_OK;
}

// End of n_new appends to N0 points (syncs): a failed pivot of step k reads N0 + k + 1 in dInfo.  N counts the points up to
// and including the first failing step (*added); after a failure the caller must refactorise, else alpha is refreshed.
static int finish_appends(gpmpc_handle_t h, const char* fn, int N0, int n_new, int* added)
{
    const int nl = h->nloc;
    std::vector<int> inf(nl, 0);
    CUDA_TRY(cudaMemcpyAsync(inf.data(), h->dInfo, nl * sizeof(int), cudaMemcpyDeviceToHost, h->st));
    CUDA_TRY(cudaStreamSynchronize(h->st));
    int fail = n_new, bad = -1;
    for (int a = 0; a < nl; ++a)
        if (inf[a] && inf[a] - N0 - 1 < fail) { fail = inf[a] - N0 - 1; bad = a; }
    *added = (bad >= 0) ? fail + 1 : n_new;
    h->N = N0 + *added;
    if (bad >= 0) {
        factor_stale(h);
        set_error(h, "%s: output %d lost positive definiteness at pick %d (refactorise, jitter applies there)", fn,
                  h->a0 + bad, *added - 1);
        return GPMPC_ERR_NOTPD;
    }
    return refresh_alpha(h);
}

extern "C" int gpmpc_append(gpmpc_handle_t h, const double* x_new, const double* y_new)
{
    if (!h || !x_new || !y_new) return GPMPC_ERR_ARG;
    int rc = model_guard(h, __func__, NEED_FACTOR);
    if (rc) return rc;
    if (h->N >= h->Npad) { set_error(h, "gpmpc_append: capacity %d reached, refit on a new handle", h->Npad); return GPMPC_ERR_STATE; }
    rc = predict_prepare(h, __func__, 1, false);
    if (rc) return rc;
    const int N = h->N, Nx = h->Nx, np = h->Npad, nl = h->nloc;
    // k(X, x_new) for every owned output through the predict ks kernel (H = 1): row 0 of KS^T
    CUDA_TRY(cudaMemcpyAsync(h->dZ, x_new, Nx * 8, cudaMemcpyHostToDevice, h->st));
    CUDA_TRY(launch_ks(h, h->dZ, 1));
    // l = Li k (rows < N)
    rc = ensure_rows(h);
    if (rc) return rc;
    dim3 g1((np + 7) / 8, 1, nl);
    trmv_lower_kernel<<<g1, 256, 0, h->st>>>(h->dLi, np, slab(h), h->dKST, (long long)HB * np, h->dV, (long long)HB * np, N);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemsetAsync(h->dInfo, 0, nl * sizeof(int), h->st));
    rc = append_rows(h, N, nullptr);
    if (rc) return rc;
    // the new point joins X^T (column N) and Y
    for (int d = 0; d < Nx; ++d) CUDA_TRY(cudaMemcpyAsync(h->dXT + (long long)d * np + N, x_new + d, 8, cudaMemcpyHostToDevice, h->st));
    for (int a = 0; a < nl; ++a) CUDA_TRY(cudaMemcpyAsync(h->dY + (long long)a * np + N, y_new + h->a0 + a, 8, cudaMemcpyHostToDevice, h->st));
    int added = 0;
    rc = finish_appends(h, __func__, N, 1, &added);
    if (h->N > N) {                                   // counted even when the pivot failed
        h->hX.insert(h->hX.end(), x_new, x_new + Nx);
        h->mu_stale = true;
    }
    return rc;
}

// The solved rows v = L^-1 k(X, z) of the H points at dZ (device, (H, Nx)) for every owned output into dst: row h of
// output a at dst + a * sdst + h * Npad.  HB-point chunks through the ks kernel and the predict product.  mean (may be
// null): ks^T alpha of every point, (nloc, H), summed from each chunk's ks partials before the next chunk's ks launch
// overwrites them, in the predict product's order (gpmpc_predict's mean bit for bit).
static int solve_rows(gpmpc_handle_t h, const double* dZ, int H, double* dst, long long sdst, double* mean = nullptr)
{
    const int np = h->Npad, Nx = h->Nx, nl = h->nloc;
    int rc = ensure_rows(h);
    if (rc) return rc;
    for (int h0 = 0; h0 < H; h0 += HB) {
        const int Hc = std::min(HB, H - h0);
        const double* dZc = dZ + (long long)h0 * Nx;
        CUDA_TRY(launch_ks(h, dZc, Hc));
        rc = tri_product(h, h->dKST, h->dLi, Hc, h->dV);
        if (rc) return rc;
        copy2d_kernel<<<dim3(16, std::min(Hc, 64), nl), 128, 0, h->st>>>(h->dV, np, (long long)HB * np,
                                                                     dst + (long long)h0 * np, np, sdst, Hc, np);
        CUDA_TRY(cudaGetLastError());
        if (mean) {
            ks_mean_kernel<<<(nl * Hc + 255) / 256, 256, 0, h->st>>>(h->dPMJ, ks_blocks(h), Nx, Hc, nl, mean + h0, H);
            CUDA_TRY(cudaGetLastError());
        }
    }
    return GPMPC_OK;
}

extern "C" int gpmpc_posterior_cov(gpmpc_handle_t h, int H, const double* Z, double* out)
{
    if (!h || !Z || !out || H < 1) return GPMPC_ERR_ARG;
    int rc = model_guard(h, __func__, NEED_FACTOR);
    if (rc) return rc;
    rc = predict_prepare(h, __func__, H, false);
    if (rc) return rc;
    const int np = h->Npad, Nx = h->Nx, nl = h->nloc;
    const long long sVall = (long long)H * np;
    ENSURE(h->dCovOut, (long long)nl * H * H);
    ENSURE(h->dCovV, (long long)nl * sVall);              // pooled on the handle (grown on demand), not per call
    CUDA_TRY(cudaMemcpyAsync(h->dZ, Z, (size_t)H * Nx * 8, cudaMemcpyHostToDevice, h->st));
    rc = solve_rows(h, h->dZ, H, h->dCovV, sVall);
    if (rc) return rc;
    gram_cov_kernel<<<dim3(H, H, nl), 256, 0, h->st>>>(h->dCovV, np, sVall, np, h->dHyp, Nx + 2, Nx, H, h->dCovOut);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(out, h->dCovOut, (size_t)nl * H * H * 8, cudaMemcpyDeviceToHost, h->st));
    CUDA_TRY(cudaStreamSynchronize(h->st));
    return GPMPC_OK;
}

// A conditional variance at or below SAMPLE_DELTA sf2 is rounding: the point is a function of the earlier ones (DESIGN 4.12)
#define SAMPLE_DELTA 1e-12

// Sampled roll-outs (kernels.cuh, sample_cond_kernel): per step the V rows of the B current inputs go to slot t of the
// store (solve_rows, with their means), one CTA per (trajectory, output) draws f_t conditioned on the trajectory's
// earlier kept points, and rollout_feedback_kernel forms the next input from f_t.  All steps are enqueued back to back;
// one D2H copy and one synchronisation at the end.  With dsamples (gpmpc_rollout_sample_grad, DESIGN 4.16) each step
// also runs the derivative chain on the same points (J, dvar_dz, and beta rows into slot t of the beta store), then after
// the draw sample_cross_kernel, sample_next_kernel (step t's input tangents) and sample_tangent_kernel; without it the
// launches are exactly those of the draw alone.
static int rollout_sample(gpmpc_handle_t h, const char* fn, int B, int Nt, const double* z0, const double* U,
                          const double* eps, const double* xi, const double* scale, const double* K, const double* x_ref,
                          const double* uscale, double* samples, double* z_out, int* kept, bool tg, double* dsamples)
{
    int rc = predict_guard(h, fn, GPMPC_METHOD_ME, 1);
    if (rc) return rc;
    const int Nx = h->Nx, Ny = h->Ny, Nu = Nx - Ny, np = h->Npad, nl = h->nloc;
    rc = rollout_args(h, fn, B, Nt, !z0 || !eps || !samples, U, K);
    if (rc) return rc;
    const int cond_smem = sample_cond_smem(Nt).bytes;
    if (cond_smem > 48 * 1024) { set_error(h, "%s: Nt = %d steps exceed the conditioning kernel's shared memory", fn, Nt); return GPMPC_ERR_ARG; }
    if (tg && !dsamples) { set_error(h, "%s: null dsamples", fn); return GPMPC_ERR_ARG; }
    if (tg && Nt > SAMPLE_GRAD_NT_MAX) {
        set_error(h, "%s: Nt = %d steps exceed the tangent kernel's shared memory (Nt <= %d)", fn, Nt, SAMPLE_GRAD_NT_MAX);
        return GPMPC_ERR_ARG;
    }
    rc = predict_prepare(h, fn, B, true);
    if (rc) return rc;
    NvtxRange nvtx_r(tg ? "gpmpc.rollout_sample_grad" : "gpmpc.rollout_sample");
    const size_t Bs = (size_t)B, nE = Bs * Nt * Ny, nX = xi ? nE : 0, o_xi = nE, o_u = o_xi + nX;
    const size_t o_z = rollout_policy(B, Nt, Ny, Nu, U, scale, K, x_ref, uscale, o_u);
    const size_t o_s = o_z + (size_t)Nt * Bs * Nx, o_kp = o_s + nE;
    const size_t o_m = o_kp + nE, o_r = o_m + (size_t)nl * Bs, tot = o_r + (size_t)nl * Bs * Nt * Nt;
    const long long sVa = (long long)Nt * B * np;          // V rows of one output: (Nt, B, Npad)
    ENSURE(h->dSmV, nl * sVa);
    ENSURE(h->dSmp, tot);
    // tangent slab [G (nloc,B,Nt,2,Nx) | dR (nloc,B,P,Nt,Nt) | dz (Nt,B,P,Nx) | dsamples (Nt,B,Ny,P)]; the beta store is
    // laid out like the V store.  dsamples is mirrored in the pinned buffer after the draw's outputs.
    const size_t P = tg ? rollout_params(Nx, Ny, Nt, K != nullptr) : 0;
    const size_t o_dr = (size_t)nl * Bs * Nt * 2 * Nx, o_dz = o_dr + (size_t)nl * Bs * P * Nt * Nt;
    const size_t o_ds = o_dz + (size_t)Nt * Bs * P * Nx, nDs = tg ? (size_t)Nt * Bs * Ny * P : 0;
    const int tg_smem = sample_tangent_smem(Nt).bytes, nx_smem = sample_next_smem(Ny).bytes;
    DerivSlabs ds;
    if (tg) {
        rc = derivs_prepare(h, B, false, &ds);
        if (rc) return rc;
        ENSURE(h->dSmB, nl * sVa);
        ENSURE(h->dSmTg, o_ds + nDs);
    }
    rc = ensure_pinned(h, (o_m + nDs) * 8);
    if (rc) return rc;
    double* pin = h->hPinned;
    memcpy(pin, eps, nE * 8);
    if (nX) memcpy(pin + o_xi, xi, nX * 8);
    double* d = h->dSmp;
    RolloutPolicy pol;
    rollout_policy(B, Nt, Ny, Nu, U, scale, K, x_ref, uscale, o_u, pin, d, &pol);
    memcpy(pin + o_z, z0, Bs * Nx * 8);                     // slot 0 of the input history
    CUDA_TRY(cudaMemcpyAsync(d, pin, (o_z + Bs * Nx) * 8, cudaMemcpyHostToDevice, h->st));
    const int fb_smem = rollout_feedback_smem(Ny, Nu, K != nullptr, false).bytes;
    double* g = tg ? h->dSmTg.p : nullptr;
    for (int t = 0; t < Nt; ++t) {
        double* Zt = d + o_z + (size_t)t * Bs * Nx;
        rc = solve_rows(h, Zt, B, h->dSmV + (long long)t * B * np, sVa, d + o_m);
        if (rc) return rc;
        if (tg) {                                           // J_t, dvar_dz_t and the beta rows of the step's points
            rc = derivs_enqueue(h, GPMPC_METHOD_ME, B, Zt, nullptr, 1, ds, h->dSmB + (long long)t * B * np, sVa);
            if (rc) return rc;
        }
        sample_cond_kernel<<<dim3(B, nl), 256, cond_smem, h->st>>>(h->dSmV, sVa, np, h->N, d + o_m, d + o_z, h->dHyp, Nx + 2,
                                                                 Nx, Ny, d, xi ? d + o_xi : nullptr, d + o_r, d + o_kp,
                                                                 d + o_s, Nt, t, SAMPLE_DELTA);
        CUDA_TRY(cudaGetLastError());
        if (tg) {
            if (t > 0) {
                sample_cross_kernel<<<dim3(B, nl, t), 256, 0, h->st>>>(h->dSmB, sVa, np, h->dXT, np, h->N, d + o_z, h->dHyp,
                                                                       Nx + 2, Nx, Ny, d + o_kp, g, Nt, t);
                CUDA_TRY(cudaGetLastError());
            }
            double* ds_t = g + o_ds + (size_t)t * Bs * Ny * P;
            sample_next_kernel<<<B, ROLL_TG_WARPS * 32, nx_smem, h->st>>>(Ny, Nu, (int)P, t, d + o_s + (size_t)(t > 0 ? t - 1 : 0) * Bs * Ny,
                                                               ds_t - (t > 0 ? Bs * Ny * P : 0), pol.scale, pol.K, pol.x_ref,
                                                               pol.uscale, g + o_dz + (size_t)t * Bs * P * Nx);
            CUDA_TRY(cudaGetLastError());
            sample_tangent_kernel<<<dim3(B, nl), ROLL_TG_WARPS * 32, tg_smem, h->st>>>(h->dSmV, sVa, np, h->N, d + o_z, h->dHyp, Nx + 2,
                                                                           Nx, Ny, d, d + o_r, d + o_kp, h->dJ, ds.dvar, g,
                                                                           g + o_dz, g + o_dr, ds_t, (int)P, Nt, t);
            CUDA_TRY(cudaGetLastError());
        }
        if (t + 1 < Nt) {
            rollout_feedback_kernel<<<B, 256, fb_smem, h->st>>>(d + o_s + (size_t)t * Bs * Ny, nullptr, d + o_u + (size_t)(t + 1) * Nu,
                                                                (long long)Nt * Nu, pol.scale, pol.K, pol.x_ref, pol.uscale,
                                                                Ny, Nu, Zt + Bs * Nx, nullptr);
            CUDA_TRY(cudaGetLastError());
        }
    }
    CUDA_TRY(cudaMemcpyAsync(pin + o_z, d + o_z, (o_m - o_z) * 8, cudaMemcpyDeviceToHost, h->st));
    if (tg) CUDA_TRY(cudaMemcpyAsync(pin + o_m, g + o_ds, nDs * 8, cudaMemcpyDeviceToHost, h->st));
    CUDA_TRY(cudaStreamSynchronize(h->st));
    rows_by_trajectory(samples, pin + o_s, B, Nt, Ny);
    if (z_out) rows_by_trajectory(z_out, pin + o_z, B, Nt, Nx);
    if (kept)
        for (size_t b = 0; b < Bs; ++b)
            for (int t = 0; t < Nt; ++t) {
                const size_t src = (size_t)t * Bs + b, dst = b * Nt + t;
                for (int a = 0; a < Ny; ++a) kept[dst * Ny + a] = pin[o_kp + src * Ny + a] != 0.0 ? 1 : 0;
            }
    if (tg) rows_by_trajectory(dsamples, pin + o_m, B, Nt, (size_t)Ny * P);
    return GPMPC_OK;
}

extern "C" int gpmpc_rollout_sample(gpmpc_handle_t h, int B, int Nt, const double* z0, const double* U, const double* eps,
                                    const double* xi, const double* scale, const double* K, const double* x_ref,
                                    const double* uscale, double* samples, double* z_out, int* kept)
{
    return rollout_sample(h, __func__, B, Nt, z0, U, eps, xi, scale, K, x_ref, uscale, samples, z_out, kept, false, nullptr);
}

// gpmpc_rollout_sample plus the pathwise derivatives of every draw (see include/gpmpc.h)
extern "C" int gpmpc_rollout_sample_grad(gpmpc_handle_t h, int B, int Nt, const double* z0, const double* U, const double* eps,
                                         const double* xi, const double* scale, const double* K, const double* x_ref,
                                         const double* uscale, double* samples, double* z_out, int* kept, double* dsamples)
{
    return rollout_sample(h, __func__, B, Nt, z0, U, eps, xi, scale, K, x_ref, uscale, samples, z_out, kept, true, dsamples);
}

// Greedy max-variance selection (kernels.cuh, greedy_*): the pool's V and variances are formed once, then each step
// appends the candidate with the largest combined variance by the rank-1 update of gpmpc_append and downdates the rest.
// Every step is enqueued back to back (Nk = N + k is known here); one synchronisation at the end.
extern "C" int gpmpc_append_greedy(gpmpc_handle_t h, int n, const double* Xc, const double* Yc, int n_new,
                                   int* picked, double* score, int* n_added)
{
    if (!h) return GPMPC_ERR_ARG;
    if (!Xc || !Yc || !picked || !n_added) { set_error(h, "gpmpc_append_greedy: null Xc / Yc / picked / n_added"); return GPMPC_ERR_ARG; }
    *n_added = 0;
    if (n < 1 || n_new < 0 || n_new > n) { set_error(h, "gpmpc_append_greedy: need n >= 1 and 0 <= n_new <= n (n = %d, n_new = %d)", n, n_new); return GPMPC_ERR_ARG; }
    int rc = model_guard(h, __func__, NEED_FACTOR);
    if (rc) return rc;
    rc = predict_prepare(h, __func__, 1, true);
    if (rc) return rc;
    if (h->N + n_new > h->Npad) {
        set_error(h, "gpmpc_append_greedy: N + n_new = %d exceeds the capacity %d (reserve it with gpmpc_create_reserve)", h->N + n_new, h->Npad);
        return GPMPC_ERR_STATE;
    }
    if (n_new == 0) return GPMPC_OK;
    NvtxRange nvtx_r("gpmpc.append_greedy");
    const int N = h->N, Nx = h->Nx, np = h->Npad, nl = h->nloc;
    const long long sV = (long long)n * np, sl = (long long)HB * np;
    ENSURE(h->dGrD, (long long)nl * n + (long long)n * (Nx + nl) + n_new);
    ENSURE(h->dGrI, (long long)n + n_new + 1);
    double* dVar = h->dGrD;
    double* dXc = dVar + (long long)nl * n;
    double* dYc = dXc + (long long)n * Nx;
    double* dScore = dYc + (long long)n * nl;
    int* dAct = h->dGrI;
    int* dPick = dAct + n;
    int* dStop = dPick + n_new;
    {
        const std::vector<int> ones(n, 1);
        CUDA_TRY(cudaMemcpyAsync(dAct, ones.data(), (size_t)n * sizeof(int), cudaMemcpyHostToDevice, h->st));
    }
    CUDA_TRY(cudaMemcpyAsync(dXc, Xc, (size_t)n * Nx * 8, cudaMemcpyHostToDevice, h->st));
    CUDA_TRY(cudaMemcpyAsync(dYc, Yc, (size_t)n * nl * 8, cudaMemcpyHostToDevice, h->st));
    CUDA_TRY(cudaMemsetAsync(dStop, 0, sizeof(int), h->st));
    CUDA_TRY(cudaMemsetAsync(h->dInfo, 0, nl * sizeof(int), h->st));
    ENSURE(h->dCovV, (long long)nl * sV);
    rc = solve_rows(h, dXc, n, h->dCovV, sV);
    if (rc) return rc;
    const dim3 gw((n + 7) / 8, nl);
    greedy_var_kernel<<<gw, 256, 0, h->st>>>(h->dCovV, np, sV, N, n, h->dHyp, Nx + 2, Nx, dVar);
    CUDA_TRY(cudaGetLastError());
    for (int k = 0; k < n_new; ++k) {
        const int Nk = N + k;
        greedy_pick_kernel<<<1, 1024, 0, h->st>>>(dVar, n, nl, dAct, dXc, dYc, Nx, h->dXT, h->dY, np, Nk, h->dInfo, dStop,
                                                 dPick, dScore, k);
        CUDA_TRY(cudaGetLastError());
        greedy_gather_kernel<<<dim3((np + 255) / 256, nl), 256, 0, h->st>>>(h->dCovV, np, sV, dPick, k, Nk, h->dV, sl, np, dStop);
        CUDA_TRY(cudaGetLastError());
        rc = append_rows(h, Nk, dStop);     // after a failed pivot r is computed and never read
        if (rc) return rc;
        greedy_downdate_kernel<<<gw, 256, 0, h->st>>>(h->dCovV, np, sV, dVar, n, dAct, h->dV, sl, h->dL, np, slab(h), dXc, Nx,
                                                     h->dHyp, Nx + 2, dPick, k, Nk, h->dInfo, nl);
        CUDA_TRY(cudaGetLastError());
    }
    std::vector<int> pk(n_new, 0);
    std::vector<double> sc(n_new, 0.0);
    CUDA_TRY(cudaMemcpyAsync(pk.data(), dPick, n_new * sizeof(int), cudaMemcpyDeviceToHost, h->st));
    CUDA_TRY(cudaMemcpyAsync(sc.data(), dScore, n_new * 8, cudaMemcpyDeviceToHost, h->st));
    rc = finish_appends(h, __func__, N, n_new, n_added);
    for (int k = 0; k < *n_added; ++k) {
        picked[k] = pk[k];
        if (score) score[k] = sc[k];
        h->hX.insert(h->hX.end(), Xc + (size_t)pk[k] * Nx, Xc + (size_t)(pk[k] + 1) * Nx);
    }
    if (*n_added > 0) h->mu_stale = true;
    return rc;
}

// Removal of training points by rank-1 updates of the trailing blocks of L and L^-1 (kernels.cuh, remove_*), one point
// at a time in descending index order.  Per point: p, d, g for every output, then per output the L rows into dU, the
// L^-1 rows into dKinv (partials over row blocks in the W1 workspace), the copy back with the identity tail row; then
// the point leaves X^T and Y.  alpha and logdet are refreshed once, at the end.
extern "C" int gpmpc_remove(gpmpc_handle_t h, int n, const int* idx)
{
    int rc = model_guard(h, __func__, NEED_FACTOR);
    if (rc) return rc;
    if (n < 0 || (n > 0 && !idx)) { set_error(h, "gpmpc_remove: need n >= 0 and idx non-null for n > 0 (n = %d)", n); return GPMPC_ERR_ARG; }
    if (n == 0) return GPMPC_OK;
    const int N = h->N, Nx = h->Nx, np = h->Npad, nl = h->nloc;
    if (n >= N) { set_error(h, "gpmpc_remove: removing %d of %d points leaves none", n, N); return GPMPC_ERR_ARG; }
    std::vector<int> order(idx, idx + n);
    std::sort(order.begin(), order.end(), [](int u, int v) { return u > v; });
    if (order[0] >= N || order[n - 1] < 0) { set_error(h, "gpmpc_remove: index out of range [0, %d)", N); return GPMPC_ERR_ARG; }
    for (int k = 1; k < n; ++k)
        if (order[k] == order[k - 1]) { set_error(h, "gpmpc_remove: index %d given twice", order[k]); return GPMPC_ERR_ARG; }
    rc = ensure_kinv_scratch(h);          // dU / dKinv: the work slabs of the new rows
    if (rc) return rc;
    ENSURE(h->dRm, (long long)nl * 3 * np);
    NvtxRange nvtx_r("gpmpc.remove");
    panel_stale(h, -1, order[n - 1]);     // rows from the smallest removed index on move up
    const dim3 gcol((np + 255) / 256);
    for (int k = 0; k < n; ++k) {
        const int i = order[k], Nk = N - k, m = Nk - i - 1;     // m trailing points
        if (m > 0) {
            remove_coef_kernel<<<nl, 1024, 0, h->st>>>(h->dL, h->dLi, np, slab(h), i, m, h->dRm);
            CUDA_TRY(cudaGetLastError());
        }
        for (int a = 0; a < nl; ++a) {
            double* L = h->dL + (long long)a * slab(h);
            double* Li = h->dLi + (long long)a * slab(h);
            const double* coef = h->dRm + (long long)a * 3 * np;
            if (m > 0) {
                const int nb = (m + RM_RB - 1) / RM_RB;
                remove_l_rows_kernel<<<m, 256, 0, h->st>>>(L, h->dU, np, coef, i, m);
                CUDA_TRY(cudaGetLastError());
                remove_li_part_kernel<<<dim3(gcol.x, nb), 256, 0, h->st>>>(Li, np, coef, i, m, h->dW1);
                CUDA_TRY(cudaGetLastError());
                remove_li_scan_kernel<<<gcol, 256, 0, h->st>>>(h->dW1, np, nb);
                CUDA_TRY(cudaGetLastError());
                remove_li_apply_kernel<<<dim3(gcol.x, nb), 256, 0, h->st>>>(Li, h->dKinv, np, coef, i, m, h->dW1);
                CUDA_TRY(cudaGetLastError());
            }
            remove_commit_kernel<<<m + 1, 256, 0, h->st>>>(L, Li, h->dU, h->dKinv, np, i, Nk);
            CUDA_TRY(cudaGetLastError());
        }
        remove_shift_kernel<<<Nx + nl, 256, 0, h->st>>>(h->dXT, Nx, h->dY, np, i, Nk);
        CUDA_TRY(cudaGetLastError());
    }
    // the host copy follows X^T only once every removal is enqueued, so an early error return leaves hX and N consistent
    for (int k = 0; k < n; ++k)           // descending indices: row order kept, as in X^T
        h->hX.erase(h->hX.begin() + (size_t)order[k] * Nx, h->hX.begin() + (size_t)(order[k] + 1) * Nx);
    h->mu_stale = true;
    h->N = N - n;
    return refresh_alpha(h);
}

// ------------------------------------------------------------------------------------
// multi-GPU
// ------------------------------------------------------------------------------------
extern "C" int gpmpc_comm_unique_id(void* id128)
{
    if (!id128) return GPMPC_ERR_ARG;
    if (!nccl_load(g_create_err, sizeof(g_create_err))) return GPMPC_ERR_NCCL;
    nccl_uid_t id;
    int r = g_nccl.GetUniqueId(&id);
    if (r) { snprintf(g_create_err, sizeof(g_create_err), "ncclGetUniqueId failed (%d)", r); return GPMPC_ERR_NCCL; }
    memcpy(id128, &id, 128);
    return GPMPC_OK;
}

extern "C" int gpmpc_comm_init(gpmpc_handle_t h, const void* id128, int rank, int world)
{
    if (!h || !id128 || world < 1 || rank < 0 || rank >= world) return GPMPC_ERR_ARG;
    CUDA_TRY(cudaSetDevice(h->device));
    const int nlm = (h->Ny + world - 1) / world;
    if (h->a0 != std::min(h->Ny, rank * nlm) || h->nloc > nlm) {
        set_error(h, "gpmpc_comm_init: rank %d of %d must own outputs starting at %d (at most %d); handle owns [%d,%d)",
                  rank, world, rank * nlm, nlm, h->a0, h->a0 + h->nloc);
        return GPMPC_ERR_ARG;
    }
    if (world > 1) {
        if (!nccl_load(h->err, sizeof(h->err))) return GPMPC_ERR_NCCL;
        nccl_uid_t id;
        memcpy(&id, id128, 128);
        int r = g_nccl.CommInitRank(&h->comm, world, id, rank);
        if (r) { set_error(h, "ncclCommInitRank failed: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?"); return GPMPC_ERR_NCCL; }
    }
    h->rank = rank; h->world = world; h->nloc_max = nlm;
    h->Hcap = 0;      // gather buffer must be re-sized for the padded output count
    return GPMPC_OK;
}

extern "C" int gpmpc_peer_export(gpmpc_handle_t h, int Hcap, void* handle64)
{
    if (!h || !handle64 || Hcap < 1) return GPMPC_ERR_ARG;
    CUDA_TRY(cudaSetDevice(h->device));
    if (h->world > GPMPC_MAXW) { set_error(h, "peer exchange supports at most %d ranks", GPMPC_MAXW); return GPMPC_ERR_ARG; }
    if (h->dPeerBlock) { set_error(h, "gpmpc_peer_export: already exported"); return GPMPC_ERR_STATE; }
    const int nyp = h->nloc_max * h->world;
    h->peerGsz = (long long)nyp * Hcap * (h->Nx + 2);
    h->peerHcap = Hcap;
    ENSURE(h->dPeerBlock, 2 * GPMPC_MAXW + 2 * h->peerGsz);
    if (!h->dPeerStatus) {     // status word in mapped pinned host memory: the host reads it without a copy
        CUDA_TRY(cudaHostAlloc((void**)&h->hPeerStatus, sizeof(int), cudaHostAllocMapped));
        *h->hPeerStatus = 0;
        CUDA_TRY(cudaHostGetDevicePointer((void**)&h->dPeerStatus, h->hPeerStatus, 0));
    }
    CUDA_TRY(cudaStreamSynchronize(h->st));
    cudaIpcMemHandle_t mh;
    CUDA_TRY(cudaIpcGetMemHandle(&mh, h->dPeerBlock));
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    memcpy(handle64, &mh, 64);
    return GPMPC_OK;
}

extern "C" int gpmpc_peer_attach(gpmpc_handle_t h, const void* handles)
{
    if (!h || !handles) return GPMPC_ERR_ARG;
    if (!h->dPeerBlock) { set_error(h, "gpmpc_peer_attach: call gpmpc_peer_export first"); return GPMPC_ERR_STATE; }
    CUDA_TRY(cudaSetDevice(h->device));
    for (int r = 0; r < h->world; ++r) {
        if (r == h->rank) { h->peerBase[r] = h->dPeerBlock; continue; }
        cudaIpcMemHandle_t mh;
        memcpy(&mh, (const char*)handles + 64 * r, 64);
        void* ptr = nullptr;
        CUDA_TRY(cudaIpcOpenMemHandle(&ptr, mh, cudaIpcMemLazyEnablePeerAccess));
        h->peerBase[r] = (double*)ptr; h->peerOpened[r] = true;
    }
    h->peer_ready = true; h->peer_step = 0;
    return GPMPC_OK;
}

extern "C" int gpmpc_get_size(gpmpc_handle_t h, int* N, int* Nx, int* Ny)
{
    if (!h) return GPMPC_ERR_ARG;
    if (N) *N = h->N;
    if (Nx) *Nx = h->Nx;
    if (Ny) *Ny = h->Ny;
    return GPMPC_OK;
}

extern "C" void* gpmpc_stream(gpmpc_handle_t h) { return h ? (void*)h->st : nullptr; }

extern "C" int gpmpc_synchronize(gpmpc_handle_t h)
{
    if (!h) return GPMPC_ERR_ARG;
    CUDA_TRY(cudaSetDevice(h->device));
    CUDA_TRY(cudaStreamSynchronize(h->st));
    return peer_status_check(h);
}

// gpmpc_profile_balance / _tail (fn): two stamped runs of the predict product over the last predict call's operands, the
// second one warm.  setup(p, tail) adds what the entry profiles; t = {start, end} of the grid CTAs, then n_tail stamps.
template <typename Setup>
static int profile_product(gpmpc_handle_t h, const char* fn, int H, const double* out, bool all_outputs, int n_tail,
                           Setup&& setup, std::vector<unsigned long long>& t, int* grid)
{
    if (!h || !out || H < 1 || H > HB) return GPMPC_ERR_ARG;
    int rc = predict_guard(h, fn, GPMPC_METHOD_TA, H);
    if (rc) return rc;
    rc = predict_prepare(h, fn, HB, all_outputs);
    if (rc) return rc;
    PredictParams p;
    psk_base(h, p, H);
    *grid = psk_schedule(h, p, h->dLi);
    DevBuf<unsigned long long> dbg;
    ENSURE(dbg, (long long)*grid * 2 + n_tail);
    p.dbg = dbg;
    setup(p, dbg + 2 * *grid);
    for (int rep = 0; rep < 2; ++rep) {
        const cudaError_t e = psk_launch(h, p, h->dKST, h->dLi);
        if (e != cudaSuccess) { set_error(h, "%s: %s", fn, cudaGetErrorString(e)); return GPMPC_ERR_CUDA; }
    }
    t.resize((size_t)*grid * 2 + n_tail);
    cudaMemcpyAsync(t.data(), dbg, t.size() * 8, cudaMemcpyDeviceToHost, h->st);
    cudaStreamSynchronize(h->st);
    return GPMPC_OK;
}

// load balance of the persistent predict product: per-CTA busy time (globaltimer at CTA start / end)
//   out = {shortest CTA, longest CTA, mean CTA, first start -> last end} in microseconds
extern "C" int gpmpc_profile_balance(gpmpc_handle_t h, int H, double* out4)
{
    std::vector<unsigned long long> t; int grid = 0;
    const int rc = profile_product(h, __func__, H, out4, false, 0, [](PredictParams&, unsigned long long*) {}, t, &grid);
    if (rc) return rc;
    unsigned long long lo = ~0ull, hi = 0; double mn = 1e300, mx = 0.0, sum = 0.0;
    for (int c = 0; c < grid; ++c) {
        const double d = (double)(t[2 * c + 1] - t[2 * c]) * 1e-3;
        mn = std::min(mn, d); mx = std::max(mx, d); sum += d;
        lo = std::min(lo, t[2 * c]); hi = std::max(hi, t[2 * c + 1]);
    }
    out4[0] = mn; out4[1] = mx; out4[2] = sum / grid; out4[3] = (double)(hi - lo) * 1e-3;
    return GPMPC_OK;
}

// phase stamps of the fused kernel's serial tail (the CTA that completes the step): out8 = microseconds, relative to the
// latest end of every OTHER CTA, of {last output complete, records built, step counter passed, records staged,
// J Sigma done, outputs written}, then the kernel's span and the tail CTA's own span.  Needs a predict call before it.
extern "C" int gpmpc_profile_tail(gpmpc_handle_t h, int H, double* out8)
{
    std::vector<unsigned long long> t; int grid = 0;
    auto setup = [&](PredictParams& p, unsigned long long* tail) {
        psk_finalize(h, p, H, 0);
        p.as = assemble_args(h, H, GPMPC_METHOD_TA, h->dSigma, 0, h->dMean, h->dVar, h->dJ, h->dCov);
        p.as.dbg = tail;
        p.do_assemble = 1;
    };
    const int rc = profile_product(h, __func__, H, out8, true, 8, setup, t, &grid);
    if (rc) return rc;
    unsigned long long lo = ~0ull, hi = 0, hi2 = 0; int cmax = 0;
    for (int c = 0; c < grid; ++c) {
        lo = std::min(lo, t[2 * c]);
        if (t[2 * c + 1] > hi) { hi2 = hi; hi = t[2 * c + 1]; cmax = c; } else hi2 = std::max(hi2, t[2 * c + 1]);
    }
    for (int k = 0; k < 6; ++k) out8[k] = ((double)t[2 * grid + k] - (double)hi2) * 1e-3;
    out8[6] = (double)(hi - lo) * 1e-3;
    out8[7] = (double)(t[2 * cmax + 1] - t[2 * cmax]) * 1e-3;
    return GPMPC_OK;
}

// phase clock stamps of one 128x128 leaf (potrf + trtri): out15 = clock64 at
// {start, loaded, first panel, after block steps 1..7, L stored, inverse levels 16/32/64, Linv stored}
extern "C" int gpmpc_profile_leaf(gpmpc_handle_t h, double* out15)
{
    if (!h || !out15) return GPMPC_ERR_ARG;
    int rc = model_guard(h, __func__, NEED_HYPER);
    if (rc) return rc;
    DevBuf<long long> d;
    ENSURE(d, 16);
    CUDA_TRY(cudaMemcpyToSymbol(d_leaf_prof, &d.p, sizeof(d.p)));
    for (int rep = 0; rep < 2 && rc == GPMPC_OK; ++rep) {           // second run: warm instruction cache
        rc = launch_kbuild(h, h->dHyp, h->dJit, h->dL, 1, 0);
        if (rc == GPMPC_OK) rc = potrf_inv_rec(h, h->dL, h->dLi, slab(h), slab(h), h->dInfo, 0, 128, 1, 1, h->dW1, h->dW2);
    }
    cudaStreamSynchronize(h->st);
    long long hst[16];
    cudaMemcpy(hst, d, sizeof(hst), cudaMemcpyDeviceToHost);
    long long* nul = nullptr;
    cudaMemcpyToSymbol(d_leaf_prof, &nul, sizeof(nul));
    for (int k = 0; k < 15; ++k) out15[k] = (double)(hst[k] - hst[0]);
    factor_stale(h);
    return rc;
}

// ------------------------------------------------------------------------------------
// kernel-level timing for the roofline report (CUDA events on the handle's stream)
// ------------------------------------------------------------------------------------
extern "C" int gpmpc_profile(gpmpc_handle_t h, int what, int n, int reps, double* ms_out)
{
    if (!h || !ms_out || reps < 1) return GPMPC_ERR_ARG;
    int rc = model_guard(h, __func__, NEED_HYPER);
    if (rc) return rc;
    const int np = h->Npad, Hc = (n > 0 && n <= HB) ? n : 56;       // Hc: test points of the product selectors
    float ms = 0.f;
    auto run = [&]() -> int {
        switch (what) {
        case GPMPC_PROF_KBUILD_FULL: return launch_kbuild(h, h->dHyp, h->dJit, h->dL, 1, 1);
        case GPMPC_PROF_KBUILD_LOWER: return launch_kbuild(h, h->dHyp, h->dJit, h->dL, 1, 0);
        case GPMPC_PROF_SYRK: {
            // trailing update shape of the top recursion level: C(n2 x n2, lower) -= P P^T, K = n1
            const int nn = (n > 0 && n <= np) ? n / 128 * 128 : np;
            const int n1 = (nn / 128 / 2) * 128, n2 = nn - n1;
            if (n1 < 128) { set_error(h, "gpmpc_profile: SYRK needs N >= 256"); return GPMPC_ERR_ARG; }
            GemmParams p;
            memset(&p, 0, sizeof(p));
            p.A = h->dW1; p.lda = n1; p.B = h->dW1; p.ldb = n1;
            p.C = h->dLi; p.ldc = np; p.Cin = h->dLi; p.ldcin = np;
            p.mt = n2 / 128; p.nt = n2 / 128; p.K = n1; p.alpha = -1e-30; p.beta = 1.0; p.lower = 1;
            cudaError_t e = gemm128(h, h->st, true, p, 1, 1);
            if (e != cudaSuccess) { set_error(h, "profile syrk: %s", cudaGetErrorString(e)); return GPMPC_ERR_CUDA; }
            return GPMPC_OK;
        }
        case GPMPC_PROF_FACTORIZE: {
            int r = launch_kbuild(h, h->dHyp, h->dJit, h->dL, 1, 0);
            if (r) return r;
            return potrf_inv_rec(h, h->dL, h->dLi, slab(h), slab(h), h->dInfo, 0, np, 1, 1, h->dW1, h->dW2);
        }
        case GPMPC_PROF_TRIGEMM: return tri_product(h, h->dKST, h->dLi, Hc, nullptr);
        case GPMPC_PROF_PANEL: panel_stale(h, -1, 0); return panel_refresh(h);
        case GPMPC_PROF_KS: {             // the ks / mean / Jacobian partial kernel alone (Z = the last batch's inputs)
            cudaError_t e = launch_ks(h, h->dZ, Hc);
            if (e != cudaSuccess) { set_error(h, "profile ks: %s", cudaGetErrorString(e)); return GPMPC_ERR_CUDA; }
            return GPMPC_OK;
        }
        case GPMPC_PROF_PREDICT_TAIL: {   // the fused kernel WITH finalize + assembly, without the ks kernel in front
            PredictParams p;
            psk_base(h, p, Hc);
            psk_finalize(h, p, Hc, 0);
            p.as = assemble_args(h, Hc, GPMPC_METHOD_TA, h->dSigma, 0, h->dMean, h->dVar, h->dJ, h->dCov);
            p.do_assemble = (h->world == 1 && h->nloc == h->Ny) ? 1 : 0;
            cudaError_t e = psk_launch(h, p, h->dKST, h->dLi);
            if (e != cudaSuccess) { set_error(h, "profile predict tail: %s", cudaGetErrorString(e)); return GPMPC_ERR_CUDA; }
            return GPMPC_OK;
        }
        default: set_error(h, "gpmpc_profile: unknown selector %d", what); return GPMPC_ERR_ARG;
        }
    };
    // the product selectors run on the predict buffers; the others use the factor's slabs as scratch
    const bool product = what == GPMPC_PROF_TRIGEMM || what == GPMPC_PROF_KS || what == GPMPC_PROF_PREDICT_TAIL ||
                         what == GPMPC_PROF_PANEL;
    if (product) {
        rc = ensure_predict_bufs(h, HB);
        if (rc == GPMPC_OK) rc = panel_refresh(h);
        if (rc) return rc;
    } else {
        panel_stale(h, -1, 0);
    }
    CUDA_TRY(cudaMemsetAsync(h->dJit, 0, h->nloc * sizeof(double), h->st));
    rc = run();
    if (rc) return rc;
    CUDA_TRY(cudaStreamSynchronize(h->st));
    CUDA_TRY(cudaEventRecord(h->ev0, h->st));
    for (int r = 0; r < reps; ++r) { rc = run(); if (rc) return rc; }
    CUDA_TRY(cudaEventRecord(h->ev1, h->st));
    CUDA_TRY(cudaEventSynchronize(h->ev1));
    CUDA_TRY(cudaEventElapsedTime(&ms, h->ev0, h->ev1));
    ms_out[0] = (double)ms / reps;
    if (!product) factor_stale(h);
    return GPMPC_OK;
}
