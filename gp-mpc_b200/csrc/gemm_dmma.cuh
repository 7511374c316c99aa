// fp64 tensor-core (DMMA m8n8k4) GEMM family used by every O(N^3) / O(N^2 H) step of the
// GP hot path: Cholesky trailing updates (SYRK), explicit-inverse panel solves, the
// triangular inverse assembly and K^-1 = Linv^T Linv.  The fp64 tensor path (Hopper
// wgmma has no fp64 kind) is mma.sync.m8n8k4 (SASS DMMA.8x8x4) fed by a 4-stage cp.async
// shared-memory pipeline.  (The predictive v = Linv * ks product, predict_streamk.cuh,
// issues DMMA.16x8x16.)
//
//   C[i][j] = alpha * sum_k A[i][k] * Bop[k][j] + beta * Cin[i][j]
//   A   : row-major M x K (K contiguous)
//   BT  : B is row-major N x K  (C = A * B^T, "NT")
//   !BT : B is row-major K x N  (C = A * B,   "NN")
//
// All dimensions are multiples of the tile sizes (every matrix in the engine is padded
// to GPMPC_TILE with an identity tail), so there is no bounds handling anywhere.
#pragma once
#include "common.cuh"

enum : int {
    GEMM_KI_LE = 1,   // A[i][k] == 0 for k >  i  (A lower-triangular)  -> k_hi <= (it+1)*BM
    GEMM_KI_GE = 2,   // A[i][k] == 0 for k <  i  (A upper-triangular)  -> k_lo >= it*BM
    GEMM_KJ_LE = 4,   // Bop[k][j] == 0 for k > j                       -> k_hi <= (jt+1)*BN
    GEMM_KJ_GE = 8,   // Bop[k][j] == 0 for k < j                       -> k_lo >= jt*BN
};

struct GemmParams {
    const double* A; const double* B; double* C; const double* Cin;
    int lda, ldb, ldc, ldcin;
    long long sA, sB, sC, sCin;     // batch strides in elements (blockIdx.z)
    int mt, nt;                      // tile counts in M and N
    int K;
    double alpha, beta;
    int kflags;
    int lower;                       // compute tiles it >= jt only; mask col > row on diagonal tiles
};

constexpr int GEMM_BK = 16;

template <int BM, int BN, bool BT, int STAGES>
struct GemmSmem {
    static constexpr int LDA_S = GEMM_BK + 4;                 // 160 B rows: (g*32 + t*8) mod 128 distinct
    static constexpr int LDB_S = BT ? (GEMM_BK + 4) : (BN + 4);
    static constexpr int A_STAGE = BM * LDA_S;
    static constexpr int B_STAGE = BT ? BN * LDB_S : GEMM_BK * LDB_S;
    static constexpr int BYTES = STAGES * (A_STAGE + B_STAGE) * 8;
};

template <int BM, int BN, int WM, int WN, bool BT, int STAGES, int MINB>
__global__ void __launch_bounds__(WM * WN * 32, MINB)
gemm_dmma_kernel(const GemmParams p)
{
    using SM = GemmSmem<BM, BN, BT, STAGES>;
    constexpr int BK = GEMM_BK, NT = WM * WN * 32;
    constexpr int RL = BM / BN;                       // lower mode: row tile `it` owns column tiles [0, RL*(it+1))
    static_assert(BM % BN == 0 || BM < BN, "lower mode needs BM to be a multiple of BN");
    constexpr int LDA_S = SM::LDA_S, LDB_S = SM::LDB_S, A_STAGE = SM::A_STAGE, B_STAGE = SM::B_STAGE;
    constexpr int WTM = BM / WM, WTN = BN / WN, MF = WTM / 8, NF = WTN / 8;
    static_assert(WTM % 8 == 0 && WTN % 8 == 0, "warp tile must be a multiple of the 8x8 MMA");

    extern __shared__ __align__(16) double smem[];
    double* As = smem;
    double* Bs = smem + STAGES * A_STAGE;

    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t = lane & 3;
    const int wm = warp / WN, wn = warp % WN;

    int it, jt;
    const long long bz = blockIdx.z;
    if (p.lower) {
        const int tt = blockIdx.x;
        constexpr int R = RL > 0 ? RL : 1;
        it = (int)((sqrt(8.0 * (double)tt / R + 1.0) - 1.0) * 0.5);
        while (R * it * (it + 1) / 2 > tt) --it;
        while (R * (it + 1) * (it + 2) / 2 <= tt) ++it;
        jt = tt - R * it * (it + 1) / 2;
    } else {
        it = blockIdx.x / p.nt;
        jt = blockIdx.x - it * p.nt;
    }

    int k_lo = 0, k_hi = p.K;
    if (p.kflags & GEMM_KI_LE) k_hi = min(k_hi, (it + 1) * BM);
    if (p.kflags & GEMM_KI_GE) k_lo = max(k_lo, it * BM);
    if (p.kflags & GEMM_KJ_LE) k_hi = min(k_hi, (jt + 1) * BN);
    if (p.kflags & GEMM_KJ_GE) k_lo = max(k_lo, jt * BN);
    const int nk = (k_hi - k_lo) / BK;

    const double* Ag = p.A + bz * p.sA + (long long)it * BM * p.lda;
    const double* Bg = BT ? (p.B + bz * p.sB + (long long)jt * BN * p.ldb)
                          : (p.B + bz * p.sB + (long long)jt * BN);

    auto load_stage = [&](int s, int k0) {
        double* as = As + s * A_STAGE;
        double* bs = Bs + s * B_STAGE;
#pragma unroll
        for (int c = tid; c < BM * 8; c += NT) {
            const int r = c >> 3, ch = c & 7;
            cp_async16(as + r * LDA_S + ch * 2, Ag + (long long)r * p.lda + k0 + ch * 2);
        }
        if (BT) {
#pragma unroll
            for (int c = tid; c < BN * 8; c += NT) {
                const int r = c >> 3, ch = c & 7;
                cp_async16(bs + r * LDB_S + ch * 2, Bg + (long long)r * p.ldb + k0 + ch * 2);
            }
        } else {
#pragma unroll
            for (int c = tid; c < BK * (BN / 2); c += NT) {
                const int r = c / (BN / 2), ch = c % (BN / 2);
                cp_async16(bs + r * LDB_S + ch * 2, Bg + (long long)(k0 + r) * p.ldb + ch * 2);
            }
        }
    };

    double acc[MF][NF][2];
#pragma unroll
    for (int mi = 0; mi < MF; ++mi)
#pragma unroll
        for (int ni = 0; ni < NF; ++ni) { acc[mi][ni][0] = 0.0; acc[mi][ni][1] = 0.0; }

#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) {
        if (s < nk) load_stage(s, k_lo + s * BK);
        cp_async_commit();
    }

    for (int kt = 0; kt < nk; ++kt) {
        cp_async_wait<STAGES - 2>();
        __syncthreads();
        {   // prefetch the stage that was consumed in the previous iteration
            const int kn = kt + STAGES - 1;
            if (kn < nk) load_stage(kn % STAGES, k_lo + kn * BK);
            cp_async_commit();
        }
        const int s = kt % STAGES;
        const double* as = As + s * A_STAGE + (wm * WTM + g) * LDA_S + t;
        const double* bs = BT ? (Bs + s * B_STAGE + (wn * WTN + g) * LDB_S + t)
                              : (Bs + s * B_STAGE + t * LDB_S + wn * WTN + g);
#pragma unroll
        for (int kk = 0; kk < BK / 4; ++kk) {
            double a[MF], b[NF];
#pragma unroll
            for (int mi = 0; mi < MF; ++mi) a[mi] = as[mi * 8 * LDA_S + kk * 4];
#pragma unroll
            for (int ni = 0; ni < NF; ++ni)
                b[ni] = BT ? bs[ni * 8 * LDB_S + kk * 4] : bs[kk * 4 * LDB_S + ni * 8];
#pragma unroll
            for (int mi = 0; mi < MF; ++mi)
#pragma unroll
                for (int ni = 0; ni < NF; ++ni)
                    dmma884(acc[mi][ni][0], acc[mi][ni][1], a[mi], b[ni]);
        }
    }
    cp_async_wait<0>();

    // epilogue: each lane owns two adjacent columns of every 8x8 fragment -> 16-byte accesses
    double* Cg = p.C + bz * p.sC;
    const double* Cing = p.Cin ? (p.Cin + bz * p.sCin) : nullptr;
    const bool diag = p.lower && ((jt + 1) * BN > it * BM);      // tile reaches the diagonal
#pragma unroll
    for (int mi = 0; mi < MF; ++mi) {
        const int row = it * BM + wm * WTM + mi * 8 + g;
#pragma unroll
        for (int ni = 0; ni < NF; ++ni) {
            const int col = jt * BN + wn * WTN + ni * 8 + 2 * t;
            double2 c;
            c.x = p.alpha * acc[mi][ni][0];
            c.y = p.alpha * acc[mi][ni][1];
            if (diag && col > row) continue;
            if (p.beta != 0.0) {
                const double2 cin = *reinterpret_cast<const double2*>(Cing + (long long)row * p.ldcin + col);
                c.x += p.beta * cin.x;
                c.y += p.beta * cin.y;
            }
            double* dst = Cg + (long long)row * p.ldc + col;
            if (diag && col + 1 > row) dst[0] = c.x;
            else *reinterpret_cast<double2*>(dst) = c;
        }
    }
}

template <int BM, int BN, int WM, int WN, bool BT, int STAGES, int MINB>
static cudaError_t gemm_launch(const GemmParams& p, int batch, cudaStream_t st)
{
    using SM = GemmSmem<BM, BN, BT, STAGES>;
    auto kern = gemm_dmma_kernel<BM, BN, WM, WN, BT, STAGES, MINB>;
    constexpr int BYTES = SM::BYTES;
    const cudaError_t e = smem_opt_in<gemm_dmma_kernel<BM, BN, WM, WN, BT, STAGES, MINB>>(BYTES);
    if (e != cudaSuccess) return e;
    constexpr int R = (BM >= BN) ? BM / BN : 1;
    const int tiles = p.lower ? R * p.mt * (p.mt + 1) / 2 : p.mt * p.nt;
    kern<<<dim3(tiles, 1, batch), WM * WN * 32, BYTES, st>>>(p);
    return cudaGetLastError();
}

// =======================================================================================
// Tile-granular TMA feed (NT products): one cp.async.bulk.tensor (SASS UTMALDG) per operand
// per stage moves a {16 doubles x BM rows} box into a 128B-swizzled, un-padded shared tile
// and completes on the stage's mbarrier.  Fragment loads use the k-permutation
//     step kk, lane t  ->  k = 2 kk + (t & 1) + 8 (t >> 1)
// (the MMA sums over k, so any permutation applied to A and B alike is valid); with the
// 128B swizzle  chunk' = chunk ^ (row & 7)  the 16 lanes of a half-warp hit 16 distinct
// 8-byte banks.  Same tiling / k-range / epilogue logic as gemm_dmma_kernel.
// =======================================================================================
#include <cuda.h>
#include <mutex>

__device__ __forceinline__ void tma_tile_g2s_3d(void* smem_dst, const CUtensorMap* tm, int c0, int c1, int c2, uint64_t* bar)
{
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];\n"
                 :: "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tm)), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
                 : "memory");
}

__device__ __forceinline__ void tma_tile_g2s_3d_hint(void* smem_dst, const CUtensorMap* tm, int c0, int c1, int c2, uint64_t* bar, uint64_t policy)
{
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%2, %3, %4}], [%5], %6;\n"
                 :: "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tm)), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar)), "l"(policy)
                 : "memory");
}

// non-tensor bulk copy (SASS UBLKCP) of `bytes` contiguous bytes (multiple of 16, both ends 16-byte aligned), same barrier
__device__ __forceinline__ void bulk_g2s_hint(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar, uint64_t policy)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;\n"
                 :: "r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
                 : "memory");
}

template <int BM, int BN, int WM, int WN, int STAGES, int MINB>
__global__ void __launch_bounds__(WM * WN * 32, MINB)
gemm_dmma_tmap_kernel(const GemmParams p, const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB)
{
    constexpr int BK = GEMM_BK;
    constexpr int RL = BM / BN;
    constexpr int WTM = BM / WM, WTN = BN / WN, MF = WTM / 8, NF = WTN / 8;
    constexpr int A_STAGE = BM * BK, B_STAGE = BN * BK;            // doubles, rows of 128 B, no padding
    constexpr uint32_t STAGE_TX = (BM + BN) * BK * 8;
    static_assert((BM * 128) % 1024 == 0 && (BN * 128) % 1024 == 0, "tiles must be whole swizzle atoms");

    extern __shared__ __align__(16) double smem_raw[];
    double* smem = smem_align1024(smem_raw);
    double* As = smem;
    double* Bs = smem + STAGES * A_STAGE;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * (A_STAGE + B_STAGE));

    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, t = lane & 3;
    const int wm = warp / WN, wn = warp % WN;

    int it, jt;
    const long long bz = blockIdx.z;
    if (p.lower) {
        const int tt = blockIdx.x;
        constexpr int R = RL > 0 ? RL : 1;
        it = (int)((sqrt(8.0 * (double)tt / R + 1.0) - 1.0) * 0.5);
        while (R * it * (it + 1) / 2 > tt) --it;
        while (R * (it + 1) * (it + 2) / 2 <= tt) ++it;
        jt = tt - R * it * (it + 1) / 2;
    } else {
        it = blockIdx.x / p.nt;
        jt = blockIdx.x - it * p.nt;
    }
    int k_lo = 0, k_hi = p.K;
    if (p.kflags & GEMM_KI_LE) k_hi = min(k_hi, (it + 1) * BM);
    if (p.kflags & GEMM_KI_GE) k_lo = max(k_lo, it * BM);
    if (p.kflags & GEMM_KJ_LE) k_hi = min(k_hi, (jt + 1) * BN);
    if (p.kflags & GEMM_KJ_GE) k_lo = max(k_lo, jt * BN);
    const int nk = (k_hi - k_lo) / BK;

    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < STAGES; ++s) mbar_init(full + s, 1);
        mbar_fence_init();
    }
    __syncthreads();

    auto load_stage = [&](int s, int k0) {
        if (tid == 0) {
            mbar_arrive_expect_tx(full + s, STAGE_TX);
            tma_tile_g2s_3d(As + s * A_STAGE, &tmA, k0, it * BM, (int)bz, full + s);
            tma_tile_g2s_3d(Bs + s * B_STAGE, &tmB, k0, jt * BN, (int)bz, full + s);
        }
    };

    double acc[MF][NF][2];
#pragma unroll
    for (int mi = 0; mi < MF; ++mi)
#pragma unroll
        for (int ni = 0; ni < NF; ++ni) { acc[mi][ni][0] = 0.0; acc[mi][ni][1] = 0.0; }

#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s)
        if (s < nk) load_stage(s, k_lo + s * BK);

    // swizzled fragment offsets (doubles): row r -> r*16 + ((chunk ^ (r & 7)) * 2) + (t & 1); (r & 7) == g
    const int kperm_hi = 4 * (t >> 1), kpar = t & 1;
    for (int kt = 0; kt < nk; ++kt) {
        mbar_wait(full + kt % STAGES, (kt / STAGES) & 1);
        __syncthreads();                                   // everyone is done with the stage refilled below
        {
            const int kn = kt + STAGES - 1;
            if (kn < nk) load_stage(kn % STAGES, k_lo + kn * BK);
        }
        const int s = kt % STAGES;
        const double* as = As + s * A_STAGE + (wm * WTM + g) * 16 + kpar;
        const double* bs = Bs + s * B_STAGE + (wn * WTN + g) * 16 + kpar;
#pragma unroll
        for (int kk = 0; kk < BK / 4; ++kk) {
            const int coff = (((kk + kperm_hi) ^ g) << 1);
            double a[MF], b[NF];
#pragma unroll
            for (int mi = 0; mi < MF; ++mi) a[mi] = as[mi * 8 * 16 + coff];
#pragma unroll
            for (int ni = 0; ni < NF; ++ni) b[ni] = bs[ni * 8 * 16 + coff];
#pragma unroll
            for (int mi = 0; mi < MF; ++mi)
#pragma unroll
                for (int ni = 0; ni < NF; ++ni)
                    dmma884(acc[mi][ni][0], acc[mi][ni][1], a[mi], b[ni]);
        }
    }

    double* Cg = p.C + bz * p.sC;
    const double* Cing = p.Cin ? (p.Cin + bz * p.sCin) : nullptr;
    const bool diag = p.lower && ((jt + 1) * BN > it * BM);
#pragma unroll
    for (int mi = 0; mi < MF; ++mi) {
        const int row = it * BM + wm * WTM + mi * 8 + g;
#pragma unroll
        for (int ni = 0; ni < NF; ++ni) {
            const int col = jt * BN + wn * WTN + ni * 8 + 2 * t;
            double2 c;
            c.x = p.alpha * acc[mi][ni][0];
            c.y = p.alpha * acc[mi][ni][1];
            if (diag && col > row) continue;
            if (p.beta != 0.0) {
                const double2 cin = *reinterpret_cast<const double2*>(Cing + (long long)row * p.ldcin + col);
                c.x += p.beta * cin.x;
                c.y += p.beta * cin.y;
            }
            double* dst = Cg + (long long)row * p.ldc + col;
            if (diag && col + 1 > row) dst[0] = c.x;
            else *reinterpret_cast<double2*>(dst) = c;
        }
    }
}

typedef CUresult (*tmap_encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// 3-D map {K, rows, batch} over a row-major fp64 operand; box {16, box_rows, 1}, 128B swizzle.
// Encoding is a pure function of its arguments: a small cache keeps the predict path (same
// operands every step) free of driver calls.
struct TmapKey { const double* base; int K, rows, ld, batch, box_rows; long long bstride; };
static bool tmap_make(CUtensorMap* tm, const double* base, int K, int rows, int ld, long long batch_stride, int batch, int box_rows)
{
    static tmap_encode_fn enc = nullptr;
    static TmapKey keys[64];
    static CUtensorMap maps[64];
    static int used = 0, next = 0;
    static std::mutex mtx;                                       // handles on different threads share the cache
    std::lock_guard<std::mutex> lock(mtx);
    const TmapKey key = {base, K, rows, ld, batch, box_rows, batch_stride};
    for (int i = 0; i < used; ++i)
        if (keys[i].base == key.base && keys[i].K == key.K && keys[i].rows == key.rows && keys[i].ld == key.ld &&
            keys[i].batch == key.batch && keys[i].box_rows == key.box_rows && keys[i].bstride == key.bstride) { *tm = maps[i]; return true; }
    if (!enc) {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn) return false;
        enc = (tmap_encode_fn)fn;
    }
    cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)rows, (cuuint64_t)batch};
    cuuint64_t strides[2] = {(cuuint64_t)ld * 8, (cuuint64_t)(batch > 1 ? batch_stride : (long long)rows * ld) * 8};
    cuuint32_t box[3] = {16, (cuuint32_t)box_rows, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    if (enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 3, (void*)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) return false;
    const int slot = (used < 64) ? used++ : (next++ & 63);
    keys[slot] = key; maps[slot] = *tm;
    return true;
}

template <int BM, int BN, int WM, int WN, int STAGES, int MINB>
static cudaError_t gemm_tmap_launch(const GemmParams& p, int batch, cudaStream_t st)
{
    auto kern = gemm_dmma_tmap_kernel<BM, BN, WM, WN, STAGES, MINB>;
    constexpr int BYTES = STAGES * (BM + BN) * GEMM_BK * 8 + STAGES * 8 + 1024;
    const cudaError_t e = smem_opt_in<gemm_dmma_tmap_kernel<BM, BN, WM, WN, STAGES, MINB>>(BYTES);
    if (e != cudaSuccess) return e;
    CUtensorMap tmA, tmB;
    if (!tmap_make(&tmA, p.A, p.K, p.mt * BM, p.lda, p.sA, batch, BM)) return cudaErrorInvalidValue;
    if (!tmap_make(&tmB, p.B, p.K, p.nt * BN, p.ldb, p.sB, batch, BN)) return cudaErrorInvalidValue;
    constexpr int R = (BM >= BN) ? BM / BN : 1;
    const int tiles = p.lower ? R * p.mt * (p.mt + 1) / 2 : p.mt * p.nt;
    kern<<<dim3(tiles, 1, batch), WM * WN * 32, BYTES, st>>>(p, tmA, tmB);
    return cudaGetLastError();
}
