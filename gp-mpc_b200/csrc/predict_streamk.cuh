// Fused predict step (a8-a10, gp_functions.py:111-147, :167-171):  one persistent kernel does
//   v = L^-1 ks  (fp64 DMMA fed by TMA tensor maps)         -> sum_i v_i^2      (never stored)
//   var = sf2 - v^T v, mean = ks^T alpha, J                 -> gather records [mean,var,J..]
//   (multi-GPU) records stored straight into every peer's gather buffer over NVLink, flags published
//   cov = diag(var) (+ J Sigma J^T)                         -> mean / var / J / cov outputs
//
// Scheduling is stream-K: the triangular product's work is the list of BK=16 k-steps of every
// (output a, PSK_BN-row tile jt) pair -- tile jt has min((jt+1) BN, Npad) / 16 steps because L^-1 is
// lower triangular -- and the persistent grid cuts that list into equal contiguous
// ranges, so every CTA issues the same number of DMMAs regardless of where tile borders fall
// (the static split-K grid it replaces lost a visible share to the tail at one output per GPU).  A tile cut
// by a range border is completed by its LAST-ARRIVING contributor: everyone else parks its partial
// accumulators in a per-CTA slot and bumps the tile's counter; the last one adds the parked
// partials in contributor order (fixed order => bit-reproducible), squares and row-reduces.
// A lower-mode product of L^-1 from its panel whose tile pairs fill the grid runs the paired schedule instead
// (psk_pair_units): whole tiles, paired long with short so every unit has the same length, dealt to the CTAs round-robin
// so the CTAs of one output walk its ks^T in step; no tile is cut.
// The same "last arriver" idea chains the rest of the step: the CTA that finishes an output's last
// tile builds that output's [mean,var,J] records (and stores them to the peers), the CTA that
// finishes the last output publishes the peer flags and assembles the covariances.
// All counters are self-cleaning (reset by their last arriver): no memset between steps.
#pragma once
#include "common.cuh"
#include "gemm_dmma.cuh"

#define GPMPC_MAXW 16
// The product kernel: PSK_CW warps of 32 L-rows each (tile height PSK_BN).  Registers are handed out per SM
// sub-partition (a quarter of the resident warps each, 512 per thread slot): at 8 warps per SM every warp can hold the
// 2 x BM / 8 x 4 fp64 accumulators with no spill, a 9th (producer) warp would cap all of them at 168 and spill.
// One 256-row CTA per SM (5 stages of 39-41 KB) measured faster at C5 than two 128-row CTAs per SM (4 stages each).
#define PSK_CW 8
#define PSK_BN (32 * PSK_CW)
#define PSK_STAGES 5
#define PSK_CTAS_PER_SM 1
#define PSK_THREADS (32 * PSK_CW)

// doubles of the product kernel's stage buffers at bm test points (the fused tail reuses them as scratch)
__host__ __device__ constexpr long long psk_pipe_doubles(int bm) { return (long long)PSK_STAGES * (bm + PSK_BN) * GEMM_BK; }


// Peer ("fused epilogue + all-gather") mode: instead of writing into the local gather buffer and
// calling ncclAllGather, every rank stores its [mean,var,J] records directly into the gather
// buffer of EVERY rank (peer pointers mapped with CUDA IPC, NVLink/NVSwitch P2P stores), then
// publishes a per-source flag on every peer (release at system scope).  The consumer acquires all
// `world` flags before reading.  Buffers are double-buffered by step parity; in-order streams make
// that sufficient (DESIGN.md 4.7).
struct PeerArgs {
    double* base[GPMPC_MAXW];         // peer-mapped base of each rank's exchange block (own = local)
    int world, rank;
    long long goff;                   // offset (doubles) of this step's gather buffer inside the block
    int flag_idx;                     // parity * GPMPC_MAXW + rank
    unsigned long long step;
    long long timeout_clocks;         // consumer gives up (status word, no assembly) after this many clock64 ticks
};

struct AssembleArgs {
    const double* G;                  // gather buffer [Ny_pad][H][2+Nx]
    int Ny, Nx, H, method_ta;
    const double* Sigma; int sigma_per_point;
    double *mean, *var, *J, *cov;
    const unsigned long long* flags;  // peer mode: this step's flag row (world entries), else null
    int world; unsigned long long step; int* status;
    long long timeout_clocks;
    unsigned long long* dbg;          // profiling: globaltimer stamps of the tail's phases (null in production)
    int stage_g;                      // fused tail: the gather records fit the pipeline's shared memory next to J Sigma
};

struct PredictParams {
    int nloc, nt, Hc;                 // local outputs, 128-column groups per output (Npad / 128), valid rows of this chunk
    int ntb, nk;                      // PSK_BN-row tiles per output (the last one 128 rows high when nt is odd), Npad / 16
    int upper;                        // 0: B lower triangular (k <= j, v = Linv ks); 1: B upper (k >= j, beta = Linv^T v)
    const double* Lp;                 // lower mode, B = L^-1: its panel copy (panel_pack_kernel), one bulk copy per stage; else null
    long long T, G;                   // k-steps per output (psk_steps_per_output), total = nloc * T
    int upo;                          // paired schedule: units (tile pairs) per output (psk_pair_units); 0: stream-K
    double* part;                     // [grid][2][BM*PSK_BN] parked partial accumulators (fragment-major)
    unsigned int* tile_cnt;           // [nloc*ntb]
    unsigned int* out_cnt;            // [nloc]
    unsigned int* done_cnt;           // [1]
    double* SQ;                       // [nloc][64][nt] per-tile sums of squares
    double* Vout; long long sV; int ldv;     // optional: the solved rows themselves (refinement, GP.covar, append)
    int finalize;                     // 0: product only (Vout / SQ), 1: build the gather records
    const double* PMJ; int nblk_mj;   // partial mean / Jacobian sums of ks_mean_jac_kernel
    const double* hyp; int hyp_ld, Nx;
    double* Gloc; int slot0, Htot, h0;
    PeerArgs pa; int use_peers, publish;
    AssembleArgs as; int do_assemble;
    unsigned long long* dbg;          // optional [grid][2]: globaltimer at CTA start / end (load-balance diagnostics)
};

// ---- stage 5: assemble mean (H,Ny), var (H,Ny), J (H,Ny,Nx) and the covariance for test point h:
// 'ME' diag(var) (gp_functions.py:142); 'TA' diag(var) + J Sigma J^T (build_TA_cov, :167-171).
__device__ __forceinline__ void tail_stamp(unsigned long long* dbg, int k, int tid)
{
    if (dbg && tid == 0) { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); dbg[k] = t; }
}

template <bool WARP>
__device__ __forceinline__ void assemble_point(const AssembleArgs& A, int h, double* sh, int tid, int nth)
{
    const int Ny = A.Ny, Nx = A.Nx, H = A.H;
    double* Jh = sh; double* JS = sh + Ny * Nx; double* vh = sh + 2 * Ny * Nx;
    for (int idx = tid; idx < Ny * Nx; idx += nth) {
        const int a = idx / Nx, d = idx % Nx;
        const double v = __ldcg(A.G + (((long long)a) * H + h) * (Nx + 2) + 2 + d);
        Jh[idx] = v;
        if (A.J) A.J[((long long)h * Ny + a) * Nx + d] = v;
    }
    for (int a = tid; a < Ny; a += nth) {
        const double* g = A.G + (((long long)a) * H + h) * (Nx + 2);
        const double m = __ldcg(g), v = __ldcg(g + 1);
        if (A.mean) A.mean[(long long)h * Ny + a] = m;
        if (A.var) A.var[(long long)h * Ny + a] = v;
        vh[a] = v;
    }
    if (WARP) __syncwarp(); else __syncthreads();
    if (A.cov) {
        if (A.method_ta) {
            const double* Sg = A.Sigma + (A.sigma_per_point ? (long long)h * Nx * Nx : 0);
            for (int idx = tid; idx < Ny * Nx; idx += nth) {
                const int a = idx / Nx, e = idx % Nx;
                double s = 0.0;
                for (int d = 0; d < Nx; ++d) s = fma(Jh[a * Nx + d], Sg[d * Nx + e], s);
                JS[idx] = s;
            }
            if (WARP) __syncwarp(); else __syncthreads();
        }
        for (int idx = tid; idx < Ny * Ny; idx += nth) {
            const int a = idx / Ny, b = idx % Ny;
            double s = (a == b) ? vh[a] : 0.0;
            if (A.method_ta) {
                double t = 0.0;
                for (int e = 0; e < Nx; ++e) t = fma(JS[a * Nx + e], Jh[b * Nx + e], t);
                s += t;
            }
            A.cov[((long long)h * Ny + a) * Ny + b] = s;
        }
    }
    if (WARP) __syncwarp(); else __syncthreads();
}

// all H points at once by one CTA (the fused tail of the product kernel).  One CTA at 2 warps per scheduler is
// latency-bound -- a dependent L2 load costs far more than a dependent fp64 op -- so the tail is organised around
// independent work per thread:
//   assemble_rows (stage_g: records + J Sigma fit the pipeline's shared memory): the gather records are copied to shared
//     memory in batches of independent loads, re-laid [point][output][field] with odd strides (conflict-free); then a
//     thread owns one (point, output) row and keeps 8 independent accumulators (8 columns of J Sigma, then 8 columns of
//     cov), several times faster than the flat loops below at C5 (8 outputs); outputs are written coalesced.
//   assemble_flat_global: the r2 mid-round flat loops straight from L2 (any size).
// Both use the summation order of assemble_point (ascending d, then ascending e).
__device__ __forceinline__ void assemble_flat_global(const AssembleArgs& A, double* JS, int tid, int nth)
{
    const int Ny = A.Ny, Nx = A.Nx, H = A.H, NyNx = Ny * Nx;
    const bool ta = A.cov && A.method_ta;
    for (int idx = tid; idx < H * NyNx; idx += nth) {
        const int h = idx / NyNx, r = idx - h * NyNx, a = r / Nx, e = r - a * Nx;
        const double* g = A.G + (((long long)a) * H + h) * (Nx + 2) + 2;
        if (A.J) A.J[idx] = __ldcg(g + e);                      // (h, a, e) is the output's own layout
        if (ta) {
            const double* Sg = A.Sigma + (A.sigma_per_point ? (long long)h * Nx * Nx : 0);
            double s = 0.0;
            for (int d = 0; d < Nx; ++d) s = fma(__ldcg(g + d), Sg[d * Nx + e], s);
            JS[idx] = s;
        }
    }
    for (int idx = tid; idx < H * Ny; idx += nth) {
        const int h = idx / Ny, a = idx - h * Ny;
        const double* g = A.G + (((long long)a) * H + h) * (Nx + 2);
        if (A.mean) A.mean[idx] = __ldcg(g);
        if (A.var) A.var[idx] = __ldcg(g + 1);
    }
    __syncthreads();
    if (A.cov) {
        for (int idx = tid; idx < H * Ny * Ny; idx += nth) {
            const int h = idx / (Ny * Ny), r = idx - h * Ny * Ny, a = r / Ny, b = r - a * Ny;
            double s = (a == b) ? __ldcg(A.G + (((long long)a) * H + h) * (Nx + 2) + 1) : 0.0;
            if (ta) {
                const double* gb = A.G + (((long long)b) * H + h) * (Nx + 2) + 2;
                const double* js = JS + (h * Ny + a) * Nx;
                double t = 0.0;
                for (int e = 0; e < Nx; ++e) t = fma(js[e], __ldcg(gb + e), t);
                s += t;
            }
            A.cov[idx] = s;
        }
    }
}

// shared-memory doubles assemble_rows needs (host side: AssembleArgs::stage_g)
__host__ __device__ inline long long assemble_rows_doubles(int H, int Ny, int Nx)
{
    return (long long)H * Ny * (((Nx + 2) | 1) + (Nx | 1)) + (long long)Nx * Nx;
}

__device__ __forceinline__ void assemble_rows(const AssembleArgs& A, double* sh, int tid, int nth)
{
    const int Ny = A.Ny, Nx = A.Nx, H = A.H, F = Nx + 2, FP = F | 1, NP = Nx | 1, R = H * Ny;
    const bool ta = A.cov && A.method_ta;
    double* Gs = sh;                                   // [H Ny][FP]: mean, var, J_0.. of (point, output)
    double* JS = Gs + R * FP;                          // [H Ny][NP]: (J Sigma) row, later the cov row
    double* Ss = JS + R * NP;                          // [Nx][Nx]: one Sigma for every point
    const bool sig_s = ta && !A.sigma_per_point;
    {
        const int tot = R * F, HF = H * F;
        if (sig_s) for (int i = tid; i < Nx * Nx; i += nth) Ss[i] = A.Sigma[i];
        constexpr int SB = 20;                                  // C5, 8 outputs: 4800 records words = 19 per thread
        for (int idx = tid; idx < tot; idx += SB * nth) {      // all loads of a batch first
            double v[SB];
#pragma unroll
            for (int k = 0; k < SB; ++k) v[k] = (idx + k * nth < tot) ? __ldcg(A.G + idx + k * nth) : 0.0;
#pragma unroll
            for (int k = 0; k < SB; ++k) {
                const int o = idx + k * nth;
                if (o < tot) {
                    const int a = o / HF, rem = o - a * HF, h = rem / F, q = rem - h * F;
                    Gs[(h * Ny + a) * FP + q] = v[k];
                }
            }
        }
        __syncthreads();
    }
    tail_stamp(A.dbg, 3, tid);
    if (A.J) for (int i = tid; i < R * Nx; i += nth) { const int row = i / Nx; A.J[i] = Gs[row * FP + 2 + (i - row * Nx)]; }
    for (int idx = tid; idx < R; idx += nth) {
        const double* g = Gs + idx * FP;
        if (A.mean) A.mean[idx] = g[0];
        if (A.var) A.var[idx] = g[1];
        if (ta) {
            const int h = idx / Ny;
            const double* Sg = sig_s ? Ss : A.Sigma + (long long)h * Nx * Nx;
            for (int e0 = 0; e0 < Nx; e0 += 8) {
                double acc[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) acc[k] = 0.0;
                for (int d = 0; d < Nx; ++d) {
                    const double jd = g[2 + d];
#pragma unroll
                    for (int k = 0; k < 8; ++k) if (e0 + k < Nx) acc[k] = fma(jd, Sg[d * Nx + e0 + k], acc[k]);
                }
#pragma unroll
                for (int k = 0; k < 8; ++k) if (e0 + k < Nx) JS[idx * NP + e0 + k] = acc[k];
            }
        }
    }
    __syncthreads();
    tail_stamp(A.dbg, 4, tid);
    if (A.cov) {
        const bool via_smem = Ny <= 8 && Ny <= NP;        // the finished cov row replaces the thread's own J Sigma row
        for (int idx = tid; idx < R; idx += nth) {
            const int h = idx / Ny, a = idx - h * Ny;
            const double var = Gs[idx * FP + 1];
            for (int b0 = 0; b0 < Ny; b0 += 8) {
                double acc[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) acc[k] = 0.0;
                if (ta) {
                    for (int e = 0; e < Nx; ++e) {
                        const double je = JS[idx * NP + e];
#pragma unroll
                        for (int k = 0; k < 8; ++k) if (b0 + k < Ny) acc[k] = fma(je, Gs[(h * Ny + b0 + k) * FP + 2 + e], acc[k]);
                    }
                }
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    if (b0 + k < Ny) {
                        const double c = ((a == b0 + k) ? var : 0.0) + acc[k];
                        if (via_smem) JS[idx * NP + k] = c; else A.cov[(long long)idx * Ny + b0 + k] = c;
                    }
                }
            }
        }
        if (via_smem) {
            __syncthreads();
            for (int i = tid; i < R * Ny; i += nth) { const int row = i / Ny; A.cov[i] = JS[row * NP + (i - row * Ny)]; }
        }
    }
}

__device__ __forceinline__ void assemble_flat(const AssembleArgs& A, double* sh, int tid, int nth)
{
    if (A.stage_g) assemble_rows(A, sh, tid, nth);
    else assemble_flat_global(A, sh, tid, nth);
}

// peer mode: acquire every source rank's flag for this step; false = a rank never showed up
__device__ __forceinline__ bool peer_acquire(const AssembleArgs& A, int tid, int* sh_ok)
{
    if (!A.flags) return true;
    if (tid == 0) *sh_ok = 1;
    __syncthreads();
    if (tid < A.world) {
        const long long t0 = clock64();
        unsigned long long v;
        do {
            asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(A.flags + tid) : "memory");
            if (v >= A.step) break;
            if (clock64() - t0 > A.timeout_clocks) {      // status lives in mapped host memory
                *reinterpret_cast<volatile int*>(A.status) = 1 + tid;
                *reinterpret_cast<volatile int*>(sh_ok) = 0;
                break;
            }
            __nanosleep(64);
        } while (true);
    }
    __syncthreads();
    return *reinterpret_cast<volatile int*>(sh_ok) != 0;
}

// stand-alone assembly (H above one chunk, or after the NCCL all-gather fallback)
__global__ void __launch_bounds__(128)
assemble_kernel(const AssembleArgs A)
{
    extern __shared__ double sh[];          // Jh[Ny][Nx], JS[Ny][Nx], varh[Ny]
    __shared__ int ok;
    if (!peer_acquire(A, threadIdx.x, &ok)) return;
    for (int h = blockIdx.x; h < A.H; h += gridDim.x) assemble_point<false>(A, h, sh, threadIdx.x, blockDim.x);
}

// The k-step list of one output.  Lower: tile jt covers k < min((jt+1) BN, Npad).  Upper: list position jt stands for
// column tile ntb-1-jt, which covers k in [(ntb-1-jt) BN, Npad).  Only a tile that reaches Npad can be short (the half
// tile of an odd Npad / 128: the L-side map's row bound zero-fills its upper half), so with d = SB ntb - nk (0 or 8)
// position jt has SB (jt+1) steps in lower mode, except the last one (SB ntb - d), and SB (jt+1) - d in upper mode.
// The two modes' totals differ when d != 0.
#define PSK_SB (PSK_BN / GEMM_BK)     // k-steps per full tile height
__host__ __device__ inline long long psk_kstart(int ntb, int nk, int upper, int jt)   // first step of position jt
{
    const long long full = (long long)(PSK_SB / 2) * jt * (jt + 1), d = (long long)PSK_SB * ntb - nk;
    return upper ? full - jt * d : (jt == ntb ? full - d : full);
}
__host__ __device__ inline long long psk_steps_per_output(int ntb, int nk, int upper) { return psk_kstart(ntb, nk, upper, ntb); }
__device__ __forceinline__ long long psk_kstart(const PredictParams& p, int jt) { return psk_kstart(p.ntb, p.nk, p.upper, jt); }
// A tile's k range reaches 128 columns past the diagonal of its first (lower) / before the diagonal of its second (upper)
// 128-row half.  Only the leaf kernel's diagonal 128 x 128 blocks are stored with explicit zeros on their far side; the
// off-diagonal block beyond is not kept zero (a full K build leaves K's upper triangle in the L slab), so the warps of
// that half skip those 8 k-steps in the product kernel's main loop and never read it.
__host__ __device__ inline int psk_ksteps(int ntb, int nk, int upper, int jt)
{
    return upper ? nk - PSK_SB * (ntb - 1 - jt) : (PSK_SB * (jt + 1) < nk ? PSK_SB * (jt + 1) : nk);
}
__device__ __forceinline__ int psk_ksteps(const PredictParams& p, int jt) { return psk_ksteps(p.ntb, p.nk, p.upper, jt); }

// The paired schedule (lower mode).  Unit p of an output is tiles ntb-1-p (long, first) and p (short), so every unit has
// SB (ntb + 1) k-steps -- the middle tile of an odd ntb is a unit alone, and the pair with the half tile of an odd Npad / 128
// is 8 steps shorter.  Unit u = a upo + p goes to CTA u mod C: the CTAs of one output start its long tiles at k = 0 together
// and advance at the same rate, so one fetch of a ks^T box serves all of them and only the few outputs in flight keep ks^T
// in L2.  Each tile is one accumulation chain from k = 0 inside one CTA, so the bits do not depend on C.
// psk_pair_units: units per output when this schedule applies, else 0.  It applies when every CTA of the grid owns at least
// one unit and the rounds of units fill at least 7/8 of the grid's unit slots: a CTA's time is its unit count, so 136
// units on 132 CTAs would take two rounds for the work of one and stay on stream-K (C5 on 132 SMs: 256 units, 0.97).
__host__ __device__ inline int psk_pair_units(int nloc, int ntb, int grid)
{
    const long long upo = (ntb + 1) / 2, units = nloc * upo, rounds = (units + grid - 1) / grid;
    return (units >= grid && 8 * units >= 7 * rounds * grid) ? (int)upo : 0;
}
// the automatic grid of the paired schedule: the fewest CTAs that need no more rounds of units than `grid` CTAs would, so
// the CTAs' unit counts are equal or one apart and no SM starts a unit it cannot finish with the others (C5 on 132 SMs:
// 128 CTAs of 2 units each, measured faster than 132 of 2 or 1)
__host__ __device__ inline int psk_pair_grid(long long units, int grid)
{
    const long long rounds = (units + grid - 1) / grid;
    return (int)((units + rounds - 1) / rounds);
}
__host__ __device__ inline int psk_unit_steps(int ntb, int nk, int pu)
{
    const int jl = ntb - 1 - pu;
    return psk_ksteps(ntb, nk, 0, jl) + (pu != jl ? psk_ksteps(ntb, nk, 0, pu) : 0);
}
// k-steps of CTA c of C
__host__ __device__ inline long long psk_pair_cta_steps(int nloc, int ntb, int nk, int upo, long long c, long long C)
{
    long long n = 0;
    for (long long u = c; u < (long long)nloc * upo; u += C) n += psk_unit_steps(ntb, nk, (int)(u % upo));
    return n;
}
// the long tile of unit u, where CTA u starts
__host__ __device__ inline void psk_pair_first(int ntb, int upo, long long u, int& a, int& jt)
{
    a = (int)(u / upo);
    jt = ntb - 1 - (int)(u - (long long)a * upo);
}
// the tile after tile (a, jt) in a CTA's sequence: the short tile of the same unit, or the long tile of unit u + C
__host__ __device__ inline void psk_pair_next(int ntb, int upo, long long C, int& a, int& jt)
{
    if (2 * jt > ntb - 1) jt = ntb - 1 - jt;
    else psk_pair_first(ntb, upo, (long long)a * upo + jt + C, a, jt);
}

struct PskIter { int a, jt, s, ks; };

// the first step of CTA c of C: unit c (paired), or position G c / C of the list (stream-K)
__device__ __forceinline__ void psk_iter_init(PskIter& it, const PredictParams& p, long long c, long long C)
{
    if (p.upo) {
        psk_pair_first(p.ntb, p.upo, c, it.a, it.jt);
        it.s = 0; it.ks = psk_ksteps(p, it.jt);
        return;
    }
    const long long g = p.G * c / C;
    it.a = (int)(g / p.T);
    const long long r = g - (long long)it.a * p.T;            // (SB/2) jt (jt+1) <= r, about
    int jt = (int)((sqrt(8.0 * (double)r / PSK_SB + 1.0) - 1.0) * 0.5);
    jt = max(0, min(jt, p.ntb - 1));
    while (jt > 0 && psk_kstart(p, jt) > r) --jt;
    while (jt + 1 < p.ntb && psk_kstart(p, jt + 1) <= r) ++jt;
    it.jt = jt; it.s = (int)(r - psk_kstart(p, jt)); it.ks = psk_ksteps(p, jt);
}
__device__ __forceinline__ void psk_iter_next(PskIter& it, const PredictParams& p)
{
    if (++it.s == it.ks) {
        it.s = 0;
        if (p.upo) psk_pair_next(p.ntb, p.upo, gridDim.x, it.a, it.jt);
        else if (++it.jt == p.ntb) { it.jt = 0; ++it.a; }
        it.ks = psk_ksteps(p, it.jt);
    }
}

// The L^-1 panel (dLiP): each output's lower-mode k-step list, block after block in the order the product consumes it.
// Block g = a T + psk_kstart(jt) + s (PSK_BN x 16 doubles) holds rows jt BN .. jt BN + BN-1 and columns 16 s .. 16 s + 15
// of output a's L^-1 exactly as the tensor map lands them in a stage: 128-byte rows, the 16-byte chunk c of row r at
// chunk c ^ (r & 7), rows past Npad (the half tile) zero.  Each tile, and a stream-K CTA's whole range of the list, is then
// one contiguous stretch of memory.  The far-side 128 x 128 block the upper-half warps skip is copied as L^-1 holds it.
// psk_panel_chunk: offset (doubles) in one output's panel of chunk c (columns 16 s + 2c, +1) of row r of tile jt, step s.
__host__ __device__ inline long long psk_panel_chunk(int ntb, int nk, int jt, int s, int r, int c)
{
    return (psk_kstart(ntb, nk, 0, jt) + s) * (PSK_BN * GEMM_BK) + r * GEMM_BK + 2 * (c ^ (r & 7));
}

// grid (nk, ntb - jt0): block (s, jt - jt0) of output Li, 8 threads per row with one 16-byte load and store each
__global__ void __launch_bounds__(256)
panel_pack_kernel(const double* __restrict__ Li, int np, double* __restrict__ P, int ntb, int jt0)
{
    const int s = blockIdx.x, jt = jt0 + blockIdx.y, nk = np / GEMM_BK, c = threadIdx.x & 7;
    if (s >= psk_ksteps(ntb, nk, 0, jt)) return;
#pragma unroll 4
    for (int r = threadIdx.x >> 3; r < PSK_BN; r += 32) {
        const long long row = (long long)jt * PSK_BN + r;
        const double2 v = row < np ? __ldcs(reinterpret_cast<const double2*>(Li + row * np + s * GEMM_BK) + c) : make_double2(0.0, 0.0);
        *reinterpret_cast<double2*>(P + psk_panel_chunk(ntb, nk, jt, s, r, c)) = v;
    }
}

// Records [mean, var, J_0..] of (output a, test point h), built in two places:
//   psk_reduce_mj: mean and J from the partial sums of ks_rows_kernel (gp_functions.py:119-120,135,146-147).  They do
//     not depend on the product, so the fused kernel spreads these sums over ALL its CTAs and runs them while the first
//     TMA stages are in flight (item = (a, h, field), one thread each, its nblk loads issued in batches of 16).
//   psk_finalize_output: var = sf2 - sum_jt SQ (gp_functions.py:125-126,136) by the CTA that completes the output: 4 lanes
//     per test point, each one chain of nt/4 tile sums, combined (s0+s1)+(s2+s3) by two shuffles.
// A serial load -> add loop costs one L2 round trip per iteration on one in-order warp, which made the r2 mid-round tail
// (one CTA, both jobs, divergent per-field branches) slow; splitting the jobs keeps the var part short.
__device__ __forceinline__ void psk_store_record(const PredictParams& p, int a, int h, int q, double val)
{
    const long long off = (((long long)(p.slot0 + a)) * p.Htot + p.h0 + h) * (p.Nx + 2) + q;
    if (!p.use_peers) p.Gloc[off] = val;
    else for (int r = 0; r < p.pa.world; ++r) p.pa.base[r][p.pa.goff + off] = val;
}

// items [i_begin, i_end) of the flat (a, h, field) space, field 0 = mean, 1 + d = J_d; threads [t0, t0 + nthr) of the CTA
__device__ __forceinline__ void psk_reduce_mj(const PredictParams& p, int i_begin, int i_end, int t, int nthr)
{
    const int F1 = p.Nx + 1;
    for (int i = i_begin + t; i < i_end; i += nthr) {
        const int ah = i / F1, qq = i - ah * F1, a = ah / p.Hc, h = ah - a * p.Hc;
        const double* pm = p.PMJ + ((long long)ah * p.nblk_mj) * F1 + qq;
        double s0 = 0.0, s1 = 0.0;                         // even / odd blocks, fixed association
        int b = 0;
        for (; b + 16 <= p.nblk_mj; b += 16) {
            double v[16];
#pragma unroll
            for (int k = 0; k < 16; ++k) v[k] = __ldcg(pm + (long long)(b + k) * F1);
#pragma unroll
            for (int k = 0; k < 16; k += 2) { s0 += v[k]; s1 += v[k + 1]; }
        }
        for (; b + 2 <= p.nblk_mj; b += 2) { s0 += __ldcg(pm + (long long)b * F1); s1 += __ldcg(pm + (long long)(b + 1) * F1); }
        if (b < p.nblk_mj) s0 += __ldcg(pm + (long long)b * F1);
        psk_store_record(p, a, h, qq == 0 ? 0 : qq + 1, s0 + s1);
    }
}

__device__ __forceinline__ void psk_finalize_output(const PredictParams& p, int a, int tid, int nth)
{
    const int Nx = p.Nx;
    const double sf = p.hyp[(long long)a * p.hyp_ld + Nx];
    for (int base = 0; base < p.Hc; base += nth / 4) {         // nth is a multiple of 32
        const int h = base + (tid >> 2), j0 = tid & 3;
        double sj = 0.0;
        if (h < p.Hc) {
            const double* sq = p.SQ + ((long long)a * 64 + h) * p.nt;
            int j = j0;
            for (; j + 4 * 15 < p.nt; j += 4 * 16) {
                double v[16];
#pragma unroll
                for (int k = 0; k < 16; ++k) v[k] = __ldcg(sq + j + 4 * k);
#pragma unroll
                for (int k = 0; k < 16; ++k) sj += v[k];
            }
            for (; j < p.nt; j += 4) sj += __ldcg(sq + j);
        }
        sj += __shfl_xor_sync(0xffffffffu, sj, 1);            // s0 + s1 | s2 + s3
        sj += __shfl_xor_sync(0xffffffffu, sj, 2);            // (s0 + s1) + (s2 + s3)
        if (h < p.Hc && j0 == 0) psk_store_record(p, a, h, 1, sf * sf - sj);
    }
    if (p.use_peers) __threadfence_system(); else __threadfence();
}

// after an output's records are written: the CTA that completes the step's last output publishes
// the peer flags and (optionally) assembles.  Must be called by every thread of the CTA.
__device__ __forceinline__ void psk_step_tail(const PredictParams& p, double* sh, int tid, int nth,
                                              unsigned int* s_flag, int* s_ok)
{
    __syncthreads();
    if (tid == 0) {
        const unsigned int old = atomicAdd(p.done_cnt, 1u);
        const unsigned int last = (old == (unsigned int)(p.nloc - 1)) ? 1u : 0u;
        if (last) *p.done_cnt = 0u;
        *s_flag = last;
    }
    __syncthreads();
    if (*s_flag == 0u) return;
    if (p.finalize && p.use_peers && p.publish && tid == 0) {
        __threadfence_system();
        for (int r = 0; r < p.pa.world; ++r) {
            unsigned long long* f = reinterpret_cast<unsigned long long*>(p.pa.base[r]) + p.pa.flag_idx;
            asm volatile("st.release.sys.global.u64 [%0], %1;" :: "l"(f), "l"(p.pa.step) : "memory");
        }
    }
    tail_stamp(p.as.dbg, 2, tid);
    if (p.do_assemble) {
        __threadfence();
        if (peer_acquire(p.as, tid, s_ok)) assemble_flat(p.as, sh, tid, nth);
    }
    __syncthreads();
    tail_stamp(p.as.dbg, 5, tid);
}

// refinement path: the solved rows were corrected outside the product (v = v1 + Li r), so the
// squared norms are taken from V itself; then the common finalize / publish / assemble tail.
// grid (nt, Hc, nloc): SQ[a][h][jt] = sum of squares of the 128 columns of tile jt
__global__ void __launch_bounds__(128)
sq_rows_kernel(const double* __restrict__ V, int ldv, long long sV, double* __restrict__ SQ, int nt)
{
    __shared__ double red[4];
    const int jt = blockIdx.x, h = blockIdx.y, a = blockIdx.z;
    const double v = V[(long long)a * sV + (long long)h * ldv + jt * 128 + threadIdx.x];
    const double s = warp_sum(v * v);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) SQ[((long long)a * 64 + h) * nt + jt] = (red[0] + red[1]) + (red[2] + red[3]);
}

__global__ void __launch_bounds__(PSK_THREADS)
finalize_kernel(const PredictParams p)
{
    extern __shared__ double sh[];
    __shared__ unsigned int s_flag;
    __shared__ int s_ok;
    const int per = p.Hc * (p.Nx + 1);
    psk_reduce_mj(p, blockIdx.x * per, (blockIdx.x + 1) * per, threadIdx.x, PSK_THREADS);
    psk_finalize_output(p, blockIdx.x, threadIdx.x, PSK_THREADS);
    psk_step_tail(p, sh, threadIdx.x, PSK_THREADS, &s_flag, &s_ok);
}

// The product on DMMA.16x8x16 (dmma16816).  tmA delivers the BM x 16 box of ks^T (test points x k), tmB the BN x 16
// box of the L-side matrix (L^-1, U in upper mode, L in the refinement), both in rows of 128 bytes with the 128B
// swizzle: the 16-byte chunk c of row r sits at chunk c ^ (r & 7).  A lower-mode product of L^-1 (p.Lp) copies the same
// bytes from the panel instead (panel_pack_kernel).
//   Per k-step (16 k) warp w computes the 32 x BM block V^T[L-rows 32w .. 32w+31][points] as two MMA A
//   operands (mi = 0, 1: L-rows 32w + 16 mi .. +15, row layout) against ks^T as the B operand (col layout, N = 8
//   points per fragment, BM / 8 fragments).  Each B fragment feeds both A fragments: 16 + 4 BM / 8 LDS.64 per 2 BM / 8
//   DMMAs, where 16 L-rows per warp needed 8 + 4 BM / 8 per BM / 8.
//   k-permutation: lane (g, t) puts k = 2j + (t & 1) + 8 (t >> 1) into register slot j (the one gemm_dmma_tmap_kernel
//   uses per 4-k step), i.e. logical chunk j + 4 (t >> 1), half t & 1.  Each value is one LDS.64 straight into its
//   MMA register, and the 16 lanes of a half-warp hit 16 distinct 8-byte banks under the swizzle (rows g, g + 8,
//   g + 16, g + 24 of a warp all sit at swizzle phase g).
//   A: av[mi][2j] = L-row 32w + 16 mi + g, av[mi][2j+1] = the row 8 below;  B: point row 8 ni + g.
//   accumulators acc[mi][ni][i]: L-row 32w + 16 mi + g + 8 (i >> 1), point 8 ni + 2t + (i & 1).
//   (Contiguous k = 4t + j would allow LDS.128, but the MMA pairs rows g and g + 8 in adjacent A registers, so every
//   A load then needs register moves; ptxas kept two copies of the A fragment and spilled.)
// Every BM uses this one instruction shape, k-permutation and reduction order (per 128-column group: sum of squares
// over the thread's two L-rows, xor shuffles over g, then the group's eight 16-row blocks in order), so a point's var
// does not depend on BM or on its row in the chunk.
template <int BM>
__global__ void __launch_bounds__(PSK_THREADS, PSK_CTAS_PER_SM)
predict_streamk_kernel(const PredictParams p, const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB)
{
    constexpr int BK = GEMM_BK, BN = PSK_BN, STAGES = PSK_STAGES, CW = PSK_CW, NT = PSK_THREADS;
    constexpr int NF = BM / 8;                                     // 8-point fragments; CW warps x 32 L-rows = BN
    static_assert(BK == 16 && BN == 32 * CW && BN % 128 == 0, "one m16n8k16 per fragment and k-step, 32 L-rows per warp");
    constexpr int GR = BN / 128;                                   // 128-column groups per tile
    constexpr int A_STAGE = BM * BK, B_STAGE = BN * BK;           // doubles, 128-byte rows, 128B swizzle
    constexpr uint32_t STAGE_TX = (BM + BN) * BK * 8;
    static_assert(BM % 8 == 0 && BM >= 8 && BM <= 64, "BM");

    extern __shared__ __align__(16) double smem_raw[];
    double* smem = smem_align1024(smem_raw);
    double* As = smem;
    double* Bs = smem + STAGES * A_STAGE;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * (A_STAGE + B_STAGE));
    uint64_t* empty = full + STAGES;
    __shared__ double red[BN / 16][64];
    __shared__ unsigned int s_flag;
    __shared__ int s_ok;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const long long C = gridDim.x, c = blockIdx.x;
    const int nsteps = p.upo ? (int)psk_pair_cta_steps(p.nloc, p.ntb, p.nk, p.upo, c, C)    // this CTA's share of the
                             : (int)(p.G * (c + 1) / C - p.G * c / C);                      // k-step list
    if (nsteps <= 0) return;
    if (p.dbg && threadIdx.x == 0) { unsigned long long t0; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0)); p.dbg[2 * blockIdx.x] = t0; }

    // producer state lives in shared memory: only thread 0 touches it, so it costs no registers
    __shared__ PskIter s_pit;
    __shared__ int s_pg;
    __shared__ uint64_t s_pol[2];
    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < STAGES; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, CW); }
        mbar_fence_init();
    }
    __syncthreads();

    // Pipeline without CTA-wide barriers: stage s is FULL when its two TMA boxes have landed and EMPTY when all CW warps
    // have read it.  Thread 0 refills AHEAD = STAGES - 2 steps ahead: the stage it overwrites at step i was last read at
    // step i - 2, so its empty-wait is almost never a real wait and the warps may drift up to a step apart.
    auto issue = [&]() {               // thread 0: TMA loads of step s_pg into stage s_pg % STAGES
        PskIter it = s_pit;
        const int pg = s_pg, s = pg % STAGES;
        if (pg >= STAGES) mbar_wait(empty + s, (uint32_t)(((pg / STAGES) - 1) & 1));
        mbar_arrive_expect_tx(full + s, STAGE_TX);
        const int jta = p.upper ? p.ntb - 1 - it.jt : it.jt;
        const int k0 = (p.upper ? jta * BN : 0) + it.s * BK;
        // ks^T (A) is re-read by every column tile: keep it in L2; L^-1 (B) is streamed exactly once.  Also when ks^T is
        // larger than the L2 (8 outputs at N=16384 on H100: 59 MB vs 50 MB) evict_last measured no slower than evict_normal
        tma_tile_g2s_3d_hint(As + s * A_STAGE, &tmA, k0, 0, it.a, full + s, s_pol[1]);
        // the panel holds the step as the tensor map would land it: one contiguous 32 KB copy instead of 256 rows
        if (p.Lp) bulk_g2s_hint(Bs + s * B_STAGE, p.Lp + ((long long)it.a * p.T + psk_kstart(p, it.jt) + it.s) * B_STAGE,
                                B_STAGE * 8, full + s, s_pol[0]);
        else tma_tile_g2s_3d_hint(Bs + s * B_STAGE, &tmB, k0, jta * BN, it.a, full + s, s_pol[0]);
        psk_iter_next(it, p);
        s_pit = it;
        s_pg = pg + 1;
    };
    constexpr int AHEAD = STAGES - 2;  // prefetch distance in steps
    // programmatic dependent launch: everything above overlapped the tail of the ks kernel; its output
    // (KS^T, the partial mean / Jacobian sums) is only touched below this point.  A no-op when the
    // kernel was launched without the attribute.
    asm volatile("griddepcontrol.wait;" ::: "memory");
    if (tid == 0) {
        PskIter it;
        psk_iter_init(it, p, c, C);
        s_pit = it; s_pg = 0;
        s_pol[0] = l2_policy_evict_first(); s_pol[1] = l2_policy_evict_last();
#pragma unroll
        for (int s = 0; s < AHEAD; ++s)
            if (s_pg < nsteps) issue();
    }
    if (p.finalize) {
        // this CTA's share of the mean / Jacobian records (warps 1..; thread 0 is the TMA producer), while the first
        // stages are in flight.  Ordered before the step's publication by the fence + counter chain every CTA's tiles
        // go through (each CTA owns at least one k-step).
        const int tot = p.nloc * p.Hc * (p.Nx + 1), per = (tot + (int)C - 1) / (int)C;
        if (tid >= 32) {
            psk_reduce_mj(p, min(tot, (int)c * per), min(tot, ((int)c + 1) * per), tid - 32, NT - 32);
            if (p.use_peers) __threadfence_system();
        }
    }

    PskIter cit;
    psk_iter_init(cit, p, c, C);
    int cj[4];                                                      // slot j: k = 2j + (t & 1) + 8 (t >> 1)
#pragma unroll
    for (int j = 0; j < 4; ++j) cj[j] = (((j + 4 * (t >> 1)) ^ g) << 1) + (t & 1);
    int i = 0;
    while (i < nsteps) {
        const int a = cit.a, jt = cit.jt, s_begin = cit.s, ksteps = cit.ks;
        const int seg = min(ksteps - s_begin, nsteps - i);
        // steps [st_lo, st_hi) of the tile touch this warp's 128-row half below (lower) / above (upper) the diagonal; the
        // others would read the 128 x 128 block on the wrong side of it, which no caller keeps zero (psk_ksteps)
        const int hh = warp / (128 / 32);
        const int st_lo = p.upper ? (128 / BK) * hh : 0;
        const int st_hi = p.upper ? ksteps : PSK_SB * jt + (128 / BK) * (hh + 1);
        double acc[2][NF][4];
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
            for (int ni = 0; ni < NF; ++ni)
#pragma unroll
                for (int r = 0; r < 4; ++r) acc[mi][ni][r] = 0.0;

        for (int q = 0; q < seg; ++q, ++i) {
            const int s = i % STAGES;
            if (tid == 0 && i + AHEAD < nsteps) issue();  // s_pg == i + AHEAD
            mbar_wait(full + s, (uint32_t)((i / STAGES) & 1));
            const int st = s_begin + q;
            if (st >= st_lo && st < st_hi) {
                const double* ls = Bs + s * B_STAGE + (warp * 32 + g) * 16;    // L-rows 32w + g (+ 8, 16, 24: 128 doubles apart)
                const double* ps = As + s * A_STAGE + g * 16;                  // point rows 8 ni + g
                double av[2][8];
#pragma unroll
                for (int mi = 0; mi < 2; ++mi)
#pragma unroll
                    for (int j = 0; j < 4; ++j) { av[mi][2 * j] = ls[256 * mi + cj[j]]; av[mi][2 * j + 1] = ls[256 * mi + 128 + cj[j]]; }
#pragma unroll
                for (int ni = 0; ni < NF; ++ni) {
                    double bv[4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) bv[j] = ps[ni * 8 * 16 + cj[j]];
                    dmma16816(acc[0][ni], av[0], bv);
                    dmma16816(acc[1][ni], av[1], bv);
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(empty + s);        // this warp is done reading stage s
        }
        cit.s = s_begin + seg - 1;
        psk_iter_next(cit, p);

        // ---- tile fix-up: a tile cut by a range border is finished by its last-arriving contributor
        bool have_tile = true;
        if (seg != ksteps) {
            const long long tg0 = (long long)a * p.T + psk_kstart(p, jt), tg1 = tg0 + ksteps;
            const long long Cf = gridDim.x;                           // re-read: keeps C and c out of the loop's registers
            const int c_first = (int)(((tg0 + 1) * Cf - 1) / p.G), c_last = (int)((tg1 * Cf - 1) / p.G);
            double2* mine = reinterpret_cast<double2*>(p.part + ((long long)blockIdx.x * 2 + (s_begin == 0 ? 1 : 0)) * (BM * BN)) + tid;
#pragma unroll
            for (int mi = 0; mi < 2; ++mi)
#pragma unroll
                for (int ni = 0; ni < NF; ++ni)
#pragma unroll
                    for (int hf = 0; hf < 2; ++hf)
                        __stcg(mine + ((mi * NF + ni) * 2 + hf) * NT, make_double2(acc[mi][ni][2 * hf], acc[mi][ni][2 * hf + 1]));
            __threadfence();
            __syncthreads();
            if (tid == 0) {
                unsigned int* cnt = p.tile_cnt + (long long)a * p.ntb + jt;
                const unsigned int old = atomicAdd(cnt, 1u);
                const unsigned int last = (old == (unsigned int)(c_last - c_first)) ? 1u : 0u;
                if (last) *cnt = 0u;                      // self-cleaning: every contributor has arrived
                s_flag = last;
            }
            __syncthreads();
            have_tile = s_flag != 0u;
            if (have_tile) {
                __threadfence();
#pragma unroll
                for (int mi = 0; mi < 2; ++mi)
#pragma unroll
                    for (int ni = 0; ni < NF; ++ni)
#pragma unroll
                        for (int r = 0; r < 4; ++r) acc[mi][ni][r] = 0.0;
                for (int cc = c_first; cc <= c_last; ++cc) {          // contributor (= ascending k) order
                    const double2* src = reinterpret_cast<const double2*>(p.part + ((long long)cc * 2 + (cc == c_first ? 1 : 0)) * (BM * BN)) + tid;
#pragma unroll
                    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
                        for (int ni = 0; ni < NF; ++ni)
#pragma unroll
                            for (int hf = 0; hf < 2; ++hf) {
                                const double2 v = __ldcg(src + ((mi * NF + ni) * 2 + hf) * NT);
                                acc[mi][ni][2 * hf] += v.x; acc[mi][ni][2 * hf + 1] += v.y;
                            }
                }
            }
        }
        if (!have_tile) continue;

        // ---- complete tile: optional store of the solved rows, squared row norms of each 128-column group
        const int jta = p.upper ? p.ntb - 1 - jt : jt;
        const int row0 = jta * BN + warp * 32;                       // this warp's first L-row
        if (p.Vout && row0 < p.nk * BK) {                             // none past Npad (the half tile's zero rows)
            double* vo = p.Vout + (long long)a * p.sV + row0 + g;
#pragma unroll
            for (int mi = 0; mi < 2; ++mi)
#pragma unroll
                for (int ni = 0; ni < NF; ++ni)
#pragma unroll
                    for (int r = 0; r < 4; ++r)
                        vo[(long long)(ni * 8 + 2 * t + (r & 1)) * p.ldv + 16 * mi + 8 * (r >> 1)] = acc[mi][ni][r];
        }
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
            for (int ni = 0; ni < NF; ++ni)
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    double r = acc[mi][ni][j] * acc[mi][ni][j];       // L-row g, then g + 8
                    r = fma(acc[mi][ni][j + 2], acc[mi][ni][j + 2], r);
                    r += __shfl_xor_sync(0xffffffffu, r, 4);
                    r += __shfl_xor_sync(0xffffffffu, r, 8);
                    r += __shfl_xor_sync(0xffffffffu, r, 16);
                    if (g == 0) red[2 * warp + mi][ni * 8 + 2 * t + j] = r;   // 16-row block 2w + mi of the tile
                }
        __syncthreads();
        for (int idx = tid; idx < GR * BM; idx += NT) {             // (group, point): blocks 8 gr .. 8 gr + 7 in order
            const int gr = idx / BM, pt = idx - gr * BM, col = jta * GR + gr;
            if (col < p.nt) {
                double r = 0.0;
#pragma unroll
                for (int b = 0; b < 8; ++b) r += red[8 * gr + b][pt];
                __stcg(p.SQ + ((long long)a * 64 + pt) * p.nt + col, r);
            }
        }
        __threadfence();
        __syncthreads();
        if (tid == 0) {
            unsigned int* cnt = p.out_cnt + a;
            const unsigned int old = atomicAdd(cnt, 1u);
            const unsigned int last = (old == (unsigned int)(p.ntb - 1)) ? 1u : 0u;
            if (last) *cnt = 0u;
            s_flag = last;
        }
        __syncthreads();
        if (s_flag == 0u) continue;

        // ---- this CTA completed output a: build its records; last output => publish / assemble
        __threadfence();
        tail_stamp(p.as.dbg, 0, tid);
        if (p.finalize) psk_finalize_output(p, a, tid, NT);
        tail_stamp(p.as.dbg, 1, tid);
        psk_step_tail(p, smem, tid, NT, &s_flag, &s_ok);
    }
    if (p.dbg && threadIdx.x == 0) { unsigned long long t1; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1)); p.dbg[2 * blockIdx.x + 1] = t1; }
}
