// Device kernels of the GP hot path other than the DMMA GEMM family.
// Reference semantics are cited as file:line of helgeanl/GP-MPC.
#pragma once
#include <type_traits>
#include "common.cuh"

// hyper layout per output (device copy): [ell_0..ell_{Nx-1}, sf, sn]  (gp_class.py:139-142)
#define KB_TILE 64

// ---------------------------------------------------------------------------------------
// a1/a2  K = sf2 exp(-1/2 sum_d ((x_id - x_jd)/ell_d)^2) + (sn2 + jitter) I   (gp_functions.py:17-22,
//   optimize.py:303-319, :342-344), with the pairwise distances on the fp64 TENSOR pipe.
//   With u_i = sqrt(log2 e) (x_i - mu)/ell and q_i = -1/2 |u_i|^2 + 1/2 log2 sf2,
//       log2 k(x_i, x_j) = q_i + q_j + u_i . u_j            (= log2 sf2 - log2(e)/2 |xs_i - xs_j|^2)
//   so the O(N^2 Nx) part is a rank-Nx product done with DMMA m8n8k4 (tensor pipe), leaving the
//   fp64 pipe only ~12 instructions per pair (two adds, clamp, a two-level-table exp2 with a
//   degree-4 polynomial).  a profile of the first (direct-difference, libm exp) kernel showed the fp64 pipe and DRAM
//   traffic not overlapping: the two pipes now overlap and the kernel becomes write-bandwidth bound.
//   The kernel is translation invariant, so inputs are centred on the column means mu of the current X (set_data,
//   and recomputed after appends and removals): the expansion's cancellation error is eps*|u|^2 with |u| measured from
//   the data centre
//   (<= 6e-16 relative on both reference fixtures, same as direct differences; the reference's
//   own numpy path uses the un-centred expansion, optimize.py:315-319).
//   One CTA = one 128x128 tile of the lower triangle; off-diagonal tiles also store the
//   mirrored tile (each exp2 serves two outputs).  q_i + q_j and the k-ordered dot product are
//   commutative, so K is bitwise symmetric, including inside diagonal tiles.
// ---------------------------------------------------------------------------------------
// 2^(k/16) and 2^(m/256), k, m = 0..15, correctly rounded (generated with 40-digit arithmetic)
__constant__ double c_exp2_tab[16] = {
    1.0, 1.0442737824274138, 1.0905077326652577, 1.1387886347566916, 1.189207115002721,
    1.241857812073484, 1.2968395546510096, 1.3542555469368927, 1.4142135623730951,
    1.4768261459394993, 1.5422108254079407, 1.6104903319492543, 1.681792830507429,
    1.7562521603732995, 1.8340080864093424, 1.9152065613971474};
// Two-level table: 2^t = 2^e * T1[(n >> 4) & 15] * T2[n & 15] * 2^f with n = rint(256 t), T1[k] = 2^(k/16), T2[m] = 2^(m/256),
// |f| <= 1/512 (degree-4 polynomial, truncation 3.8e-17).  Both tables have ONE entry per shared-memory bank, so the
// lookups are conflict-free whatever the lane pattern (a flat 256-entry table replays ~3x), and the polynomial needs four
// coefficients where a single 16-entry table needs seven (each costs two UMOVs in the loop on this target).  At most
// 2.75 ulp (measured against mpmath on an exact restatement, tests/test_kernel_range_cpu.py).
// Valid for -1020 <= t <= ~1000: the CALLER clamps (rint(256 t) must fit the low word and the exponent stay normal).
// T32 is a shared-memory copy of both tables: T32[0..15] = c_exp2_tab, T32[16..31] = c_exp2_tab2.
__constant__ double c_exp2_tab2[16] = {
    1, 1.0027112750502025, 1.0054299011128027, 1.0081558981184175, 1.0108892860517005, 1.0136300849514894,
    1.0163783149109531, 1.0191339960777379, 1.0218971486541166, 1.0246677928971357, 1.0274459491187637,
    1.030231637686041, 1.0330248790212284, 1.0358256936019572, 1.0386341019613787, 1.0414501246883161};
__device__ __forceinline__ double exp2_t2lvl(double t, const double* __restrict__ T32)
{
    const double SH = 6755399441055744.0;            // 1.5 * 2^52: rint(256 t) lands in the low word
    const double s = fma(t, 256.0, SH);
    const int n = __double2loint(s);
    const double f = fma(s - SH, -0.00390625, t);    // |f| <= 1/512, exact
    double p = 0.009618129107628477;                 // (ln 2)^k / k!, k = 4..1
    p = fma(p, f, 0.05550410866482158);
    p = fma(p, f, 0.24022650695910072);
    p = fma(p, f, 0.6931471805599453);
    p = fma(p, f, 1.0);
    p *= T32[(n >> 4) & 15];
    p *= T32[16 + (n & 15)];
    return __hiloint2double(__double2hiint(p) + ((n >> 8) << 20), __double2loint(p));
}

struct KbTrue { __device__ constexpr operator bool() const { return true; } };
struct KbFalse { __device__ constexpr operator bool() const { return false; } };

#define KB2_TILE 128
template <bool FULL>
__global__ void __launch_bounds__(256)
kbuild_dmma_kernel(const double* __restrict__ XT, int ldx, int N, int Nx, const double* __restrict__ mu,
                   const double* __restrict__ hyp, int hyp_ld, const double* __restrict__ jitter,
                   double* __restrict__ K, int ld, long long sK)
{
    extern __shared__ double sm[];
    const int KD = (Nx + 3) & ~3;                         // k extent of the MMA, zero padded
    const int S = ((KD >> 2) & 1) ? KD : KD + 4;          // row stride: S/4 odd => conflict-free frags
    double* Ui = sm;                                      // [128][S]
    double* Uj = Ui + KB2_TILE * S;                       // [128][S]
    double* qi = Uj + KB2_TILE * S;                       // [128]
    double* qj = qi + KB2_TILE;                           // [128]
    double* T256 = qj + KB2_TILE;                         // [256]

    const int a = blockIdx.z;
    const double* hp = hyp + (long long)a * hyp_ld;
    const int tt = blockIdx.x;
    int bi = (int)((sqrt(8.0 * (double)tt + 1.0) - 1.0) * 0.5);
    while (bi * (bi + 1) / 2 > tt) --bi;
    while ((bi + 1) * (bi + 2) / 2 <= tt) ++bi;
    const int bj = tt - bi * (bi + 1) / 2;
    const int i0 = bi * KB2_TILE, j0 = bj * KB2_TILE;
    const int tid = threadIdx.x;
    const double sf2 = hp[Nx] * hp[Nx];
    const double l2sf2 = log2(sf2);

    __shared__ double sc[36], mus[36];                    // sqrt(log2 e) / ell_d and the column means: one division per dimension per CTA
    if (tid < S) {
        sc[tid] = (tid < Nx) ? 1.2011224087864498 / hp[tid] : 0.0;
        mus[tid] = (tid < Nx) ? mu[tid] : 0.0;
    }
    // two 16-entry tables (exp2_t2lvl): conflict-free lookups and a degree-4 polynomial
    if (tid < 16) T256[tid] = c_exp2_tab[tid];
    else if (tid < 32) T256[tid] = c_exp2_tab2[tid - 16];
    __syncthreads();
    {   // scaled, centred coordinates of the 128 row points (tid < 128) / column points
        const int p = (tid < KB2_TILE) ? i0 + tid : j0 + tid - KB2_TILE;
        double* U = (tid < KB2_TILE) ? Ui + tid * S : Uj + (tid - KB2_TILE) * S;
        double nrm = 0.0;
        for (int d = 0; d < S; ++d) {
            double u = 0.0;
            if (d < Nx) u = (XT[(long long)d * ldx + p] - mus[d]) * sc[d];
            U[d] = u;
            nrm = fma(u, u, nrm);
        }
        ((tid < KB2_TILE) ? qi : qj)[tid & (KB2_TILE - 1)] = fma(-0.5, nrm, 0.5 * l2sf2);
    }
    __syncthreads();

    const int warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const double dg = hp[Nx + 1] * hp[Nx + 1] + (jitter ? jitter[a] : 0.0);
    double* Ka = K + (long long)a * sK;
    const bool offdiag = (bi != bj);
    const bool mirror = FULL && offdiag;
    // tiles that touch the diagonal or the identity tail take the checked epilogue
    const bool special = !offdiag || (i0 + KB2_TILE > N) || (j0 + KB2_TILE > N);
    const int nk4 = KD >> 2;
    // SP = tile touches the diagonal or the identity tail (checked epilogue, upper clamp); MR = mirrored tile stored too.
    // Both are CTA-uniform.  No fmin/fmax anywhere (their NaN semantics cost ~7 instructions each on this target; a plain
    // compare-select is 3).
    auto tile_body = [&](auto sp_tag, auto mr_tag) {
        const bool SP = sp_tag, MR = mr_tag;      // KbTrue / KbFalse fold at compile time, plain bools stay run-time
#pragma unroll 1
        for (int mi = 0; mi < 2; ++mi) {
            const int rl = warp * 16 + mi * 8 + g;            // local row of this lane's accumulators
            const int row = i0 + rl;
            const double* ua = Ui + rl * S + t;
            const double qr = qi[rl];
            double* drow = Ka + (long long)row * ld + j0 + 2 * t;              // direct:  K[row][j0 + cl]
            double* mcol = Ka + (long long)(j0 + 2 * t) * ld + row;            // mirror:  K[j0 + cl][row]
#pragma unroll 1
            for (int ng = 0; ng < 4; ++ng) {
                double acc[4][2];
#pragma unroll
                for (int q = 0; q < 4; ++q) { acc[q][0] = 0.0; acc[q][1] = 0.0; }
                const double* ub = Uj + (ng * 32 + g) * S + t;
                for (int kk = 0; kk < nk4; ++kk) {
                    const double av = ua[kk * 4];
#pragma unroll
                    for (int q = 0; q < 4; ++q) dmma884(acc[q][0], acc[q][1], av, ub[q * 8 * S + kk * 4]);
                }
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int cl0 = ng * 32 + q * 8;          // + 2t folded into the base pointers
                    const double2 qc = *reinterpret_cast<const double2*>(qj + cl0 + 2 * t);
                    // log2 k, clamped from below (far-apart points under tiny length scales: SLSQP probes them; 2^-1020 ~ 0)
                    double t0 = (qr + qc.x) + acc[q][0], t1 = (qr + qc.y) + acc[q][1];
                    t0 = (t0 < -1020.0) ? -1020.0 : t0;
                    t1 = (t1 < -1020.0) ? -1020.0 : t1;
                    if (SP) {                                 // k <= sf2 despite rounding: only where the distance can be 0
                        t0 = (t0 > l2sf2) ? l2sf2 : t0;
                        t1 = (t1 > l2sf2) ? l2sf2 : t1;
                    }
                    double v0 = exp2_t2lvl(t0, T256), v1 = exp2_t2lvl(t1, T256);
                    if (SP) {
                        const int col = j0 + cl0 + 2 * t;
                        if (row == col) v0 += dg;
                        if (row == col + 1) v1 += dg;
                        if (row >= N || col >= N) v0 = (row == col) ? 1.0 : 0.0;
                        if (row >= N || col + 1 >= N) v1 = (row == col + 1) ? 1.0 : 0.0;
                    }
                    *reinterpret_cast<double2*>(drow + cl0) = make_double2(v0, v1);
                    if (MR) {
                        double* m = mcol + (long long)cl0 * ld;        // independent address per store pair (no serial pointer chain)
                        m[0] = v0;
                        m[ld] = v1;
                    }
                }
            }
        }
    };
    if (FULL) {
        // store-bound: one body with run-time flags (four specialised copies measured slower: CTAs of different kinds
        // share an SM and the instruction working set quadruples)
        tile_body(special, mirror);
    } else if (special) {
        tile_body(KbTrue{}, KbFalse{});
    } else {
        tile_body(KbFalse{}, KbFalse{});      // instruction-bound: the hot path carries no checks at all
    }
}

// ---------------------------------------------------------------------------------------
// a3 leaf: 128x128 diagonal block  ->  L (in place, zeros above the diagonal) and L^-1.
//   np.linalg.cholesky at optimize.py:346/485; a non-positive pivot is reported LAPACK
//   style (1-based global index) so the host can apply the reference's single 1e-8
//   jitter retry (optimize.py:347-350).  One CTA per batch entry; whole block in smem.
//   Blocked (nb = 16) right-looking Cholesky + triangular inverse; the trailing updates and the
//   inverse assembly run on DMMA fragments read straight from shared memory (row stride
//   LF_LD = 132 doubles: (g*32 + t*8) mod 128 is conflict-free).  The 128-pivot dependency chain
//   is the only thing on the critical path:
//   * per 16-column block step the chain is  potrf16 (warp 0, registers + shuffles, two pivots
//     per step)  ->  panel by FORWARD SUBSTITUTION with the 16x16 factor (one
//     thread per row, the factor is broadcast from shared memory; no 16x16 inverse needed)  ->
//     DMMA update of the next block column;
//   * everything else runs beside it: warps 2..7 finish the trailing update of the previous step
//     and warp 1 inverts the previous 16x16 diagonal block (needed only by the inverse assembly)
//     while warp 0 factorises the next one;
//   * the triangular inverse is assembled by recursive doubling with four independent DMMA
//     accumulator chains per warp;
//   * 16-byte global loads / stores.
// ---------------------------------------------------------------------------------------
#define LEAF_N 128
#define LF_LD 132
#define LF_NB 16
// optional phase clock stamps of CTA 0 (diagnostics: gpmpc_profile_leaf)
__device__ long long* d_leaf_prof = nullptr;
#define LEAF_STAMP(k) do { if (d_leaf_prof && blockIdx.x == 0 && threadIdx.x == 0) d_leaf_prof[k] = clock64(); } while (0)

__device__ __forceinline__ double rsqrt_seeded(double d)
{
    // rsqrt.approx.f64 (SASS MUFU.RSQ64H on the high word, ~2^-22, no fp32 round trip) + two Newton steps in
    // fp64: relative error ~1e-15; tiny / huge / non-positive arguments take the library routine
    if (!(d > 1e-290 && d < 1e290)) return rsqrt(d);
    double y;
    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(d));
    double e = fma(-(d * y), y, 1.0);
    y = fma(0.5 * y, e, y);
    e = fma(-(d * y), y, 1.0);
    y = fma(0.5 * y, e, y);
    return y;
}

// 16x16 Cholesky in registers (lane r and r+16 hold row r); writes the factor back (lower part) and
// the reciprocal pivots to ipd[16].  TWO columns per step: the pivots' reciprocal square roots are the
// longest dependent chain of the whole factorisation (about nine dependent fp64 operations per pivot).  For columns
// j, j+1 with Schur-complement entries p = S_jj, q = S_j+1,j, r = S_j+1,j+1 the second pivot is
// s = r - q^2/p = det/p with det = p r - q^2, so  1/sqrt(s) = rsqrt(det) * sqrt(p):  rsqrt(p) and rsqrt(det)
// are independent and run concurrently -- 11 dependent operations per two pivots instead of 18.  Arithmetic is
// the standard Cholesky recurrence (same stability: s inherits the relative error eps p r / det either way).
__device__ __forceinline__ void warp_potrf16x2(double* D, double* ipd, int* info, int info_val0, int lane)
{
    const unsigned full = 0xffffffffu;
    const int r = lane & 15;
    double a[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) a[k] = D[r * LF_LD + k];
#pragma unroll
    for (int j = 0; j < 16; j += 2) {
        const double p = __shfl_sync(full, a[j], j);
        const double q = __shfl_sync(full, a[j], j + 1);
        const double rr = __shfl_sync(full, a[j + 1], j + 1);
        const double det = fma(p, rr, -(q * q));
        if (lane == 0) {
            if (!(p > 0.0)) atomicCAS(info, 0, info_val0 + j + 1);
            else if (!(det > 0.0)) atomicCAS(info, 0, info_val0 + j + 2);
        }
        double yp = rsqrt_seeded(p), yd = rsqrt_seeded(det);            // independent chains
        double sp = p * yp;
        sp = fma(fma(-sp, sp, p), 0.5 * yp, sp);                         // sqrt(p)
        if (!(p > 0.0)) { sp = sqrt(p); yp = 1.0 / sp; }
        const double c21 = q * yp;                                       // L[j+1][j]
        double ys = yd * sp;                                             // 1 / sqrt(s)
        const double s2 = fma(-c21, c21, rr);                            // s by the standard formula: diagonal entry only (off the chain)
        double ss = s2 * ys;
        ss = fma(fma(-ss, ss, s2), 0.5 * ys, ss);                        // sqrt(s)
        if (!(det > 0.0) || !(p > 0.0)) { ss = sqrt(s2); ys = 1.0 / ss; }
        const double lj = (r == j) ? sp : a[j] * yp;                     // column j
        const double t = fma(-lj, c21, a[j + 1]);
        const double lj1 = (r == j + 1) ? ss : t * ys;                   // column j+1 (row j: above the diagonal, never read)
        a[j] = lj; a[j + 1] = lj1;
        if (lane == 0) { ipd[j] = yp; ipd[j + 1] = ys; }
#pragma unroll
        for (int k = j + 2; k < 16; ++k) {
            const double lkj = __shfl_sync(full, lj, k);
            const double lkj1 = __shfl_sync(full, lj1, k);
            a[k] = fma(-lj1, lkj1, fma(-lj, lkj, a[k]));               // meaningful for r >= k
        }
    }
    __syncwarp();
    if (lane < 16) {
#pragma unroll
        for (int k = 0; k < 16; ++k) if (k <= r) D[r * LF_LD + k] = a[k];
    }
    __syncwarp();
}

// inverse of a factorised 16x16 block (off the critical path): lane r computes column r by forward
// substitution; two partial sums shorten the dependent FMA chain
__device__ __forceinline__ void warp_trtri16(const double* D, const double* ipd, double* Dinv, int lane)
{
    const int r = lane & 15;
    double x[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        double s0 = 0.0, s1 = 0.0;
#pragma unroll
        for (int k = 0; k < i; ++k) {
            const double l = D[i * LF_LD + k];              // broadcast read
            if (k & 1) s1 = fma(l, x[k], s1); else s0 = fma(l, x[k], s0);
        }
        const double ip = ipd[i];
        x[i] = (i < r) ? 0.0 : ((i == r) ? ip : -(s0 + s1) * ip);
        if (lane < 16) Dinv[i * 17 + r] = x[i];
    }
}

#define LEAF_SMEM_DOUBLES (LEAF_N * LF_LD + 8 * 16 * 17 + 8 * 16 + 64 * 68 + 64)
__global__ void __launch_bounds__(256, 1)
leaf_potrf_trtri_kernel(double* __restrict__ A, int lda, long long sA,
                        double* __restrict__ Li, int ldi, long long sLi,
                        int* __restrict__ info, int info_base)
{
    extern __shared__ __align__(16) double S[];                // [128][132]
    double* DinvAll = S + LEAF_N * LF_LD;                      // [8][16][17]
    double* ipdAll = DinvAll + 8 * 16 * 17;                    // [8][16] reciprocal pivots
    double* T1 = ipdAll + 8 * 16;                              // inverse-assembly scratch: npair x sz x (sz+4) <= 64 x 68
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    double* Ab = A + (long long)blockIdx.x * sA;
    double* Lb = Li + (long long)blockIdx.x * sLi;
    LEAF_STAMP(0);
    {   // 128 x 128 block -> shared memory, 16-byte loads, 16 in flight per thread
        double2 v[16];
#pragma unroll
        for (int half = 0; half < 2; ++half) {
#pragma unroll
            for (int q = 0; q < 16; ++q) {
                const int idx = tid + 256 * (q + 16 * half);       // double2 index: row = idx >> 6, col2 = idx & 63
                v[q] = *reinterpret_cast<const double2*>(Ab + (long long)(idx >> 6) * lda + 2 * (idx & 63));
            }
#pragma unroll
            for (int q = 0; q < 16; ++q) {
                const int idx = tid + 256 * (q + 16 * half);
                *reinterpret_cast<double2*>(S + (idx >> 6) * LF_LD + 2 * (idx & 63)) = v[q];
            }
        }
    }
    __syncthreads();
    LEAF_STAMP(1);

    auto panel = [&](int c0, const double* ipd) {
        // rows below the diagonal block: x = a D^-T by forward substitution (x_j = (a_j - sum_{k<j} x_k L_jk)/L_jj)
        const int rr = c0 + LF_NB + tid;
        if (rr < LEAF_N) {
            double* row = S + rr * LF_LD + c0;
            const double* Dk = S + c0 * LF_LD + c0;
            double a[16];
#pragma unroll
            for (int k = 0; k < 16; ++k) a[k] = row[k];
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                a[j] *= ipd[j];
#pragma unroll
                for (int k = j + 1; k < 16; ++k) a[k] = fma(-a[j], Dk[k * LF_LD + j], a[k]);
            }
#pragma unroll
            for (int k = 0; k < 16; ++k) row[k] = a[k];
        }
    };
    auto update_tile = [&](int c0, int ti, int tj) {      // C(8x8 at tile ti,tj of the trailing block) -= P_R P_C^T
        const int R0 = c0 + LF_NB + 8 * ti, C0 = c0 + LF_NB + 8 * tj;
        double* cp = S + (R0 + g) * LF_LD + C0 + 2 * t;
        double acc0 = cp[0], acc1 = cp[1];
        const double* pa = S + (R0 + g) * LF_LD + c0 + t;
        const double* pb = S + (C0 + g) * LF_LD + c0 + t;
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) dmma884(acc0, acc1, -pa[kk * 4], pb[kk * 4]);
        cp[0] = acc0; cp[1] = acc1;
    };
    if (warp == 0) warp_potrf16x2(S, ipdAll, info + blockIdx.x, info_base, lane);
    __syncthreads();
    panel(0, ipdAll);
    __syncthreads();
    LEAF_STAMP(2);
    for (int kb = 0; kb < 7; ++kb) {
        const int c0 = kb * LF_NB, b0 = c0 + LF_NB;
        const int nt8 = (LEAF_N - b0) >> 3;
        // C1: the two 8-wide tile columns of the next block column
        for (int tl = warp; tl < 2 * nt8; tl += 8) {
            const int ti = tl >> 1, tj = tl & 1;
            if (tj <= ti) update_tile(c0, ti, tj);
        }
        __syncthreads();
        if (warp == 0) {
            warp_potrf16x2(S + b0 * LF_LD + b0, ipdAll + (kb + 1) * 16, info + blockIdx.x, info_base + b0, lane);
        } else if (warp == 1) {
            warp_trtri16(S + c0 * LF_LD + c0, ipdAll + kb * 16, DinvAll + kb * 16 * 17, lane);
        } else {
            // C2: tiles 2 <= tj <= ti < nt8 on warps 2..7
            const int m = nt8 - 2;
            const int ntile = m > 0 ? m * (m + 1) / 2 : 0;
            for (int tl = warp - 2; tl < ntile; tl += 6) {
                int ti = (int)((sqrtf(8.0f * (float)tl + 1.0f) - 1.0f) * 0.5f);
                while (ti * (ti + 1) / 2 > tl) --ti;
                while ((ti + 1) * (ti + 2) / 2 <= tl) ++ti;
                const int tj = tl - ti * (ti + 1) / 2;
                update_tile(c0, ti + 2, tj + 2);
            }
        }
        __syncthreads();
        panel(b0, ipdAll + (kb + 1) * 16);
        __syncthreads();
        LEAF_STAMP(3 + kb);
    }
    if (warp == 1) warp_trtri16(S + 112 * LF_LD + 112, ipdAll + 7 * 16, DinvAll + 7 * 16 * 17, lane);
    // L out (exact zeros above the diagonal), 16-byte stores; warp 1 joins after its last 16x16 inverse
    for (int idx = tid; idx < LEAF_N * LEAF_N / 2; idx += 256) {
        const int r = idx >> 6, c = 2 * (idx & 63);
        double2 v = *reinterpret_cast<const double2*>(S + r * LF_LD + c);
        if (c > r) v.x = 0.0;
        if (c + 1 > r) v.y = 0.0;
        *reinterpret_cast<double2*>(Ab + (long long)r * lda + c) = v;
    }
    __syncthreads();
    LEAF_STAMP(10);

    // ---------------- triangular inverse by recursive doubling ----------------
    {
        const int r = tid >> 4, c = tid & 15;               // 16 x 16 threads
        for (int kb = 0; kb < 8; ++kb)                      // exact zeros above the diagonal: DMMA k-ranges read them
            S[(kb * 16 + r) * LF_LD + kb * 16 + c] = (c <= r) ? DinvAll[kb * 16 * 17 + r * 17 + c] : 0.0;
    }
    __syncthreads();
    for (int sz = 16; sz < LEAF_N; sz <<= 1) {
        const int npair = LEAF_N / (2 * sz), t8 = sz >> 3, ldt = sz + 4;
        const int gw = (t8 < 4) ? t8 : 4;                   // tiles per group (same tile row, consecutive tile columns)
        const int ngrp = npair * t8 * (t8 / gw);
        // T1 = B * Ainv   (Ainv lower: k >= j; the group starts at its first column's k)
        for (int gi = warp; gi < ngrp; gi += 8) {
            const int per = t8 * (t8 / gw);
            const int pr = gi / per, rem = gi % per, ti = rem / (t8 / gw), tj0 = (rem % (t8 / gw)) * gw;
            const int p0 = pr * 2 * sz;
            const double* pa = S + (p0 + sz + 8 * ti + g) * LF_LD + p0 + t;            // B rows
            const double* pb = S + (p0 + t) * LF_LD + p0 + 8 * tj0 + g;                // Ainv[k][n]
            double acc[4][2];
#pragma unroll
            for (int q = 0; q < 4; ++q) { acc[q][0] = 0.0; acc[q][1] = 0.0; }
            for (int k0 = 8 * tj0; k0 < sz; k0 += 4) {
                const double av = pa[k0];
#pragma unroll
                for (int q = 0; q < 4; ++q)       // column tile tj0+q only has k >= 8 (tj0+q): above that Ainv is zero by
                    if (q < gw && k0 >= 8 * (tj0 + q))   // structure, but the storage there holds stale values
                        dmma884(acc[q][0], acc[q][1], av, pb[k0 * LF_LD + 8 * q]);
            }
#pragma unroll
            for (int q = 0; q < 4; ++q)
                if (q < gw) {
                    double* tp = T1 + pr * sz * ldt + (8 * ti + g) * ldt + 8 * (tj0 + q) + 2 * t;
                    tp[0] = acc[q][0]; tp[1] = acc[q][1];
                }
        }
        __syncthreads();
        // X = -Cinv * T1  (Cinv lower: k <= i), written over B
        for (int gi = warp; gi < ngrp; gi += 8) {
            const int per = t8 * (t8 / gw);
            const int pr = gi / per, rem = gi % per, ti = rem / (t8 / gw), tj0 = (rem % (t8 / gw)) * gw;
            const int p0 = pr * 2 * sz;
            const double* pa = S + (p0 + sz + 8 * ti + g) * LF_LD + p0 + sz + t;       // Cinv rows
            const double* pb = T1 + pr * sz * ldt + t * ldt + 8 * tj0 + g;             // T1[k][n]
            double acc[4][2];
#pragma unroll
            for (int q = 0; q < 4; ++q) { acc[q][0] = 0.0; acc[q][1] = 0.0; }
            for (int k0 = 0; k0 < 8 * ti + 8; k0 += 4) {
                const double av = -pa[k0];
#pragma unroll
                for (int q = 0; q < 4; ++q)
                    if (q < gw) dmma884(acc[q][0], acc[q][1], av, pb[k0 * ldt + 8 * q]);
            }
#pragma unroll
            for (int q = 0; q < 4; ++q)
                if (q < gw) {
                    double* xp = S + (p0 + sz + 8 * ti + g) * LF_LD + p0 + 8 * (tj0 + q) + 2 * t;
                    xp[0] = acc[q][0]; xp[1] = acc[q][1];
                }
        }
        __syncthreads();
        LEAF_STAMP(sz == 16 ? 11 : (sz == 32 ? 12 : 13));
    }
    for (int idx = tid; idx < LEAF_N * LEAF_N / 2; idx += 256) {
        const int r = idx >> 6, c = 2 * (idx & 63);
        double2 v = *reinterpret_cast<const double2*>(S + r * LF_LD + c);
        if (c > r) v.x = 0.0;
        if (c + 1 > r) v.y = 0.0;
        *reinterpret_cast<double2*>(Lb + (long long)r * ldi + c) = v;
    }
    LEAF_STAMP(14);
}

// batched 2-D copy  dst[b][r][c] = src[b][r][c]   (cols multiple of 2, 16-byte aligned)
__global__ void copy2d_kernel(const double* __restrict__ src, int lds, long long ss,
                              double* __restrict__ dst, int ldd, long long sd, int rows, int cols)
{
    const double* s = src + (long long)blockIdx.z * ss;
    double* d = dst + (long long)blockIdx.z * sd;
    const int c2 = cols >> 1;
    for (int r = blockIdx.y; r < rows; r += gridDim.y)
        for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < c2; c += gridDim.x * blockDim.x)
            reinterpret_cast<double2*>(d + (long long)r * ldd)[c] =
                reinterpret_cast<const double2*>(s + (long long)r * lds)[c];
}

// U = Linv^T for the lower tiles of Linv (32x32 smem transpose), one slab per blockIdx.z (strides sLi, sU); U's strictly
// lower tiles are written as zeros, so U is exactly upper-triangular whatever the slab held before.
__global__ void transpose_lower_kernel(const double* __restrict__ Li, long long sLi, double* __restrict__ U, long long sU,
                                       int ld, int nt32)
{
    __shared__ double tile[32][33];
    const int bi = blockIdx.y, bj = blockIdx.x;
    if (bj > bi) return;
    Li += (long long)blockIdx.z * sLi;
    U += (long long)blockIdx.z * sU;
    const int tx = threadIdx.x, ty = threadIdx.y;   // 32 x 8
    for (int r = ty; r < 32; r += 8) tile[r][tx] = Li[(long long)(bi * 32 + r) * ld + bj * 32 + tx];
    __syncthreads();
    for (int r = ty; r < 32; r += 8) U[(long long)(bj * 32 + r) * ld + bi * 32 + tx] = tile[tx][r];
    if (bj < bi)      // keep U exactly upper-triangular (the buffer doubles as a staging area)
        for (int r = ty; r < 32; r += 8) U[(long long)(bi * 32 + r) * ld + bj * 32 + tx] = 0.0;
}

// w = T * y with T lower-triangular (one warp per row).   a5: alpha = L^-T (L^-1 y)
__global__ void trmv_lower_kernel(const double* __restrict__ T, int ld, long long sT,
                                  const double* __restrict__ y, long long sy,
                                  double* __restrict__ w, long long sw, int n)
{
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= n) return;
    const double* Tr = T + (long long)blockIdx.z * sT + (long long)row * ld;
    const double* yy = y + (long long)blockIdx.z * sy;
    double s = 0.0;
    for (int k = lane; k <= row; k += 32) s = fma(Tr[k], yy[k], s);
    s = warp_sum(s);
    if (lane == 0) w[(long long)blockIdx.z * sw + row] = s;
}

// out = T^T * w with T lower-triangular: out[k] = sum_{i>=k} T[i][k] w[i]; 32 columns per CTA
__global__ void __launch_bounds__(256)
trmv_lower_T_kernel(const double* __restrict__ T, int ld, long long sT,
                    const double* __restrict__ w, long long sw,
                    double* __restrict__ out, long long so, int n)
{
    __shared__ double red[8][33];
    const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
    const int k = blockIdx.x * 32 + lane;
    const double* Tb = T + (long long)blockIdx.z * sT;
    const double* ww = w + (long long)blockIdx.z * sw;
    double s = 0.0;
    for (int i = blockIdx.x * 32 + wp; i < n; i += 8)
        if (i >= k) s = fma(Tb[(long long)i * ld + k], ww[i], s);
    red[wp][lane] = s;
    __syncthreads();
    if (wp == 0) {
        double r = 0.0;
#pragma unroll
        for (int q = 0; q < 8; ++q) r += red[q][lane];
        out[(long long)blockIdx.z * so + k] = r;
    }
}

// out = T^T * w in row chunks of TRT_ROWS: grid (n/32, ceil(n/TRT_ROWS), batch); block (k-block, c)
// sums rows [c*TRT_ROWS, (c+1)*TRT_ROWS) of its 32 columns into P[batch][c][k].  Chunks entirely
// above the diagonal are skipped; the consumer sums chunks c >= k/TRT_ROWS in ascending order
// (deterministic).  The one-block-per-32-columns kernel above needs N/32 >= #SMs*4 to fill the GPU
// at moderate N; this one has N^2/16384 blocks.
#define TRT_ROWS 512
__global__ void __launch_bounds__(256)
trmv_lower_T_part_kernel(const double* __restrict__ T, int ld, long long sT,
                         const double* __restrict__ w, long long sw,
                         double* __restrict__ P, long long sP, int n)
{
    __shared__ double red[8][33];
    const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
    const int k0 = blockIdx.x * 32, c = blockIdx.y;
    const int r1 = min(n, (c + 1) * TRT_ROWS);
    if (r1 <= k0) return;
    const int r0 = max(c * TRT_ROWS, k0);
    const int k = k0 + lane;
    const double* Tb = T + (long long)blockIdx.z * sT;
    const double* ww = w + (long long)blockIdx.z * sw;
    double s = 0.0;
    for (int i = r0 + wp; i < r1; i += 8)
        if (i >= k) s = fma(Tb[(long long)i * ld + k], ww[i], s);
    red[wp][lane] = s;
    __syncthreads();
    if (wp == 0) {
        double r = 0.0;
#pragma unroll
        for (int q = 0; q < 8; ++q) r += red[q][lane];
        P[(long long)blockIdx.z * sP + (long long)c * n + k] = r;
    }
}

// alpha[k] = sum of the row-chunk partials; res[0] = 2 sum_i log L_ii (a4, optimize.py:352), res[1] = y . alpha
__global__ void __launch_bounds__(1024)
alpha_logdet_kernel(const double* __restrict__ P, long long sP, int nch,
                    const double* __restrict__ L, int ld, long long sL,
                    const double* __restrict__ y, long long sy,
                    double* __restrict__ al, long long sal, int n, double* __restrict__ res)
{
    __shared__ double r0[32], r1[32];
    const double* Lb = L + (long long)blockIdx.x * sL;
    const double* Pb = P + (long long)blockIdx.x * sP;
    double s0 = 0.0, s1 = 0.0;
    for (int i = threadIdx.x; i < n; i += 1024) {
        double a = 0.0;
        for (int c = i / TRT_ROWS; c < nch; ++c) a += Pb[(long long)c * n + i];
        al[(long long)blockIdx.x * sal + i] = a;
        s0 += log(fabs(Lb[(long long)i * ld + i]));
        s1 = fma(y[(long long)blockIdx.x * sy + i], a, s1);
    }
    s0 = warp_sum(s0); s1 = warp_sum(s1);
    if ((threadIdx.x & 31) == 0) { r0[threadIdx.x >> 5] = s0; r1[threadIdx.x >> 5] = s1; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0.0, b = 0.0;
        for (int q = 0; q < 32; ++q) { a += r0[q]; b += r1[q]; }
        res[2 * blockIdx.x] = 2.0 * a;
        res[2 * blockIdx.x + 1] = b;
    }
}

// per batch entry: res[0] = sum_i log(L_ii) * 2 (a4, optimize.py:352), res[1] = y . alpha
__global__ void __launch_bounds__(256)
logdet_dot_kernel(const double* __restrict__ L, int ld, long long sL,
                  const double* __restrict__ y, long long sy,
                  const double* __restrict__ al, long long sal, int n, double* __restrict__ res)
{
    __shared__ double r0[8], r1[8];
    const double* Lb = L + (long long)blockIdx.x * sL;
    double s0 = 0.0, s1 = 0.0;
    for (int i = threadIdx.x; i < n; i += 256) {
        s0 += log(fabs(Lb[(long long)i * ld + i]));
        s1 = fma(y[(long long)blockIdx.x * sy + i], al[(long long)blockIdx.x * sal + i], s1);
    }
    s0 = warp_sum(s0); s1 = warp_sum(s1);
    if ((threadIdx.x & 31) == 0) { r0[threadIdx.x >> 5] = s0; r1[threadIdx.x >> 5] = s1; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0.0, b = 0.0;
        for (int q = 0; q < 8; ++q) { a += r0[q]; b += r1[q]; }
        res[2 * blockIdx.x] = 2.0 * a;
        res[2 * blockIdx.x + 1] = b;
    }
}

// ---------------------------------------------------------------------------------------
// a8/a9 stage 1: ks, partial mean and partial Jacobian for every (output, test point).
//   ks_i = covSE(X_i, z)               gp_functions.py:114-117,132
//   mean = ks^T alpha                  gp_functions.py:119-120,135
//   J_d  = sum_i alpha_i ks_i (X_id - z_d)/ell_d^2   (closed form of ca.jacobian, :146-147)
//   KST[a][h][i] (h-major) is the A operand of the v = Linv ks tensor-core product; rows h >= H are zero-filled.
// One CTA = 8 test points x CH training points of one output.  A thread owns ONE test point (lane / 4) and every 32nd
// training point of the chunk (subset 4 warp + lane % 4) for the whole loop, so the mean / Jacobian partial sums stay in
// its registers and are reduced across lanes and warps ONCE per CTA.  (The r2 mid-round kernel looped test points per CTA
// and ran a 13-value warp reduction per test point, several times the instructions per covariance evaluation of this
// shape.)  The chunk of X^T is staged in shared memory pre-scaled by 1/ell
// (dimension-major: staging stores and the broadcast reads are both conflict-free), alpha next to it; a quarter-warp
// reads 4 consecutive training points, a warp stores 8 rows x 32 B of KS^T per step.
// grid (Npad/CH, BM/8, outputs); PMJ[a][h][blk][1 + Nx].
// ---------------------------------------------------------------------------------------
template <int NXP, int CH>
__global__ void __launch_bounds__(256, (NXP <= 12 ? 2 : 1))
ks_tile_kernel(const double* __restrict__ XT, int ldx, int N, int Nx,
               const double* __restrict__ hyp, int hyp_ld,
               const double* __restrict__ alpha, long long sal,
               const double* __restrict__ Z, int H,
               double* __restrict__ KST, int ldk, long long sK,
               double* __restrict__ PMJ, int nblk)
{
    extern __shared__ double sm[];                         // xs[NXP][CH] (x / ell), als[CH]
    __shared__ double red[8][8][NXP + 1];
    __shared__ double ie[NXP], zs[8][NXP], T32s[32], l2sf2_s;
    double* xs = sm;
    double* als = sm + NXP * CH;
    // let the dependent product kernel start launching once every CTA of this grid is resident (it waits
    // for this grid's completion before reading KS^T): hides its launch latency and prologue
    asm volatile("griddepcontrol.launch_dependents;");
    const int a = blockIdx.z, rg = blockIdx.y, blk = blockIdx.x, tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    const int i0 = blk * CH;
    const double* hp = hyp + (long long)a * hyp_ld;
    // every global load of the prologue is issued before the first dependent instruction (in-order issue: a
    // load -> scale -> store loop pays one L2 round trip per iteration)
    constexpr int RP = (CH + 255) / 256;
    double xv[RP][NXP], av[RP];
#pragma unroll
    for (int q = 0; q < RP; ++q) {
        const int rr = tid + 256 * q;
        const bool in = (CH % 256 == 0 || rr < CH) && (i0 + rr < N);
#pragma unroll
        for (int d = 0; d < NXP; ++d) xv[q][d] = (in && d < Nx) ? XT[(long long)d * ldx + i0 + rr] : 0.0;
        av[q] = in ? alpha[(long long)a * sal + i0 + rr] : 0.0;
    }
    if (tid < NXP) ie[tid] = (tid < Nx) ? 1.0 / hp[tid] : 0.0;
    if (tid >= 64 && tid < 80) T32s[tid - 64] = c_exp2_tab[tid - 64];
    else if (tid >= 80 && tid < 96) T32s[tid - 64] = c_exp2_tab2[tid - 80];
    if (tid == 96) l2sf2_s = 2.0 * log2(fabs(hp[Nx]));
    for (int idx = tid; idx < 8 * NXP; idx += 256) {       // Z may live in mapped host memory: one read per CTA
        const int rr = idx / NXP, d = idx - rr * NXP, hh = rg * 8 + rr;
        zs[rr][d] = (hh < H && d < Nx) ? Z[(long long)hh * Nx + d] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < RP; ++q) {
        const int rr = tid + 256 * q;
        if (CH % 256 == 0 || rr < CH) {
#pragma unroll
            for (int d = 0; d < NXP; ++d) xs[d * CH + rr] = xv[q][d] * ie[d];
            als[rr] = av[q];
        }
    }
    const int r = lane >> 2, s = warp * 4 + (lane & 3);
    const int h = rg * 8 + r;
    const bool active = h < H;
    double z[NXP], aj[NXP], am = 0.0;
#pragma unroll
    for (int d = 0; d < NXP; ++d) {
        z[d] = zs[r][d] * ie[d];
        aj[d] = 0.0;
    }
    const double l2sf2 = l2sf2_s;
    __syncthreads();
    double* krow = KST + (long long)a * sK + (long long)h * ldk + i0;
    if (active) {
#pragma unroll 2
        for (int il = s; il < CH; il += 32) {
            double df[NXP], d0 = 0.0, d1 = 0.0;
#pragma unroll
            for (int d = 0; d < NXP; d += 2) {
                df[d] = xs[d * CH + il] - z[d];
                df[d + 1] = xs[(d + 1) * CH + il] - z[d + 1];
                d0 = fma(df[d], df[d], d0);
                d1 = fma(df[d + 1], df[d + 1], d1);
            }
            // sf2 exp(-dist/2) = 2^(log2 sf2 - log2(e)/2 dist) with the two-level table exp2 of the K build (<= 2.75 ulp)
            double te = fma(-0.72134752044448170, d0 + d1, l2sf2);
            te = (te < -1020.0) ? -1020.0 : te;
            double ks = exp2_t2lvl(te, T32s);
            if (i0 + il >= N) ks = 0.0;
            const double w = als[il] * ks;
            am += w;
#pragma unroll
            for (int d = 0; d < NXP; ++d) aj[d] = fma(w, df[d], aj[d]);
            if (i0 + il < ldk) krow[il] = ks;
        }
    } else {
        for (int il = s; il < CH; il += 32)
            if (i0 + il < ldk) krow[il] = 0.0;               // padding rows of the A operand: zeros
    }
    // one reduction per CTA: the 4 subsets of a row inside the warp, then the 8 warps through shared memory
    am += __shfl_xor_sync(0xffffffffu, am, 1);
    am += __shfl_xor_sync(0xffffffffu, am, 2);
#pragma unroll
    for (int d = 0; d < NXP; ++d) {
        aj[d] += __shfl_xor_sync(0xffffffffu, aj[d], 1);
        aj[d] += __shfl_xor_sync(0xffffffffu, aj[d], 2);
    }
    if ((lane & 3) == 0) {
        red[warp][r][0] = am;
#pragma unroll
        for (int d = 0; d < NXP; ++d) red[warp][r][d + 1] = aj[d];
    }
    __syncthreads();
    // 8 (Nx + 1) values: more than the 256 threads at Nx = 32
    for (int idx = tid; idx < 8 * (Nx + 1); idx += 256) {
        const int rr = idx / (Nx + 1), f = idx - rr * (Nx + 1), hh = rg * 8 + rr;
        double sacc = ((red[0][rr][f] + red[1][rr][f]) + (red[2][rr][f] + red[3][rr][f])) +
                      ((red[4][rr][f] + red[5][rr][f]) + (red[6][rr][f] + red[7][rr][f]));
        if (f > 0) sacc *= ie[f - 1];                        // df was scaled by 1/ell: one more 1/ell makes (x - z)/ell^2
        if (hh < H) PMJ[(((long long)a * H + hh) * nblk + blk) * (Nx + 1) + f] = sacc;
    }
}

// ---------------------------------------------------------------------------------------
// a6/a7 analytic NLML gradient, fused with a K rebuild so dK/dtheta is never stored:
//   dNLL/dtheta = 1/2 tr((K^-1 - alpha alpha^T) dK/dtheta)   (R&W eq. 5.9; objective of
//   optimize.py:322-356).  theta = [ell.., sf, sn] are standard deviations (q1):
//   dK/dell_d = Kf (x_id-x_jd)^2/ell_d^3,  dK/dsf = 2 Kf/sf,  dK/dsn = 2 sn I.
//   One CTA per 64x64 lower tile of K^-1; partial sums [tile][Nx+2].  blockIdx.y selects one
//   batch entry: its hyper row, K^-1 slab, alpha and partials at the strides shp, sK, sal, sp.
// ---------------------------------------------------------------------------------------
template <int NXP>
__global__ void __launch_bounds__(256)
nlml_grad_kernel(const double* __restrict__ XT, int ldx, int N, int Nx,
                 const double* __restrict__ hp, long long shp, const double* __restrict__ Kinv, int ld, long long sK,
                 const double* __restrict__ alpha, long long sal, double* __restrict__ partial, long long sp)
{
    hp += blockIdx.y * shp;
    Kinv += blockIdx.y * sK;
    alpha += blockIdx.y * sal;
    partial += blockIdx.y * sp;
    extern __shared__ double sm[];
    double* Xi = sm; double* Xj = sm + Nx * KB_TILE;
    __shared__ double red[8][NXP + 2];
    const int tt = blockIdx.x;
    int bi = (int)((sqrt(8.0 * (double)tt + 1.0) - 1.0) * 0.5);
    while (bi * (bi + 1) / 2 > tt) --bi;
    while ((bi + 1) * (bi + 2) / 2 <= tt) ++bi;
    const int bj = tt - bi * (bi + 1) / 2;
    const int i0 = bi * KB_TILE, j0 = bj * KB_TILE;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    for (int idx = tid; idx < Nx * KB_TILE; idx += 256) {
        const int d = idx / KB_TILE, r = idx % KB_TILE;
        Xi[idx] = XT[(long long)d * ldx + i0 + r];
        Xj[idx] = XT[(long long)d * ldx + j0 + r];
    }
    __syncthreads();
    const double sf2 = hp[Nx] * hp[Nx];
    double g[NXP + 2];
#pragma unroll
    for (int d = 0; d < NXP + 2; ++d) g[d] = 0.0;
    double ie2[NXP];
#pragma unroll
    for (int d = 0; d < NXP; ++d) ie2[d] = (d < Nx) ? 1.0 / (hp[d] * hp[d]) : 0.0;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int row = i0 + ty + 16 * r;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int col = j0 + tx + 16 * c;
            if (row >= N || col >= N || col > row) continue;
            double dist = 0.0, d2[NXP];
#pragma unroll
            for (int d = 0; d < NXP; ++d) {
                d2[d] = 0.0;
                if (d < Nx) {
                    const double df = Xi[d * KB_TILE + ty + 16 * r] - Xj[d * KB_TILE + tx + 16 * c];
                    d2[d] = df * df;
                    dist = fma(d2[d], ie2[d], dist);
                }
            }
            const double kf = sf2 * exp(-0.5 * dist);
            const double w = Kinv[(long long)row * ld + col] - alpha[row] * alpha[col];
            const double mult = (row == col) ? 1.0 : 2.0;
            const double wk = mult * w * kf;
#pragma unroll
            for (int d = 0; d < NXP; ++d) g[d] = fma(wk, d2[d], g[d]);
            g[NXP] += wk;
            if (row == col) g[NXP + 1] += w;
        }
    }
#pragma unroll
    for (int d = 0; d < NXP + 2; ++d) g[d] = warp_sum(g[d]);
    if ((tid & 31) == 0) {
#pragma unroll
        for (int d = 0; d < NXP + 2; ++d) red[tid >> 5][d] = g[d];
    }
    __syncthreads();
    if (tid < Nx + 2) {
        const int src = (tid < Nx) ? tid : (NXP + (tid - Nx));
        double s = 0.0;
        for (int q = 0; q < 8; ++q) s += red[q][src];
        partial[(long long)tt * (Nx + 2) + tid] = s;
    }
}

// deterministic column sums of partial[ntile][m] -> grad[m], with the theta scalings; blockIdx.y selects one batch
// entry (partials at stride sp, hyper row at stride shp, gradient at stride Nx+2)
__global__ void __launch_bounds__(256)
nlml_grad_final_kernel(const double* __restrict__ partial, long long sp, int ntile, int Nx,
                       const double* __restrict__ hp, long long shp, double* __restrict__ grad)
{
    __shared__ double red[8];
    partial += blockIdx.y * sp;
    hp += blockIdx.y * shp;
    grad += blockIdx.y * (Nx + 2);
    const int q = blockIdx.x;
    double s = 0.0;
    for (int t = threadIdx.x; t < ntile; t += 256) s += partial[(long long)t * (Nx + 2) + q];
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double r = 0.0;
        for (int w = 0; w < 8; ++w) r += red[w];
        if (q < Nx) r = 0.5 * r / (hp[q] * hp[q] * hp[q]);
        else if (q == Nx) r = 0.5 * r * 2.0 / hp[Nx];
        else r = 0.5 * r * 2.0 * hp[Nx + 1];
        grad[q] = r;
    }
}

// extract an N x N block out of a padded slab; mode 0 = as is, 1 = lower triangle with
// exact zeros above the diagonal (the stored-model convention, SURVEY 8a-a3),
// 2 = symmetric from the lower triangle
__global__ void extract_kernel(const double* __restrict__ src, int ld, double* __restrict__ dst, int N, int mode)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x, r = blockIdx.y;
    if (c >= N) return;
    double v;
    if (mode == 1) v = (c <= r) ? src[(long long)r * ld + c] : 0.0;
    else if (mode == 2) v = (c <= r) ? src[(long long)r * ld + c] : src[(long long)c * ld + r];
    else v = src[(long long)r * ld + c];
    dst[(long long)r * N + c] = v;
}

// Gram matrix of the solved columns: out[a][h1][h2] = sf2_a - sum_i V[a][h1][i] V[a][h2][i]
// (GP.covar, gp_class.py:380: kss - v.T @ v with the scalar kss).  grid (H, H, outputs).
__global__ void __launch_bounds__(256)
gram_cov_kernel(const double* __restrict__ V, int ldv, long long sV, int n,
                const double* __restrict__ hyp, int hyp_ld, int Nx, int H, double* __restrict__ out)
{
    __shared__ double red[8];
    const int a = blockIdx.z, h1 = blockIdx.y, h2 = blockIdx.x;
    if (h2 > h1) return;                                   // symmetric: lower half computed, both written
    const double* v1 = V + (long long)a * sV + (long long)h1 * ldv;
    const double* v2 = V + (long long)a * sV + (long long)h2 * ldv;
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += 256) s = fma(v1[i], v2[i], s);
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double r = 0.0;
        for (int q = 0; q < 8; ++q) r += red[q];
        const double sf = hyp[(long long)a * hyp_ld + Nx];
        const double c = sf * sf - r;
        out[((long long)a * H + h1) * H + h2] = c;
        out[((long long)a * H + h2) * H + h1] = c;
    }
}

// ---------------------------------------------------------------------------------------
// 'EM' exact moment matching  (gp_exact_moment, gp_functions.py:344-418), one test point
// per launch set.  Host prepares the Nx x Nx quantities (gpmpc.cu, em_prepare_point):
//   per output a :  iR_a = (Sigma + Lambda_a)^-1 ,  c_a = sf2_a prod(ell_a) / sqrt(det(Sigma+Lambda_a))
//   per pair a>=b:  Qm = (Sigma (iL_a+iL_b) + I)^-1 Sigma/2 ,  t_ab = det(...)^-1/2
// EMP layout (doubles): [a: iR (Nx*Nx), c, G_a (Nx*Nx), lc_a] * Ny, then [pair: Qm (Nx*Nx), t, a, b, const_ab] * npairs
// A launch set covers a chunk of points: every buffer below holds one slice per point at the strides of EmStrides, and the
// point is blockIdx.z (em_pair_kernel's pair sums: blockIdx.z / npairs; em_trdot_kernel: blockIdx.y; em_finalize_kernel:
// blockIdx.x).  A point's arithmetic does not depend on its slot, so its bits do not depend on the chunk.
// ---------------------------------------------------------------------------------------
struct EmStrides {
    long long z, emp;           // test point (Nx), em_prepare_point block
    long long mpart, pair, w;   // mean partials (Ny nblk); E, F, E2, F2 (npairs ldn each); W, IJ (npairs Nx ldn each)
    long long lq, part, q;      // log q (Ny ldn); pair-sum partials (npairs T T); Q~ and L^-1 Q~ slabs (ld^2)
    long long tr, vec;          // trace partials (Ny ntr); [qv (ldn) | L^-1 qv (ldn) | |L^-1 qv|^2 (Ny)]
};

template <int NXP>
__global__ void __launch_bounds__(256)
em_prep_kernel(const double* __restrict__ XT, int ldx, int N, int Nx, int Ny, int npairs,
               const double* __restrict__ hyp, int hyp_ld, const double* __restrict__ alpha, long long sal,
               const double* __restrict__ z, const double* __restrict__ EMP,
               double* __restrict__ meanPart, int nblk,
               double* __restrict__ E, double* __restrict__ F, double* __restrict__ W, double* __restrict__ IJ, int ldn,
               double* __restrict__ LQ, double* __restrict__ E2, double* __restrict__ F2, EmStrides s)
{
    __shared__ double M[NXP * NXP], Ga[NXP * NXP], Gb[NXP * NXP];
    __shared__ double red[8];
    const int role = blockIdx.y, tid = threadIdx.x;
    const long long pt = blockIdx.z;
    z += pt * s.z; EMP += pt * s.emp; meanPart += pt * s.mpart;
    E += pt * s.pair; F += pt * s.pair; E2 += pt * s.pair; F2 += pt * s.pair;
    W += pt * s.w; IJ += pt * s.w; LQ += pt * s.lq;
    const int i = blockIdx.x * 256 + tid;
    const int nn = Nx * Nx;
    double v[NXP];
#pragma unroll
    for (int d = 0; d < NXP; ++d) v[d] = (d < Nx && i < N) ? XT[(long long)d * ldx + i] - z[d] : 0.0;
    if (role < Ny) {                                        // mean of output a (:381-388)
        const int a = role;
        const double* P = EMP + (long long)a * (2 * nn + 2);
        for (int q = tid; q < nn; q += 256) M[q] = P[q];
        __syncthreads();
        double quad = 0.0;
#pragma unroll
        for (int d = 0; d < NXP; ++d) {
            if (d < Nx) {
                double tacc = 0.0;
#pragma unroll
                for (int e = 0; e < NXP; ++e) if (e < Nx) tacc = fma(M[d * Nx + e], v[e], tacc);
                quad = fma(v[d], tacc, quad);
            }
        }
        // log q_i = log c_a - 1/2 v^T (Sigma+Lambda_a)^-1 v: kept so the pair sums can form
        // t Q_ij - q_i q_j = q_i q_j expm1(.) without cancellation (em_pair_kernel)
        if (i < ldn) LQ[(long long)a * ldn + i] = (i < N) ? log(P[nn]) - 0.5 * quad : 0.0;
        double q = (i < N) ? P[nn] * exp(-0.5 * quad) * alpha[(long long)a * sal + i] : 0.0;
        q = warp_sum(q);
        if ((tid & 31) == 0) red[tid >> 5] = q;
        __syncthreads();
        if (tid == 0) {
            double r = 0.0;
            for (int w = 0; w < 8; ++w) r += red[w];
            meanPart[(long long)a * nblk + blockIdx.x] = r;
        }
        return;
    }
    const int p = role - Ny;
    const double* P = EMP + (long long)Ny * (2 * nn + 2) + (long long)p * (nn + 4);
    const int a = (int)P[nn + 1], b = (int)P[nn + 2];
    for (int q = tid; q < nn; q += 256) {
        M[q] = P[q];
        Ga[q] = EMP[(long long)a * (2 * nn + 2) + nn + 1 + q];      // G_a = Lambda_a^-1 Sigma (Sigma + Lambda_a)^-1
        Gb[q] = EMP[(long long)b * (2 * nn + 2) + nn + 1 + q];
    }
    __syncthreads();
    if (i >= ldn) return;
    const double* ha = hyp + (long long)a * hyp_ld;
    const double* hb = hyp + (long long)b * hyp_ld;
    double lka = 2.0 * log(ha[Nx]), lkb = 2.0 * log(hb[Nx]);      // log_k (:389-391)
    double ii[NXP], ij[NXP];
#pragma unroll
    for (int d = 0; d < NXP; ++d) {
        ii[d] = 0.0; ij[d] = 0.0;
        if (d < Nx) {
            const double sa = v[d] / ha[d], sb = v[d] / hb[d];
            lka = fma(-0.5 * sa, sa, lka); lkb = fma(-0.5 * sb, sb, lkb);
            ii[d] = v[d] / (ha[d] * ha[d]); ij[d] = v[d] / (hb[d] * hb[d]);
        }
    }
    // e2 / f2: the SMALL parts only, for the cancellation-free pair sums:
    //   log(t Q_ij) - log q_i - log q_j = const_ab + e2_i + f2_j + 2 ii^T M ij,
    //   e2_i = ii^T M ii - 1/2 v^T G_a v   (log k_a(x_i) - log q^a_i = const - 1/2 v^T G_a v by Woodbury)
    double e2 = 0.0, f2 = 0.0;
#pragma unroll
    for (int e = 0; e < NXP; ++e) {
        if (e < Nx) {
            double wi = 0.0, wj = 0.0, ga = 0.0, gb = 0.0;
#pragma unroll
            for (int d = 0; d < NXP; ++d)
                if (d < Nx) {
                    wi = fma(ii[d], M[d * Nx + e], wi); wj = fma(ij[d], M[d * Nx + e], wj);
                    ga = fma(v[d], Ga[d * Nx + e], ga); gb = fma(v[d], Gb[d * Nx + e], gb);
                }
            e2 = fma(wi, ii[e], e2); f2 = fma(wj, ij[e], f2);
            e2 = fma(-0.5 * ga, v[e], e2); f2 = fma(-0.5 * gb, v[e], f2);
            W[((long long)p * Nx + e) * ldn + i] = wi;
            IJ[((long long)p * Nx + e) * ldn + i] = ij[e];
        }
    }
    // E / F (with the big log k terms) serve the Q matrix of the trace term only
    double ei = lka, fj = lkb;
#pragma unroll
    for (int e = 0; e < NXP; ++e)
        if (e < Nx) {
            double wi = 0.0, wj = 0.0;
#pragma unroll
            for (int d = 0; d < NXP; ++d) if (d < Nx) { wi = fma(ii[d], M[d * Nx + e], wi); wj = fma(ij[d], M[d * Nx + e], wj); }
            ei = fma(wi, ii[e], ei); fj = fma(wj, ij[e], fj);
        }
    E[(long long)p * ldn + i] = ei;
    F[(long long)p * ldn + i] = fj;
    E2[(long long)p * ldn + i] = (i < N) ? e2 : 0.0;
    F2[(long long)p * ldn + i] = (i < N) ? f2 : 0.0;
}

// The 64x64 tiles of the 'EM' pair sums (em_pair_kernel, em_pair_rec_kernel), 4x4 per thread: acc[r][c] = sum_d
// Ws[d][ty + 16 r] Js[d][tx + 16 c] over the staged W rows of the i block and IJ rows of the j block (stride 64).
__device__ __forceinline__ void em_tile(const double* Ws, const double* Js, int Nx, int tx, int ty, double (&acc)[4][4])
{
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] = 0.0;
    for (int d = 0; d < Nx; ++d) {
        double wv[4], jv[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) wv[r] = Ws[d * 64 + ty + 16 * r];
#pragma unroll
        for (int c = 0; c < 4; ++c) jv[c] = Js[d * 64 + tx + 16 * c];
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[r][c] = fma(wv[r], jv[c], acc[r][c]);
    }
}

// The cross term of pair p = (a, b) at (i, j) without cancellation: beta_i beta_j (t Q_ij - q_i q_j) =
// w_ij expm1(x_ij) with w_ij = (beta_i q_i)(beta_j q_j) and x_ij = log t + log Q_ij - log q_i - log q_j -- the
// reference's  t beta^T Q beta - mean_a mean_b  (:412,416) term by term, before the sums cancel.  The exponent is
// assembled from its small parts only (never as a difference of O(10) logarithms).
__device__ __forceinline__ double em_cross_w(const double* __restrict__ alpha, long long sal, const double* __restrict__ LQ,
                                             int ldn, int a, int b, int i, int j)
{
    const double la = LQ[(long long)a * ldn + i], lb = LQ[(long long)b * ldn + j];
    return (alpha[(long long)a * sal + i] * exp(la)) * (alpha[(long long)b * sal + j] * exp(lb));
}
__device__ __forceinline__ double em_cross_x(double cab, const double* __restrict__ E2, const double* __restrict__ F2,
                                             int ldn, int p, int i, int j, double acc)
{
    return cab + E2[(long long)p * ldn + i] + F2[(long long)p * ldn + j] + 2.0 * acc;
}

// The part of Q_aa (pair p = (a, a)) beyond its rank-one backbone: Q_ij = e^{E_i} e^{F_j} (1 + expm1(2 acc_ij))
__device__ __forceinline__ double em_rem(const double* __restrict__ E, const double* __restrict__ F, int ldn, int p,
                                         int i, int j, double acc)
{
    return exp(E[(long long)p * ldn + i] + F[(long long)p * ldn + j]) * expm1(2.0 * acc);
}

// sum_ij beta_a,i beta_b,j (t Q_ij - q_i q_j) for one pair; 64x64 tile per CTA, 4x4 per thread (:394-416).
// The reference subtracts invK from beta beta^T on the diagonal pairs before the sum (:410-411),
// which cancels 6-8 digits at cond(K) ~ 1e8-1e10 (negative variances on the car fixture, SURVEY
// q18).  Here that term is evaluated separately and stably as tr(L^-1 Q L^-T) (em_q_kernel +
// DMMA product + em_trdot_kernel): a trace of a positive semi-definite matrix, formed from the
// Cholesky factor like var = sf2 - |L^-1 ks|^2 -- no explicit K^-1 anywhere.
// mode 0: partial sums of beta_i beta_j q_ij into `part`; mode 1: q_ij itself into Qout (ld ldq,
// zero outside N) for the pair's output a == b.
__global__ void __launch_bounds__(256)
em_pair_kernel(int N, int Nx, int Ny, const double* __restrict__ EMP,
               const double* __restrict__ alpha, long long sal,
               const double* __restrict__ E, const double* __restrict__ F, const double* __restrict__ W,
               const double* __restrict__ IJ, int ldn, const double* __restrict__ LQ,
               const double* __restrict__ E2, const double* __restrict__ F2, double* __restrict__ part,
               int mode, int pair_q, double* __restrict__ Qout, int ldq, EmStrides st)
{
    extern __shared__ double sm[];
    double* Ws = sm; double* Js = sm + Nx * 64;
    __shared__ double red[8];
    const int npairs = Ny * (Ny + 1) / 2;
    const long long pt = mode ? blockIdx.z : blockIdx.z / npairs;
    const int p = mode ? pair_q : blockIdx.z - (int)pt * npairs, nn = Nx * Nx;
    EMP += pt * st.emp; LQ += pt * st.lq;
    E += pt * st.pair; F += pt * st.pair; E2 += pt * st.pair; F2 += pt * st.pair;
    W += pt * st.w; IJ += pt * st.w;
    if (mode) Qout += pt * st.q; else part += pt * st.part;
    const double* P = EMP + (long long)Ny * (2 * nn + 2) + (long long)p * (nn + 4);
    const int a = (int)P[nn + 1], b = (int)P[nn + 2];
    const double cab = P[nn + 3];       // log t + (log sf2_a - log c_a) + (log sf2_b - log c_b), from determinants of I + small
    const int i0 = blockIdx.y * 64, j0 = blockIdx.x * 64;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    for (int idx = tid; idx < Nx * 64; idx += 256) {
        const int d = idx >> 6, r = idx & 63;
        Ws[idx] = (i0 + r < ldn) ? W[((long long)p * Nx + d) * ldn + i0 + r] : 0.0;
        Js[idx] = (j0 + r < ldn) ? IJ[((long long)p * Nx + d) * ldn + j0 + r] : 0.0;
    }
    __syncthreads();
    double acc[4][4];
    em_tile(Ws, Js, Nx, tx, ty, acc);
    double s = 0.0;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int i = i0 + ty + 16 * r;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int j = j0 + tx + 16 * c;
            // mode 1 stores only the part of Q beyond its rank-one backbone (em_rem); the backbone's trace term |L^-1 e^E|^2 is formed like the ME variance (em_qvec_kernel + trmv), which keeps
            // EM -> ME exact to ~1e-11 as Sigma -> 0 instead of amplifying the full Q through L^-1 twice
            if (mode) { if (i < ldq && j < ldq) Qout[(long long)i * ldq + j] = (i < N && j < N) ? em_rem(E, F, ldn, p, i, j, acc[r][c]) : 0.0; }
            else if (i < N && j < N)
                s = fma(em_cross_w(alpha, sal, LQ, ldn, a, b, i, j), expm1(em_cross_x(cab, E2, F2, ldn, p, i, j, acc[r][c])), s);
        }
    }
    if (mode) return;
    s = warp_sum(s);
    if ((tid & 31) == 0) red[tid >> 5] = s;
    __syncthreads();
    if (tid == 0) {
        double r = 0.0;
        for (int w = 0; w < 8; ++w) r += red[w];
        part[((long long)p * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x] = r;
    }
}

// rank-one backbone of Q_aa: qv_i = exp(E_i) (i < N, else 0); point blockIdx.z
__global__ void em_qvec_kernel(const double* __restrict__ E, int N, int n, double* __restrict__ qv, EmStrides s)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    E += blockIdx.z * s.pair; qv += blockIdx.z * s.vec;
    if (i < n) qv[i] = (i < N) ? exp(E[i]) : 0.0;
}

// out[0] = sum_i v_i^2 (one block per vector, fixed order): vector blockIdx.x at v + blockIdx.x sv, its sum at out + blockIdx.x so
__global__ void __launch_bounds__(256)
sumsq_kernel(const double* __restrict__ v, long long sv, int n, double* __restrict__ out, long long so)
{
    __shared__ double red[8];
    v += blockIdx.x * sv; out += blockIdx.x * so;
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += 256) s = fma(v[i], v[i], s);
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double r = 0.0;
        for (int w = 0; w < 8; ++w) r += red[w];
        out[0] = r;
    }
}

// tr(L^-1 Q L^-T) = sum_{k >= j} Wm[k][j] Li[k][j] with Wm = L^-1 Q (lower tiles): block partial sums,
// grid (n/64 * (n/64+1)/2) lower 64x64 tiles, point blockIdx.y (Wm and part at its slices; Li shared)
__global__ void __launch_bounds__(256)
em_trdot_kernel(const double* __restrict__ Wm, const double* __restrict__ Li, int ld, double* __restrict__ part, EmStrides st)
{
    __shared__ double red[8];
    const int tt = blockIdx.x;
    Wm += blockIdx.y * st.q; part += blockIdx.y * st.tr;
    int bi = (int)((sqrt(8.0 * (double)tt + 1.0) - 1.0) * 0.5);
    while (bi * (bi + 1) / 2 > tt) --bi;
    while ((bi + 1) * (bi + 2) / 2 <= tt) ++bi;
    const int bj = tt - bi * (bi + 1) / 2;
    const int tid = threadIdx.x, tx = tid & 63, ty = tid >> 6;
    double s = 0.0;
    for (int r = ty; r < 64; r += 4) {
        const int row = bi * 64 + r, col = bj * 64 + tx;
        if (col <= row) s = fma(Wm[(long long)row * ld + col], Li[(long long)row * ld + col], s);
    }
    s = warp_sum(s);
    if ((tid & 31) == 0) red[tid >> 5] = s;
    __syncthreads();
    if (tid == 0) {
        double r = 0.0;
        for (int w = 0; w < 8; ++w) r += red[w];
        part[tt] = r;
    }
}

// mean (Ny), cov (Ny,Ny): t_ab * sum (+ sf2 on the diagonal) - mean mean^T   (:412-416)
__global__ void em_finalize_kernel(int Nx, int Ny, int npairs, const double* __restrict__ EMP,
                                   const double* __restrict__ hyp, int hyp_ld,
                                   const double* __restrict__ meanPart, int nblk,
                                   const double* __restrict__ part, int ntile2,
                                   const double* __restrict__ trPart, int ntr, const double* __restrict__ trVec,
                                   double* __restrict__ mean, double* __restrict__ var, double* __restrict__ cov, EmStrides st)
{
    const int tid = threadIdx.x, nn = Nx * Nx;
    const long long pt = blockIdx.x;     // one CTA per point; mean / var / cov at strides Ny / Ny / Ny^2
    EMP += pt * st.emp; meanPart += pt * st.mpart; part += pt * st.part; trPart += pt * st.tr; trVec += pt * st.vec;
    if (mean) mean += pt * Ny;
    if (var) var += pt * Ny;
    if (cov) cov += pt * Ny * Ny;
    if (tid < Ny && mean) {
        double s = 0.0;
        for (int b = 0; b < nblk; ++b) s += meanPart[(long long)tid * nblk + b];
        mean[tid] = s;
    }
    if (tid < npairs) {
        const double* P = EMP + (long long)Ny * (2 * nn + 2) + (long long)tid * (nn + 4);
        const int a = (int)P[nn + 1], b = (int)P[nn + 2];
        double s = 0.0;
        for (int q = 0; q < ntile2; ++q) s += part[(long long)tid * ntile2 + q];
        double c = s;       // = t beta_a^T Q beta_b - mean_a mean_b, summed term by term without the cancellation
        if (a == b) {
            // + expected variance  sf2 - t tr(K^-1 Q_aa)  from the Cholesky-based trace (two positive numbers)
            double tr = trVec[a];                                 // |L^-1 e^E|^2: the rank-one backbone
            for (int q = 0; q < ntr; ++q) tr += trPart[(long long)a * ntr + q];
            const double sf = hyp[(long long)a * hyp_ld + Nx];
            c += sf * sf - P[nn] * tr;
        }
        if (cov) { cov[a * Ny + b] = c; cov[b * Ny + a] = c; }
        if (a == b && var) var[a] = c;
    }
}

// out[rec][q] = sum over the nb block partials of rec, in block order
__global__ void em_sum_parts_kernel(const double* __restrict__ part, int nb, int RL, double* __restrict__ out)
{
    const long long rec = blockIdx.x;
    for (int q = threadIdx.x; q < RL; q += blockDim.x) {
        double s = 0.0;
        for (int b = 0; b < nb; ++b) s += part[(rec * nb + b) * RL + q];
        out[rec * RL + q] = s;
    }
}

// ---------------------------------------------------------------------------------------
// 'EM' derivative records (gpmpc_predict_em_grad: D = 2, gpmpc_predict_em_hess: D = 4).  Every O(N) / O(N^2) sum ends in
// a record over a weight m and v_k = x_k - z: per owner index k, features F_k,f over the other index (f runs over the
// unique monomials of degree <= D/2 of the other index's v: 1, v_d, and for D = 4 v_d v_e with d <= e), and the entries
//   sum_k mono_mo(v_k) F_k,f   for every unique owner monomial mo of degree <= D with deg mo + deg f <= D.
// Monomials are numbered by degree, then lexicographically over sorted index tuples; MONO[4 m + s] holds monomial m's
// indices (-1 past its degree), ENT[2 q], ENT[2 q + 1] record entry q's (mo, f).  Both tables come from the host
// (gpmpc.cu, EmTables).  One partial per 64-index owner block, summed by em_sum_parts_kernel.
// ---------------------------------------------------------------------------------------
// monomials of degree <= k (k <= 2) in n variables: the feature count of a record of total degree 2k
__host__ __device__ constexpr int em_nmono(int n, int k) { return k <= 0 ? 1 : (k == 1 ? 1 + n : 1 + n + n * (n + 1) / 2); }

__device__ __forceinline__ double em_mono(const int* __restrict__ MONO, int m, const double* __restrict__ V, int k)
{
    double r = 1.0;
#pragma unroll
    for (int s = 0; s < 4; ++s) {
        const int d = MONO[4 * m + s];
        if (d >= 0) r *= V[d * 64 + k];
    }
    return r;
}

// record entries of one owner block: Vown [Nx][64], Fown [64][ldf] (features f < nf; entries with f >= nf are zero)
__device__ __forceinline__ void em_record(const double* __restrict__ Vown, const double* __restrict__ Fown, int ldf, int nf,
                                          const int* __restrict__ MONO, const int* __restrict__ ENT, int nent,
                                          double* __restrict__ out)
{
    for (int q = threadIdx.x; q < nent; q += blockDim.x) {
        const int mo = ENT[2 * q], f = ENT[2 * q + 1];
        const int d0 = MONO[4 * mo], d1 = MONO[4 * mo + 1], d2 = MONO[4 * mo + 2], d3 = MONO[4 * mo + 3];
        double s = 0.0;
        if (f < nf)
            for (int k = 0; k < 64; ++k) {
                double r = Fown[k * ldf + f];
                if (d0 >= 0) r *= Vown[d0 * 64 + k];
                if (d1 >= 0) r *= Vown[d1 * 64 + k];
                if (d2 >= 0) r *= Vown[d2 * 64 + k];
                if (d3 >= 0) r *= Vown[d3 * 64 + k];
                s += r;
            }
        out[q] = s;
    }
}

// Owner records with per-owner features: F_k,f = x1_k exp(x2_k) Fc[f][k] (null x1 / Fc count as 1, nf = 1 without Fc),
// v_k = V[d][k] - z[d] (null z counts as 0), k < n.  One 64-index block per CTA (blockIdx.x), one record per blockIdx.y
// (x1, x2 offset by sx, Fc by sfc, record by srec).  Serves the mean records (x1 = alpha_a, x2 = log q_a), the trace
// backbone (x2 = E, Fc = K^-1 e for D = 2, K^-1 (e o features) for D = 4) and the backbone Gram (V = L^-1 rows, z null).
template <int NXP, int D>
__global__ void __launch_bounds__(256)
em_owner_rec_kernel(const double* __restrict__ V, int ldv, int n, int Nx, const double* __restrict__ z,
                    const double* __restrict__ x1, const double* __restrict__ x2, long long sx,
                    const double* __restrict__ Fc, long long sfc, int ldfc, int nf,
                    const int* __restrict__ MONO, const int* __restrict__ ENT, int nent,
                    double* __restrict__ part, long long srec)
{
    constexpr int NFP = em_nmono(NXP, D / 2);
    extern __shared__ double sm[];
    double* Vown = sm;                     // [NXP][64]
    double* Fown = Vown + NXP * 64;        // [64][NFP]
    const int tid = threadIdx.x, k0 = blockIdx.x * 64;
    if (x1) x1 += blockIdx.y * sx;
    if (x2) x2 += blockIdx.y * sx;
    if (Fc) Fc += blockIdx.y * sfc;
    for (int idx = tid; idx < NXP * 64; idx += 256) {
        const int d = idx >> 6, k = k0 + (idx & 63);
        Vown[idx] = (d < Nx && k < n) ? V[(long long)d * ldv + k] - (z ? z[d] : 0.0) : 0.0;
    }
    for (int idx = tid; idx < 64 * nf; idx += 256) {
        const int kl = idx / nf, f = idx % nf, k = k0 + kl;
        double w = 0.0;
        if (k < n) w = (x1 ? x1[k] : 1.0) * (x2 ? exp(x2[k]) : 1.0) * (Fc ? Fc[(long long)f * ldfc + k] : 1.0);
        Fown[kl * NFP + f] = w;
    }
    __syncthreads();
    em_record(Vown, Fown, NFP, nf, MONO, ENT, nent, part + blockIdx.y * srec + (long long)blockIdx.x * nent);
}

// Pair sums of one 64-index owner block (blockIdx.x) against every other block, the 64x64 tiles recomputed as
// em_pair_kernel does (no N x N array is written):
//   mode 0, pair p = blockIdx.y, orientation o = blockIdx.z: the cross term's m_ij = w_ij expm1(x_ij) (em_cross_w,
//     em_cross_x); owner = rows i (o = 0) or columns j (o = 1); record rec0 + 2p + o.
//   mode 1, output a = blockIdx.y (pair (a,a)): m_ij = K^-1_ij Qt_ij with Qt the O(Sigma) remainder of Q_aa (em_rem);
//     Kinv = full symmetric K^-1 per output (stride ldn^2); owner rows; record rec0 + a.
// The owner's feature sums over the other index, F_k,f = sum m mono_f(v_other), stay in registers across the tiles
// (fixed order); the record then sums over the owner block in index order.
template <int NXP, int D>
__global__ void __launch_bounds__(256)
em_pair_rec_kernel(int N, int Nx, int Ny, const double* __restrict__ EMP,
                   const double* __restrict__ alpha, long long sal,
                   const double* __restrict__ XT, int ldx, const double* __restrict__ z,
                   const double* __restrict__ E, const double* __restrict__ F, const double* __restrict__ W,
                   const double* __restrict__ IJ, int ldn, const double* __restrict__ LQ,
                   const double* __restrict__ E2, const double* __restrict__ F2,
                   const double* __restrict__ Kinv, int mode, int rec0,
                   const int* __restrict__ MONO, const int* __restrict__ ENT, int nent, double* __restrict__ part, int nb)
{
    constexpr int NFP = em_nmono(NXP, D / 2);
    constexpr int KF = (NFP + 3) / 4;                 // features per thread: f = g + 4q
    extern __shared__ double sm[];
    double* Wo = sm;                                  // [NXP][64] W rows of the i block
    double* Jo = Wo + NXP * 64;                       // [NXP][64] IJ rows of the j block
    double* Vown = Jo + NXP * 64;                     // [NXP][64] v of the owner block
    double* Ms = Vown + NXP * 64;                     // [64][65] m tile, owner-major
    double* Foth = Ms + 64 * 65;                      // [NFP][64] features of the other block; then [64][NFP] of the owner
    double* Voth = Foth + 64;                         // v of the other block: feature rows 1..Nx, behind the row of ones
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int o = mode ? 0 : blockIdx.z;
    // column owners (o = 1) serve only the entries of owner degree > D/2, whose features have degree < D/2
    const int nn = Nx * Nx, nf = em_nmono(Nx, o ? D / 2 - 1 : D / 2);
    const int p = mode ? blockIdx.y * (blockIdx.y + 1) / 2 + blockIdx.y : blockIdx.y;
    const double* P = EMP + (long long)Ny * (2 * nn + 2) + (long long)p * (nn + 4);
    const int a = (int)P[nn + 1], b = (int)P[nn + 2];
    const double cab = P[nn + 3];
    const double* Ka = mode ? Kinv + (long long)a * ldn * ldn : nullptr;
    const int own0 = blockIdx.x * 64, T = (N + 63) / 64;
    for (int idx = tid; idx < NXP * 64; idx += 256) {
        const int d = idx >> 6, k = own0 + (idx & 63);
        const bool ok = d < Nx && k < N;
        Vown[idx] = ok ? XT[(long long)d * ldx + k] - z[d] : 0.0;
        if (o == 0) Wo[idx] = ok ? W[((long long)p * Nx + d) * ldn + k] : 0.0;
        else Jo[idx] = ok ? IJ[((long long)p * Nx + d) * ldn + k] : 0.0;
    }
    if (tid < 64) Foth[tid] = 1.0;
    const int ko = tid & 63, g = tid >> 6;
    double acc2[KF];
#pragma unroll
    for (int q = 0; q < KF; ++q) acc2[q] = 0.0;
    for (int t = 0; t < T; ++t) {
        const int oth0 = t * 64;
        __syncthreads();                              // previous tile's readers are done
        for (int idx = tid; idx < Nx * 64; idx += 256) {
            const int d = idx >> 6, k = oth0 + (idx & 63);
            const bool ok = k < N;
            Voth[idx] = ok ? XT[(long long)d * ldx + k] - z[d] : 0.0;
            if (o == 0) Jo[idx] = ok ? IJ[((long long)p * Nx + d) * ldn + k] : 0.0;
            else Wo[idx] = ok ? W[((long long)p * Nx + d) * ldn + k] : 0.0;
        }
        __syncthreads();
        for (int idx = (1 + Nx) * 64 + tid; idx < nf * 64; idx += 256) Foth[idx] = em_mono(MONO, idx >> 6, Voth, idx & 63);
        const int i0 = o ? oth0 : own0, j0 = o ? own0 : oth0;
        double acc[4][4];
        em_tile(Wo, Jo, Nx, tx, ty, acc);
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int il = ty + 16 * r, i = i0 + il;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const int jl = tx + 16 * c, j = j0 + jl;
                double m = 0.0;
                if (i < N && j < N)
                    m = mode ? Ka[(long long)i * ldn + j] * em_rem(E, F, ldn, p, i, j, acc[r][c])
                             : em_cross_w(alpha, sal, LQ, ldn, a, b, i, j) * expm1(em_cross_x(cab, E2, F2, ldn, p, i, j, acc[r][c]));
                if (o == 0) Ms[il * 65 + jl] = m; else Ms[jl * 65 + il] = m;
            }
        }
        __syncthreads();
        for (int x = 0; x < 64; ++x) {
            const double mv = Ms[ko * 65 + x];
#pragma unroll
            for (int q = 0; q < KF; ++q) {
                const int f = g + 4 * q;
                if (f < nf) acc2[q] = fma(mv, Foth[f * 64 + x], acc2[q]);
            }
        }
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < KF; ++q) {
        const int f = g + 4 * q;
        if (f < nf) Foth[ko * NFP + f] = acc2[q];     // owner-major: F_k,f
    }
    __syncthreads();
    const int rec = rec0 + (mode ? (int)blockIdx.y : 2 * p + o);
    em_record(Vown, Foth, NFP, nf, MONO, ENT, nent, part + ((long long)rec * nb + blockIdx.x) * nent);
}

// ---------------------------------------------------------------------------------------
// 'EM' second derivatives from the records (gpmpc_predict_em_hess, DESIGN 4.8).  Dense symmetric tensors of order k <= 4
// over Nx (row-major), a "family" holds orders 0..4 back to back (offsets emh_off, total emh_off(5)).  The z-derivatives
// of a Gaussian term are Hermite polynomials He_k(y; S): He_2 = y y - S, He_3 = y y y - (3 placements of S y),
// He_4 = y^4 - (6 placements of S y y) + (3 pairings of S S); MID (family layout) maps an index tuple to its monomial,
// ENTPOS[m * nf + f] a (monomial, feature) pair to its record entry.  Every step is block-cooperative (ends synchronised).
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ int emh_pow(int Nx, int k) { int r = 1; for (int q = 0; q < k; ++q) r *= Nx; return r; }
__device__ __forceinline__ int emh_off(int Nx, int k) { int s = 0, r = 1; for (int q = 0; q < k; ++q) { s += r; r *= Nx; } return s; }
__device__ __forceinline__ void emh_digits(int f, int Nx, int k, int* d) { for (int q = k - 1; q >= 0; --q) { d[q] = f % Nx; f /= Nx; } }
__device__ __forceinline__ int emh_sorted(const int* d, int k, int Nx)
{
    // a sorting network on four registers, the missing indices above every real one
    int a0 = d[0], a1 = k > 1 ? d[1] : 1 << 30, a2 = k > 2 ? d[2] : 1 << 30, a3 = k > 3 ? d[3] : 1 << 30;
#define EMH_CS(x, y) { const int lo_ = min(x, y), hi_ = max(x, y); x = lo_; y = hi_; }
    EMH_CS(a0, a1) EMH_CS(a2, a3) EMH_CS(a0, a2) EMH_CS(a1, a3) EMH_CS(a1, a2)
#undef EMH_CS
    int f = a0;
    if (k > 1) f = f * Nx + a1;
    if (k > 2) f = f * Nx + a2;
    if (k > 3) f = f * Nx + a3;
    return f;
}

// dst = (M_0 x ... x M_{k-1}) src (matrix M_s on axis s); tmp: scratch of Nx^k; src aliases neither
__device__ void emh_modes(const double* src, double* dst, double* tmp, int Nx, int k, const double* const* M)
{
    const int n = emh_pow(Nx, k);
    if (k == 0) { if (threadIdx.x == 0) dst[0] = src[0]; __syncthreads(); return; }
    const double* in = src;
    for (int s = 0; s < k; ++s) {
        double* out = ((k - 1 - s) % 2 == 0) ? dst : tmp;
        const int inner = emh_pow(Nx, k - 1 - s);
        const double* Ms = M[s];
        for (int f = threadIdx.x; f < n; f += blockDim.x) {
            const int lo = f % inner, hi = f / (inner * Nx), d = (f / inner) % Nx;
            double acc = 0.0;
            for (int e = 0; e < Nx; ++e) acc = fma(Ms[d * Nx + e], in[(hi * Nx + e) * inner + lo], acc);
            out[f] = acc;
        }
        __syncthreads();
        in = out;
    }
}

// X[p][q] (i-side axes first) from a record with owner i, or the transposed record with owner j; r2 (optional) is added
__device__ void emh_expand(const double* r, const double* r2, int pi, int qj, bool owner_j, int Nx,
                           const int* MID, const int* ENTPOS, int nf, double* X)
{
    const int nq = emh_pow(Nx, qj), n = emh_pow(Nx, pi) * nq;
    const int* ti = MID + emh_off(Nx, pi);
    const int* tj = MID + emh_off(Nx, qj);
    for (int x = threadIdx.x; x < n; x += blockDim.x) {
        const int mi = ti[x / nq], mj = tj[x % nq];
        const int e = owner_j ? ENTPOS[mj * nf + mi] : ENTPOS[mi * nf + mj];
        X[x] = r[e] + (r2 ? r2[e] : 0.0);
    }
    __syncthreads();
}

// sum over the placements of S on two of the k axes of index d, T (order k - 2) on the rest
__device__ double emh_place(const double* S, const double* T, int Nx, int k, const int* d)
{
    double s = 0.0;
    for (int i = 0; i < k; ++i)
        for (int j = i + 1; j < k; ++j) {
            int r = 0;
            for (int q = 0; q < k; ++q) if (q != i && q != j) r = r * Nx + d[q];
            s += S[d[i] * Nx + d[j]] * T[r];
        }
    return s;
}

// the three pairings S1 (x) S2 of four axes, each symmetrised over which matrix takes which pair
__device__ double emh_pairings(const double* S1, const double* S2, int Nx, const int* d)
{
    const int pr[3][4] = {{0, 1, 2, 3}, {0, 2, 1, 3}, {0, 3, 1, 2}};
    double s = 0.0;
    for (int q = 0; q < 3; ++q) {
        const int* p = pr[q];
        s += 0.5 * (S1[d[p[0]] * Nx + d[p[1]]] * S2[d[p[2]] * Nx + d[p[3]]] + S2[d[p[0]] * Nx + d[p[1]]] * S1[d[p[2]] * Nx + d[p[3]]]);
    }
    return s;
}

// in place: G_k = sum W y^(x)k  ->  sum W He_k(y; S)  (order 4 first: it reads G_2 and G_0)
__device__ void emh_hermite(double* G, const double* S, int Nx)
{
    const double g0 = G[0];
    int d[4];
    for (int x = threadIdx.x; x < emh_pow(Nx, 4); x += blockDim.x) {
        emh_digits(x, Nx, 4, d);
        G[emh_off(Nx, 4) + x] += emh_pairings(S, S, Nx, d) * g0 - emh_place(S, G + emh_off(Nx, 2), Nx, 4, d);
    }
    for (int x = threadIdx.x; x < emh_pow(Nx, 3); x += blockDim.x) {
        emh_digits(x, Nx, 3, d);
        G[emh_off(Nx, 3) + x] -= emh_place(S, G + 1, Nx, 3, d);
    }
    __syncthreads();
    for (int x = threadIdx.x; x < Nx * Nx; x += blockDim.x) G[emh_off(Nx, 2) + x] -= S[x] * g0;
    __syncthreads();
}

// G_k = sum W (Mi v_i + Mj v_j)^(x)k from the pair records: over the axis subsets, (Mi.. x Mj..) X_{p,q}.  Records with
// owner i serve q <= 2, with owner j q >= 3.  Scratch: X (Nx^4), Y (5 Nx^4), tmp (Nx^4).
__device__ void emh_gmoments(const double* ri, const double* ri2, const double* rj, const double* rj2, const double* Mi,
                             const double* Mj, int Nx, const int* MID, const int* ENTPOS, int nf,
                             double* G, double* X, double* Y, double* tmp)
{
    const int Q = emh_pow(Nx, 4);
    for (int k = 0; k <= 4; ++k) {
        for (int pi = 0; pi <= k; ++pi) {
            const int qj = k - pi;
            emh_expand(qj <= 2 ? ri : rj, qj <= 2 ? ri2 : rj2, pi, qj, qj > 2, Nx, MID, ENTPOS, nf, X);
            const double* Ms[4];
            for (int s = 0; s < k; ++s) Ms[s] = s < pi ? Mi : Mj;
            emh_modes(X, Y + (size_t)pi * Q, tmp, Nx, k, Ms);
        }
        int d[4];
        for (int x = threadIdx.x; x < emh_pow(Nx, k); x += blockDim.x) {
            emh_digits(x, Nx, k, d);
            double s = 0.0;
            for (int S = 0; S < (1 << k); ++S) {
                int fs = 0, fc = 0, ns = 0;
                for (int q = 0; q < k; ++q) {
                    if (S >> q & 1) { fs = fs * Nx + d[q]; ++ns; }
                    else fc = fc * Nx + d[q];
                }
                s += Y[(size_t)ns * Q + fs * emh_pow(Nx, k - ns) + fc];
            }
            G[emh_off(Nx, k) + x] = s;
        }
        __syncthreads();
    }
}

// Delta_k = sum u [He_k(F v; sF) - He_k(iR v; iR)] from the v-moments mu (family), telescoped so that every term carries
// X = F - iR (F^(x)k - iR^(x)k = sum_j F.. X iR..):  no difference of O(1) tensors.  muF: family scratch (orders 1, 2),
// tj, tmp: Nx^4 scratch.
__device__ void emh_delta(const double* mu, const double* iR, const double* F, const double* Xm, const double* sX,
                          const double* sF, int Nx, double* Dl, double* muF, double* tj, double* tmp)
{
    for (int k = 0; k <= 4; ++k) {
        const int n = emh_pow(Nx, k), o = emh_off(Nx, k);
        for (int x = threadIdx.x; x < n; x += blockDim.x) Dl[o + x] = 0.0;
        __syncthreads();
        const double* Ms[4];
        if (k == 1 || k == 2) {
            for (int s = 0; s < k; ++s) Ms[s] = F;
            emh_modes(mu + o, muF + o, tmp, Nx, k, Ms);
        }
        for (int j = 0; j < k; ++j) {
            for (int s = 0; s < k; ++s) Ms[s] = s < j ? F : (s == j ? Xm : iR);
            emh_modes(mu + o, tj, tmp, Nx, k, Ms);
            for (int x = threadIdx.x; x < n; x += blockDim.x) Dl[o + x] += tj[x];
            __syncthreads();
        }
    }
    const double u0 = mu[0];
    int d[4];
    for (int x = threadIdx.x; x < emh_pow(Nx, 4); x += blockDim.x) {      // reads Delta_2 before it is adjusted
        emh_digits(x, Nx, 4, d);
        Dl[emh_off(Nx, 4) + x] += (emh_pairings(sX, sF, Nx, d) + emh_pairings(iR, sX, Nx, d)) * u0
                                  - emh_place(sX, muF + emh_off(Nx, 2), Nx, 4, d) - emh_place(iR, Dl + emh_off(Nx, 2), Nx, 4, d);
    }
    for (int x = threadIdx.x; x < emh_pow(Nx, 3); x += blockDim.x) {
        emh_digits(x, Nx, 3, d);
        Dl[emh_off(Nx, 3) + x] -= emh_place(sX, muF + 1, Nx, 3, d) + emh_place(iR, Dl + 1, Nx, 3, d);
    }
    __syncthreads();
    for (int x = threadIdx.x; x < Nx * Nx; x += blockDim.x) Dl[emh_off(Nx, 2) + x] -= sX[x] * u0;
    __syncthreads();
}

// Mean part, one CTA per (output a = blockIdx.x, point blockIdx.y): the v-moments mu (family) from the mean record,
// D = sum u He_k(iR v; iR) (d^k mean_a / dz^k), and the three mean blocks (each entry read at its sorted index).
// EMP: the point's em_prepare_point block (stride per), REC: its records (stride nrec * RL), scratch: Nx^4 per CTA.
__global__ void __launch_bounds__(256)
em_hess_mean_finish_kernel(int Nx, int Ny, const double* __restrict__ EMP, long long per, const double* __restrict__ REC,
                           int nrec, int RL, const int* __restrict__ MID, const int* __restrict__ ENTPOS, int nf,
                           double* __restrict__ MU, double* __restrict__ D, double* __restrict__ scratch,
                           double* __restrict__ o2, double* __restrict__ o3, double* __restrict__ o4)
{
    __shared__ double iR[256];
    const int a = blockIdx.x, h = blockIdx.y, nn = Nx * Nx, TS = emh_off(Nx, 5);
    for (int q = threadIdx.x; q < nn; q += blockDim.x) iR[q] = EMP[h * per + (long long)a * (2 * nn + 2) + q];
    const double* rec = REC + ((long long)h * nrec + a) * RL;
    double* mu = MU + ((long long)h * Ny + a) * TS;
    double* Da = D + ((long long)h * Ny + a) * TS;
    double* tmp = scratch + ((long long)h * Ny + a) * emh_pow(Nx, 4);
    __syncthreads();
    const double* Ms[4] = {iR, iR, iR, iR};
    for (int k = 0; k <= 4; ++k) {
        emh_expand(rec, nullptr, k, 0, false, Nx, MID, ENTPOS, nf, mu + emh_off(Nx, k));
        emh_modes(mu + emh_off(Nx, k), Da + emh_off(Nx, k), tmp, Nx, k, Ms);
    }
    emh_hermite(Da, iR, Nx);
    int d[4];
    const long long ha = (long long)h * Ny + a;
    for (int x = threadIdx.x; x < nn; x += blockDim.x) { emh_digits(x, Nx, 2, d); o2[ha * nn + x] = Da[emh_off(Nx, 2) + emh_sorted(d, 2, Nx)]; }
    for (int x = threadIdx.x; x < nn * Nx; x += blockDim.x) { emh_digits(x, Nx, 3, d); o3[ha * nn * Nx + x] = 0.5 * Da[emh_off(Nx, 3) + emh_sorted(d, 3, Nx)]; }
    for (int x = threadIdx.x; x < nn * nn; x += blockDim.x) { emh_digits(x, Nx, 4, d); o4[ha * nn * nn + x] = 0.25 * Da[emh_off(Nx, 4) + emh_sorted(d, 4, Nx)]; }
}

// Covariance part, one CTA per (pair p = blockIdx.x, point h0 + blockIdx.y): d^k cov_ab / dz^k (k = 2..4) =
//   sum m He_k(g; CP)                                      (cross records, expm1 weights)
// + sum_S Delta_a,|S| (x) (D_b + Delta_b)_|S'| + D_a,|S| (x) Delta_b,|S'|   (w = u_a u_b^T by the Hermite addition formula)
// - t sum K^-1 Q He_k(g; CP)                               (a = b: trace backbone + remainder records)
// and the three cov blocks from it and D (heat equation, product rule), each entry formed once per orbit of its index
// symmetries and written to (a,b) and (b,a).  EHP per (point, pair): [Fa Fb CP At Bt sAt sBt sFa sFb] (Nx^2 each), t.
__global__ void __launch_bounds__(256, 1)
em_hess_pair_finish_kernel(int Nx, int Ny, int h0, const double* __restrict__ EMP, long long per, const double* __restrict__ EHP,
                           const double* __restrict__ REC, int nrec, int RL, const int* __restrict__ MID,
                           const int* __restrict__ ENTPOS, int nf, const double* __restrict__ MU, const double* __restrict__ D,
                           double* __restrict__ scratch, double* __restrict__ o2, double* __restrict__ o3, double* __restrict__ o4)
{
    __shared__ double Mt[11 * 256];
    const int p = blockIdx.x, h = h0 + blockIdx.y, nn = Nx * Nx, TS = emh_off(Nx, 5), Q = emh_pow(Nx, 4);
    const int npairs = gridDim.x;
    int a = 0;
    while ((a + 1) * (a + 2) / 2 <= p) ++a;
    const int b = p - a * (a + 1) / 2;
    const double* ehp = EHP + ((long long)h * npairs + p) * (9 * nn + 1);
    for (int q = threadIdx.x; q < 9 * nn; q += blockDim.x) Mt[q] = ehp[q];
    for (int q = threadIdx.x; q < nn; q += blockDim.x) {
        Mt[9 * nn + q] = EMP[h * per + (long long)a * (2 * nn + 2) + q];
        Mt[10 * nn + q] = EMP[h * per + (long long)b * (2 * nn + 2) + q];
    }
    const double t = ehp[9 * nn];
    const double *Fa = Mt, *Fb = Mt + nn, *CP = Mt + 2 * nn, *At = Mt + 3 * nn, *Bt = Mt + 4 * nn, *sAt = Mt + 5 * nn;
    const double *sBt = Mt + 6 * nn, *sFa = Mt + 7 * nn, *sFb = Mt + 8 * nn, *iRa = Mt + 9 * nn, *iRb = Mt + 10 * nn;
    double* G = scratch + (long long)blockIdx.y * npairs * (6LL * TS + 8LL * Q) + (long long)p * (6LL * TS + 8LL * Q);
    double *Tr = G + TS, *Da = Tr + TS, *Db = Da + TS, *muF = Db + TS, *X = muF + TS, *Y = X + Q, *tmp = Y + 5 * Q, *tj = tmp + Q;
    const double* rec = REC + (long long)h * nrec * RL;
    const int r_cross = Ny, r_tr = Ny + 2 * npairs, r_bb = r_tr + Ny;
    __syncthreads();
    emh_gmoments(rec + (long long)(r_cross + 2 * p) * RL, nullptr, rec + (long long)(r_cross + 2 * p + 1) * RL, nullptr,
                 Fa, Fb, Nx, MID, ENTPOS, nf, G, X, Y, tmp);
    emh_hermite(G, CP, Nx);
    const double* mua = MU + ((long long)h * Ny + a) * TS;
    const double* mub = MU + ((long long)h * Ny + b) * TS;
    const double* DA = D + ((long long)h * Ny + a) * TS;
    const double* DB = D + ((long long)h * Ny + b) * TS;
    emh_delta(mua, iRa, Fa, At, sAt, sFa, Nx, Da, muF, tj, tmp);
    emh_delta(mub, iRb, Fb, Bt, sBt, sFb, Nx, Db, muF, tj, tmp);
    int d[4];
    for (int k = 2; k <= 4; ++k) {
        for (int x = threadIdx.x; x < emh_pow(Nx, k); x += blockDim.x) {
            emh_digits(x, Nx, k, d);
            double s = 0.0;
            for (int S = 0; S < (1 << k); ++S) {
                int fs = 0, fc = 0, ns = 0;
                for (int q = 0; q < k; ++q) {
                    if (S >> q & 1) { fs = fs * Nx + d[q]; ++ns; }
                    else fc = fc * Nx + d[q];
                }
                const int os = emh_off(Nx, ns), oc = emh_off(Nx, k - ns);
                s += Da[os + fs] * (DB[oc + fc] + Db[oc + fc]) + DA[os + fs] * Db[oc + fc];
            }
            G[emh_off(Nx, k) + x] += s;
        }
    }
    __syncthreads();
    if (a == b) {
        const double* rt = rec + (long long)(r_tr + a) * RL;
        const double* rb = rec + (long long)(r_bb + a) * RL;
        emh_gmoments(rt, rb, rt, rb, Fa, Fa, Nx, MID, ENTPOS, nf, Tr, X, Y, tmp);
        emh_hermite(Tr, CP, Nx);
        for (int x = threadIdx.x; x < TS; x += blockDim.x) if (x >= emh_off(Nx, 2)) G[x] -= t * Tr[x];
        __syncthreads();
    }
    const double *Ja = DA + 1, *Jb = DB + 1, *Ha = DA + emh_off(Nx, 2), *Hb = DB + emh_off(Nx, 2);
    const double *M3a = DA + emh_off(Nx, 3), *M3b = DB + emh_off(Nx, 3);
    const double *C2 = G + emh_off(Nx, 2), *C3 = G + emh_off(Nx, 3), *C4 = G + emh_off(Nx, 4);
    const long long ab = ((long long)h * Ny + a) * Ny + b, ba = ((long long)h * Ny + b) * Ny + a;
    for (int x = threadIdx.x; x < nn; x += blockDim.x) {
        emh_digits(x, Nx, 2, d);
        o2[ab * nn + x] = o2[ba * nn + x] = C2[emh_sorted(d, 2, Nx)];
    }
    for (int x = threadIdx.x; x < nn * Nx; x += blockDim.x) {
        emh_digits(x, Nx, 3, d);
        const int dd = min(d[0], d[1]), e = max(d[0], d[1]), f = d[2];
        const int s3[3] = {dd, e, f};
        const double v = 0.5 * C3[emh_sorted(s3, 3, Nx)]
                       + 0.5 * (Ha[dd * Nx + f] * Jb[e] + Ja[dd] * Hb[e * Nx + f] + Hb[dd * Nx + f] * Ja[e] + Jb[dd] * Ha[e * Nx + f]);
        o3[ab * nn * Nx + x] = o3[ba * nn * Nx + x] = v;
    }
    for (int x = threadIdx.x; x < nn * nn; x += blockDim.x) {
        emh_digits(x, Nx, 4, d);
        // canonical representative under d <-> e, f <-> g and (d,e) <-> (f,g)
        int p1a = min(d[0], d[1]), p1b = max(d[0], d[1]), p2a = min(d[2], d[3]), p2b = max(d[2], d[3]);
        if (p2a < p1a || (p2a == p1a && p2b < p1b)) { int u = p1a; p1a = p2a; p2a = u; u = p1b; p1b = p2b; p2b = u; }
        const int dd = p1a, e = p1b, f = p2a, g = p2b;
        const int s4[4] = {dd, e, f, g};
        auto m3 = [&](const double* T, int i, int j, int k) { const int s[3] = {i, j, k}; return T[emh_sorted(s, 3, Nx)]; };
        const double lab = m3(M3a, f, dd, e) * Jb[g] + Ha[f * Nx + dd] * Hb[g * Nx + e] + Ha[f * Nx + e] * Hb[g * Nx + dd] + Ja[f] * m3(M3b, g, dd, e);
        const double lba = m3(M3b, f, dd, e) * Ja[g] + Hb[f * Nx + dd] * Ha[g * Nx + e] + Hb[f * Nx + e] * Ha[g * Nx + dd] + Jb[f] * m3(M3a, g, dd, e);
        const double v = 0.25 * C4[emh_sorted(s4, 4, Nx)] + 0.25 * (lab + lba)
                       + 0.25 * (m3(M3a, dd, f, g) * Jb[e] + Ja[dd] * m3(M3b, e, f, g) + m3(M3b, dd, f, g) * Ja[e] + Jb[dd] * m3(M3a, e, f, g));
        o4[ab * nn * nn + x] = o4[ba * nn * nn + x] = v;
    }
}

// backbone feature rows of Q_aa for L^-1: R[f][i] = e_i mono_f(v_i) (f < nf: the record's features); zero for i >= N
__global__ void em_backbone_rows_kernel(const double* __restrict__ XT, int ldx, int N, int Nx, const double* __restrict__ z,
                                        const double* __restrict__ E, int n, const int* __restrict__ MONO, int nf,
                                        double* __restrict__ R)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double e = (i < N) ? exp(E[i]) : 0.0;
    for (int f = 0; f < nf; ++f) {
        double r = e;
        for (int s = 0; s < 4; ++s) {
            const int d = MONO[4 * f + s];
            if (d >= 0) r *= (i < N) ? XT[(long long)d * ldx + i] - z[d] : 0.0;
        }
        R[(long long)f * n + i] = r;
    }
}

// full symmetric copy of a lower-stored matrix (32x32 tiles, every entry taken from the lower triangle)
__global__ void sym_from_lower_kernel(const double* __restrict__ Kl, double* __restrict__ Kf, int ld)
{
    __shared__ double tile[32][33];
    const int bi = blockIdx.y, bj = blockIdx.x;
    if (bj > bi) return;
    const int tx = threadIdx.x, ty = threadIdx.y;   // 32 x 8
    for (int r = ty; r < 32; r += 8) tile[r][tx] = Kl[(long long)(bi * 32 + r) * ld + bj * 32 + tx];
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {
        const double lo = (bi > bj || r >= tx) ? tile[r][tx] : tile[tx][r];
        Kf[(long long)(bi * 32 + r) * ld + bj * 32 + tx] = lo;
        if (bi > bj) Kf[(long long)(bj * 32 + r) * ld + bi * 32 + tx] = tile[tx][r];
    }
}

// ---------------------------------------------------------------------------------------
// Rank-1 append of one training point (SURVEY 8f row 3; the reference's update_data,
// gp_class.py:384-471, is self-declared broken -- this is the textbook update):
//   l = L^-1 k(X, x_new);  lambda = sqrt(k(x_new,x_new) + sn2 + jitter - l^T l)
//   L    <- [[L, 0], [l^T, lambda]]          L^-1 <- [[L^-1, 0], [-(l^T L^-1)/lambda, 1/lambda]]
// lvec = L^-1 k, rvec = (L^-1)^T lvec are produced by the trmv kernels; this kernel writes
// row N of both factors (the identity tail row it replaces).  jit[a]: the jitter output a's factorisation put on every
// diagonal entry of K, which the new one gets as well.  One CTA per output.  stop (may be null): a greedy selection
// step after a failed pivot, nothing is written.
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
append_row_kernel(double* __restrict__ L, double* __restrict__ Li, int ld, long long sL,
                  const double* __restrict__ lvec, const double* __restrict__ rvec, long long sv,
                  const double* __restrict__ hyp, int hyp_ld, int Nx, const double* __restrict__ jit, int N,
                  int* __restrict__ info, const int* __restrict__ stop)
{
    __shared__ double red[8];
    __shared__ double lam_s;
    if (stop && *stop) return;
    const int a = blockIdx.x, tid = threadIdx.x;
    const double* lv = lvec + (long long)a * sv;
    const double* rv = rvec + (long long)a * sv;
    double s = 0.0;
    for (int i = tid; i < N; i += 256) s = fma(lv[i], lv[i], s);
    s = warp_sum(s);
    if ((tid & 31) == 0) red[tid >> 5] = s;
    __syncthreads();
    if (tid == 0) {
        double r = 0.0;
        for (int w = 0; w < 8; ++w) r += red[w];
        const double sf = hyp[(long long)a * hyp_ld + Nx], sn = hyp[(long long)a * hyp_ld + Nx + 1];
        const double d = sf * sf + sn * sn + jit[a] - r;
        if (!(d > 0.0)) atomicCAS(info + a, 0, N + 1);
        lam_s = sqrt(d);
    }
    __syncthreads();
    const double lam = lam_s, il = 1.0 / lam;
    double* Lr = L + (long long)a * sL + (long long)N * ld;
    double* Lir = Li + (long long)a * sL + (long long)N * ld;
    for (int j = tid; j < N; j += 256) { Lr[j] = lv[j]; Lir[j] = -rv[j] * il; }
    if (tid == 0) { Lr[N] = lam; Lir[N] = il; }
}

// ---------------------------------------------------------------------------------------
// Greedy max-variance selection from a pool of n candidates (gpmpc_append_greedy).  V[a][c][0..Npad) = L_a^-1 k_a(X, c)
// (row stride ldv, output stride sV), var[a][c] = sf2_a - |V[a][c]|^2 (noise free, q3).  Step k (Nk = N + k points):
//   pick c* -> gather l_a = V[a][c*] -> trmv_lower_T + append_row (row Nk of L, L^-1) -> downdate the active candidates:
//   w = (k_a(x*, c) - l_a . v_ac) / L_a[Nk][Nk],  v_ac[Nk] = w,  var[a][c] -= w^2
// Every dot product runs in a fixed order (two calls give the same bits).  Once a pivot failed (info != 0 on any
// output) the kernels of the later steps return at once: nothing is written past the failing row.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ bool greedy_failed(const int* __restrict__ info, int nloc)
{
    for (int a = 0; a < nloc; ++a)
        if (info[a]) return true;
    return false;
}

// sum of a row of n doubles times another, lane-strided with four accumulators (fixed order); every lane gets it
__device__ __forceinline__ double warp_dot(const double* __restrict__ x, const double* __restrict__ y, int n)
{
    const int lane = threadIdx.x & 31;
    double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
    int i = lane;
    for (; i + 96 < n; i += 128) {
        s0 = fma(x[i], y[i], s0);
        s1 = fma(x[i + 32], y[i + 32], s1);
        s2 = fma(x[i + 64], y[i + 64], s2);
        s3 = fma(x[i + 96], y[i + 96], s3);
    }
    for (; i < n; i += 32) s0 = fma(x[i], y[i], s0);
    return warp_sum((s0 + s1) + (s2 + s3));
}

// var[a][c] = sf2_a - |V[a][c][0..N)|^2; one warp per (candidate, output), grid (ceil(n/8), nloc)
__global__ void __launch_bounds__(256)
greedy_var_kernel(const double* __restrict__ V, int ldv, long long sV, int N, int n,
                  const double* __restrict__ hyp, int hyp_ld, int Nx, double* __restrict__ var)
{
    const int c = blockIdx.x * 8 + (threadIdx.x >> 5), a = blockIdx.y;
    if (c >= n) return;
    const double* v = V + (long long)a * sV + (long long)c * ldv;
    const double s = warp_dot(v, v, N);
    if ((threadIdx.x & 31) == 0) {
        const double sf = hyp[(long long)a * hyp_ld + Nx];
        var[(long long)a * n + c] = sf * sf - s;
    }
}

// true if (s1, i1) beats (s2, i2): larger score, ties to the lower index; index n is "none"
__device__ __forceinline__ bool greedy_better(double s1, int i1, double s2, int i2, int n)
{
    return i1 != n && (i2 == n || s1 > s2 || (s1 == s2 && i1 < i2));
}

// One CTA: score[c] = sum_a var[a][c] (outputs in order) over the active candidates, argmax with ties to the lowest
// index.  Records c* and its score, deactivates it, writes x* into column Nk of X^T and y* into row Nk of Y.  After a
// failed pivot it only raises `stop` for the rest of the step.
__global__ void __launch_bounds__(1024)
greedy_pick_kernel(const double* __restrict__ var, int n, int nloc, int* __restrict__ active,
                   const double* __restrict__ Xc, const double* __restrict__ Yc, int Nx,
                   double* __restrict__ XT, double* __restrict__ Y, int ld, int Nk,
                   const int* __restrict__ info, int* __restrict__ stop,
                   int* __restrict__ picked, double* __restrict__ score, int k)
{
    __shared__ double bs[32];
    __shared__ int bi[32];
    const int tid = threadIdx.x, lane = tid & 31, wp = tid >> 5;
    if (greedy_failed(info, nloc)) {
        if (tid == 0) *stop = 1;
        return;
    }
    double best = 0.0;
    int bidx = n;
    for (int c = tid; c < n; c += 1024) {        // ascending c: the first of equal scores stays
        if (!active[c]) continue;
        double s = 0.0;
        for (int a = 0; a < nloc; ++a) s += var[(long long)a * n + c];
        if (bidx == n || s > best) { best = s; bidx = c; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double s2 = __shfl_xor_sync(0xffffffffu, best, o);
        const int i2 = __shfl_xor_sync(0xffffffffu, bidx, o);
        if (greedy_better(s2, i2, best, bidx, n)) { best = s2; bidx = i2; }
    }
    if (lane == 0) { bs[wp] = best; bi[wp] = bidx; }
    __syncthreads();
    if (wp == 0) {
        best = bs[lane]; bidx = bi[lane];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double s2 = __shfl_xor_sync(0xffffffffu, best, o);
            const int i2 = __shfl_xor_sync(0xffffffffu, bidx, o);
            if (greedy_better(s2, i2, best, bidx, n)) { best = s2; bidx = i2; }
        }
        if (bidx < n) {                           // always: the host asks for at most n picks
            if (lane == 0) { picked[k] = bidx; score[k] = best; active[bidx] = 0; }
            if (lane < Nx) XT[(long long)lane * ld + Nk] = Xc[(long long)bidx * Nx + lane];
            for (int a = lane; a < nloc; a += 32) Y[(long long)a * ld + Nk] = Yc[(long long)bidx * nloc + a];
        }
    }
}

// l_a[i] = V[a][c*][i] for i < Nk, 0 up to ld (as gpmpc_append leaves its l); grid (ceil(ld/256), nloc)
__global__ void __launch_bounds__(256)
greedy_gather_kernel(const double* __restrict__ V, int ldv, long long sV, const int* __restrict__ picked, int k, int Nk,
                     double* __restrict__ l, long long sl, int ld, const int* __restrict__ stop)
{
    if (*stop) return;
    const int a = blockIdx.y, i = blockIdx.x * 256 + threadIdx.x;
    if (i >= ld) return;
    l[(long long)a * sl + i] = (i < Nk) ? V[(long long)a * sV + (long long)picked[k] * ldv + i] : 0.0;
}

// w = (k_a(x*, c) - l_a . v_ac) / lambda_a for every active candidate c, one warp per (candidate, output),
// grid (ceil(n/8), nloc); lambda_a = L_a[Nk][Nk] as append_row_kernel wrote it
__global__ void __launch_bounds__(256)
greedy_downdate_kernel(double* __restrict__ V, int ldv, long long sV, double* __restrict__ var, int n,
                       const int* __restrict__ active, const double* __restrict__ l, long long sl,
                       const double* __restrict__ L, int ld, long long sL, const double* __restrict__ Xc, int Nx,
                       const double* __restrict__ hyp, int hyp_ld, const int* __restrict__ picked, int k, int Nk,
                       const int* __restrict__ info, int nloc)
{
    const int lane = threadIdx.x & 31, c = blockIdx.x * 8 + (threadIdx.x >> 5), a = blockIdx.y;
    if (c >= n || !active[c] || greedy_failed(info, nloc)) return;
    const double* hp = hyp + (long long)a * hyp_ld;
    double* v = V + (long long)a * sV + (long long)c * ldv;
    const double s = warp_dot(l + (long long)a * sl, v, Nk);
    const int cs = picked[k];
    double q = 0.0;
    if (lane < Nx) {                              // Nx <= 32
        const double df = (Xc[(long long)cs * Nx + lane] - Xc[(long long)c * Nx + lane]) / hp[lane];
        q = df * df;
    }
    q = warp_sum(q);
    if (lane == 0) {
        const double sf = hp[Nx];
        const double w = (sf * sf * exp(-0.5 * q) - s) / L[(long long)a * sL + (long long)Nk * ld + Nk];
        v[Nk] = w;
        var[(long long)a * n + c] -= w * w;
    }
}

// ---------------------------------------------------------------------------------------
// Sampled roll-outs (gpmpc_rollout_sample): trajectory b, output a, step t is one draw of the GP posterior conditioned on
// the values the same draw took at the earlier kept points z_s of b (DESIGN 4.12).  With v_t = L_a^-1 k_a(X, z_t):
//   m_t = k_a(X, z_t)^T alpha_a,   c_s = k_a(z_t, z_s) - v_t . v_s (kept s < t),   c_tt = sf2_a - |v_t|^2
//   w = R^-1 c,  d = c_tt - |w|^2,  f_t = m_t + sum_j w_j eps_j + sqrt(d) eps_t
// R (lower, at most Nt x Nt per (b, a)) is the Cholesky factor of the joint covariance of the kept points, row by row
// [w, sqrt(d)], so that f - m = R eps over the kept points.  d <= delta sf2: f_t = m_t + sum_j w_j eps_j, not kept.
// ---------------------------------------------------------------------------------------
// m[a][r] = ks_r^T alpha_a for the H points of one ks launch: the sum of the ks kernel's block partials PMJ[a][r][blk][0]
// with the association of the predict product's psk_reduce_mj (even / odd blocks in ascending order, then their sum), so
// m is gpmpc_predict's mean bit for bit.  One thread per (output, row), grid (ceil(nloc H / 256)).
__global__ void __launch_bounds__(256)
ks_mean_kernel(const double* __restrict__ PMJ, int nblk, int Nx, int H, int nloc, double* __restrict__ m, long long sm)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= nloc * H) return;
    const int a = i / H, r = i - a * H;
    const double* pm = PMJ + (long long)i * nblk * (Nx + 1);
    double s0 = 0.0, s1 = 0.0;
    int b = 0;
    for (; b + 2 <= nblk; b += 2) { s0 += pm[(long long)b * (Nx + 1)]; s1 += pm[(long long)(b + 1) * (Nx + 1)]; }
    if (b < nblk) s0 += pm[(long long)b * (Nx + 1)];
    m[(long long)a * sm + r] = s0 + s1;
}

// Steps of a differentiated sampled roll-out (gpmpc_rollout_sample_grad): the tangent kernel keeps R (Nt^2 doubles) and
// per-warp rows in shared memory under 48 KB
#define SAMPLE_GRAD_NT_MAX 64

// Warps of a CTA of the roll-outs' tangent stage (rollout_tangent_kernel, rollout_tangent_em_kernel, sample_next_kernel,
// sample_tangent_kernel): each warp owns one parameter column at a time and a slice of the dynamic shared memory
#define ROLL_TG_WARPS 8

// The dynamic shared memory of the sampled roll-outs' kernels, written once for the kernel that carves it and for the
// launch that sizes it: offsets in doubles from the start of the buffer, and the launch's bytes.  The offsets are 64-bit
// sums of int terms, the address arithmetic of stepping a pointer term by term, which keeps the kernels' registers.
// sample_cond_kernel: c (Nt + 1) | conditioning steps (Nt ints)
struct SampleCondSmem { long long idx; int bytes; };
__host__ __device__ __forceinline__ SampleCondSmem sample_cond_smem(int Nt)
{
    return {(long long)Nt + 1, (Nt + 1) * 8 + Nt * 4};
}

// sample_tangent_kernel: c (Nt + 1) | R (Nt Nt) | per warp dw (Nt) | conditioning steps (Nt ints)
struct SampleTangentSmem { long long R, tw, idx; int bytes; };
__host__ __device__ __forceinline__ SampleTangentSmem sample_tangent_smem(int Nt)
{
    const long long R = (long long)Nt + 1, tw = R + Nt * Nt, idx = tw + ROLL_TG_WARPS * Nt;
    return {R, tw, idx, (int)idx * 8 + Nt * 4};
}

// The conditioning steps of (b, a) before step t into idx (thread 0; the caller synchronises), and their count
__device__ __forceinline__ int sample_cond_steps(const double* __restrict__ kept, int B, int b, int Ny, int a, int t, int* idx)
{
    int k = 0;
    for (int s = 0; s < t; ++s)
        if (kept[((long long)s * B + b) * Ny + a] != 0.0) idx[k++] = s;
    return k;
}

// c[j] = k(z_t, z_s) - v_t . v_s for the k conditioning steps s = idx[j] and c[k] = sf2 - |v_t|^2, one warp per j (every
// thread of a CTA of ROLL_TG_WARPS warps calls it; the caller synchronises).  Va: the V rows of output a; hp: its hyper row.  The
// arithmetic of sample_cond_kernel's own loop, bit for bit (that kernel keeps its inline copy: calling these helpers
// from it costs it a spill).
__device__ __forceinline__ void sample_cond_c(const double* __restrict__ Va, int ldv, int N, const double* __restrict__ Zh,
                                              const double* __restrict__ hp, int Nx, int B, int b, int t, int k,
                                              const int* idx, double sf2, double* c)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const double* vt = Va + ((long long)t * B + b) * ldv;
    const double* zt = Zh + ((long long)t * B + b) * Nx;
    for (int j = warp; j <= k; j += ROLL_TG_WARPS) {      // j = k: the point itself
        const int s = (j < k) ? idx[j] : t;
        const double dot = warp_dot(vt, Va + ((long long)s * B + b) * ldv, N);
        double q = 0.0;
        if (j < k && lane < Nx) {                         // Nx <= 32; direct differences
            const double df = (zt[lane] - Zh[((long long)s * B + b) * Nx + lane]) / hp[lane];
            q = df * df;
        }
        q = warp_sum(q);
        if (lane == 0) c[j] = ((j < k) ? sf2 * exp(-0.5 * q) : sf2) - dot;
    }
}

// One CTA per (trajectory b, output a) at step t, grid (B, nloc).  V rows of (a, s, b) at V + a sVa + (s B + b) ldv;
// Zh (Nt, B, Nx); m (nloc, B) of this step; eps, xi (B, Nt, Ny) (xi may be null); Rf (nloc, B, Nt, Nt);
// kept, samp (Nt, B, Ny).  Dynamic shared memory: sample_cond_smem.
__global__ void __launch_bounds__(256)
sample_cond_kernel(const double* __restrict__ V, long long sVa, int ldv, int N, const double* __restrict__ m,
                   const double* __restrict__ Zh, const double* __restrict__ hyp, int hyp_ld, int Nx, int Ny,
                   const double* __restrict__ eps, const double* __restrict__ xi, double* __restrict__ Rf,
                   double* __restrict__ kept, double* __restrict__ samp, int Nt, int t, double delta)
{
    extern __shared__ double sc_sh[];
    __shared__ int nk_s;
    const int b = blockIdx.x, a = blockIdx.y, B = gridDim.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    double* c = sc_sh;
    int* idx = reinterpret_cast<int*>(sc_sh + sample_cond_smem(Nt).idx);
    const double* hp = hyp + (long long)a * hyp_ld;
    const double* Va = V + (long long)a * sVa;
    const double* vt = Va + ((long long)t * B + b) * ldv;
    const double* zt = Zh + ((long long)t * B + b) * Nx;
    if (tid == 0) {
        int k = 0;
        for (int s = 0; s < t; ++s)
            if (kept[((long long)s * B + b) * Ny + a] != 0.0) idx[k++] = s;
        nk_s = k;
    }
    __syncthreads();
    const int k = nk_s;
    const double sf2 = hp[Nx] * hp[Nx];
    for (int j = warp; j <= k; j += 8) {                  // j = k: the point itself
        const int s = (j < k) ? idx[j] : t;
        const double dot = warp_dot(vt, Va + ((long long)s * B + b) * ldv, N);
        double q = 0.0;
        if (j < k && lane < Nx) {                         // Nx <= 32; direct differences
            const double df = (zt[lane] - Zh[((long long)s * B + b) * Nx + lane]) / hp[lane];
            q = df * df;
        }
        q = warp_sum(q);
        if (lane == 0) c[j] = ((j < k) ? sf2 * exp(-0.5 * q) : sf2) - dot;
    }
    __syncthreads();
    if (tid != 0) return;
    double* R = Rf + ((long long)a * B + b) * Nt * Nt;
    const double* e = eps + (long long)b * Nt * Ny + a;  // eps of (b, s, a) at e[s Ny]
    double ww = 0.0, we = 0.0;
    for (int j = 0; j < k; ++j) {                         // forward substitution in place: c[j] <- w_j
        double w = c[j];
        for (int i = 0; i < j; ++i) w -= R[j * Nt + i] * c[i];
        w /= R[j * Nt + j];
        c[j] = w;
        ww += w * w;
        we += w * e[(long long)idx[j] * Ny];
    }
    const double d = c[k] - ww;
    const bool keep = d > delta * sf2;
    double f = m[(long long)a * B + b] + we;
    if (keep) {
        const double sd = sqrt(d);
        f += sd * e[(long long)t * Ny];
        for (int j = 0; j < k; ++j) R[k * Nt + j] = c[j];
        R[k * Nt + k] = sd;
    }
    const long long o = ((long long)t * B + b) * Ny + a;
    kept[o] = keep ? 1.0 : 0.0;
    samp[o] = xi ? f + hp[Nx + 1] * xi[((long long)b * Nt + t) * Ny + a] : f;
}

// Pathwise derivatives of the draws (gpmpc_rollout_sample_grad, DESIGN 4.16).  With beta_s = K_a^-1 ks_s and
// d_e ks_t[i] = -(z_t,e - x_i,e) / ell_e^2 ks_t[i], the derivative of c_ts = k(z_t, z_s) - ks_t^T K^-1 ks_s is
// g(t,s) . dz_t + g(s,t) . dz_s with
//   g(t,s)_e = -(z_t,e - z_s,e) / ell_e^2 k(z_t, z_s) + sum_i (z_t,e - x_i,e) ks_t[i] beta_s[i] / ell_e^2.
// One CTA per (trajectory b, output a, j-th conditioning step s of step t), grid (B, nloc, t); a CTA with j past the
// conditioning set exits.  ks_t and ks_s are recomputed from X^T (direct differences, as the ks kernel forms them) in
// tiles of 256 points: each thread forms ks_t[i] beta_s[i] and ks_s[i] beta_t[i] of one point, then warp w sums the
// products with (z - x_i) for e = w, w + 8, ...  Beta rows of (a, s, b) at Beta + a sBa + (s B + b) ldb; XT (Nx, ldx);
// Zh (Nt, B, Nx); G (nloc, B, Nt, 2, Nx): [g(t,s) | g(s,t)] at row j.  Every sum runs in a fixed order.
__global__ void __launch_bounds__(256)
sample_cross_kernel(const double* __restrict__ Beta, long long sBa, int ldb, const double* __restrict__ XT, int ldx, int N,
                    const double* __restrict__ Zh, const double* __restrict__ hyp, int hyp_ld, int Nx, int Ny,
                    const double* __restrict__ kept, double* __restrict__ G, int Nt, int t)
{
    __shared__ double wk[2][256], zts[32], zss[32], il2[32];
    __shared__ int idx[SAMPLE_GRAD_NT_MAX];
    __shared__ int s_s;
    const int b = blockIdx.x, a = blockIdx.y, j = blockIdx.z, B = gridDim.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) {
        const int k = sample_cond_steps(kept, B, b, Ny, a, t, idx);
        s_s = j < k ? idx[j] : -1;
    }
    __syncthreads();
    const int s = s_s;
    if (s < 0) return;                                    // uniform over the CTA
    const double* hp = hyp + (long long)a * hyp_ld;
    if (tid < Nx) {
        zts[tid] = Zh[((long long)t * B + b) * Nx + tid];
        zss[tid] = Zh[((long long)s * B + b) * Nx + tid];
        il2[tid] = 1.0 / (hp[tid] * hp[tid]);
    }
    __syncthreads();
    const double sf2 = hp[Nx] * hp[Nx];
    const double* bt = Beta + (long long)a * sBa + ((long long)t * B + b) * ldb;
    const double* bs = Beta + (long long)a * sBa + ((long long)s * B + b) * ldb;
    double acc1[4] = {0.0, 0.0, 0.0, 0.0}, acc2[4] = {0.0, 0.0, 0.0, 0.0};   // e = warp + 8 r, Nx <= 32
    for (int i0 = 0; i0 < N; i0 += 256) {
        const int i = i0 + tid;
        double w1 = 0.0, w2 = 0.0;
        if (i < N) {
            double qt = 0.0, qs = 0.0;
            for (int e = 0; e < Nx; ++e) {
                const double x = XT[(long long)e * ldx + i];
                const double dt = (zts[e] - x) / hp[e], ds = (zss[e] - x) / hp[e];
                qt = fma(dt, dt, qt);
                qs = fma(ds, ds, qs);
            }
            w1 = sf2 * exp(-0.5 * qt) * bs[i];
            w2 = sf2 * exp(-0.5 * qs) * bt[i];
        }
        __syncthreads();                                  // the previous tile's products are consumed
        wk[0][tid] = w1;
        wk[1][tid] = w2;
        __syncthreads();
        const int n = min(256, N - i0);
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int e = warp + 8 * r;
            if (e < Nx)
                for (int ii = lane; ii < n; ii += 32) {
                    const double x = XT[(long long)e * ldx + i0 + ii];
                    acc1[r] = fma(zts[e] - x, wk[0][ii], acc1[r]);
                    acc2[r] = fma(zss[e] - x, wk[1][ii], acc2[r]);
                }
        }
    }
    double q = 0.0;
    if (lane < Nx) {
        const double df = (zts[lane] - zss[lane]) / hp[lane];
        q = df * df;
    }
    const double kts = sf2 * exp(-0.5 * warp_sum(q));
    double* g = G + (((long long)a * B + b) * Nt + j) * 2 * Nx;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int e = warp + 8 * r;
        const double s1 = warp_sum(acc1[r]), s2 = warp_sum(acc2[r]);
        if (lane == 0 && e < Nx) {
            const double dz = zts[e] - zss[e];
            g[e] = (s1 - dz * kts) * il2[e];
            g[Nx + e] = (s2 + dz * kts) * il2[e];
        }
    }
}

// The tangent stage of one sampled step, one CTA per (trajectory b, output a), grid (B, nloc), ROLL_TG_WARPS warps over
// the P parameter columns.  With w = R^-1 c and d = c_tt - |w|^2 re-formed as sample_cond_kernel forms them and the kept flag of
// step t (the branch the draw took), per column p:
//   dm = J_t dz_t,  dc_tt = dvar_dz_t . dz_t,  dc_j = g(t,s_j) . dz_t + g(s_j,t) . dz_{s_j},
//   dw = R^-1 (dc - dR w),  dd = dc_tt - 2 w . dw,  df = dm + dw . eps_S (+ dd / (2 sqrt d) eps_t when kept),
// and when kept the new row [dw, dd / (2 sqrt d)] of dR.  J, dvar (B, Ny, Nx) of the derivative chain at the step's points;
// G of sample_cross_kernel; dZh (Nt, B, P, Nx) the tangent history; dRf (nloc, B, P, Nt, Nt); dsamp (B, Ny, P) of step t.
// Every sum runs in index order in one thread.  Dynamic shared memory: sample_tangent_smem.
__global__ void __launch_bounds__(ROLL_TG_WARPS * 32)
sample_tangent_kernel(const double* __restrict__ V, long long sVa, int ldv, int N, const double* __restrict__ Zh,
                      const double* __restrict__ hyp, int hyp_ld, int Nx, int Ny, const double* __restrict__ eps,
                      const double* __restrict__ Rf, const double* __restrict__ kept, const double* __restrict__ J,
                      const double* __restrict__ dvar, const double* __restrict__ G, const double* __restrict__ dZh,
                      double* __restrict__ dRf, double* __restrict__ dsamp, int P, int Nt, int t)
{
    extern __shared__ double st_sh[];
    __shared__ int nk_s;
    const int b = blockIdx.x, a = blockIdx.y, B = gridDim.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const SampleTangentSmem L = sample_tangent_smem(Nt);
    double* c = st_sh;
    double* sR = st_sh + L.R;
    double* tw = st_sh + L.tw + warp * Nt;
    int* idx = reinterpret_cast<int*>(st_sh + L.idx);
    const double* hp = hyp + (long long)a * hyp_ld;
    const double* R = Rf + ((long long)a * B + b) * Nt * Nt;
    if (tid == 0) nk_s = sample_cond_steps(kept, B, b, Ny, a, t, idx);
    __syncthreads();
    const int k = nk_s;
    const double sf2 = hp[Nx] * hp[Nx];
    sample_cond_c(V + (long long)a * sVa, ldv, N, Zh, hp, Nx, B, b, t, k, idx, sf2, c);
    for (int i = tid; i < k * Nt; i += ROLL_TG_WARPS * 32) sR[i] = R[i];
    __syncthreads();
    if (tid == 0) {                                       // w and d with sample_cond_kernel's arithmetic
        double ww = 0.0;
        for (int j = 0; j < k; ++j) {
            double w = c[j];
            for (int i = 0; i < j; ++i) w -= sR[j * Nt + i] * c[i];
            w /= sR[j * Nt + j];
            c[j] = w;
            ww += w * w;
        }
        c[k] -= ww;
    }
    __syncthreads();
    const bool keep = kept[((long long)t * B + b) * Ny + a] != 0.0;
    const double sd2 = keep ? 2.0 * sqrt(c[k]) : 1.0;
    const double* e = eps + (long long)b * Nt * Ny + a;   // eps of (b, s, a) at e[s Ny]
    const double* Ja = J + ((long long)b * Ny + a) * Nx;
    const double* dva = dvar + ((long long)b * Ny + a) * Nx;
    const double* Gab = G + ((long long)a * B + b) * Nt * 2 * Nx;
    for (int p = warp; p < P; p += ROLL_TG_WARPS) {
        const double* dzt = dZh + (((long long)t * B + b) * P + p) * Nx;
        double* dR = dRf + (((long long)a * B + b) * P + p) * Nt * Nt;
        for (int j = lane; j < k; j += 32) {              // dc_j - (dR w)_j
            const double* g = Gab + (long long)j * 2 * Nx;
            const double* dzs = dZh + (((long long)idx[j] * B + b) * P + p) * Nx;
            double s = 0.0;
            for (int q = 0; q < Nx; ++q) s = fma(g[q], dzt[q], s);
            for (int q = 0; q < Nx; ++q) s = fma(g[Nx + q], dzs[q], s);
            for (int i = 0; i <= j; ++i) s = fma(-dR[j * Nt + i], c[i], s);
            tw[j] = s;
        }
        __syncwarp();
        if (lane == 0) {
            double dm = 0.0, dct = 0.0;
            for (int q = 0; q < Nx; ++q) {
                dm = fma(Ja[q], dzt[q], dm);
                dct = fma(dva[q], dzt[q], dct);
            }
            double wdw = 0.0, df = dm;
            for (int j = 0; j < k; ++j) {                 // dw = R^-1 (dc - dR w), in place
                double s = tw[j];
                for (int i = 0; i < j; ++i) s = fma(-sR[j * Nt + i], tw[i], s);
                s /= sR[j * Nt + j];
                tw[j] = s;
                wdw = fma(c[j], s, wdw);
                df = fma(s, e[(long long)idx[j] * Ny], df);
            }
            if (keep) {
                const double dq = (dct - 2.0 * wdw) / sd2;
                df = fma(dq, e[(long long)t * Ny], df);
                dR[k * Nt + k] = dq;
            }
            dsamp[((long long)b * Ny + a) * P + p] = df;
        }
        __syncwarp();
        if (keep)
            for (int j = lane; j < k; j += 32) dR[k * Nt + j] = tw[j];
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------------------
// Removal of training point i from an N-point factorisation (gpmpc_remove), O(N^2) per output.  With lambda = L[i][i],
// n = N - i - 1 trailing points (r, s, j, k index them: old row / column i + 1 + r):
//   p_r = -lambda Li[i+1+r][i] (= L33^-1 l32),  t_-1 = 1,  t_r = t_{r-1} + p_r^2,
//   d_r = sqrt(t_r / t_{r-1}),  g_r = p_r / sqrt(t_r t_{r-1})
// chol(I + p p^T) = diag(d) + strict_lower(p g^T), its inverse diag(1/d) - strict_lower(g p^T).  New rows i + r:
//   L'[i+r][c]   = L[i+1+r][c] (c < i),   L'[i+r][i+j] = d_j L[i+1+r][i+1+j] + g_j sum_{j<k<=r} p_k L[i+1+r][i+1+k]
//   R_r = Li[i+1+r][.] + p_r Li[i][.]  (its column i vanishes and is dropped),
//   Li'[i+r][.]  = R_r / d_r - g_r sum_{s<r} p_s R_s
// A rank-1 update of the trailing block (every t_r >= 1): it cannot lose positive definiteness.  The L rows are
// suffix scans along each row, the L^-1 rows prefix scans down each column (row blocks of RM_RB: partials, their scan
// over blocks, the apply pass).  Both write rows i .. N-2 into a work slab (a row moves up over the row another CTA
// still reads), which remove_commit_kernel copies back.  Rows are written up to the end of their 128-wide diagonal
// block, zeros right of the diagonal; the strictly-upper 128-tiles are never written.  Every sum runs in a fixed order.
// ---------------------------------------------------------------------------------------
#define RM_RB 64

// Exclusive prefix sum of v over the CTA's threads in thread order, and the CTA total (*total), in a fixed order: warp
// shuffles, then the warp totals scanned in warp order.  sh: 33 doubles of shared memory; every thread must call it.
__device__ __forceinline__ double block_exclusive_scan(double v, double* sh, double* total)
{
    const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    double x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    double ex = __shfl_up_sync(0xffffffffu, x, 1);
    if (lane == 0) ex = 0.0;
    if (lane == 31) sh[wp] = x;
    __syncthreads();
    if (wp == 0) {
        double w = lane < nw ? sh[lane] : 0.0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const double y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += y;
        }
        double wex = __shfl_up_sync(0xffffffffu, w, 1);
        if (lane == 0) wex = 0.0;
        __syncwarp();
        sh[lane] = wex;
        if (lane == 31) sh[32] = w;
    }
    __syncthreads();
    const double r = ex + sh[wp];
    *total = sh[32];
    __syncthreads();                              // sh is free for the next call
    return r;
}

// p, d, g of the removal of point i for every output (one CTA each): coef[a] = [p (ld) | d (ld) | g (ld)]
__global__ void __launch_bounds__(1024)
remove_coef_kernel(const double* __restrict__ L, const double* __restrict__ Li, int ld, long long sL, int i, int n,
                   double* __restrict__ coef)
{
    __shared__ double sh[33];
    const double* Lib = Li + (long long)blockIdx.x * sL;
    double* p = coef + (long long)blockIdx.x * 3 * ld;
    double* d = p + ld;
    double* g = d + ld;
    const double lam = L[(long long)blockIdx.x * sL + (long long)i * ld + i];
    const int C = (n + 1023) / 1024, r0 = threadIdx.x * C, r1 = min(n, r0 + C);   // contiguous chunk per thread
    double s = 0.0;
    for (int r = r0; r < r1; ++r) {
        const double pr = -lam * Lib[(long long)(i + 1 + r) * ld + i];
        p[r] = pr;
        s = fma(pr, pr, s);
    }
    double tot;
    double tp = 1.0 + block_exclusive_scan(s, sh, &tot);
    for (int r = r0; r < r1; ++r) {
        const double pr = p[r], t = fma(pr, pr, tp);
        d[r] = sqrt(t / tp);
        g[r] = pr / sqrt(t * tp);
        tp = t;
    }
}

// New rows i .. i+n-1 of L into W (one CTA per row, the longest first): the moved columns < i, the suffix scan of
// p_k L[i+1+r][i+1+k] from the diagonal leftwards in 256-element segments, zeros up to the diagonal block's end
__global__ void __launch_bounds__(256)
remove_l_rows_kernel(const double* __restrict__ L, double* __restrict__ W, int ld, const double* __restrict__ coef,
                     int i, int n)
{
    __shared__ double sh[33];
    const int tid = threadIdx.x, r = n - 1 - blockIdx.x, R = i + r;
    const double* src = L + (long long)(R + 1) * ld;
    double* dst = W + (long long)R * ld;
    const double* p = coef;
    const double* d = coef + ld;
    const double* g = coef + 2 * ld;
    for (int c = tid; c < i; c += 256) dst[c] = src[c];
    const int be = (R / 128 + 1) * 128;
    for (int c = R + 1 + tid; c < be; c += 256) dst[c] = 0.0;
    double carry = 0.0;                            // sum of p_k a_k over the segments already done (larger k)
    for (int hi = r + 1; hi > 0; hi -= 256) {
        const int j = hi - 1 - tid;               // thread order = descending j: a prefix over threads is a suffix in j
        const double a = j >= 0 ? src[i + 1 + j] : 0.0;
        const double pa = j >= 0 ? p[j] * a : 0.0;
        double tot;
        const double s = block_exclusive_scan(pa, sh, &tot);
        if (j >= 0) dst[i + j] = fma(g[j], carry + s, d[j] * a);
        carry += tot;
    }
}

// Q[b][c] = sum_{r in row block b} p_r R_r[c'] for new column c (old column c' = c + (c >= i)); grid (ceil(ld/256), nb)
__global__ void __launch_bounds__(256)
remove_li_part_kernel(const double* __restrict__ Li, int ld, const double* __restrict__ coef, int i, int n,
                      double* __restrict__ Q)
{
    const int c = blockIdx.x * 256 + threadIdx.x, b = blockIdx.y;
    const int r0 = b * RM_RB, r1 = min(n, r0 + RM_RB);
    if (c >= ld) return;
    const double* p = coef;
    const int oc = c + (c >= i);
    const double li = c < i ? Li[(long long)i * ld + c] : 0.0;
    double q = 0.0;
    for (int r = max(r0, c - i); r < r1; ++r) {  // new row i + r holds column c from r >= c - i on
        const double x = fma(p[r], li, Li[(long long)(i + 1 + r) * ld + oc]);
        q = fma(p[r], x, q);
    }
    Q[(long long)b * ld + c] = q;
}

// exclusive scan of Q over the nb row blocks, per column (in place)
__global__ void __launch_bounds__(256)
remove_li_scan_kernel(double* __restrict__ Q, int ld, int nb)
{
    const int c = blockIdx.x * 256 + threadIdx.x;
    if (c >= ld) return;
    double e = 0.0;
    for (int b = 0; b < nb; ++b) {
        const double q = Q[(long long)b * ld + c];
        Q[(long long)b * ld + c] = e;
        e += q;
    }
}

// New rows i + r of L^-1 into W for the rows of block b, from the scanned partials Q; grid as remove_li_part_kernel
__global__ void __launch_bounds__(256)
remove_li_apply_kernel(const double* __restrict__ Li, double* __restrict__ W, int ld, const double* __restrict__ coef,
                       int i, int n, const double* __restrict__ Q)
{
    const int c = blockIdx.x * 256 + threadIdx.x, b = blockIdx.y;
    const int r0 = b * RM_RB, r1 = min(n, r0 + RM_RB);
    if (c >= ld || c >= ((i + r1 - 1) / 128 + 1) * 128) return;   // right of the last row's diagonal block
    const double* p = coef;
    const double* d = coef + ld;
    const double* g = coef + 2 * ld;
    const int oc = c + (c >= i);
    const double li = c < i ? Li[(long long)i * ld + c] : 0.0;
    double P = Q[(long long)b * ld + c];
    for (int r = r0; r < r1; ++r) {
        const int R = i + r;
        if (c >= (R / 128 + 1) * 128) continue;
        double o = 0.0;
        if (c <= R) {
            const double x = fma(p[r], li, Li[(long long)(i + 1 + r) * ld + oc]);
            o = fma(-g[r], P, x / d[r]);
            P = fma(p[r], x, P);
        }
        W[(long long)R * ld + c] = o;
    }
}

// Rows i .. N-2 of L and L^-1 from the work slabs (columns up to the diagonal block's end), row N-1 the identity tail
// row; one CTA per row
__global__ void __launch_bounds__(256)
remove_commit_kernel(double* __restrict__ L, double* __restrict__ Li, const double* __restrict__ WL,
                     const double* __restrict__ WLi, int ld, int i, int N)
{
    const int R = i + blockIdx.x, be2 = (R / 128 + 1) * 64;
    double2* l = reinterpret_cast<double2*>(L + (long long)R * ld);
    double2* li = reinterpret_cast<double2*>(Li + (long long)R * ld);
    if (R == N - 1) {
        for (int c = threadIdx.x; c < be2; c += 256) {
            const double2 v = make_double2(2 * c == R ? 1.0 : 0.0, 2 * c + 1 == R ? 1.0 : 0.0);
            l[c] = v; li[c] = v;
        }
        return;
    }
    const double2* wl = reinterpret_cast<const double2*>(WL + (long long)R * ld);
    const double2* wli = reinterpret_cast<const double2*>(WLi + (long long)R * ld);
    for (int c = threadIdx.x; c < be2; c += 256) { l[c] = wl[c]; li[c] = wli[c]; }
}

// Entry i leaves each of the `rows` rows of stride ld (X^T, then Y): later entries move down one, entry N-1 becomes 0.
// One CTA per row; each segment is read before any of it is written, so the in-place move is race-free.
__global__ void __launch_bounds__(256)
remove_shift_kernel(double* __restrict__ XT, int nx, double* __restrict__ Y, int ld, int i, int N)
{
    double* x = blockIdx.x < nx ? XT + (long long)blockIdx.x * ld : Y + (long long)(blockIdx.x - nx) * ld;
    for (int c0 = i; c0 < N - 1; c0 += 256) {
        const int c = c0 + threadIdx.x;
        const double v = c < N - 1 ? x[c + 1] : 0.0;
        __syncthreads();
        if (c < N - 1) x[c] = v;
    }
    if (threadIdx.x == 0) x[N - 1] = 0.0;
}

// ---------------------------------------------------------------------------------------
// First derivatives of the prediction w.r.t. the test input z (SURVEY 8f row 1: what CasADi's
// AD produces for the MPC's NLP from the symbolic build_gp / build_TA_cov graphs,
// gp_functions.py:111-173; mpc_class.py:390-412 differentiates them inside nlpsol):
//   d ks_i / d z_d = ks_i (X_id - z_d)/ell_d^2
//   d var / d z_d  = -2 sum_i beta_i ks_i (X_id - z_d)/ell_d^2 ,  beta = K^-1 ks = L^-T (L^-1 ks)
//   Hm_de = d^2 mean / dz_d dz_e = sum_i alpha_i ks_i s_id s_ie - delta_de mean/ell_d^2 ,
//           s_id = (X_id - z_d)/ell_d^2
// Stage 1 (this kernel): per (output, test point, 1024-point block) partial sums
//   PDV[d] = sum_i beta_i ks_i s_id            PH[q(d<=e)] = sum_i alpha_i ks_i s_id s_ie
// ks is read back from KST (written by ks_mean_jac_kernel), beta rows from the second product.
// grid (Npad/1024, Hc, outputs), 256 threads.
// ---------------------------------------------------------------------------------------
#define GR_CHUNK 1024
template <int NXP>
__global__ void __launch_bounds__(256)
grad_reduce_kernel(const double* __restrict__ XT, int ldx, int N, int Nx,
                   const double* __restrict__ hyp, int hyp_ld,
                   const double* __restrict__ alpha, long long sal,
                   const double* __restrict__ Z,
                   const double* __restrict__ KST, const double* __restrict__ BETA, int ldk, long long sK,
                   double* __restrict__ PDV, double* __restrict__ PH, int nblk, int Hc)
{
    extern __shared__ double gsm[];                 // S[Nx][257], WA[256]
    __shared__ double red[8][NXP];
    __shared__ double zs[NXP], ie2[NXP];
    const int a = blockIdx.z, h = blockIdx.y, blk = blockIdx.x, tid = threadIdx.x;
    double* S = gsm; double* WA = gsm + Nx * 257;
    const double* hp = hyp + (long long)a * hyp_ld;
    if (tid < NXP) {
        const double e = (tid < Nx) ? hp[tid] : 1.0;
        zs[tid] = (tid < Nx) ? Z[(long long)h * Nx + tid] : 0.0;
        ie2[tid] = 1.0 / (e * e);
    }
    __syncthreads();
    const int npairs = Nx * (Nx + 1) / 2;
    const double* ks = KST + (long long)a * sK + (long long)h * ldk;
    const double* be = BETA + (long long)a * sK + (long long)h * ldk;
    const double* al = alpha + (long long)a * sal;
    double dv[NXP];
#pragma unroll
    for (int d = 0; d < NXP; ++d) dv[d] = 0.0;
    double hacc[3] = {0.0, 0.0, 0.0};               // pairs tid, tid+256, tid+512 (NX_MAX = 32: 528 pairs)
    for (int sub = 0; sub < GR_CHUNK / 256; ++sub) {
        const int i = blk * GR_CHUNK + sub * 256 + tid;
        double k = 0.0, wb = 0.0, wa = 0.0;
        if (i < N) { k = ks[i]; wb = be[i] * k; wa = al[i] * k; }
#pragma unroll
        for (int d = 0; d < NXP; ++d) {
            if (d < Nx) {
                const double sd = (i < N) ? (XT[(long long)d * ldx + i] - zs[d]) * ie2[d] : 0.0;
                S[d * 257 + tid] = sd;
                dv[d] = fma(wb, sd, dv[d]);
            }
        }
        WA[tid] = wa;
        __syncthreads();
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const int q = tid + 256 * r;
            if (q < npairs) {
                // q -> (d <= e), row-major upper packing: q = d*Nx - d(d-1)/2 + (e - d)
                int d = 0, base = 0;
                while (base + (Nx - d) <= q) { base += Nx - d; ++d; }
                const int e = d + (q - base);
                const double* sd = S + d * 257; const double* se = S + e * 257;
                double acc = 0.0;
                for (int t = 0; t < 256; ++t) acc = fma(WA[t] * sd[t], se[t], acc);
                hacc[r] += acc;
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int d = 0; d < NXP; ++d) dv[d] = warp_sum(dv[d]);
    if ((tid & 31) == 0) {
#pragma unroll
        for (int d = 0; d < NXP; ++d) red[tid >> 5][d] = dv[d];
    }
    __syncthreads();
    const long long rec = ((long long)a * Hc + h) * nblk + blk;
    if (tid < Nx) {
        double sacc = 0.0;
        for (int w = 0; w < 8; ++w) sacc += red[w][tid];
        PDV[rec * Nx + tid] = sacc;
    }
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const int q = tid + 256 * r;
        if (q < npairs) PH[rec * npairs + q] = hacc[r];
    }
}

// Stage 2: per (test point h of the chunk, output a): dvar_dz (Nx) and the mean Hessian (Nx,Nx)
// from the block partials; grid (Hc, outputs), 128 threads.  mean comes from the gather record.
__global__ void __launch_bounds__(128)
grad_finalize_kernel(const double* __restrict__ PDV, const double* __restrict__ PH, int nblk, int Hc,
                     const double* __restrict__ hyp, int hyp_ld, int Nx, int Ny,
                     const double* __restrict__ G, int Htot, int h0,
                     double* __restrict__ dvar, double* __restrict__ hess)
{
    const int h = blockIdx.x, a = blockIdx.y, tid = threadIdx.x;
    const int npairs = Nx * (Nx + 1) / 2;
    const long long rec = ((long long)a * Hc + h) * nblk;
    const double* hp = hyp + (long long)a * hyp_ld;
    const double mean = G[(((long long)a) * Htot + h0 + h) * (Nx + 2)];
    for (int d = tid; d < Nx; d += 128) {
        double sacc = 0.0;
        for (int b = 0; b < nblk; ++b) sacc += PDV[(rec + b) * Nx + d];
        dvar[(((long long)(h0 + h)) * Ny + a) * Nx + d] = -2.0 * sacc;
    }
    for (int q = tid; q < npairs; q += 128) {
        int d = 0, base = 0;
        while (base + (Nx - d) <= q) { base += Nx - d; ++d; }
        const int e = d + (q - base);
        double sacc = 0.0;
        for (int b = 0; b < nblk; ++b) sacc += PH[(rec + b) * npairs + q];
        if (d == e) sacc -= mean / (hp[d] * hp[d]);
        double* Hm = hess + (((long long)(h0 + h)) * Ny + a) * Nx * Nx;
        Hm[d * Nx + e] = sacc;
        Hm[e * Nx + d] = sacc;
    }
}

// Stage 3: d cov[a][b] / d z_e for every test point (grid H, 128 threads):
//   'ME': delta_ab dvar_a[e]
//   'TA': delta_ab dvar_a[e] + sum_d Hm_a[d][e] (Sigma J_b)[d] + sum_d (J_a Sigma)[d] Hm_b[d][e]
//   (derivative of diag(var) + J Sigma J^T, gp_functions.py:167-171; Sigma need not be symmetric)
__global__ void __launch_bounds__(128)
grad_cov_kernel(int Ny, int Nx, int method_ta, const double* __restrict__ Sigma, int sigma_per_point,
                const double* __restrict__ J, const double* __restrict__ dvar, const double* __restrict__ hess,
                double* __restrict__ dcov)
{
    extern __shared__ double sh[];                  // SJ[Ny][Nx] = Sigma J_b, JS[Ny][Nx] = J_a Sigma
    double* SJ = sh; double* JS = sh + Ny * Nx;
    const int h = blockIdx.x, tid = threadIdx.x;
    const double* Jh = J + (long long)h * Ny * Nx;
    if (method_ta) {
        const double* Sg = Sigma + (sigma_per_point ? (long long)h * Nx * Nx : 0);
        for (int idx = tid; idx < Ny * Nx; idx += 128) {
            const int a = idx / Nx, d = idx % Nx;
            double s1 = 0.0, s2 = 0.0;
            for (int e = 0; e < Nx; ++e) {
                s1 = fma(Sg[d * Nx + e], Jh[a * Nx + e], s1);          // (Sigma J_a)[d]
                s2 = fma(Jh[a * Nx + e], Sg[e * Nx + d], s2);          // (J_a Sigma)[d]
            }
            SJ[idx] = s1; JS[idx] = s2;
        }
    }
    __syncthreads();
    const double* dv = dvar + (long long)h * Ny * Nx;
    const double* Hh = hess + (long long)h * Ny * Nx * Nx;
    double* out = dcov + (long long)h * Ny * Ny * Nx;
    for (int idx = tid; idx < Ny * Ny * Nx; idx += 128) {
        const int e = idx % Nx, b = (idx / Nx) % Ny, a = idx / (Nx * Ny);
        double s = (a == b) ? dv[a * Nx + e] : 0.0;
        if (method_ta) {
            const double* Ha = Hh + (long long)a * Nx * Nx; const double* Hb = Hh + (long long)b * Nx * Nx;
            for (int d = 0; d < Nx; ++d) {
                s = fma(Ha[d * Nx + e], SJ[b * Nx + d], s);
                s = fma(JS[a * Nx + d], Hb[d * Nx + e], s);
            }
        }
        out[idx] = s;
    }
}

// ---------------------------------------------------------------------------------------
// Second derivatives of the prediction w.r.t. the test input (gpmpc_predict_hess: what CasADi's AD
// produces when IPOPT uses the exact Hessian of the MPC's NLP, mpc_class.py:390-412, :496-513).  Per
// output a and test point z, s_id = (X_id - z_d)/ell_d^2, beta = K^-1 ks, J / Hm the mean Jacobian / Hessian:
//   d3 mean / dz_d dz_e dz_f = M3_def - d_de J_f/ell_d^2 - d_df J_e/ell_d^2 - d_ef J_d/ell_e^2
//   d2 var / dz_d dz_e       = -2 [G_de + B2_de - d_de (ks^T K^-1 ks)/ell_d^2]
//   M3_def = sum_i alpha_i ks_i s_id s_ie s_if     B2_de = sum_i beta_i ks_i s_id s_ie
//   G_de = (L^-1 d_d ks)^T (L^-1 d_e ks)           ks^T K^-1 ks = sf2 - var
// The rows d_d ks of R = 64/Nx test points at a time go through the predict product (V_d = L^-1 d_d ks);
// everything else is fixed-order block partials like grad_reduce / grad_finalize.
// ---------------------------------------------------------------------------------------

// packed index q -> (d <= e <= f): d-major, then e, then f (the pair order of grad_reduce within each d)
__device__ __forceinline__ void triple_of(int q, int Nx, int& d, int& e, int& f)
{
    int base = 0;
    d = 0;
    while (base + (Nx - d) * (Nx - d + 1) / 2 <= q) { base += (Nx - d) * (Nx - d + 1) / 2; ++d; }
    const int r = q - base, m = Nx - d;
    int e0 = 0, b2 = 0;
    while (b2 + (m - e0) <= r) { b2 += m - e0; ++e0; }
    e = d + e0;
    f = e + (r - b2);
}

__device__ __forceinline__ void pair_of(int q, int Nx, int& d, int& e)
{
    int base = 0;
    d = 0;
    while (base + (Nx - d) <= q) { base += Nx - d; ++d; }
    e = d + (q - base);
}

// A operand of the derivative product: row pt*Nx + d of output a = d_d ks of test point p0 + pt of the chunk
// (h-major like KST, zero for i >= N).  grid (ceil(Npad/256), points of the pass, outputs), 256 threads.
__global__ void __launch_bounds__(256)
hess_rows_kernel(const double* __restrict__ XT, int ldx, int N, int Nx, const double* __restrict__ hyp, int hyp_ld,
                 const double* __restrict__ Z, const double* __restrict__ KST, int ldk, long long sK,
                 double* __restrict__ D, int p0)
{
    const int a = blockIdx.z, pt = blockIdx.y, i = blockIdx.x * 256 + threadIdx.x;
    if (i >= ldk) return;
    const int h = p0 + pt;
    const double* hp = hyp + (long long)a * hyp_ld;
    const double k = (i < N) ? KST[(long long)a * sK + (long long)h * ldk + i] : 0.0;
    double* out = D + (long long)a * sK + (long long)pt * Nx * ldk + i;
    for (int d = 0; d < Nx; ++d) {
        const double e = hp[d], ie2 = 1.0 / (e * e);
        const double sd = (i < N) ? (XT[(long long)d * ldx + i] - Z[(long long)h * Nx + d]) * ie2 : 0.0;
        out[(long long)d * ldk] = k * sd;
    }
}

// Stage 1 per (output, test point of the pass, 1024-point block): partial sums
//   PG[q(d<=e)] = sum_i V_d,i V_e,i    PB[q] = sum_i beta_i ks_i s_id s_ie    PM[t(d<=e<=f)] = sum_i alpha_i ks_i s_id s_ie s_if
// V rows from the derivative product, ks from KST, beta from the second product of predict_grad.
// grid (Npad/1024, points of the pass, outputs), 256 threads; NX_MAX = 32: 528 pairs, 5984 triples.
template <int NXP>
__global__ void __launch_bounds__(256)
hess_reduce_kernel(const double* __restrict__ XT, int ldx, int N, int Nx,
                   const double* __restrict__ hyp, int hyp_ld,
                   const double* __restrict__ alpha, long long sal,
                   const double* __restrict__ Z,
                   const double* __restrict__ KST, const double* __restrict__ BETA, const double* __restrict__ VD,
                   int ldk, long long sK,
                   double* __restrict__ PG, double* __restrict__ PB, double* __restrict__ PM, int nblk, int Hc, int p0)
{
    constexpr int NPR = (NXP * (NXP + 1) / 2 + 255) / 256;
    constexpr int NTR = (NXP * (NXP + 1) * (NXP + 2) / 6 + 255) / 256;
    extern __shared__ double hsm[];                 // S[Nx][257] (s_id), W[Nx][257] (V rows), WA[256], WB[256]
    __shared__ double zs[NXP], ie2[NXP];
    const int a = blockIdx.z, pt = blockIdx.y, blk = blockIdx.x, tid = threadIdx.x, h = p0 + pt;
    double* S = hsm; double* W = hsm + Nx * 257; double* WA = W + Nx * 257; double* WB = WA + 256;
    const double* hp = hyp + (long long)a * hyp_ld;
    if (tid < NXP) {
        const double e = (tid < Nx) ? hp[tid] : 1.0;
        zs[tid] = (tid < Nx) ? Z[(long long)h * Nx + tid] : 0.0;
        ie2[tid] = 1.0 / (e * e);
    }
    const int npairs = Nx * (Nx + 1) / 2, ntri = Nx * (Nx + 1) * (Nx + 2) / 6;
    int pc[NPR], tc[NTR];                           // (d, e[, f]) of this thread's pairs / triples, 5 bits each
#pragma unroll
    for (int r = 0; r < NPR; ++r) {
        int d = 0, e = 0;
        if (tid + 256 * r < npairs) pair_of(tid + 256 * r, Nx, d, e);
        pc[r] = d | (e << 5);
    }
#pragma unroll
    for (int r = 0; r < NTR; ++r) {
        int d = 0, e = 0, f = 0;
        if (tid + 256 * r < ntri) triple_of(tid + 256 * r, Nx, d, e, f);
        tc[r] = d | (e << 5) | (f << 10);
    }
    __syncthreads();
    const double* ks = KST + (long long)a * sK + (long long)h * ldk;
    const double* be = BETA + (long long)a * sK + (long long)h * ldk;
    const double* vd = VD + (long long)a * sK + (long long)pt * Nx * ldk;
    const double* al = alpha + (long long)a * sal;
    double gacc[NPR], bacc[NPR], macc[NTR];
#pragma unroll
    for (int r = 0; r < NPR; ++r) { gacc[r] = 0.0; bacc[r] = 0.0; }
#pragma unroll
    for (int r = 0; r < NTR; ++r) macc[r] = 0.0;
    for (int sub = 0; sub < GR_CHUNK / 256; ++sub) {
        const int i = blk * GR_CHUNK + sub * 256 + tid;
        double k = 0.0, wb = 0.0, wa = 0.0;
        if (i < N) { k = ks[i]; wb = be[i] * k; wa = al[i] * k; }
#pragma unroll
        for (int d = 0; d < NXP; ++d) {
            if (d < Nx) {
                S[d * 257 + tid] = (i < N) ? (XT[(long long)d * ldx + i] - zs[d]) * ie2[d] : 0.0;
                W[d * 257 + tid] = (i < N) ? vd[(long long)d * ldk + i] : 0.0;
            }
        }
        WA[tid] = wa; WB[tid] = wb;
        __syncthreads();
#pragma unroll
        for (int r = 0; r < NPR; ++r) {
            if (tid + 256 * r < npairs) {
                const double* sd = S + (pc[r] & 31) * 257; const double* se = S + (pc[r] >> 5) * 257;
                const double* vd_ = W + (pc[r] & 31) * 257; const double* ve = W + (pc[r] >> 5) * 257;
                double g = 0.0, b = 0.0;
                for (int t = 0; t < 256; ++t) {
                    g = fma(vd_[t], ve[t], g);
                    b = fma(WB[t] * sd[t], se[t], b);
                }
                gacc[r] += g; bacc[r] += b;
            }
        }
#pragma unroll
        for (int r = 0; r < NTR; ++r) {
            if (tid + 256 * r < ntri) {
                const double* sd = S + (tc[r] & 31) * 257; const double* se = S + ((tc[r] >> 5) & 31) * 257;
                const double* sf = S + (tc[r] >> 10) * 257;
                double m = 0.0;
                for (int t = 0; t < 256; ++t) m = fma(WA[t] * sd[t] * se[t], sf[t], m);
                macc[r] += m;
            }
        }
        __syncthreads();
    }
    const long long rec = ((long long)a * Hc + h) * nblk + blk;
#pragma unroll
    for (int r = 0; r < NPR; ++r) {
        const int q = tid + 256 * r;
        if (q < npairs) { PG[rec * npairs + q] = gacc[r]; PB[rec * npairs + q] = bacc[r]; }
    }
#pragma unroll
    for (int r = 0; r < NTR; ++r) {
        const int q = tid + 256 * r;
        if (q < ntri) PM[rec * ntri + q] = macc[r];
    }
}

// Stage 2 per (test point h of the chunk, output a): d2var (Nx,Nx) and d3mean (Nx,Nx,Nx) from the block
// partials, each value written to every symmetric position (exactly symmetric).  grid (Hc, outputs), 128 threads.
__global__ void __launch_bounds__(128)
hess_finalize_kernel(const double* __restrict__ PG, const double* __restrict__ PB, const double* __restrict__ PM,
                     int nblk, int Hc, const double* __restrict__ hyp, int hyp_ld, int Nx, int Ny,
                     const double* __restrict__ G, int Htot, int h0,
                     double* __restrict__ d2var, double* __restrict__ d3mean)
{
    const int h = blockIdx.x, a = blockIdx.y, tid = threadIdx.x;
    const int npairs = Nx * (Nx + 1) / 2, ntri = Nx * (Nx + 1) * (Nx + 2) / 6;
    const long long rec = ((long long)a * Hc + h) * nblk;
    const double* hp = hyp + (long long)a * hyp_ld;
    const double* g = G + (((long long)a) * Htot + h0 + h) * (Nx + 2);     // [mean, var, J]
    const double sf = hp[Nx], q_kk = sf * sf - g[1];                       // ks^T K^-1 ks
    double* V2 = d2var + (((long long)(h0 + h)) * Ny + a) * Nx * Nx;
    double* T3 = d3mean + (((long long)(h0 + h)) * Ny + a) * Nx * Nx * Nx;
    for (int q = tid; q < npairs; q += 128) {
        int d, e;
        pair_of(q, Nx, d, e);
        double sg = 0.0, sb = 0.0;
        for (int b = 0; b < nblk; ++b) { sg += PG[(rec + b) * npairs + q]; sb += PB[(rec + b) * npairs + q]; }
        double s = sg + sb;
        if (d == e) s -= q_kk / (hp[d] * hp[d]);
        s *= -2.0;
        V2[d * Nx + e] = s;
        V2[e * Nx + d] = s;
    }
    for (int q = tid; q < ntri; q += 128) {
        int d, e, f;
        triple_of(q, Nx, d, e, f);
        double s = 0.0;
        for (int b = 0; b < nblk; ++b) s += PM[(rec + b) * ntri + q];
        if (d == e) s -= g[2 + f] / (hp[d] * hp[d]);
        if (d == f) s -= g[2 + e] / (hp[d] * hp[d]);
        if (e == f) s -= g[2 + d] / (hp[e] * hp[e]);
        T3[(d * Nx + e) * Nx + f] = s; T3[(d * Nx + f) * Nx + e] = s;
        T3[(e * Nx + d) * Nx + f] = s; T3[(e * Nx + f) * Nx + d] = s;
        T3[(f * Nx + d) * Nx + e] = s; T3[(f * Nx + e) * Nx + d] = s;
    }
}

// Stage 3: d2 cov[a][b] / dz_f dz_g for every test point (grid H, 128 threads), the second-order analogue of
// grad_cov_kernel (diag(var) + J Sigma J^T, gp_functions.py:167-171; Sigma need not be symmetric):
//   'ME': delta_ab d2var_a[f][g]
//   'TA': delta_ab d2var_a[f][g] + sum_d T_a[d][f][g] (Sigma J_b)[d] + sum_d (J_a Sigma)[d] T_b[d][f][g]
//         + P_ab[f][g] + P_ab[g][f],   P_ab = Hm_a^T Sigma Hm_b  (SH_b = Sigma Hm_b staged in SHg, (H,Ny,Nx,Nx))
// computed for f <= g and written to both halves.
__global__ void __launch_bounds__(128)
hess_cov_kernel(int Ny, int Nx, int method_ta, const double* __restrict__ Sigma, int sigma_per_point,
                const double* __restrict__ J, const double* __restrict__ hess, const double* __restrict__ d2var,
                const double* __restrict__ d3mean, double* __restrict__ SHg, double* __restrict__ d2cov)
{
    extern __shared__ double sh[];                  // SJ[Ny][Nx] = Sigma J_b, JS[Ny][Nx] = J_a Sigma
    double* SJ = sh; double* JS = sh + Ny * Nx;
    const int h = blockIdx.x, tid = threadIdx.x, nxx = Nx * Nx;
    const double* Jh = J + (long long)h * Ny * Nx;
    const double* Hh = hess + (long long)h * Ny * nxx;
    double* SH = SHg + (long long)h * Ny * nxx;
    if (method_ta) {
        const double* Sg = Sigma + (sigma_per_point ? (long long)h * nxx : 0);
        for (int idx = tid; idx < Ny * Nx; idx += 128) {
            const int a = idx / Nx, d = idx % Nx;
            double s1 = 0.0, s2 = 0.0;
            for (int e = 0; e < Nx; ++e) {
                s1 = fma(Sg[d * Nx + e], Jh[a * Nx + e], s1);          // (Sigma J_a)[d]
                s2 = fma(Jh[a * Nx + e], Sg[e * Nx + d], s2);          // (J_a Sigma)[d]
            }
            SJ[idx] = s1; JS[idx] = s2;
        }
        for (int idx = tid; idx < Ny * nxx; idx += 128) {
            const int b = idx / nxx, d = (idx / Nx) % Nx, g = idx % Nx;
            const double* Hb = Hh + (long long)b * nxx;
            double s = 0.0;
            for (int e = 0; e < Nx; ++e) s = fma(Sg[d * Nx + e], Hb[e * Nx + g], s);
            SH[idx] = s;
        }
    }
    __syncthreads();
    const int npairs = Nx * (Nx + 1) / 2;
    const double* V2 = d2var + (long long)h * Ny * nxx;
    const double* T3 = d3mean + (long long)h * Ny * nxx * Nx;
    double* out = d2cov + (long long)h * Ny * Ny * nxx;
    for (int idx = tid; idx < Ny * Ny * npairs; idx += 128) {
        const int q = idx % npairs, b = (idx / npairs) % Ny, a = idx / (npairs * Ny);
        int f, g;
        pair_of(q, Nx, f, g);
        double s = (a == b) ? V2[(long long)a * nxx + f * Nx + g] : 0.0;
        if (method_ta) {
            const double* Ta = T3 + (long long)a * nxx * Nx; const double* Tb = T3 + (long long)b * nxx * Nx;
            const double* Ha = Hh + (long long)a * nxx; const double* SHb = SH + (long long)b * nxx;
            double t = 0.0, pfg = 0.0, pgf = 0.0;
            for (int d = 0; d < Nx; ++d) {
                t = fma(Ta[d * nxx + f * Nx + g], SJ[b * Nx + d], t);
                t = fma(JS[a * Nx + d], Tb[d * nxx + f * Nx + g], t);
                pfg = fma(Ha[d * Nx + f], SHb[d * Nx + g], pfg);
                pgf = fma(Ha[d * Nx + g], SHb[d * Nx + f], pgf);
            }
            s += t + (pfg + pgf);
        }
        double* o = out + ((long long)a * Ny + b) * nxx;
        o[f * Nx + g] = s;
        o[g * Nx + f] = s;
    }
}

// ---------------------------------------------------------------------------------------
// Leave-one-out cross-validation (gpmpc_loo, gpmpc_loo_nlpp; R&W section 5.4.2, eqs. 5.10-5.14).  With C = K^-1 =
// Li^T Li, alpha = C y and c_i = C_ii = sum_{k >= i} Li[k][i]^2 (the column norms of Li):
//   LOO mean  y_i - alpha_i / c_i,   LOO variance 1 / c_i,
//   NLPP = sum_i [ 1/2 log 2pi - 1/2 log c_i + alpha_i^2 / (2 c_i) ]
//   dNLPP/dtheta_j = tr(W dK/dtheta_j),  W = C diag(w) C - sym(b alpha^T),
//   w_i = (1 + alpha_i^2 / c_i) / (2 c_i),  u = alpha / c,  b = C u,  sym(M) = (M + M^T) / 2.
// The trace runs through nlml_grad_kernel with W in place of K^-1 and a zero vector in place of alpha.
// ---------------------------------------------------------------------------------------

// Column-norm partials of Li, only its lower triangle up to n read: grid (ceil(n/32), ceil(n/TRT_ROWS), batch).  Block
// (k-block, chunk c) sums Li[i][k]^2 over rows [c*TRT_ROWS, (c+1)*TRT_ROWS), i >= k, of its 32 columns into P[batch][c][k]
// (the layout of trmv_lower_T_part_kernel): each warp reads 32 consecutive entries of a row.  Chunks entirely above the
// diagonal are skipped; loo_point_kernel sums chunks c >= k/TRT_ROWS in ascending order.
__global__ void __launch_bounds__(256)
loo_colnorm_part_kernel(const double* __restrict__ Li, int ld, long long sL, double* __restrict__ P, long long sP, int n)
{
    __shared__ double red[8][33];
    const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
    const int k0 = blockIdx.x * 32, c = blockIdx.y;
    const int r1 = min(n, (c + 1) * TRT_ROWS);
    if (r1 <= k0) return;
    const int r0 = max(c * TRT_ROWS, k0);
    const int k = k0 + lane;
    const double* Lb = Li + (long long)blockIdx.z * sL;
    double s = 0.0;
    for (int i = r0 + wp; i < r1; i += 8)
        if (i >= k) {
            const double v = Lb[(long long)i * ld + k];
            s = fma(v, v, s);
        }
    red[wp][lane] = s;
    __syncthreads();
    if (wp == 0 && k < n) {
        double r = 0.0;
#pragma unroll
        for (int q = 0; q < 8; ++q) r += red[q][lane];
        P[(long long)blockIdx.z * sP + (long long)c * n + k] = r;
    }
}

// Per output (one CTA of 1024 threads each): c_i from the partials, the LOO mean and variance of the N points, and
// nlpp[b] = the sum of the per-point terms in a fixed order.  sw / u (single output, may be null): sqrt(w_i) and
// alpha_i / c_i for i < N, zero up to ldv.
__global__ void __launch_bounds__(1024)
loo_point_kernel(const double* __restrict__ P, long long sP, int nch,
                 const double* __restrict__ alpha, const double* __restrict__ y, long long sv, int N,
                 double* __restrict__ mean, double* __restrict__ var, double* __restrict__ nlpp,
                 double* __restrict__ sw, double* __restrict__ u, int ldv)
{
    __shared__ double red[32];
    const double* Pb = P + (long long)blockIdx.x * sP;
    const double* al = alpha + (long long)blockIdx.x * sv;
    const double* yy = y + (long long)blockIdx.x * sv;
    double s = 0.0;
    for (int i = threadIdx.x; i < N; i += 1024) {
        double c = 0.0;
        for (int q = i / TRT_ROWS; q < nch; ++q) c += Pb[(long long)q * N + i];
        const double a = al[i], r = a / c;
        mean[(long long)blockIdx.x * N + i] = yy[i] - r;
        var[(long long)blockIdx.x * N + i] = 1.0 / c;
        s += 0.91893853320467274178 - 0.5 * log(c) + 0.5 * a * r;       // 1/2 log 2pi - 1/2 log c + alpha^2 / (2c)
        if (sw) {
            sw[i] = sqrt(fma(a, r, 1.0) / (2.0 * c));
            u[i] = r;
        }
    }
    if (sw)
        for (int i = N + threadIdx.x; i < ldv; i += 1024) { sw[i] = 0.0; u[i] = 0.0; }
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int q = 0; q < 32; ++q) t += red[q];
        nlpp[blockIdx.x] = t;
    }
}

// S = C diag(sw), full and square, from the lower-stored symmetric C (32x32 tiles through shared memory, grid
// (ld/32, ld/32), block (32, 8)); rows and columns >= N are zero.
__global__ void loo_mirror_scale_kernel(const double* __restrict__ C, int ld, const double* __restrict__ sw,
                                        double* __restrict__ S, int N)
{
    __shared__ double tile[32][33];
    const int bi = blockIdx.y, bj = blockIdx.x;
    if (bj > bi) return;
    const int tx = threadIdx.x, ty = threadIdx.y;
    for (int r = ty; r < 32; r += 8)          // only the lower triangle of a diagonal tile holds C
        if (bi != bj || tx <= r) tile[r][tx] = C[(long long)(bi * 32 + r) * ld + bj * 32 + tx];
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {
        const int row = bi * 32 + r, col = bj * 32 + tx;
        const double v = (bi == bj && tx > r) ? tile[tx][r] : tile[r][tx];
        S[(long long)row * ld + col] = (row < N && col < N) ? v * sw[col] : 0.0;
        if (bi != bj) {        // the mirrored tile: S[bj*32 + r][bi*32 + tx] = C[bi*32 + tx][bj*32 + r] sw[bi*32 + tx]
            const int row2 = bj * 32 + r, col2 = bi * 32 + tx;
            S[(long long)row2 * ld + col2] = (row2 < N && col2 < N) ? tile[tx][r] * sw[col2] : 0.0;
        }
    }
}

// W = G - sym(b alpha^T) in place on the lower triangle of the first N rows (grid (ceil(N/256), N))
__global__ void __launch_bounds__(256)
loo_w_kernel(double* __restrict__ W, int ld, const double* __restrict__ b, const double* __restrict__ alpha, int N)
{
    const int r = blockIdx.y, c = blockIdx.x * 256 + threadIdx.x;
    if (c > r) return;
    W[(long long)r * ld + c] -= 0.5 * fma(b[r], alpha[c], alpha[r] * b[c]);
}
