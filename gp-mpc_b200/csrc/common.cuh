// Shared helpers for the gpmpc CUDA translation unit (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>

#define GPMPC_TILE 128          // all internal matrices are padded to a multiple of this
#define GPMPC_MAX_DEVICES 64

// Lets kernel Kern use `bytes` of dynamic shared memory (a launch above 48 KB needs it).  The attribute is per device, so
// it is set once per device; setting it twice is harmless.  Devices past GPMPC_MAX_DEVICES set it at every call.
template <auto Kern>
static cudaError_t smem_opt_in(int bytes)
{
    static std::atomic<bool> done[GPMPC_MAX_DEVICES];
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    const bool cached = dev >= 0 && dev < GPMPC_MAX_DEVICES;
    if (cached && done[dev].load(std::memory_order_acquire)) return cudaSuccess;
    e = cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess && cached) done[dev].store(true, std::memory_order_release);
    return e;
}

#define CUDA_TRY(expr)                                                        \
    do {                                                                      \
        cudaError_t _e = (expr);                                              \
        if (_e != cudaSuccess) {                                              \
            set_error(h, "%s:%d %s -> %s", __FILE__, __LINE__, #expr,         \
                      cudaGetErrorString(_e));                                \
            return GPMPC_ERR_CUDA;                                            \
        }                                                                     \
    } while (0)

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// The dynamic shared buffer rounded up to the 1024-byte period of the TMA 128B swizzle.  The rounding is taken on the
// 32-bit shared address and applied as an element offset from smem_raw, so the pointer keeps the shared state space
// and fragment reads compile to LDS.  (Rounding the generic pointer through uintptr_t loses it: every read becomes a
// generic LD.E with 64-bit address arithmetic.)
__device__ __forceinline__ double* smem_align1024(double* smem_raw) {
    const uint32_t b = smem_u32(smem_raw);
    return smem_raw + ((((b + 1023u) & ~1023u) - b) >> 3);
}

// 16-byte asynchronous global->shared copy (LDGSTS), L2-only caching: tiles are
// streamed once per CTA, reuse happens in L2 across CTAs.
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n"
                 :: "r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() {
    asm volatile("cp.async.commit_group;\n" ::: "memory");
}
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;\n" :: "n"(N) : "memory");
}

// fp64 tensor-core MMA: D(8x8) = A(8x4,row) * B(4x8,col) + C.  SASS: DMMA.8x8x4.
// lane l holds A[l/4][l%4], B[k=l%4][n=l/4], C/D[l/4][2*(l%4)+{0,1}].
__device__ __forceinline__ void dmma884(double& d0, double& d1, double a, double b) {
    asm volatile(
        "mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
        : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}

// fp64 tensor-core MMA: D(16x8) = A(16x16,row) * B(16x8,col) + C.  SASS: DMMA.16x8x16 (8x the work of DMMA.8x8x4).
// lane l = 4 g + t holds A[g + 8 (i & 1)][kappa(t, i >> 1)] in a[i], B[kappa(t, j)][g] in b[j] and
// C/D[g + 8 (i >> 1)][2 t + (i & 1)] in d[i].  kappa(t, j) is the k index the hardware assigns to register slot j of
// lane group t; a[2j], a[2j+1] and b[j] of a lane share it.  The MMA sums over k, so a caller may put any k into slot
// (t, j) as long as it puts the same k into A and B.
__device__ __forceinline__ void dmma16816(double (&d)[4], const double (&a)[8], const double (&b)[4]) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
        "{%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
        : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
        : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
          "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ---- mbarrier primitives for the TMA tensor-map feeds: expect_tx -> SASS SYNCS
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// bounded wait: a protocol error traps instead of hanging the GPU.  The bound is wall time
// (%globaltimer, ~20 s), not a spin count, so debuggers / compute-sanitizer / MPS time slicing
// cannot trip it.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    uint32_t ok = 0, spins = 0;
    uint64_t t0 = 0;
    do {
        asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}\n"
                     : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
        if (!ok && (++spins & 0xfffu) == 0) {
            uint64_t now;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
            if (t0 == 0) t0 = now;
            else if (now - t0 > 20000000000ull) __trap();
        }
    } while (!ok);
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" :: "r"(smem_u32(bar)) : "memory");
}
// L2 eviction-priority policies for streaming (evict_first) and re-used (evict_last) operands
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t p; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;\n" : "=l"(p)); return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
    uint64_t p; asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;\n" : "=l"(p)); return p;
}
