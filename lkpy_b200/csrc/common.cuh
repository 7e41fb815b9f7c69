// common.cuh — shared device/host helpers for the sm_90a kernels.
#pragma once

#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdio>
#include <cstring>

#include "../../include/lkpy_b200.h"

namespace lk {

void set_error(const char *fmt, ...);

#define LK_CUDA_TRY(expr)                                                                  \
    do {                                                                                   \
        cudaError_t _e = (expr);                                                           \
        if (_e != cudaSuccess) {                                                           \
            ::lk::set_error("%s failed at %s:%d: %s", #expr, __FILE__, __LINE__,           \
                            cudaGetErrorString(_e));                                       \
            return LK_ERR_CUDA;                                                            \
        }                                                                                  \
    } while (0)

#define LK_REQUIRE(cond, code, ...)       \
    do {                                  \
        if (!(cond)) {                    \
            ::lk::set_error(__VA_ARGS__); \
            return (code);                \
        }                                 \
    } while (0)

int sm_count();

// Diagnostic switches (capi.cu): defaults, overridden once from the LK_* environment variables at
// first use and afterwards only through lk_set_option.  -1 = "not set, use the built-in choice".
struct Options {
    int als_tc = 1;             // 0: SIMT ALS kernel even where the tensor-core kernel applies
    int als_tf32 = 1;           // 0: fp32 / non-uniformly weighted rows stay on the SIMT kernel
    int knn_warps = -1;         // warps per CTA of the kNN build (8, 16, 32)
    int knn_ctas = -1;          // resident CTAs per SM of the kNN build
    int knn_score_ctas = -1;    // resident CTAs per SM of the dense (all-items) scoring kernel (1..3)
};
Options &options();

constexpr unsigned FULL = 0xffffffffu;

// read-once global loads that do not allocate in L1 (streams that would otherwise evict the small tables
// every CTA keeps re-reading)
__device__ __forceinline__ int ld_stream_s32(const int32_t *p)
{
    int v;
    asm volatile("ld.global.nc.L1::no_allocate.s32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ float ld_stream_f32(const float *p)
{
    float v;
    asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
    return v;
}

// ---------------------------------------------------------------------------
// PTX wrappers: mbarrier, bulk async copy (the TMA engine's 1-D path, SASS UBLKCP) and per-lane cp.async
// ---------------------------------------------------------------------------

__device__ __forceinline__ uint32_t smem_u32(const void *p)
{
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}

__device__ __forceinline__ void mbar_fence_init()
{
    // make the inits visible to the async proxy
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
                 "r"(bytes)
                 : "memory");
}

__device__ __forceinline__ void mbar_arrive(uint64_t *bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity)
{
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}

__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
    while (!mbar_try_wait(bar, parity)) {
    }
}

// global -> shared bulk copy, completion signalled on an mbarrier (bytes % 16 == 0,
// both addresses 16-byte aligned)
__device__ __forceinline__ void bulk_g2s(void *smem_dst, const void *gmem_src, uint32_t bytes,
                                         uint64_t *bar)
{
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
        ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}

// global -> shared copy of one 16-byte granule through L2 only (cp.async.cg, SASS LDGSTS; both addresses
// 16-byte aligned).  Unlike the bulk copy it takes its operands per lane, and it writes through the generic proxy.
__device__ __forceinline__ void cp_async_16(void *smem_dst, const void *gmem_src)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}

// the lane index, read from %laneid each time: values derived from it are then recomputed where they are used
// rather than hoisted and held in registers across a whole loop
__device__ __forceinline__ uint32_t lane_id()
{
    uint32_t l;
    asm volatile("mov.u32 %0, %%laneid;" : "=r"(l));
    return l;
}

// arrive on the mbarrier once every cp.async this thread issued before has landed.  .noinc: the arrival counts
// against the count the barrier was initialised with (one per arriving thread).
__device__ __forceinline__ void cp_async_mbar_arrive(uint64_t *bar)
{
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// generic-proxy writes to smem must be fenced before the async proxy overwrites/reads them
__device__ __forceinline__ void fence_proxy_async()
{
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// next work index from an atomic counter, or INT_MAX once the (optional) cancel flag is raised — the flag is
// written by the host from another stream while the kernel runs, hence the uncached load
__device__ __forceinline__ int fetch_work(int32_t *counter, const int32_t *cancel)
{
    if (cancel != nullptr && *reinterpret_cast<const volatile int32_t *>(cancel) != 0) return 0x7fffffff;
    return atomicAdd(counter, 1);
}

__device__ __forceinline__ float warp_sum(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
    return v;
}

__device__ __forceinline__ int warp_incl_scan(int v, int lane)
{
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int t = __shfl_up_sync(FULL, v, o);
        if (lane >= o) v += t;
    }
    return v;
}

__device__ __forceinline__ float bf16_bits_to_f32(uint32_t hi16)
{
    return __uint_as_float(hi16 << 16);
}

}  // namespace lk
