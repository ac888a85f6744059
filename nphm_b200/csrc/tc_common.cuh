// wgmma / mbarrier / bulk-copy PTX helpers and the log2-unit softplus shared by the tensor-core kernels (sm_90a).
#pragma once
#include "common.cuh"
#include <cuda_fp16.h>
#include "wgmma.cuh"

namespace nphm {
namespace tc {

constexpr float kS = 144.26950408889634f;            // 100 * log2(e)

// ------------------------------------------------------------------------------------------------ PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
    const uint32_t addr = smem_u32(bar);
    uint32_t done;
    do {
        asm volatile("{\n\t.reg .pred p;\n\t"
                     "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                     "selp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(addr), "r"(parity) : "memory");
    } while (!done);
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// warpgroup MMA ordering: fence before the first wgmma that reads registers written by ordinary instructions, commit the
// issued wgmmas as one group, wait until at most N groups are in flight (their accumulators / operands are then usable)
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of an accumulator / operand register across the asynchronous MMAs
template <int N> __device__ __forceinline__ void wg_reg_fence(float (&d)[N])
{
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int N> __device__ __forceinline__ void wg_reg_fence(uint32_t (&a)[N])
{
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+r"(a[i])::"memory");
}

// wgmma shared-memory descriptor, K-major, no swizzle: 8x(16 B) core matrices of 128 contiguous bytes;
// LBO = byte distance between the two core matrices along K, SBO = between 8-row groups along M / N.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo, uint32_t sbo)
{
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo >> 4) << 16) | ((uint64_t)(sbo >> 4) << 32);
}

// Accumulator layout of a 64 x N warpgroup MMA (fp32): warp w (of the warpgroup) and lane l hold rows 16 w + l / 4 and
// 16 w + l / 4 + 8; d[4 i + 0, 1] = (row, 8 i + 2 (l % 4) + 0, 1), d[4 i + 2, 3] = (row + 8, same columns).  The register A
// operand of a k-step has the same layout: a[0] = row, k 2 (l % 4) + 0, 1 | a[1] = row + 8 | a[2], a[3]: k + 8 - so the
// accumulator columns [16 j, 16 j + 16) of one layer, split to fp16, ARE the A registers of k-step j of the next one.

// softplus in log2 units: sp'(t) = lg2(1 + 2^t) = max(t, 0) + lg2(1 + 2^-|t|)
__device__ __forceinline__ float sp_t(float t)
{
    float e, l;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-fabsf(t)));
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(l) : "f"(1.0f + e));
    return fmaxf(t, 0.0f) + l;
}

// softplus in log2 units with lg2(1 + e) on the FMA pipe: e * P5(e), |error| < 2.2e-6 log2 units = 1.5e-8 in SDF units
// (fp32 evaluation included), i.e. at the round-off level of the activations it produces.  One MUFU (ex2) instead of two.
__device__ __forceinline__ float sp_t_poly5(float t)
{
    float e;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-fabsf(t)));
    float pl = fmaf(e, -0.02645743577f, 0.1234514468f);
    pl = fmaf(pl, e, -0.2795380944f);
    pl = fmaf(pl, e, 0.4582707841f);
    pl = fmaf(pl, e, -0.7182819141f);
    pl = fmaf(pl, e, 1.442553145f);
    return fmaf(pl, e, fmaxf(t, 0.0f));
}
// every other element through the polynomial: balances the MUFU pipe (16 lanes/clk/SM) against the FMA issue slots
__device__ __forceinline__ float sp_sel(float t, int e) { return (e & 1) ? sp_t_poly5(t) : sp_t(t); }

// split two fp32 values into packed fp16 (hi, lo) pairs; element 0 in the low half (lower K index)
__device__ __forceinline__ void split2(float a, float b, uint32_t &hi, uint32_t &lo)
{
    const __half2 h = __floats2half2_rn(a, b);
    const float2 hf = __half22float2(h);
    const __half2 l = __floats2half2_rn(a - hf.x, b - hf.y);
    hi = *reinterpret_cast<const uint32_t *>(&h);
    lo = *reinterpret_cast<const uint32_t *>(&l);
}


}  // namespace tc
}  // namespace nphm
