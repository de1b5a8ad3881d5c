// gg_common.cuh -- shared device helpers for libgraphgan_b200 (sm_90a).
//
// Every arithmetic helper here executes the "canonical" operation sequence written down in
// DESIGN.md section 3, with explicit round-to-nearest intrinsics so that nvcc can neither
// contract nor reassociate anything.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/graphgan_b200.h"

namespace gg {

void set_error(const char *fmt, ...);
int check_cuda(cudaError_t e, const char *what);
int sm_count();
// in place exclusive scan of a[0..n) (device int64); a[n] and *total_out receive the sum.
int launch_exclusive_scan_i64(long long *a, long long n, long long *total_out, cudaStream_t st);

#define GG_CHECK(call)                                   \
    do {                                                 \
        int _rc = gg::check_cuda((call), #call);         \
        if (_rc) return _rc;                             \
    } while (0)
#define GG_REQUIRE(cond, msg)                            \
    do {                                                 \
        if (!(cond)) {                                   \
            gg::set_error("%s: %s", __func__, msg);      \
            return 2;                                    \
        }                                                \
    } while (0)

constexpr unsigned FULL = 0xffffffffu;

// The row strides (floats per embedding row) the kernels are built for: 32, 64, 128, 256 and 512.  Every entry point that
// takes `ld` checks it here, and sampler.pad_embedding picks the stride by the same rule.
constexpr int LD_MAX = 512;
__host__ __device__ constexpr bool ld_supported(int ld) {
    return ld == 32 || ld == 64 || ld == 128 || ld == 256 || ld == LD_MAX;
}
#define GG_LD_MESSAGE "ld must be 32, 64, 128, 256 or 512 (row stride in floats)"

// Philox4x32-10 (Salmon et al. SC'11); only the first two output words are needed.
__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                              uint32_t k0, uint32_t k1, uint32_t &o0, uint32_t &o1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
        c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    o0 = c0; o1 = c1;
}

// 53-bit uniform in [0,1): the MT19937 random_sample construction (all steps exact).
__device__ __forceinline__ double u53(uint32_t a, uint32_t b) {
    return ((double)(a >> 5) * 67108864.0 + (double)(b >> 6)) * (1.0 / 9007199254740992.0);
}

// canonical exp for x <= 0 (oracle/gg_oracle.c: ggo_exp)
__device__ __forceinline__ float exp_c(float x) {
    if (x < -86.0f) return 0.0f;
    const float MAGIC = 12582912.0f;
    const float t = __fmaf_rn(x, 1.44269504088896341f, MAGIC);
    const float n = __fsub_rn(t, MAGIC);
    float r = __fmaf_rn(n, -0.693359375f, x);
    r = __fmaf_rn(n, 2.12194440e-4f, r);
    float p = 1.9875691500e-4f;
    p = __fmaf_rn(p, r, 1.3981999507e-3f);
    p = __fmaf_rn(p, r, 8.3334519073e-3f);
    p = __fmaf_rn(p, r, 4.1665795894e-2f);
    p = __fmaf_rn(p, r, 1.6666665459e-1f);
    p = __fmaf_rn(p, r, 5.0000001201e-1f);
    const float r2 = __fmul_rn(r, r);
    float e = __fmaf_rn(p, r2, r);
    e = __fadd_rn(e, 1.0f);
    const int ni = (int)n;
    return __int_as_float(__float_as_int(e) + (ni << 23));
}

__device__ __forceinline__ float warp_sum_butterfly(float v) {
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) v = __fadd_rn(v, __shfl_xor_sync(FULL, v, off));
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) v = fmaxf(v, __shfl_xor_sync(FULL, v, off));
    return v;
}
// Kogge-Stone inclusive scan over the 32 lanes, fp64, offsets 1,2,4,8,16.
__device__ __forceinline__ double warp_scan_ks(double x, int lane) {
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const double y = __shfl_up_sync(FULL, x, off);
        if (lane >= off) x = __dadd_rn(x, y);
    }
    return x;
}
// 8-lane group reduction (xor 4,2,1) of the per-lane fmaf chains of the canonical dot.
__device__ __forceinline__ float group8_sum(float s) {
    s = __fadd_rn(s, __shfl_xor_sync(FULL, s, 4));
    s = __fadd_rn(s, __shfl_xor_sync(FULL, s, 2));
    s = __fadd_rn(s, __shfl_xor_sync(FULL, s, 1));
    return s;
}

__device__ __forceinline__ float4 ldg4(const float *p) { return __ldg(reinterpret_cast<const float4 *>(p)); }

__device__ __forceinline__ float fma4(const float4 a, const float4 b, float s) {
    s = __fmaf_rn(a.x, b.x, s);
    s = __fmaf_rn(a.y, b.y, s);
    s = __fmaf_rn(a.z, b.z, s);
    s = __fmaf_rn(a.w, b.w, s);
    return s;
}

// ---------------------------------------------------------------- TMA bulk copies + mbarrier (sm_90+; UBLKCP / SYNCS in SASS)
__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long *bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, unsigned parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, unsigned bytes, unsigned long long *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void bulk_s2g(void *dst, const void *src, unsigned bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(smem_u32(src)), "r"(bytes) : "memory");
}

}  // namespace gg
