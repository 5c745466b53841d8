// qd_common.cuh -- arithmetic and warp primitives shared by every kernel.
//
// Arithmetic contract (DESIGN.md "Bit-exactness"): the reference evaluates the
// quantization as a chain of separately rounded float32 torch ops
// (quantization/quant_functions.py:106-107, 189-191, 142-143).  Every helper
// here therefore uses the explicit round-to-nearest intrinsics (__fsub_rn,
// __fdiv_rn, __fmul_rn, __fadd_rn), which ptxas never contracts into FMAs, and
// rintf (round-half-even, like torch.round).  The translation unit is also
// built with -fmad=false and without fast-math.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "qd_b200.h"

namespace qd {

constexpr float kTolDiffZero = 1e-10f;  // ScalingFunction.tol_diff_zero (quant_functions.py:40)
constexpr unsigned kFullMask = 0xffffffffu;

// ---------------------------------------------------------------- arithmetic
// (x - beta) / alpha : sub_, div_ (quant_functions.py:106-107)
__device__ __forceinline__ float to_unit(float x, float beta, float alpha) {
    return __fdiv_rn(__fsub_rn(x, beta), alpha);
}
// round(x_hat * S) : mul_, round_ (quant_functions.py:189-190)
__device__ __forceinline__ float unit_to_level(float xh, float S) { return rintf(__fmul_rn(xh, S)); }
// (level / S) : div_ (quant_functions.py:191)
__device__ __forceinline__ float level_to_unit(float lvl, float S) { return __fdiv_rn(lvl, S); }
// y*alpha + beta : mul_, add_ (quant_functions.py:142-143)
__device__ __forceinline__ float from_unit(float y, float alpha, float beta) {
    return __fadd_rn(__fmul_rn(y, alpha), beta);
}
// alpha = max - min, tiny -> 1 (quant_functions.py:91-99).  NaN stays NaN like the reference.
__device__ __forceinline__ float make_alpha(float mn, float mx) {
    float a = __fsub_rn(mx, mn);
    return (a < kTolDiffZero) ? 1.0f : a;
}
// optional pre-ops: global mean subtraction, then clamp (quant_functions.py:66-74)
__device__ __forceinline__ float pre_op(float x, float mean, float max_el) {
    x = __fsub_rn(x, mean);
    if (max_el > 0.f) {
        x = (x > max_el) ? max_el : x;
        x = (x < -max_el) ? -max_el : x;
    }
    return x;
}

// min / max that propagate NaN the way torch.min / torch.max do
__device__ __forceinline__ float min_nan(float a, float b) {
    float r;
    asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}
__device__ __forceinline__ float max_nan(float a, float b) {
    float r;
    asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}
// Warp-wide NaN-propagating min / max (sm_90a has no float redux.sync): xor butterfly, then lane 0's value is
// broadcast so that every lane holds the same bits even where the two operands of a step are +0 and -0.
__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = min_nan(v, __shfl_xor_sync(kFullMask, v, o));
    return __shfl_sync(kFullMask, v, 0);
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = max_nan(v, __shfl_xor_sync(kFullMask, v, o));
    return __shfl_sync(kFullMask, v, 0);
}
__device__ __forceinline__ int warp_min_int(int v) { return __reduce_min_sync(kFullMask, v); }
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = __fadd_rn(v, __shfl_xor_sync(kFullMask, v, o));
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFullMask, v, o);
    return v;
}

// ---------------------------------------------------------------- memory
// Streaming 128-bit accesses: every byte is touched once, keep it out of L1.
// (no .nc: the in-place variants write the locations they have just read)
__device__ __forceinline__ float4 ld_stream4(const float* p) {
    float4 r;
    asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
                 : "l"(p));
    return r;
}
__device__ __forceinline__ float ld_stream1(const float* p) {
    float r;
    asm volatile("ld.global.L1::no_allocate.f32 %0, [%1];" : "=f"(r) : "l"(p));
    return r;
}
__device__ __forceinline__ void st_stream4(float* p, float4 v) {
    asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
                 "f"(v.w)
                 : "memory");
}
__device__ __forceinline__ void st_stream1(float* p, float v) {
    asm volatile("st.global.L1::no_allocate.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}

// L2 residency control for the two-pass variants: the first pass tags the row evict_last so that
// it survives until the second pass, everything streamed once (outputs, the second read) is
// tagged evict_first (createpolicy + .L2::cache_hint, the mechanism TMA cache hints use).
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ float4 ld_hint4(const float* p, uint64_t policy) {
    float4 r;
    asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
                 : "l"(p), "l"(policy));
    return r;
}
__device__ __forceinline__ void st_hint4(float* p, float4 v, uint64_t policy) {
    asm volatile("st.global.L1::no_allocate.L2::cache_hint.v4.f32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(p), "f"(v.x), "f"(v.y),
                 "f"(v.z), "f"(v.w), "l"(policy)
                 : "memory");
}

// Tiled helper kernels (inv_scale, pack, unpack): one CTA iteration = one contiguous tile of kTileGroups thread-groups,
// every thread owns kTileU groups of it, 256 groups apart, and issues all kTileU loads before the first use -- 64 B per
// thread in flight instead of 16 (Little: 132 SMs x 2048 threads x 16 B = 4.3 MB does not cover 3.35 TB/s x ~1.5 us).
constexpr int kTileU = 4;
constexpr int kTileGroups = 256 * kTileU;

// ---------------------------------------------------------------- Philox4x32-10
// Counter-based generator for stochastic rounding (quant_functions.py:174-187).
struct Philox {
    uint32_t key0, key1;
    __device__ __forceinline__ Philox(uint64_t seed) : key0((uint32_t)seed), key1((uint32_t)(seed >> 32)) {}
    __device__ __forceinline__ uint4 operator()(uint64_t counter) const {
        uint32_t c0 = (uint32_t)counter, c1 = (uint32_t)(counter >> 32), c2 = 0x9E3779B9u, c3 = 0xBB67AE85u;
        uint32_t k0 = key0, k1 = key1;
#pragma unroll
        for (int i = 0; i < 10; ++i) {
            uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
            uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
            uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
            c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
            k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
        }
        return make_uint4(c0, c1, c2, c3);
    }
};
// torch.rand-style uniform in [0, 1) with 24 random bits
__device__ __forceinline__ float u01(uint32_t r) { return (float)(r >> 8) * 5.9604644775390625e-08f; }

// ---------------------------------------------------------------- geometry
struct Geometry {
    int64_t n;        // elements
    int64_t row_len;  // elements per row (bucket, or n when bucket is None / n < bucket)
    int64_t rows;
};

inline int geometry_of(int64_t n, int64_t bucket, Geometry* g) {
    if (n <= 0 || bucket < 0) return QD_ERR_INVALID_ARG;
    g->n = n;
    if (bucket == 0 || n < bucket) {  // help_functions.py:69-70, 87-90
        g->row_len = n;
        g->rows = 1;
    } else {                          // help_functions.py:79-86, 93
        g->row_len = bucket;
        g->rows = (n + bucket - 1) / bucket;
    }
    return QD_OK;
}

// ---------------------------------------------------------------- fixed-width codes
// four codes in four bytes -> 4*BITS bits, low code first (the qd_pack_indices layout)
template <int BITS>
__device__ __forceinline__ uint32_t squeeze4(uint32_t w) {
    constexpr unsigned mask = (1u << BITS) - 1u;
    return (w & mask) | (((w >> 8) & mask) << BITS) | (((w >> 16) & mask) << (2 * BITS)) | (((w >> 24) & mask) << (3 * BITS));
}

// Whole-model launches: tensor t owns CTAs [cta_start[t], cta_start[t + 1]) of one grid.  The tensor of CTA b, found by
// binary search over cta_start[0..count].
__device__ __forceinline__ int model_tensor_of(const int32_t* __restrict__ cta_start, int count, int b) {
    int lo = 0, hi = count;                       // cta_start[lo] <= b < cta_start[hi]
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(cta_start + mid) <= b) lo = mid;
        else hi = mid;
    }
    return lo;
}

}  // namespace qd
