// qd_attn_tile.cuh -- the first two phases of an attention tile, shared by onmt's global attention (qd_attention.cu)
// and the Transformer's multi-head attention (qd_mha.cu): a CTA of WARPS warps owns up to TILE query rows.
//   1. tile_dots: warp w owns the keys s = w + WARPS*k, lane l the elements j = l + 32i; per row a lane-strided float32
//      sum and a butterfly over the warp.
//   2. softmax_row: one warp per row; max, sum of expf(x - max) (lane-strided, butterfly), then expf(x - max) / sum.
//      qd_mha.cu writes the same row out itself (see there).  softmax_row_bwd is its backward, as global attention's
//      two backward row kernels take it.
// The max is fmaxf, which drops a NaN operand.  qd_common.cuh's warp_max propagates NaN and would change the results
// of rows with NaN scores, so the reductions are defined here and these files do not include qd_common.cuh.
#pragma once
#include <cmath>
#include <cstdint>

namespace qd {
namespace attn {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

__device__ __forceinline__ float warp_fmax(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// For the nt rows u_t = u + t*u_stride of a tile and every key w_s = w + s*w_stride, s < count: lane 0 of the warp
// that owns s calls fin(t, s, u_t . w_s), the dot over len elements.  The sizes are references so that a caller's
// kernel-argument fields are read where the loop uses them, as before they were shared: passed by value, the MHA
// kernels compile to other instructions.
template <int TILE, int WARPS, int UNROLL, class F>
__device__ __forceinline__ void tile_dots(const float* __restrict__ u, const int64_t& u_stride, const float* __restrict__ w,
                                          const int64_t& w_stride, const int64_t& count, const int64_t& len, int nt, F&& fin) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int64_t s = warp; s < count; s += WARPS) {
        const float* ws = w + s * w_stride;
        float acc[TILE];
#pragma unroll
        for (int t = 0; t < TILE; ++t) acc[t] = 0.f;
#pragma unroll UNROLL
        for (int64_t j = lane; j < len; j += 32) {
            const float x = __ldg(ws + j);
#pragma unroll
            for (int t = 0; t < TILE; ++t)
                if (t < nt) acc[t] = __fadd_rn(acc[t], __fmul_rn(__ldg(u + t * u_stride + j), x));
        }
#pragma unroll
        for (int t = 0; t < TILE; ++t) {
            if (t < nt) {
                const float d = warp_sum(acc[t]);
                if (lane == 0) fin(t, s, d);
            }
        }
    }
}

// The softmax of the n scores in row, by the calling warp (lane: the caller's lane): store(s, y) for every s, with
// y = expf(x_s - max) / sum.
template <class F>
__device__ __forceinline__ void softmax_row(const float* row, int64_t n, int lane, F&& store) {
    float m = -INFINITY;
    for (int64_t s = lane; s < n; s += 32) m = fmaxf(m, row[s]);
    m = warp_fmax(m);
    float l = 0.f;
    for (int64_t s = lane; s < n; s += 32) l = __fadd_rn(l, expf(__fsub_rn(row[s], m)));
    l = warp_sum(l);
    for (int64_t s = lane; s < n; s += 32) store(s, __fdiv_rn(expf(__fsub_rn(row[s], m)), l));
}

// The softmax's backward of one row, by the calling warp: row[s] <- p[s] (row[s] - sum_s p[s] row[s]) for the n
// probabilities p, the sum per lane in s order, then a butterfly.
__device__ __forceinline__ void softmax_row_bwd(const float* p, float* row, int64_t n, int lane) {
    float d = 0.f;
    for (int64_t s = lane; s < n; s += 32) d = __fadd_rn(d, __fmul_rn(__ldg(p + s), row[s]));
    d = warp_sum(d);
    for (int64_t s = lane; s < n; s += 32) row[s] = __fmul_rn(__ldg(p + s), __fsub_rn(row[s], d));
}

}  // namespace attn
}  // namespace qd
