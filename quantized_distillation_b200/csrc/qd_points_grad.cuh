// qd_points_grad.cuh -- gradient of the loss w.r.t. the K centroids
// (nonUniformQuantization_variable.backward, quant_functions.py:471-506):
//
//     grad_points[k] = sum_{i : idx_i = k} fl32(g_i * alpha_row(i))
//
// The reference makes K masked passes over the tensor; here it is one pass,
// 5 B/elt (float32 g + uint8 idx).  Scatter-by-index without atomics: every lane
// owns a private column of K float32 bins in shared memory, laid out
// bins[k][lane] so that a warp's 32 read-modify-writes always hit 32 distinct
// banks whatever the indices are.  Per element that is one LDS, one FADD and
// one STS, independent of K (K <= 32 per sweep; larger K re-sweeps the data).
// Columns are flushed to float64 every 16 tiles, so float32 only ever adds a
// few hundred terms; the float64 reduction order is fixed (lane tree -> warps
// in order -> CTAs in order): the result is deterministic, which keeps
// data-parallel replicas bit-identical without communication.
#pragma once
#include "qd_common.cuh"

namespace qd {

constexpr int kPgThreads = 256;
constexpr int kPgWarps = kPgThreads / 32;
constexpr int kPgTile = 1024;      // elements per warp work item
constexpr int kPgSweep = 32;       // centroids handled per sweep over the data
constexpr int kPgFlushEvery = 16;  // tiles between float32 -> float64 flushes (<= 512 float32 adds per column)

// float32 -> float64 flush of a warp's columns: lane k (k < kcount) owns centroid k and adds the 32 per-lane
// partials of its row col[k][0..31], walking them with a lane-dependent skew so that the 32 lanes read 32
// different banks at every step.  Cost independent of kcount (32 loads + adds per lane) instead of kcount
// warp-wide float64 reductions; fixed order -> deterministic.  Returns the row sum and clears the row.
__device__ __forceinline__ double flush_column(float (*col)[32], int lane, int kcount) {
    __syncwarp();
    double s = 0.0;
    if (lane < kcount) {
#pragma unroll 8
        for (int j = 0; j < 32; ++j) {
            const int jj = (j + lane) & 31;
            s += (double)col[lane][jj];
            col[lane][jj] = 0.f;
        }
    }
    __syncwarp();
    return s;
}

template <typename IdxT>
__global__ void __launch_bounds__(kPgThreads) points_grad_partial(const float* __restrict__ g,
                                                                 const IdxT* __restrict__ idx,
                                                                 const float* __restrict__ alpha, int K, Geometry geo,
                                                                 double* __restrict__ partial /*[gridDim.x][K]*/) {
    __shared__ float s_col[kPgWarps][kPgSweep][32];
    extern __shared__ double s_acc[];  // [kPgWarps][K]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < kPgWarps * K; i += kPgThreads) s_acc[i] = 0.0;
    __syncthreads();
    float(*col)[32] = s_col[warp];

    // tile mode: 1024 consecutive elements of the flat tensor, alpha uniform per 128-element chunk
    const bool tile_mode = (geo.rows == 1) || (geo.row_len % 128 == 0);
    const int64_t tiles_per_row = (geo.row_len + kPgTile - 1) / kPgTile;
    const int64_t items = tile_mode ? (geo.n + kPgTile - 1) / kPgTile : geo.rows * tiles_per_row;
    const int64_t stride = (int64_t)gridDim.x * kPgWarps;
    const bool vec_ok = sizeof(IdxT) == 1 && ((reinterpret_cast<uintptr_t>(g) & 15) == 0) &&
                        ((reinterpret_cast<uintptr_t>(idx) & 3) == 0);

    for (int kg = 0; kg < K; kg += kPgSweep) {
        const int kcount = min(kPgSweep, K - kg);
        for (int k = 0; k < kcount; ++k) col[k][lane] = 0.f;
        __syncwarp();
        int since_flush = 0;
        for (int64_t item = (int64_t)blockIdx.x * kPgWarps + warp; item < items; item += stride) {
            if (tile_mode) {
                const int64_t start = item * kPgTile;
                const int len = (int)min((int64_t)kPgTile, geo.n - start);
                if (vec_ok && len == kPgTile) {
                    float4 gv[8];
                    uint32_t iw[8];
#pragma unroll
                    for (int j = 0; j < 8; ++j) {  // all 16 loads in flight before the first use
                        gv[j] = ld_stream4(g + start + j * 128 + lane * 4);
                        iw[j] = *reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint8_t*>(idx) + start + j * 128 + lane * 4);
                    }
                    // row of each 128-element chunk: one division per tile, then increments
                    int64_t row = (geo.rows == 1) ? 0 : start / geo.row_len;
                    int64_t rem = (geo.rows == 1) ? 0 : start - row * geo.row_len;
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const float a = alpha[row];
                        if (geo.rows != 1) {
                            rem += 128;
                            if (rem >= geo.row_len) { rem -= geo.row_len; ++row; }
                        }
                        const float pv[4] = {__fmul_rn(gv[j].x, a), __fmul_rn(gv[j].y, a), __fmul_rn(gv[j].z, a),
                                             __fmul_rn(gv[j].w, a)};  // in-place multiply of the reference (:495)
#pragma unroll
                        for (int c = 0; c < 4; ++c) {
                            const unsigned id = ((iw[j] >> (8 * c)) & 0xffu) - (unsigned)kg;
                            if (id < (unsigned)kcount) col[id][lane] += pv[c];
                        }
                    }
                } else {
                    for (int e = lane; e < len; e += 32) {
                        const int64_t ge = start + e;
                        const float a = (geo.rows == 1) ? alpha[0] : alpha[ge / geo.row_len];
                        const unsigned id = (unsigned)idx[ge] - (unsigned)kg;
                        if (id < (unsigned)kcount) col[id][lane] += __fmul_rn(g[ge], a);
                    }
                }
            } else {
                const int64_t row = item / tiles_per_row, sub = item % tiles_per_row;
                const int64_t start = row * geo.row_len + sub * kPgTile;
                const int64_t row_end = min((row + 1) * geo.row_len, geo.n);
                const int len = (int)min((int64_t)kPgTile, row_end - start);
                const float a = alpha[row];
                for (int e = lane; e < len; e += 32) {
                    const unsigned id = (unsigned)idx[start + e] - (unsigned)kg;
                    if (id < (unsigned)kcount) col[id][lane] += __fmul_rn(g[start + e], a);
                }
            }
            if (++since_flush == kPgFlushEvery) {
                since_flush = 0;
                const double s = flush_column(col, lane, kcount);
                if (lane < kcount) s_acc[warp * K + kg + lane] += s;
            }
        }
        {
            const double s = flush_column(col, lane, kcount);
            if (lane < kcount) s_acc[warp * K + kg + lane] += s;
        }
        __syncwarp();
    }
    __syncthreads();
    for (int k = threadIdx.x; k < K; k += kPgThreads) {
        double s = 0.0;
        for (int w = 0; w < kPgWarps; ++w) s += s_acc[w * K + k];
        partial[(int64_t)blockIdx.x * K + k] = s;
    }
}

// one CTA per centroid: 256 threads stride over the CTA partials (a few loads each, all in flight), then a fixed
// tree (lanes by shuffle, warps in order).  One warp per centroid on ONE CTA serialised the fold into L2 round trips
// that took a visible share of the whole op at 64 Mi elements.
__global__ void __launch_bounds__(256) points_grad_final(const double* __restrict__ partial, int nblocks, int K,
                                                         float* __restrict__ out) {
    __shared__ double s_w[8];
    const int k = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double s = 0.0;
    for (int b = threadIdx.x; b < nblocks; b += 256) s += partial[(int64_t)b * K + k];
    s = warp_sum(s);
    if (lane == 0) s_w[warp] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < 8; ++w) t += s_w[w];
        out[k] = (float)t;
    }
}

}  // namespace qd
