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
//
// This header holds what both users of the scheme share; the per-tensor kernels
// are in qd_quant.cu, the whole-model ones in qd_plan.cuh.
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

}  // namespace qd
