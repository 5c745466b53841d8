// qd_plan.cuh -- one launch over every parameter tensor of a model (SURVEY.md
// section 8 f1).  The training loop of the reference quantizes the model one
// tensor at a time (cnn_models/conv_forward_model.py:236-247: 22-60 tensors,
// ~12 stock launches each); most of those tensors are 10-500 elements and are
// pure launch latency.  A plan flattens all rows of all tensors into one row
// space; a warp maps its global row to (tensor, local row) with a binary search
// over the per-tensor row prefix held in shared memory and then runs exactly
// the single-tensor warp path on it.
#pragma once
#include "qd_points_grad.cuh"
#include "qd_warp_path.cuh"

namespace qd {

struct PlanEntry {
    const float* src;
    float* dst;
    float* save;        // optional: full-precision copy of src written by the forward launch (shadow buffer)
    float* mom;         // optional: momentum buffer of the fused optimizer step
    int64_t n;
    int64_t row_start;  // first global row of this tensor
    int64_t rows;
    int64_t row_len;
    float S;            // levels - 1
    float rS;           // RN(1/S)
    float lim;          // 0.5 - S*2^-20
    int vec;            // 16-byte aligned rows
};

constexpr int kPlanSmemEntries = 256;

// Gradient pointers of the backward launch travel BY VALUE in the kernel parameters (up to 256
// tensors = 2 KB): no host->device table copy per step, and the launch can be captured in a
// CUDA graph (a captured memcpy from a temporary host array could not).
constexpr int kPlanGradsByValue = 256;
struct GradTable {
    float* g[kPlanGradsByValue];
};

// forward of one plan row; with a shadow pointer the row is also written, untouched, to the
// master copy (save + quantize in one pass: read 4, write 4 + 4 bytes per element)
template <int R, bool VEC, bool FULL>
__device__ __forceinline__ void plan_forward_row(const Params& P, float* save, int64_t row, int lane) {
    float v[4 * R], gv[4 * R];
    Centroids cen{nullptr, nullptr, 0};
    LaneTable<OP_UNIFORM, BWD_OFF> rt;
    warp_load_row<OP_UNIFORM, BWD_OFF, R, VEC, FULL>(P, row, lane, v, gv);
    if (save != nullptr) {
        const int64_t base = row * P.geo.row_len;
        const int len = FULL ? R * 128 : (int)min(P.geo.row_len, P.geo.n - base);
        store_row<R, VEC, FULL>(save + base, len, lane, v);
    }
    warp_compute_row<OP_UNIFORM, BWD_OFF, R, VEC, FULL>(P, cen, rt, row, lane, v, gv);
}

template <int BWD, int R>
__global__ void __launch_bounds__(kWarpCtaThreads) plan_rows_kernel(const PlanEntry* __restrict__ entries, int count,
                                                                   int64_t total_rows, float* const* __restrict__ grads,
                                                                   int with_save, const __grid_constant__ GradTable gtab) {
    __shared__ int64_t s_start[kPlanSmemEntries];
    const bool in_smem = count <= kPlanSmemEntries;
    if (in_smem) {
        for (int i = threadIdx.x; i < count; i += blockDim.x) s_start[i] = entries[i].row_start;
        __syncthreads();
    }
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * kWarpsPerCta;
    Centroids cen{nullptr, nullptr, 0};
    LaneTable<OP_UNIFORM, BWD_OFF> rt;
    for (int64_t grow = (int64_t)blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5); grow < total_rows; grow += stride) {
        int lo = 0, hi = count - 1;  // largest t with row_start[t] <= grow
        while (lo < hi) {
            int mid = (lo + hi + 1) >> 1;
            int64_t s = in_smem ? s_start[mid] : entries[mid].row_start;
            if (s <= grow) lo = mid; else hi = mid - 1;
        }
        const PlanEntry en = entries[lo];
        Params P;
        P.x = en.src;
        P.q = (BWD == BWD_OFF) ? en.dst : nullptr;
        float* gptr = nullptr;
        if constexpr (BWD != BWD_OFF) gptr = (grads != nullptr) ? grads[lo] : gtab.g[lo];
        P.g = gptr;
        P.gout = gptr;
        P.xhat = nullptr; P.idx8 = nullptr; P.idx64 = nullptr;
        P.alpha = nullptr; P.beta = nullptr; P.argmin = nullptr; P.argmax = nullptr;
        P.mean = nullptr; P.max_element = 0.f; P.points = nullptr; P.num_points = 0; P.rule = 0;
        P.geo.n = en.n; P.geo.row_len = en.row_len; P.geo.rows = en.rows;
        P.S = en.S; P.rS = en.rS; P.half_minus_band = en.lim; P.stochastic = 0; P.seed = 0; P.offset = 0;
        const int64_t row = grow - en.row_start;
        bool vec = en.vec != 0;
        if constexpr (BWD != BWD_OFF) vec = vec && ((reinterpret_cast<uintptr_t>(P.g) & 15) == 0);
        const bool full = (en.row_len == R * 128) && ((row + 1) * en.row_len <= en.n);
        if constexpr (BWD == BWD_OFF) {
            float* save = with_save ? en.save : nullptr;
            if (vec && save != nullptr) vec = (reinterpret_cast<uintptr_t>(save) & 15) == 0;
            if (vec) {
                if (full) plan_forward_row<R, true, true>(P, save, row, lane);
                else plan_forward_row<R, true, false>(P, save, row, lane);
            } else {
                plan_forward_row<R, false, false>(P, save, row, lane);
            }
        } else if (vec) {
            if (full) warp_process_row<OP_UNIFORM, BWD, R, true, true>(P, cen, rt, row, lane);
            else warp_process_row<OP_UNIFORM, BWD, R, true, false>(P, cen, rt, row, lane);
        } else {
            warp_process_row<OP_UNIFORM, BWD, R, false, false>(P, cen, rt, row, lane);
        }
    }
}

}  // namespace qd

// =============================================================================================
// Differentiable-quantization loop (cnn_models/conv_forward_model.py:501-551): every step
// re-quantizes EVERY tensor of the model with its own (changing) list of points and then needs
// every tensor's centroid gradient.  Per tensor that is 3 launches (forward, gradient partials,
// gradient fold) x 22-60 tensors; here it is ONE forward launch and TWO small gradient launches
// for the whole model, all deterministic.
// =============================================================================================
namespace qd {

struct NuEntry {
    const float* src;      // the fixed full-precision tensor (pre-processed path: it never changes)
    float* dst;            // live parameter, receives the quantized values
    uint8_t* idx;          // centroid index per element (saved for the backward, :467-468)
    float* alpha;          // per-row scale (the 'scalingFactor' of the backward) and offset
    float* beta;
    const float* points;   // K ascending centroids in [0, 1], device memory, re-read every launch
    float* grad_points;    // K outputs of the backward
    int64_t n;
    int64_t row_start;     // first global row
    int64_t rows;
    int64_t row_len;
    int64_t blk_start;     // first gradient block of this tensor
    int64_t blocks;        // gradient blocks (each kNuBlockTiles tiles of 1024 elements)
    int K;                 // 1..32
    int vec;               // rows 16-byte aligned in src / dst, idx 4-byte aligned
};

// lane tables of one tensor: thresholds of the midpoint rule straight from the points (:533)
template <int KP>
__device__ __forceinline__ void nu_load_tables(LaneSearch<KP>& ls, const float* __restrict__ points, int K, int lane) {
    const float inf = __int_as_float(0x7f800000);
    const float k0 = (lane < K) ? __ldg(points + lane) : inf;
    const float k1 = (lane + 1 < K) ? __ldg(points + lane + 1) : inf;
    ls.k_lane = k0;
    ls.t_lane = (lane + 1 < K) ? __fadd_rn(k0, __fmul_rn(__fsub_rn(k1, k0), 0.5f)) : inf;
    ls.t1 = (KP >= 2) ? __shfl_sync(kFullMask, ls.t_lane, KP / 2 - 1) : 0.f;
    ls.t2lo = (KP >= 4) ? __shfl_sync(kFullMask, ls.t_lane, KP / 4 - 1) : 0.f;
    ls.t2hi = (KP >= 4) ? __shfl_sync(kFullMask, ls.t_lane, 3 * KP / 4 - 1) : 0.f;
}

template <int KP, int R>
__device__ __forceinline__ void nu_forward_row(const NuEntry& en, int64_t row, int lane) {
    Params P;
    P.x = en.src; P.g = nullptr; P.q = en.dst; P.gout = nullptr; P.xhat = nullptr;
    P.idx8 = en.idx; P.idx64 = nullptr; P.alpha = en.alpha; P.beta = en.beta; P.argmin = nullptr; P.argmax = nullptr;
    P.mean = nullptr; P.max_element = 0.f; P.points = en.points; P.num_points = en.K; P.rule = QD_RULE_MIDPOINT;
    P.geo.n = en.n; P.geo.row_len = en.row_len; P.geo.rows = en.rows;
    P.S = 0.f; P.rS = 0.f; P.half_minus_band = 0.f; P.stochastic = 0; P.seed = 0; P.offset = 0;
    LaneSearch<KP> ls;
    nu_load_tables<KP>(ls, en.points, en.K, lane);
    const Centroids cen{nullptr, nullptr, en.K};
    const bool full = (en.row_len == R * 128) && ((row + 1) * en.row_len <= en.n);
    float v[4 * R], gv[4 * R];
    if (en.vec) {
        if (full) {
            warp_load_row<OP_NONUNIFORM, KP, R, true, true>(P, row, lane, v, gv);
            warp_compute_row<OP_NONUNIFORM, KP, R, true, true>(P, cen, ls, row, lane, v, gv);
        } else {
            warp_load_row<OP_NONUNIFORM, KP, R, true, false>(P, row, lane, v, gv);
            warp_compute_row<OP_NONUNIFORM, KP, R, true, false>(P, cen, ls, row, lane, v, gv);
        }
    } else {
        warp_load_row<OP_NONUNIFORM, KP, R, false, false>(P, row, lane, v, gv);
        warp_compute_row<OP_NONUNIFORM, KP, R, false, false>(P, cen, ls, row, lane, v, gv);
    }
}

template <int R>
__global__ void __launch_bounds__(kWarpCtaThreads) plan_nonuniform_fwd_kernel(const NuEntry* __restrict__ entries, int count,
                                                                             int64_t total_rows) {
    __shared__ int64_t s_start[kPlanSmemEntries];
    const bool in_smem = count <= kPlanSmemEntries;
    if (in_smem) {
        for (int i = threadIdx.x; i < count; i += blockDim.x) s_start[i] = entries[i].row_start;
        __syncthreads();
    }
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * kWarpsPerCta;
    for (int64_t grow = (int64_t)blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5); grow < total_rows; grow += stride) {
        int lo = 0, hi = count - 1;  // largest t with row_start[t] <= grow
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            const int64_t s = in_smem ? s_start[mid] : entries[mid].row_start;
            if (s <= grow) lo = mid; else hi = mid - 1;
        }
        const NuEntry en = entries[lo];
        const int64_t row = grow - en.row_start;
        // table size class: warp-uniform (one tensor per row)
        if (en.K <= 4) nu_forward_row<4, R>(en, row, lane);
        else if (en.K <= 8) nu_forward_row<8, R>(en, row, lane);
        else if (en.K <= 16) nu_forward_row<16, R>(en, row, lane);
        else nu_forward_row<32, R>(en, row, lane);
    }
}

// ---- centroid gradients of every tensor (quant_functions.py:471-506) -----------------------
// grad_points[t][k] = sum_{i in tensor t : idx_i = k} fl32(g_i * alpha_row(i)).  A gradient BLOCK is a
// fixed run of kNuBlockTiles tiles (1024 elements each) inside ONE tensor; one warp reduces one block
// with the conflict-free per-lane column scheme of qd_points_grad.cuh into K float64 partials, a second
// launch folds each tensor's blocks in index order.  The block size is fixed when the plan is built,
// so the summation tree -- and the result -- is the same on every replica and every step.
constexpr int kNuMaxK = 32;

template <int DUMMY = 0>
__global__ void __launch_bounds__(kPgThreads) plan_points_grad_partial(const NuEntry* __restrict__ entries, int count,
                                                                      int64_t total_blocks, int block_tiles,
                                                                      const __grid_constant__ GradTable gtab,
                                                                      float* const* __restrict__ grads,
                                                                      double* __restrict__ partial /*[total_blocks][32]*/) {
    __shared__ float s_col[kPgWarps][kNuMaxK][32];
    __shared__ int64_t s_bstart[kPlanSmemEntries];
    const bool in_smem = count <= kPlanSmemEntries;
    if (in_smem) {
        for (int i = threadIdx.x; i < count; i += blockDim.x) s_bstart[i] = entries[i].blk_start;
        __syncthreads();
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float(*col)[32] = s_col[warp];
    const int64_t stride = (int64_t)gridDim.x * kPgWarps;
    for (int64_t blk = (int64_t)blockIdx.x * kPgWarps + warp; blk < total_blocks; blk += stride) {
        int lo = 0, hi = count - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            const int64_t s = in_smem ? s_bstart[mid] : entries[mid].blk_start;
            if (s <= blk) lo = mid; else hi = mid - 1;
        }
        const NuEntry en = entries[lo];
        const float* g = (grads != nullptr) ? grads[lo] : gtab.g[lo];
        const uint8_t* idx = en.idx;
        const int K = en.K;
        for (int k = 0; k < K; ++k) col[k][lane] = 0.f;
        __syncwarp();
        double acc = 0.0;  // lane k < K owns centroid k's float64 sum
        const int64_t tile0 = (blk - en.blk_start) * block_tiles;
        const bool vec_ok = ((reinterpret_cast<uintptr_t>(g) & 15) == 0) && ((reinterpret_cast<uintptr_t>(idx) & 3) == 0);
        int since_flush = 0;
        for (int tt = 0; tt < block_tiles; ++tt) {
            const int64_t start = (tile0 + tt) * kPgTile;
            if (start >= en.n) break;
            const int len = (int)min((int64_t)kPgTile, en.n - start);
            if (vec_ok && len == kPgTile && (en.rows == 1 || en.row_len % 128 == 0)) {
                float4 gv[8];
                uint32_t iw[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    gv[j] = ld_stream4(g + start + j * 128 + lane * 4);
                    iw[j] = *reinterpret_cast<const uint32_t*>(idx + start + j * 128 + lane * 4);
                }
                int64_t row = (en.rows == 1) ? 0 : start / en.row_len;
                int64_t rem = (en.rows == 1) ? 0 : start - row * en.row_len;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float a = en.alpha[row];
                    if (en.rows != 1) {
                        rem += 128;
                        if (rem >= en.row_len) { rem -= en.row_len; ++row; }
                    }
                    const float pv[4] = {__fmul_rn(gv[j].x, a), __fmul_rn(gv[j].y, a), __fmul_rn(gv[j].z, a), __fmul_rn(gv[j].w, a)};
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        const unsigned id = (iw[j] >> (8 * c)) & 0xffu;
                        if (id < (unsigned)K) col[id][lane] += pv[c];
                    }
                }
            } else {
                for (int e = lane; e < len; e += 32) {
                    const int64_t ge = start + e;
                    const float a = (en.rows == 1) ? en.alpha[0] : en.alpha[ge / en.row_len];
                    const unsigned id = idx[ge];
                    if (id < (unsigned)K) col[id][lane] += __fmul_rn(g[ge], a);
                }
            }
            if (++since_flush == kPgFlushEvery) {  // float32 columns only ever add a few hundred terms
                since_flush = 0;
                acc += flush_column(col, lane, K);
            }
        }
        acc += flush_column(col, lane, K);
        if (lane < K) partial[blk * kNuMaxK + lane] = acc;
    }
}

// Fold of one tensor's gradient blocks, shared by both outputs of the backward.  Lane k < K sums
// centroid k's block partials in index order; the store stage is picked at compile time:
//   NU_FOLD_POINTS  grad_points[k] = (float)s                     (the single-process backward)
//   NU_FOLD_SUMS    sums[t][k] = s, zeros for k >= K              (data parallel: reduced across ranks
//                                                                  in float64, cast once by the finish)
enum { NU_FOLD_POINTS = 0, NU_FOLD_SUMS = 1 };

template <int OUT>
__device__ __forceinline__ void nu_fold_tensor(const NuEntry& en, int t, const double* __restrict__ partial,
                                               double* __restrict__ sums) {
    const int lane = threadIdx.x & 31;   // read here, not passed in: keeps plan_points_grad_final's code as it was
    if (lane < en.K) {
        double s = 0.0;
        for (int64_t b = 0; b < en.blocks; ++b) s += partial[(en.blk_start + b) * kNuMaxK + lane];
        if constexpr (OUT == NU_FOLD_POINTS) en.grad_points[lane] = (float)s;
        else sums[(int64_t)t * kNuMaxK + lane] = s;
    } else if constexpr (OUT == NU_FOLD_SUMS) {
        sums[(int64_t)t * kNuMaxK + lane] = 0.0;
    }
}

// one warp per tensor: lane k folds the tensor's blocks in index order
__global__ void __launch_bounds__(256) plan_points_grad_final(const NuEntry* __restrict__ entries, int count,
                                                              const double* __restrict__ partial) {
    const int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (t >= count) return;
    const NuEntry en = entries[t];
    nu_fold_tensor<NU_FOLD_POINTS>(en, t, partial, nullptr);
}

// the same fold, float64 sums into a caller-owned [count][32] table
__global__ void __launch_bounds__(256) plan_points_grad_sums(const NuEntry* __restrict__ entries, int count,
                                                             const double* __restrict__ partial, double* __restrict__ sums) {
    const int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (t >= count) return;
    const NuEntry en = entries[t];
    nu_fold_tensor<NU_FOLD_SUMS>(en, t, partial, sums);
}

// grad_points[t][k] = (float)(sums[t][k] * scale): the one float32 rounding of a reduced table
__global__ void __launch_bounds__(256) plan_points_grad_finish(const NuEntry* __restrict__ entries, int count,
                                                               const double* __restrict__ sums, double scale) {
    const int lane = threadIdx.x & 31;
    const int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (t >= count) return;
    const NuEntry en = entries[t];
    if (lane < en.K) en.grad_points[lane] = (float)(sums[(int64_t)t * kNuMaxK + lane] * scale);
}

}  // namespace qd

// =============================================================================================
// f1, second half: the end of one quantized-distillation step and the beginning of the next in ONE
// pass over the model (cnn_models/conv_forward_model.py:302-317 then :286-287 of the next step):
//
//     g      <- gradient fix-up of the chosen style, evaluated at the full-precision master w
//     m, w   <- SGD with momentum / Nesterov / weight decay (torch.optim.SGD arithmetic, see below)
//     master <- w                     (what load_state_dict / state_dict kept alive)
//     live   <- uniformQuantization(w)   (what the next forward pass sees)
//
// 24 bytes per element (read w, g, m; write w, m, q) instead of restore 8 + fix-up 12 + SGD 20 +
// save-and-quantize 12.  FMA policy = what torch's multi-tensor SGD kernels compute on CUDA, where
// `a + alpha * b` is contracted:  gd = fma(wd, w, g);  m' = RN(RN(mu*m) + gd)  (mul_ then add_ are two
// kernels there);  gn = fma(mu, m', gd) (Nesterov) or m';  w' = fma(-lr, gn, w).  The first step
// starts from m = 0, which gives m' = gd like torch's clone of the gradient.
// =============================================================================================
namespace qd {

struct SgdParams {
    float lr, momentum, weight_decay;
    int nesterov;
};

// q of a whole row held in registers (every lane, every slot; slots past the row end hold zeros)
template <int E>
__device__ __forceinline__ void quantize_row_regs(const float (&v)[E], float alpha, float beta, float S, float rS, float lim,
                                                  float (&qv)[E]) {
    const UniformFast uf = make_uniform_fast(alpha, S);
    if (uf.ok) {
        float lv[E];
        bool unsafe = false;
#pragma unroll
        for (int i = 0; i < E; ++i) lv[i] = fast_level(v[i], beta, uf.c, lim, unsafe);
        if (__any_sync(kFullMask, unsafe)) {
#pragma unroll
            for (int i = 0; i < E; ++i) lv[i] = exact_level(v[i], beta, alpha, S);
        }
#pragma unroll
        for (int i = 0; i < E; ++i) qv[i] = from_unit(small_level_to_unit(lv[i], S, rS), alpha, beta);
    } else {
#pragma unroll
        for (int i = 0; i < E; ++i) qv[i] = exact_quantize(v[i], beta, alpha, S).x;
    }
}

template <int R, bool VEC, bool FULL>
__device__ __forceinline__ void row_min_max(const float (&v)[4 * R], int len, int lane, float& mn, float& mx) {
    mn = __int_as_float(0x7f800000);
    mx = __int_as_float(0xff800000);
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (FULL || elem_index<R, VEC>(r, j, lane) < len) {
                mn = min_nan(mn, v[4 * r + j]);
                mx = max_nan(mx, v[4 * r + j]);
            }
    mn = warp_min(mn);
    mx = warp_max(mx);
}

template <int BWD, int R, bool VEC, bool FULL>
__device__ __forceinline__ void sgd_step_row(const PlanEntry& en, float* __restrict__ grad, float* __restrict__ mom,
                                             const SgdParams& sp, int64_t row, int lane) {
    constexpr int E = 4 * R;
    const int64_t base = row * en.row_len;
    const int len = FULL ? R * 128 : (int)min(en.row_len, en.n - base);
    float w[E], g[E], m[E], q[E];
    load_row<R, VEC, FULL>(en.save + base, len, lane, w);   // full-precision master
    load_row<R, VEC, FULL>(grad + base, len, lane, g);
    load_row<R, VEC, FULL>(mom + base, len, lane, m);

    // ---- gradient fix-up at the master weights (conv_forward_model.py:249-266) ----------------
    if constexpr (BWD == BWD_TRUNC) {
#pragma unroll
        for (int i = 0; i < E; ++i) g[i] = (fabsf(w[i]) > 1.0f) ? 0.f : g[i];
    } else if constexpr (BWD == BWD_MINMAX) {
        float mn, mx;
        row_min_max<R, VEC, FULL>(w, len, lane, mn, mx);
        RowState rs;
        rs.mean = 0.f;
        rs.beta = mn;
        rs.alpha = make_alpha(mn, mx);
        quantize_row_regs<E>(w, rs.alpha, rs.beta, en.S, en.rS, en.lim, q);
        // second scaling of q (quant_functions.py:350-363): same reductions, same order as the plan's
        // backward launch (warp_compute_row), so fused and unfused steps agree bit for bit
        float qmn = __int_as_float(0x7f800000), qmx = __int_as_float(0xff800000);
#pragma unroll
        for (int r = 0; r < R; ++r)
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (FULL || elem_index<R, VEC>(r, j, lane) < len) {
                    qmn = min_nan(qmn, q[4 * r + j]);
                    qmx = max_nan(qmx, q[4 * r + j]);
                }
        qmn = warp_min(qmn);
        qmx = warp_max(qmx);
        rs.beta2 = qmn;
        rs.alpha2 = make_alpha(qmn, qmx);
        const int imin = first_equal<R, VEC, FULL>(q, qmn, len, lane);
        const int imax = first_equal<R, VEC, FULL>(q, qmx, len, lane);
        const RowDivider div2(rs.alpha2);
        const double acc = div2.ok ? minmax_lane_sum<R, VEC, FULL, true>(w, q, g, rs.beta2, rs.alpha2, div2, len, lane)
                                   : minmax_lane_sum<R, VEC, FULL, false>(w, q, g, rs.beta2, rs.alpha2, div2, len, lane);
        const float rb = (float)warp_sum(acc);
        if (imin != imax) {
#pragma unroll
            for (int r = 0; r < R; ++r)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int e = elem_index<R, VEC>(r, j, lane);
                    if (e == imax) g[4 * r + j] = __fadd_rn(g[4 * r + j], rb);
                    if (e == imin) g[4 * r + j] = __fadd_rn(g[4 * r + j], -rb);
                }
        }
    }

    // ---- torch.optim.SGD (dampening 0) ----------------------------------------------------------
#pragma unroll
    for (int i = 0; i < E; ++i) {
        float gd = g[i];
        if (sp.weight_decay != 0.f) gd = __fmaf_rn(sp.weight_decay, w[i], gd);
        float step = gd;
        if (sp.momentum != 0.f) {
            m[i] = __fadd_rn(__fmul_rn(m[i], sp.momentum), gd);
            step = sp.nesterov ? __fmaf_rn(sp.momentum, m[i], gd) : m[i];
        }
        w[i] = __fmaf_rn(-sp.lr, step, w[i]);
        if constexpr (BWD == BWD_TRUNC) w[i] = fminf(fmaxf(w[i], -1.0f), 1.0f);   // next step's p.data.clamp_(-1, 1) (:240-241)
    }
    store_row<R, VEC, FULL>(en.save + base, len, lane, w);
    if (sp.momentum != 0.f) store_row<R, VEC, FULL>(mom + base, len, lane, m);

    // ---- next step's quantization of the updated weights -----------------------------------------
    float mn, mx;
    row_min_max<R, VEC, FULL>(w, len, lane, mn, mx);
    const float alpha = make_alpha(mn, mx);
    quantize_row_regs<E>(w, alpha, mn, en.S, en.rS, en.lim, q);
    store_row<R, VEC, FULL>(en.dst + base, len, lane, q);
}

template <int BWD, int R>
__global__ void __launch_bounds__(kWarpCtaThreads) plan_sgd_step_kernel(const PlanEntry* __restrict__ entries, int count,
                                                                       int64_t total_rows, float* const* __restrict__ grads,
                                                                       const __grid_constant__ GradTable gtab,
                                                                       const SgdParams sp) {
    __shared__ int64_t s_start[kPlanSmemEntries];
    const bool in_smem = count <= kPlanSmemEntries;
    if (in_smem) {
        for (int i = threadIdx.x; i < count; i += blockDim.x) s_start[i] = entries[i].row_start;
        __syncthreads();
    }
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * kWarpsPerCta;
    for (int64_t grow = (int64_t)blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5); grow < total_rows; grow += stride) {
        int lo = 0, hi = count - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            const int64_t s = in_smem ? s_start[mid] : entries[mid].row_start;
            if (s <= grow) lo = mid; else hi = mid - 1;
        }
        const PlanEntry en = entries[lo];
        float* grad = (grads != nullptr) ? grads[lo] : gtab.g[lo];
        float* mom = en.mom;
        const int64_t row = grow - en.row_start;
        const bool vec = en.vec != 0 && ((reinterpret_cast<uintptr_t>(grad) | reinterpret_cast<uintptr_t>(mom) |
                                          reinterpret_cast<uintptr_t>(en.save)) & 15) == 0;
        const bool full = (en.row_len == R * 128) && ((row + 1) * en.row_len <= en.n);
        if (vec) {
            if (full) sgd_step_row<BWD, R, true, true>(en, grad, mom, sp, row, lane);
            else sgd_step_row<BWD, R, true, false>(en, grad, mom, sp, row, lane);
        } else {
            sgd_step_row<BWD, R, false, false>(en, grad, mom, sp, row, lane);
        }
    }
}

}  // namespace qd

// =============================================================================================
// Long-row plan: bucket_size=None (every tensor is ONE row; the post-mortem setting of the drivers,
// cifar10_test.py:113, 305-317) or rows beyond the warp path.  The per-tensor route costs three launches
// per tensor (chunk partials, fold, apply); here all tensors share them: THREE launches for the model.
//   1. every 16 K-element chunk of every tensor -> (min, max)        [one CTA per chunk]
//   2. one CTA per tensor ROW folds its chunks                        -> alpha, beta
//   3. element-wise pass over all chunks, in reverse (the tail of the model is still in L2)
// =============================================================================================
namespace qd {

constexpr int kPlanChunk = 16384;
constexpr int kPlanChunkThreads = 512;

struct LongEntry {
    const float* src;
    float* dst;
    float* save;          // optional shadow copy
    int64_t n;
    int64_t row_len;      // = n for bucket None, else the bucket
    int64_t rows;
    int64_t chunks_per_row;
    int64_t chunk_start;  // first global chunk
    int64_t row_start;    // first global row
    float S, rS, lim;
};

struct ChunkMinMax { float mn, mx; };
struct RowScale { float alpha, beta; };

__device__ __forceinline__ int plan_find(const int64_t* starts, int count, int64_t v) {
    int lo = 0, hi = count - 1;  // largest t with starts[t] <= v
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (starts[mid] <= v) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(kPlanChunkThreads) plan_long_stats_partial(const LongEntry* __restrict__ entries, int count,
                                                                            const int64_t* __restrict__ chunk_starts,
                                                                            int64_t total_chunks, ChunkMinMax* __restrict__ partial) {
    __shared__ float s_mm[2][kPlanChunkThreads / 32];
    const uint64_t pol_keep = l2_policy_evict_last();
    for (int64_t c = blockIdx.x; c < total_chunks; c += gridDim.x) {
        const LongEntry en = entries[plan_find(chunk_starts, count, c)];
        const int64_t lc = c - en.chunk_start;
        const int64_t row = lc / en.chunks_per_row, chunk = lc % en.chunks_per_row;
        const int64_t row_base = row * en.row_len;
        const int64_t row_end = min(en.row_len, en.n - row_base);
        const int64_t off = chunk * kPlanChunk;
        const int len = (int)min((int64_t)kPlanChunk, row_end - off);
        const float* src = en.src + row_base + off;
        float mn = __int_as_float(0x7f800000), mx = __int_as_float(0xff800000);
        const int vlen = ((reinterpret_cast<uintptr_t>(src) & 15) == 0) ? (len & ~3) : 0;
        for (int e = threadIdx.x * 4; e < vlen; e += kPlanChunkThreads * 4) {
            const float4 t = ld_hint4(src + e, pol_keep);
            mn = min_nan(min_nan(mn, t.x), min_nan(t.y, min_nan(t.z, t.w)));
            mx = max_nan(max_nan(mx, t.x), max_nan(t.y, max_nan(t.z, t.w)));
        }
        for (int e = vlen + threadIdx.x; e < len; e += kPlanChunkThreads) {
            const float t = src[e];
            mn = min_nan(mn, t);
            mx = max_nan(mx, t);
        }
        mn = warp_min(mn);
        mx = warp_max(mx);
        if ((threadIdx.x & 31) == 0) { s_mm[0][threadIdx.x >> 5] = mn; s_mm[1][threadIdx.x >> 5] = mx; }
        __syncthreads();
        if (threadIdx.x < 32) {
            mn = warp_min(s_mm[0][threadIdx.x & 15]);
            mx = warp_max(s_mm[1][threadIdx.x & 15]);
            if (threadIdx.x == 0) { partial[c].mn = mn; partial[c].mx = mx; }
        }
        __syncthreads();
    }
}

// one warp per global row
__global__ void __launch_bounds__(256) plan_long_stats_final(const LongEntry* __restrict__ entries, int count,
                                                             const int64_t* __restrict__ row_starts, int64_t total_rows,
                                                             const ChunkMinMax* __restrict__ partial, RowScale* __restrict__ rowscale) {
    const int lane = threadIdx.x & 31;
    const int64_t grow = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (grow >= total_rows) return;
    const LongEntry en = entries[plan_find(row_starts, count, grow)];
    const int64_t row = grow - en.row_start;
    const ChunkMinMax* p = partial + en.chunk_start + row * en.chunks_per_row;
    float mn = __int_as_float(0x7f800000), mx = __int_as_float(0xff800000);
    for (int64_t c = lane; c < en.chunks_per_row; c += 32) {
        mn = min_nan(mn, p[c].mn);
        mx = max_nan(mx, p[c].mx);
    }
    mn = warp_min(mn);
    mx = warp_max(mx);
    if (lane == 0) {
        rowscale[grow].beta = mn;
        rowscale[grow].alpha = make_alpha(mn, mx);
    }
}

// BWD_OFF: dst <- uniformQuantization(src) (+ shadow <- src);  BWD_TRUNC: grad <- (|src| > 1 ? 0 : grad)
template <int BWD>
__global__ void __launch_bounds__(kPlanChunkThreads) plan_long_apply(const LongEntry* __restrict__ entries, int count,
                                                                    const int64_t* __restrict__ chunk_starts, int64_t total_chunks,
                                                                    const RowScale* __restrict__ rowscale, int with_save,
                                                                    float* const* __restrict__ grads) {
    const uint64_t pol_stream = l2_policy_evict_first();
    for (int64_t it = blockIdx.x; it < total_chunks; it += gridDim.x) {
        const int64_t c = total_chunks - 1 - it;  // reverse: most recently read data first
        const int t = plan_find(chunk_starts, count, c);
        const LongEntry en = entries[t];
        const int64_t lc = c - en.chunk_start;
        const int64_t row = lc / en.chunks_per_row, chunk = lc % en.chunks_per_row;
        const int64_t row_base = row * en.row_len;
        const int64_t row_end = min(en.row_len, en.n - row_base);
        const int64_t g0 = row_base + chunk * kPlanChunk;
        const int len = (int)min((int64_t)kPlanChunk, row_end - chunk * kPlanChunk);
        if constexpr (BWD == BWD_TRUNC) {
            float* g = grads[t] + g0;
            const float* x = en.src + g0;
            for (int e = threadIdx.x; e < len; e += kPlanChunkThreads) {
                if (fabsf(x[e]) > 1.0f) g[e] = 0.f;
            }
            continue;
        }
        const RowScale rsc = rowscale[en.row_start + row];
        const UniformFast uf = make_uniform_fast(rsc.alpha, en.S);
        RowState rs;
        rs.mean = 0.f; rs.alpha = rsc.alpha; rs.beta = rsc.beta;
        const float* x = en.src + g0;
        float* q = en.dst + g0;
        float* sv = (with_save && en.save != nullptr) ? en.save + g0 : nullptr;
        const bool vec = ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(sv)) & 15) == 0;
        const int vlen = vec ? (len & ~3) : 0;
#pragma unroll 2
        for (int e = threadIdx.x * 4; e < vlen; e += kPlanChunkThreads * 4) {
            const float4 tv = *reinterpret_cast<const float4*>(x + e);   // L2-resident from pass 1 when the model fits
            float lv[4];
            const float4 qo = uniform_quantize_auto4(tv, rs.alpha, rs.beta, uf, en.S, en.rS, en.lim, lv);
            if (sv != nullptr) st_hint4(sv + e, tv, pol_stream);
            st_hint4(q + e, qo, pol_stream);
        }
        for (int e = vlen + threadIdx.x; e < len; e += kPlanChunkThreads) {
            const float tv = x[e];
            float lvl;
            const float qv = uniform_quantize_auto(tv, rs, uf, en.S, en.rS, en.lim, lvl);
            if (sv != nullptr) sv[e] = tv;
            q[e] = qv;
        }
    }
}

}  // namespace qd
