// qd_grid_path.cuh -- rows longer than QD_MAX_STAGED_BUCKET (in practice
// bucket_size=None on a large tensor: one row spanning the tensor).  A row does
// not fit on one SM, so the op is two streaming passes, 12 B/elt:
//
//   1. grid_stats_partial : every CTA reduces one 16 K-element chunk of a row to
//                           (min, max, first argmin, first argmax)  -> workspace
//   2. grid_stats_final   : one CTA per row folds the chunk partials in index
//                           order (first occurrence wins) -> alpha, beta
//   3. grid_apply         : element-wise pass.  Chunks are visited in REVERSE
//                           order so the tail of the tensor, still resident in
//                           the 50 MB L2 from pass 1, is consumed first.
#pragma once
#include "qd_block_path.cuh"

namespace qd {

constexpr int kGridCtaThreads = 512;
constexpr int kGridChunk = 16384;  // elements per CTA work item
constexpr int64_t kGridKeepBytes = 32ll << 20;  // tail of the tensor pinned in the 50 MB L2 between the two passes

struct ChunkPartial {
    float mn, mx;
    int64_t imin, imax;  // index inside the row
};
struct RowStat {
    float alpha, beta;
};

inline int64_t grid_chunks_per_row(const Geometry& g) { return (g.row_len + kGridChunk - 1) / kGridChunk; }

__global__ void __launch_bounds__(kGridCtaThreads) grid_stats_partial(const __grid_constant__ Params P,
                                                                     ChunkPartial* __restrict__ partial,
                                                                     int64_t chunks_per_row, int want_arg) {
    __shared__ double s_scratch[kGridCtaThreads / 32];
    const bool pre = (P.mean != nullptr) || (P.max_element > 0.f);
    const float mean = P.mean ? *P.mean : 0.f;
    const int64_t items = P.geo.rows * chunks_per_row;
    // the apply pass walks the tensor backwards: pin the last kGridKeepBytes of it in L2 (evict_last),
    // let the rest stream through (evict_first), so that the first part of pass 2 is served by L2
    const uint64_t pol_keep = l2_policy_evict_last(), pol_stream = l2_policy_evict_first();
    for (int64_t item = blockIdx.x; item < items; item += gridDim.x) {
        const int64_t row = item / chunks_per_row, chunk = item % chunks_per_row;
        const int64_t row_base = row * P.geo.row_len;
        const int64_t row_end = min(P.geo.row_len, P.geo.n - row_base);  // elements in this row
        const int64_t off = chunk * kGridChunk;
        const int len = (int)min((int64_t)kGridChunk, row_end - off);
        const float* src = P.x + row_base + off;
        const uint64_t pol = ((P.geo.n - (row_base + off)) * (int64_t)sizeof(float) <= kGridKeepBytes) ? pol_keep : pol_stream;
        float mn = __int_as_float(0x7f800000), mx = __int_as_float(0xff800000);
        const bool vec = ((reinterpret_cast<uintptr_t>(src) & 15) == 0);
        const int vlen = vec ? (len & ~3) : 0;
        for (int e = threadIdx.x * 4; e < vlen; e += kGridCtaThreads * 4) {
            float4 t = ld_hint4(src + e, pol);
            if (pre) {
                t.x = pre_op(t.x, mean, P.max_element); t.y = pre_op(t.y, mean, P.max_element);
                t.z = pre_op(t.z, mean, P.max_element); t.w = pre_op(t.w, mean, P.max_element);
            }
            mn = min_nan(min_nan(mn, t.x), min_nan(t.y, min_nan(t.z, t.w)));
            mx = max_nan(max_nan(mx, t.x), max_nan(t.y, max_nan(t.z, t.w)));
        }
        for (int e = vlen + threadIdx.x; e < len; e += kGridCtaThreads) {
            float t = ld_stream1(src + e);
            if (pre) t = pre_op(t, mean, P.max_element);
            mn = min_nan(mn, t);
            mx = max_nan(mx, t);
        }
        mn = cta_minmax<true>(mn, reinterpret_cast<float*>(s_scratch));
        mx = cta_minmax<false>(mx, reinterpret_cast<float*>(s_scratch));
        int imin = 0x7fffffff, imax = 0x7fffffff;
        if (want_arg) {  // second look at the chunk (L2-resident) for the first occurrence
            for (int e = threadIdx.x; e < len; e += kGridCtaThreads) {
                float t = src[e];
                if (pre) t = pre_op(t, mean, P.max_element);
                if (t == mn) imin = min(imin, e);
                if (t == mx) imax = min(imax, e);
            }
            imin = cta_min_int(imin, reinterpret_cast<int*>(s_scratch));
            imax = cta_min_int(imax, reinterpret_cast<int*>(s_scratch));
        }
        if (threadIdx.x == 0) {
            ChunkPartial cp;
            cp.mn = mn; cp.mx = mx;
            cp.imin = (imin == 0x7fffffff) ? -1 : off + imin;
            cp.imax = (imax == 0x7fffffff) ? -1 : off + imax;
            partial[item] = cp;
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256) grid_stats_final(const __grid_constant__ Params P,
                                                        const ChunkPartial* __restrict__ partial,
                                                        RowStat* __restrict__ rowstat, int64_t chunks_per_row) {
    __shared__ double s_scratch[8];
    const int64_t row = blockIdx.x;
    const ChunkPartial* p = partial + row * chunks_per_row;
    float mn = __int_as_float(0x7f800000), mx = __int_as_float(0xff800000);
    for (int64_t c = threadIdx.x; c < chunks_per_row; c += blockDim.x) {
        mn = min_nan(mn, p[c].mn);
        mx = max_nan(mx, p[c].mx);
    }
    mn = cta_minmax<true>(mn, reinterpret_cast<float*>(s_scratch));
    mx = cta_minmax<false>(mx, reinterpret_cast<float*>(s_scratch));
    if (threadIdx.x == 0) {
        RowStat rs;
        rs.beta = mn;
        rs.alpha = make_alpha(mn, mx);
        rowstat[row] = rs;
        if (P.alpha != nullptr) { P.alpha[row] = rs.alpha; P.beta[row] = rs.beta; }
        if (P.argmin != nullptr) {  // first chunk that attains the extreme holds the first occurrence
            int64_t imin = 0, imax = 0;
            bool fmin = false, fmax = false;
            for (int64_t c = 0; c < chunks_per_row && !(fmin && fmax); ++c) {
                if (!fmin && p[c].mn == mn && p[c].imin >= 0) { imin = p[c].imin; fmin = true; }
                if (!fmax && p[c].mx == mx && p[c].imax >= 0) { imax = p[c].imax; fmax = true; }
            }
            P.argmin[row] = imin;
            P.argmax[row] = imax;
        }
    }
}

// One complete, 16-byte aligned chunk of the centroid op: four 128-bit loads in flight, exact
// x_hat through the hoisted reciprocal with ONE slow-path branch per group of four elements.
// KP <= 32: threshold search and value lookup through the lanes of the warp (LaneSearch; every
// thread of the CTA runs the same trip count, so the shuffles are warp-uniform); larger tables
// are searched in shared memory.
template <int KP>
__device__ __forceinline__ void nonuniform_chunk(const float* __restrict__ x, float* __restrict__ q, uint8_t* __restrict__ idx8,
                                                 const Centroids& cen, const RowState& rs, const RowDivider& div,
                                                 uint64_t pol_stream) {
    constexpr int kPer = 4;
    constexpr bool LANES = KP <= 32;
    const unsigned thr_bits = __float_as_uint(div.thr()) - 1u;
    LaneSearch<LANES ? KP : 1> ls;
    float q_lane = 0.f;
    if constexpr (LANES) {
        ls.load(cen, threadIdx.x & 31);
        q_lane = ls.row_table(rs.alpha, rs.beta, false, 0.f);
    }
#pragma unroll 1
    for (int it = 0; it < kGridChunk / (kGridCtaThreads * 4 * kPer); ++it) {
        float4 xv4[kPer];
#pragma unroll
        for (int u = 0; u < kPer; ++u) xv4[u] = ld_hint4(x + (it * kPer + u) * (kGridCtaThreads * 4) + threadIdx.x * 4, pol_stream);
#pragma unroll
        for (int u = 0; u < kPer; ++u) {
            const int e = (it * kPer + u) * (kGridCtaThreads * 4) + threadIdx.x * 4;
            const float a[4] = {__fsub_rn(xv4[u].x, rs.beta), __fsub_rn(xv4[u].y, rs.beta), __fsub_rn(xv4[u].z, rs.beta),
                                __fsub_rn(xv4[u].w, rs.beta)};
            float xh[4];
            unsigned guard = 0xffffffffu;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                xh[j] = div.fast(a[j]);
                guard = RowDivider::guard_fold(guard, a[j]);
            }
            if (!div.ok || guard < thr_bits) {
#pragma unroll
                for (int j = 0; j < 4; ++j) xh[j] = RowDivider::slow_div(a[j], rs.alpha);
            }
            float qv[4];
            int id[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if constexpr (LANES) {
                    id[j] = ls.index(xh[j]);
                    qv[j] = LaneSearch<LANES ? KP : 1>::value(q_lane, id[j]);
                } else {
                    float kval;
                    id[j] = smem_index<KP>(cen.k, cen.t, xh[j], kval);
                    qv[j] = from_unit(kval, rs.alpha, rs.beta);
                }
            }
            if (q != nullptr) st_hint4(q + e, make_float4(qv[0], qv[1], qv[2], qv[3]), pol_stream);
            if (idx8 != nullptr)
                *reinterpret_cast<uint32_t*>(idx8 + e) =
                    (uint32_t)id[0] | ((uint32_t)id[1] << 8) | ((uint32_t)id[2] << 16) | ((uint32_t)id[3] << 24);
        }
    }
}

// element-wise pass; BWD_MINMAX is not offered on this path (the reference
// refuses bucket_size=None for it, quant_functions.py:332-334)
template <int OP, int BWD>
__global__ void __launch_bounds__(kGridCtaThreads) grid_apply(const __grid_constant__ Params P,
                                                             const RowStat* __restrict__ rowstat,
                                                             int64_t chunks_per_row) {
    __shared__ float s_k[OP == OP_NONUNIFORM ? 256 : 1];
    __shared__ float s_t[OP == OP_NONUNIFORM ? 256 : 1];
    Centroids cen{s_k, s_t, P.num_points};
    if constexpr (OP == OP_NONUNIFORM) {
        centroid_setup(s_k, s_t, P.points, P.num_points, P.rule);
        __syncthreads();
    }
    const bool pre = (P.mean != nullptr) || (P.max_element > 0.f);
    const float mean = P.mean ? *P.mean : 0.f;
    const int64_t items = P.geo.rows * chunks_per_row;
    const uint64_t pol_stream = l2_policy_evict_first();
    for (int64_t it = blockIdx.x; it < items; it += gridDim.x) {
        const int64_t item = items - 1 - it;  // reverse: most recently read data first
        const int64_t row = item / chunks_per_row, chunk = item % chunks_per_row;
        const int64_t row_base = row * P.geo.row_len;
        const int64_t row_end = min(P.geo.row_len, P.geo.n - row_base);
        const int64_t off = chunk * kGridChunk;
        RowState rs;
        rs.mean = mean;
        rs.alpha = rowstat[row].alpha;
        rs.beta = rowstat[row].beta;
        const UniformFast uf = make_uniform_fast(rs.alpha, P.S);
        const RowDivider rowdiv(rs.alpha);
        if constexpr (OP == OP_SCALE) {
            // padded layout: positions past the end of the tail row repeat x_hat of the last element
            const int plen = (int)min((int64_t)kGridChunk, P.geo.row_len - off);
            float lastv = P.x[P.geo.n - 1];
            if (pre) lastv = pre_op(lastv, mean, P.max_element);
            const float last = to_unit(lastv, rs.beta, rs.alpha);
            for (int e = threadIdx.x; e < plen; e += kGridCtaThreads) {
                float o = last;
                if (off + e < row_end) {
                    float t = P.x[row_base + off + e];
                    if (pre) t = pre_op(t, mean, P.max_element);
                    o = to_unit(t, rs.beta, rs.alpha);
                }
                st_stream1(P.xhat + row_base + off + e, o);
            }
            continue;
        }
        const int len = (int)min((int64_t)kGridChunk, row_end - off);
        const int64_t g0 = row_base + off;
        const bool vec = (((reinterpret_cast<uintptr_t>(P.x + g0) | reinterpret_cast<uintptr_t>(P.q + g0) |
                            reinterpret_cast<uintptr_t>(P.g + g0) | reinterpret_cast<uintptr_t>(P.gout + g0)) & 15) == 0) &&
                         ((reinterpret_cast<uintptr_t>(P.idx8 + g0) & 3) == 0);
        const int vlen = vec ? (len & ~3) : 0;
        if constexpr (OP == OP_UNIFORM) {
            // hot case: a complete, aligned chunk of the plain uniform op -- four float4 loads per
            // thread in flight before the first use, streaming stores
            if (vec && len == kGridChunk && !P.stochastic && P.idx8 == nullptr && P.idx64 == nullptr && !pre) {
                constexpr int kPer = 4;
#pragma unroll 1
                for (int it = 0; it < kGridChunk / (kGridCtaThreads * 4 * kPer); ++it) {
                    float4 xv4[kPer], gv4[kPer];
#pragma unroll
                    for (int u = 0; u < kPer; ++u) {
                        const int e = (it * kPer + u) * (kGridCtaThreads * 4) + threadIdx.x * 4;
                        xv4[u] = ld_hint4(P.x + g0 + e, pol_stream);
                        if constexpr (BWD != BWD_OFF) gv4[u] = ld_hint4(P.g + g0 + e, pol_stream);
                    }
#pragma unroll
                    for (int u = 0; u < kPer; ++u) {
                        const int e = (it * kPer + u) * (kGridCtaThreads * 4) + threadIdx.x * 4;
                        float lv4[4];
                        const float4 qo = uniform_quantize_auto4(xv4[u], rs.alpha, rs.beta, uf, P.S, P.rS, P.half_minus_band, lv4);
                        if (P.q != nullptr) st_hint4(P.q + g0 + e, qo, pol_stream);
                        if constexpr (BWD != BWD_OFF) {
                            if constexpr (BWD == BWD_TRUNC) {
                                gv4[u].x = (fabsf(xv4[u].x) > 1.0f) ? 0.f : gv4[u].x;
                                gv4[u].y = (fabsf(xv4[u].y) > 1.0f) ? 0.f : gv4[u].y;
                                gv4[u].z = (fabsf(xv4[u].z) > 1.0f) ? 0.f : gv4[u].z;
                                gv4[u].w = (fabsf(xv4[u].w) > 1.0f) ? 0.f : gv4[u].w;
                            }
                            st_hint4(P.gout + g0 + e, gv4[u], pol_stream);
                        }
                    }
                }
                continue;
            }
        }
        if constexpr (OP == OP_NONUNIFORM) {
            // same structure for the centroid op: complete aligned chunk, uint8 (or no) indices;
            // table size class and index rule are resolved once per chunk, not per element
            if (vec && len == kGridChunk && P.idx64 == nullptr && !pre) {
                const float* xs = P.x + g0;
                float* qs = P.q ? P.q + g0 : nullptr;
                uint8_t* is = P.idx8 ? P.idx8 + g0 : nullptr;
                if (cen.K <= 4) nonuniform_chunk<4>(xs, qs, is, cen, rs, rowdiv, pol_stream);
                else if (cen.K <= 8) nonuniform_chunk<8>(xs, qs, is, cen, rs, rowdiv, pol_stream);
                else if (cen.K <= 16) nonuniform_chunk<16>(xs, qs, is, cen, rs, rowdiv, pol_stream);
                else if (cen.K <= 32) nonuniform_chunk<32>(xs, qs, is, cen, rs, rowdiv, pol_stream);
                else if (cen.K <= 64) nonuniform_chunk<64>(xs, qs, is, cen, rs, rowdiv, pol_stream);
                else nonuniform_chunk<256>(xs, qs, is, cen, rs, rowdiv, pol_stream);
                continue;
            }
        }
        for (int e0 = threadIdx.x * 4; e0 < len; e0 += kGridCtaThreads * 4) {
            const bool v4 = e0 + 4 <= vlen;
            const int cnt = min(4, len - e0);
            float xv[4], gv[4] = {0.f, 0.f, 0.f, 0.f}, qv[4], lv[4];
            if (v4) {
                float4 t = *reinterpret_cast<const float4*>(P.x + g0 + e0);  // L2-resident from pass 1 when it fits
                xv[0] = t.x; xv[1] = t.y; xv[2] = t.z; xv[3] = t.w;
                if constexpr (BWD != BWD_OFF) {
                    float4 u = ld_stream4(P.g + g0 + e0);
                    gv[0] = u.x; gv[1] = u.y; gv[2] = u.z; gv[3] = u.w;
                }
            } else {
                for (int j = 0; j < 4; ++j) {
                    xv[j] = (j < cnt) ? P.x[g0 + e0 + j] : 0.f;
                    if constexpr (BWD != BWD_OFF) gv[j] = (j < cnt) ? P.g[g0 + e0 + j] : 0.f;
                }
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                float t = pre ? pre_op(xv[j], mean, P.max_element) : xv[j];
                if constexpr (OP == OP_UNIFORM) {
                    if (P.stochastic) {
                        Philox rng(P.seed);
                        const int64_t ge = g0 + e0 + j;
                        uint4 rnd = rng(P.offset + (uint64_t)(ge >> 2));
                        uint32_t w = (ge & 3) == 0 ? rnd.x : (ge & 3) == 1 ? rnd.y : (ge & 3) == 2 ? rnd.z : rnd.w;
                        qv[j] = uniform_quantize_stochastic(t, rs, P.S, u01(w), lv[j]);
                    } else {
                        qv[j] = uniform_quantize_auto(t, rs, uf, P.S, P.rS, P.half_minus_band, lv[j]);
                    }
                    if constexpr (BWD == BWD_TRUNC) gv[j] = (fabsf(t) > 1.0f) ? 0.f : gv[j];
                } else {  // OP_NONUNIFORM: exact x_hat through the hoisted reciprocal, unrolled table search
                    const float xh = rowdiv.exact(__fsub_rn(t, rs.beta));
                    float kval;
                    int id;
                    if (cen.K <= 4) id = smem_index<4>(cen.k, cen.t, xh, kval);
                    else if (cen.K <= 16) id = smem_index<16>(cen.k, cen.t, xh, kval);
                    else id = smem_index<256>(cen.k, cen.t, xh, kval);
                    lv[j] = (float)id;
                    qv[j] = from_unit(kval, rs.alpha, rs.beta);
                }
                if (pre) qv[j] = __fadd_rn(qv[j], mean);
            }
            if (v4) {
                if (P.q != nullptr) st_stream4(P.q + g0 + e0, make_float4(qv[0], qv[1], qv[2], qv[3]));
                if constexpr (BWD != BWD_OFF) st_stream4(P.gout + g0 + e0, make_float4(gv[0], gv[1], gv[2], gv[3]));
                if (P.idx8 != nullptr)
                    *reinterpret_cast<uint32_t*>(P.idx8 + g0 + e0) =
                        (uint32_t)(int)lv[0] | ((uint32_t)(int)lv[1] << 8) | ((uint32_t)(int)lv[2] << 16) |
                        ((uint32_t)(int)lv[3] << 24);
            } else {
                for (int j = 0; j < cnt; ++j) {
                    if (P.q != nullptr) P.q[g0 + e0 + j] = qv[j];
                    if constexpr (BWD != BWD_OFF) P.gout[g0 + e0 + j] = gv[j];
                    if (P.idx8 != nullptr) P.idx8[g0 + e0 + j] = (uint8_t)(int)lv[j];
                }
            }
            if (P.idx64 != nullptr)
                for (int j = 0; j < cnt; ++j) P.idx64[g0 + e0 + j] = (int64_t)lv[j];
        }
    }
}

}  // namespace qd
