// qd_warp_path.cuh -- rows of at most 1024 elements: ONE WARP PER ROW, the row
// lives in registers between the reduction and the element-wise pass, so every
// byte crosses HBM exactly once (8 B/elt forward, 16 B/elt fused fwd+bwd).
//
// Layout: lane L of the warp owns elements r*128 + 4L .. 4L+3 of the row
// (r = 0..R-1), i.e. each load/store instruction of the warp covers 512
// contiguous bytes (4 full 128-byte lines).  Rows that are not 16-byte aligned
// (bucket % 4 != 0 or an offset base pointer) use the scalar mapping
// (r*4+j)*32 + L, still fully coalesced.  Row reductions are shuffle
// butterflies of NaN-propagating min / max (warp_min / warp_max, qd_common.cuh).
//
// Consecutive warps stream consecutive rows: the uniform op launches one warp per
// row, the other ops a persistent grid that walks the rows with a grid stride
// (kRowPerWarp).
#pragma once
#include "qd_rowops.cuh"

namespace qd {

constexpr int kWarpCtaThreads = 256;
constexpr int kWarpsPerCta = kWarpCtaThreads / 32;

template <int R, bool VEC>
__device__ __forceinline__ int elem_index(int r, int j, int lane) {
    return VEC ? (r * 128 + lane * 4 + j) : ((r * 4 + j) * 32 + lane);
}

template <int R, bool VEC, bool FULL>
__device__ __forceinline__ void load_row(const float* __restrict__ p, int len, int lane, float (&v)[4 * R]) {
#pragma unroll
    for (int r = 0; r < R; ++r) {
        if (VEC && (FULL || r * 128 + lane * 4 + 4 <= len)) {
            float4 t = ld_stream4(p + r * 128 + lane * 4);
            v[4 * r + 0] = t.x; v[4 * r + 1] = t.y; v[4 * r + 2] = t.z; v[4 * r + 3] = t.w;
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                int e = elem_index<R, VEC>(r, j, lane);
                v[4 * r + j] = (e < len) ? ld_stream1(p + e) : 0.f;
            }
        }
    }
}

template <int R, bool VEC, bool FULL>
__device__ __forceinline__ void store_row(float* __restrict__ p, int len, int lane, const float (&v)[4 * R]) {
#pragma unroll
    for (int r = 0; r < R; ++r) {
        if (VEC && (FULL || r * 128 + lane * 4 + 4 <= len)) {
            st_stream4(p + r * 128 + lane * 4, make_float4(v[4 * r], v[4 * r + 1], v[4 * r + 2], v[4 * r + 3]));
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                int e = elem_index<R, VEC>(r, j, lane);
                if (e < len) st_stream1(p + e, v[4 * r + j]);
            }
        }
    }
}

template <int R, bool VEC, bool FULL>
__device__ __forceinline__ void store_row_u8(uint8_t* __restrict__ p, int len, int lane, const float (&lv)[4 * R]) {
#pragma unroll
    for (int r = 0; r < R; ++r) {
        if (VEC && (FULL || r * 128 + lane * 4 + 4 <= len) && ((reinterpret_cast<uintptr_t>(p) & 3) == 0)) {
            uint32_t w = (uint32_t)(int)lv[4 * r] | ((uint32_t)(int)lv[4 * r + 1] << 8) |
                         ((uint32_t)(int)lv[4 * r + 2] << 16) | ((uint32_t)(int)lv[4 * r + 3] << 24);
            *reinterpret_cast<uint32_t*>(p + r * 128 + lane * 4) = w;
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                int e = elem_index<R, VEC>(r, j, lane);
                if (e < len) p[e] = (uint8_t)(int)lv[4 * r + j];
            }
        }
    }
}

// first index (inside the row) whose value equals `target`; rows are < 2^31 long
template <int R, bool VEC, bool FULL>
__device__ __forceinline__ int first_equal(const float (&v)[4 * R], float target, int len, int lane) {
    int best = 0x7fffffff;
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            int e = elem_index<R, VEC>(r, j, lane);
            if ((FULL || e < len) && v[4 * r + j] == target) best = min(best, e);
        }
    return warp_min_int(best);
}

// One row, one warp.  OP / BWD / WANT_* are compile-time so the hot forward
// kernel carries no dead code.
template <int R, bool VEC, bool FULL>
__device__ __forceinline__ void store_row_u8(uint8_t* __restrict__ p, int len, int lane, const int (&lv)[4 * R]) {
#pragma unroll
    for (int r = 0; r < R; ++r) {
        if (VEC && (FULL || r * 128 + lane * 4 + 4 <= len) && ((reinterpret_cast<uintptr_t>(p) & 3) == 0)) {
            uint32_t w = (uint32_t)lv[4 * r] | ((uint32_t)lv[4 * r + 1] << 8) | ((uint32_t)lv[4 * r + 2] << 16) |
                         ((uint32_t)lv[4 * r + 3] << 24);
            *reinterpret_cast<uint32_t*>(p + r * 128 + lane * 4) = w;
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                int e = elem_index<R, VEC>(r, j, lane);
                if (e < len) p[e] = (uint8_t)lv[4 * r + j];
            }
        }
    }
}

// Fixed-width packed store of a row's levels (the layout of qd_pack_indices): element e of the tensor has its BITS-bit
// code in byte e*BITS/8 at bit (e*BITS)%8.  `p` is the row's first byte, so the row must start on a byte boundary,
// and in the 128-bit lane layout (VEC) lane L's four codes r*128+4L .. +3 are one aligned 4*BITS-bit field: one byte
// store at 2 bits, a 16-bit store at 4, a 32-bit store at 8 (the caller aligns `p` to 4 bytes).  At 1 bit the even
// lane merges its odd neighbour's nibble (one shuffle) and stores the byte.  Codes past `len` are zero and the bytes
// that hold none of the row's codes are not written, so the last byte of the tensor is exactly qd_pack_indices'.
template <int BITS, int R, bool FULL, typename T>
__device__ __forceinline__ void store_row_packed(uint8_t* __restrict__ p, int len, int lane, const T (&lv)[4 * R]) {
    static_assert(BITS == 1 || BITS == 2 || BITS == 4 || BITS == 8, "code width");
    constexpr int kPerByte = 8 / BITS;                 // codes per byte: byte b of a lane holds codes e0 + b*kPerByte ..
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const int e0 = r * 128 + lane * 4;
        uint32_t w = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (FULL || e0 + j < len) w |= (uint32_t)(int)lv[4 * r + j] << (j * BITS);
        if constexpr (BITS == 1) {
            const uint32_t odd = __shfl_down_sync(kFullMask, w, 1);
            if ((lane & 1) == 0 && (FULL || e0 < len)) __stcs(p + r * 16 + (lane >> 1), (uint8_t)(w | (odd << 4)));
        } else {
            uint8_t* dst = p + r * 16 * BITS + lane * (BITS / 2);
            if (FULL || e0 + 4 <= len) {
                if constexpr (BITS == 8) __stcs(reinterpret_cast<uint32_t*>(dst), w);
                else if constexpr (BITS == 4) __stcs(reinterpret_cast<uint16_t*>(dst), (uint16_t)w);
                else __stcs(dst, (uint8_t)w);
            } else {
#pragma unroll
                for (int b = 0; b < BITS / 2; ++b)
                    if (e0 + b * kPerByte < len) dst[b] = (uint8_t)(w >> (8 * b));
            }
        }
    }
}

// The level output of the row kernels: uint8 levels at P.idx8 + base (PACK = 0), or PACK-bit packed codes of the
// row starting at byte base*PACK/8 of P.idx8 (only in the 128-bit lane layout).
template <int PACK, int R, bool VEC, bool FULL, typename T>
__device__ __forceinline__ void store_levels(uint8_t* __restrict__ idx8, int64_t base, int len, int lane, const T (&lv)[4 * R]) {
    if constexpr (PACK == 0) {
        store_row_u8<R, VEC, FULL>(idx8 + base, len, lane, lv);
    } else {
        static_assert(VEC, "the packed store needs the 128-bit lane layout");
        store_row_packed<PACK, R, FULL>(idx8 + base * PACK / 8, len, lane, lv);
    }
}

// AUX is the backward mode for OP_UNIFORM and the centroid-table size class KP for
// OP_NONUNIFORM (power of two >= K; <= 32: table in the lanes of the warp, else shared memory).
template <int OP, int AUX>
using LaneTable = LaneSearch<(OP == OP_NONUNIFORM && AUX <= 32) ? AUX : 1>;

template <int OP, int AUX, int R, bool VEC, bool FULL>
__device__ __forceinline__ void warp_load_row(const Params& P, int64_t row, int lane, float (&v)[4 * R], float (&gv)[4 * R]) {
    constexpr int BWD = (OP == OP_UNIFORM) ? AUX : (int)BWD_OFF;
    const int64_t base = row * P.geo.row_len;
    const int len = FULL ? R * 128 : (int)min(P.geo.row_len, P.geo.n - base);
    load_row<R, VEC, FULL>(P.x + base, len, lane, v);
    if constexpr (BWD != BWD_OFF) load_row<R, VEC, FULL>(P.g + base, len, lane, gv);
}

// ACC_A: r_b accumulation of the min/max backward, chosen by the launcher from whether q is written (qd_quant.cu):
// false = minmax_lane_sum (division mode hoisted, float32 groups), true = one float64 add per element
template <int OP, int AUX, int R, bool VEC, bool FULL, bool ACC_A = false, int PACK = 0>
__device__ __forceinline__ void warp_compute_row(const Params& P, const Centroids& cen, const LaneTable<OP, AUX>& rt, int64_t row,
                                                 int lane, float (&v)[4 * R], float (&gv)[4 * R]) {
    constexpr int BWD = (OP == OP_UNIFORM) ? AUX : (int)BWD_OFF;
    constexpr int KP = (OP == OP_NONUNIFORM) ? AUX : 0;
    constexpr int E = 4 * R;
    const int64_t base = row * P.geo.row_len;
    const int len = FULL ? R * 128 : (int)min(P.geo.row_len, P.geo.n - base);

    RowState rs;
    rs.mean = 0.f;
    const bool pre = (P.mean != nullptr) || (P.max_element > 0.f);
    if (pre) {
        rs.mean = P.mean ? *P.mean : 0.f;
#pragma unroll
        for (int i = 0; i < E; ++i) v[i] = pre_op(v[i], rs.mean, P.max_element);
    }

    // ---- row reduction: beta = min, alpha = max - min ----------------------
    float mn = __int_as_float(0x7f800000), mx = __int_as_float(0xff800000);
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (FULL || elem_index<R, VEC>(r, j, lane) < len) {
                mn = min_nan(mn, v[4 * r + j]);
                mx = max_nan(mx, v[4 * r + j]);
            }
        }
    mn = warp_min(mn);
    mx = warp_max(mx);
    rs.beta = mn;
    rs.alpha = make_alpha(mn, mx);

    if (P.alpha != nullptr && lane == 0) {
        P.alpha[row] = rs.alpha;
        P.beta[row] = rs.beta;
    }
    if (P.argmin != nullptr) {  // first occurrence, like torch.min/max(dim) on CPU
        int imin = first_equal<R, VEC, FULL>(v, mn, len, lane);
        int imax = first_equal<R, VEC, FULL>(v, mx, len, lane);
        if (lane == 0) {
            P.argmin[row] = (imin == 0x7fffffff) ? 0 : imin;  // all-NaN rows: index 0
            P.argmax[row] = (imax == 0x7fffffff) ? 0 : imax;
        }
    }
    if constexpr (OP == OP_STATS) return;

    if constexpr (OP == OP_SCALE) {
        // x_hat in the padded layout: the tail row is filled with x_hat of the
        // last element (help_functions.py:75-76, 83-86)
        const int64_t pbase = row * P.geo.row_len;
        float o[E];
#pragma unroll
        for (int i = 0; i < E; ++i) o[i] = to_unit(v[i], rs.beta, rs.alpha);
        if (FULL) {
            store_row<R, VEC, true>(P.xhat + pbase, len, lane, o);
        } else {
            const int plen = (int)P.geo.row_len;  // padded row length
            if (len < plen) {
                float last = P.x[P.geo.n - 1];
                if (pre) last = pre_op(last, rs.mean, P.max_element);
                last = to_unit(last, rs.beta, rs.alpha);
#pragma unroll
                for (int r = 0; r < R; ++r)
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                        if (elem_index<R, VEC>(r, j, lane) >= len) o[4 * r + j] = last;
            }
            store_row<R, VEC, false>(P.xhat + pbase, plen, lane, o);
        }
        return;
    }

    if constexpr (OP == OP_UNIFORM_STOCH) {
        float qv[E];
        float lv[E];
        Philox rng(P.seed);
#pragma unroll
        for (int r = 0; r < R; ++r) {
            // one Philox block per 4 consecutive elements of the flat tensor
            if (VEC) {
                uint4 rnd = rng(P.offset + (uint64_t)((base + elem_index<R, VEC>(r, 0, lane)) >> 2));
                qv[4 * r + 0] = uniform_quantize_stochastic(v[4 * r + 0], rs, P.S, u01(rnd.x), lv[4 * r + 0]);
                qv[4 * r + 1] = uniform_quantize_stochastic(v[4 * r + 1], rs, P.S, u01(rnd.y), lv[4 * r + 1]);
                qv[4 * r + 2] = uniform_quantize_stochastic(v[4 * r + 2], rs, P.S, u01(rnd.z), lv[4 * r + 2]);
                qv[4 * r + 3] = uniform_quantize_stochastic(v[4 * r + 3], rs, P.S, u01(rnd.w), lv[4 * r + 3]);
            } else {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    int64_t ge = base + elem_index<R, VEC>(r, j, lane);
                    uint4 rnd = rng(P.offset + (uint64_t)(ge >> 2));
                    uint32_t w = (ge & 3) == 0 ? rnd.x : (ge & 3) == 1 ? rnd.y : (ge & 3) == 2 ? rnd.z : rnd.w;
                    qv[4 * r + j] = uniform_quantize_stochastic(v[4 * r + j], rs, P.S, u01(w), lv[4 * r + j]);
                }
            }
        }
        if (pre) {
#pragma unroll
            for (int i = 0; i < E; ++i) qv[i] = __fadd_rn(qv[i], rs.mean);
        }
        if (P.q != nullptr) store_row<R, VEC, FULL>(P.q + base, len, lane, qv);
        if (P.idx8 != nullptr) store_row_u8<R, VEC, FULL>(P.idx8 + base, len, lane, lv);
        return;
    }

    if constexpr (OP == OP_UNIFORM) {
        float qv[E];
        float lv[E];
        const UniformFast uf = make_uniform_fast(rs.alpha, P.S);
        if (uf.ok) {
            // fast level (see qd_rowops.cuh): candidates for the whole row, one warp vote, and the
            // exact IEEE chain only for rows that hold an element near a rounding boundary
            bool unsafe = false;
#pragma unroll
            for (int i = 0; i < E; ++i) lv[i] = fast_level(v[i], rs.beta, uf.c, P.half_minus_band, unsafe);
            if (__any_sync(kFullMask, unsafe)) {
#pragma unroll
                for (int i = 0; i < E; ++i) lv[i] = exact_level(v[i], rs.beta, rs.alpha, P.S);
            }
#pragma unroll
            for (int i = 0; i < E; ++i) qv[i] = from_unit(small_level_to_unit(lv[i], P.S, P.rS), rs.alpha, rs.beta);
        } else {
#pragma unroll
            for (int i = 0; i < E; ++i) {
                const float2 ql = exact_quantize(v[i], rs.beta, rs.alpha, P.S);
                qv[i] = ql.x;
                lv[i] = ql.y;
            }
        }

        if constexpr (BWD == BWD_MINMAX) {
            // Second scaling: the reference re-scales q with the same ScalingFunction
            // object, so alpha', beta', argmin', argmax' are those of q
            // (quant_functions.py:350-363).  q is monotone in the level, so
            // min q / max q are exact float reductions over qv.
            float qmn = __int_as_float(0x7f800000), qmx = __int_as_float(0xff800000);
#pragma unroll
            for (int r = 0; r < R; ++r)
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (FULL || elem_index<R, VEC>(r, j, lane) < len) {
                        qmn = min_nan(qmn, qv[4 * r + j]);
                        qmx = max_nan(qmx, qv[4 * r + j]);
                    }
            qmn = warp_min(qmn);
            qmx = warp_max(qmx);
            rs.beta2 = qmn;
            rs.alpha2 = make_alpha(qmn, qmx);
            int imin = first_equal<R, VEC, FULL>(qv, qmn, len, lane);
            int imax = first_equal<R, VEC, FULL>(qv, qmx, len, lane);
            // r_b = sum_j v_j: float32 inside a 128-bit group, float64 across groups, lanes and (fixed tree) the warp
            const RowDivider div2(rs.alpha2);
            double acc;
            if constexpr (ACC_A) {
                acc = 0.0;
#pragma unroll
                for (int r = 0; r < R; ++r)
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                        if (FULL || elem_index<R, VEC>(r, j, lane) < len)
                            acc += (double)minmax_term(v[4 * r + j], qv[4 * r + j], gv[4 * r + j], rs.beta2, div2);
            } else {
                acc = div2.ok ? minmax_lane_sum<R, VEC, FULL, true>(v, qv, gv, rs.beta2, rs.alpha2, div2, len, lane)
                              : minmax_lane_sum<R, VEC, FULL, false>(v, qv, gv, rs.beta2, rs.alpha2, div2, len, lane);
            }
            const float rb = (float)warp_sum(acc);
            if (imin != imax) {  // +r at argmax', -r at argmin' (the +1/-1 columns of grad_alpha, :380-393)
#pragma unroll
                for (int r = 0; r < R; ++r)
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        int e = elem_index<R, VEC>(r, j, lane);
                        if (e == imax) gv[4 * r + j] = __fadd_rn(gv[4 * r + j], rb);
                        if (e == imin) gv[4 * r + j] = __fadd_rn(gv[4 * r + j], -rb);
                    }
            }
            // (patching the two elements in global memory after the row store instead was measured to be slower: the
            // dependent load-after-store stalls the warp)
        } else if constexpr (BWD == BWD_TRUNC) {
#pragma unroll
            for (int i = 0; i < E; ++i) gv[i] = (fabsf(v[i]) > 1.0f) ? 0.f : gv[i];
        }

        if (P.q != nullptr) {
            if (pre) {
#pragma unroll
                for (int i = 0; i < E; ++i) qv[i] = __fadd_rn(qv[i], rs.mean);  // quant_functions.py:148
            }
            store_row<R, VEC, FULL>(P.q + base, len, lane, qv);
        }
        if (P.idx8 != nullptr) store_levels<PACK, R, VEC, FULL>(P.idx8, base, len, lane, lv);
        if constexpr (BWD != BWD_OFF) store_row<R, VEC, FULL>(P.gout + base, len, lane, gv);
        return;
    }

    if constexpr (OP == OP_NONUNIFORM) {
        float qv[E];
        int li[E];
        // x_hat = (x - beta) / alpha, bit-identical to div.rn.f32: hoisted-reciprocal sequence for the
        // whole row, one warp vote, IEEE routine for the (rare) rows holding an element outside the
        // sequence's proven domain (see RowDivider)
        const RowDivider div(rs.alpha);
        float xh[E];
        unsigned guard = 0xffffffffu;
#pragma unroll
        for (int i = 0; i < E; ++i) {
            const float a = __fsub_rn(v[i], rs.beta);
            xh[i] = div.fast(a);
            guard = RowDivider::guard_fold(guard, a);
        }
        if (__any_sync(kFullMask, div.guard_unsafe(guard))) {
#pragma unroll
            for (int i = 0; i < E; ++i) xh[i] = RowDivider::slow_div(__fsub_rn(v[i], rs.beta), rs.alpha);
        }
        // either rule is a count of per-launch thresholds (qd_rowops.cuh)
        if constexpr (KP <= 32) {
            const float q_lane = rt.row_table(rs.alpha, rs.beta, pre, rs.mean);   // lane L: k_L*alpha + beta (+ mean)
#pragma unroll
            for (int i = 0; i < E; ++i) {
                li[i] = rt.index(xh[i]);
                qv[i] = LaneTable<OP, AUX>::value(q_lane, li[i]);
            }
        } else {
#pragma unroll
            for (int i = 0; i < E; ++i) {
                float kval;
                li[i] = smem_index<KP>(cen.k, cen.t, xh[i], kval);
                qv[i] = from_unit(kval, rs.alpha, rs.beta);
                if (pre) qv[i] = __fadd_rn(qv[i], rs.mean);
            }
        }
        if (P.q != nullptr) store_row<R, VEC, FULL>(P.q + base, len, lane, qv);
        if (P.idx8 != nullptr) store_levels<PACK, R, VEC, FULL>(P.idx8, base, len, lane, li);
        if (P.idx64 != nullptr) {
#pragma unroll
            for (int r = 0; r < R; ++r)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    int e = elem_index<R, VEC>(r, j, lane);
                    if (FULL || e < len) P.idx64[base + e] = (int64_t)li[4 * r + j];
                }
        }
        return;
    }
}

template <int OP, int AUX, int R, bool VEC, bool FULL, bool ACC_A = false, int PACK = 0>
__device__ __forceinline__ void warp_process_row(const Params& P, const Centroids& cen, const LaneTable<OP, AUX>& rt, int64_t row,
                                                 int lane) {
    float v[4 * R], gv[4 * R];
    warp_load_row<OP, AUX, R, VEC, FULL>(P, row, lane, v, gv);
    warp_compute_row<OP, AUX, R, VEC, FULL, ACC_A, PACK>(P, cen, rt, row, lane, v, gv);
}

// Row order.  The uniform op (forward, every backward mode) gives every row its own warp: one CTA per 8 rows
// (warp_rows_grid) instead of a persistent grid of SMs x resident CTAs walking the rows with a grid stride.  The
// hardware then issues CTAs in row order as earlier ones retire, so the rows in flight stay one compact band.  On a
// plain copy of the headline's traffic (tools/stream_ceiling.py: 64 Mi floats in rows of 256, x and g read, q and gout
// written) that order moves 3011 GB/s against 2886 GB/s for the persistent grid at 3 CTAs per SM; 2 / 4 CTAs per SM,
// contiguous per-CTA spans, two rows per warp and L2 evict_first hints all stay at or below 2886 (H100 80GB HBM3,
// 700 W; DESIGN.md section 3).  The other ops keep the persistent grid and hold the NEXT row's loads in flight while
// the current row is reduced, quantized and stored (register double buffering): the centroid op at 384 .. 768 floats
// loses 30-80 % with one row per warp (tools/block_bench.py --small), and stats / scale / stochastic rounding were not
// measured with it.
template <int OP>
constexpr bool kRowPerWarp = (OP == OP_UNIFORM);

// minimum resident CTAs per SM the register allocator must allow: 256-element rows (every
// experiment of the reference) are tuned for 4 x 8 warps per SM (<= 64 registers) in the forward-only
// kernel; the fused min/max kernel spills at 64 registers on sm_90a and runs 3 % faster at 3 CTAs
// (<= 80 registers, no spill; one H100 at 400 W, 5 x 200 back-to-back launches, two interleaved rounds:
// 398-407 -> 385-391 us per launch, identical output bits)
// (measured per kernel: STE / truncated / non-uniform are better with ptxas's own choice, 0 = unconstrained)
template <int OP, int AUX, int R>
constexpr int kMinCtas = (OP == OP_UNIFORM && R == 2 && AUX == (int)BWD_OFF) ? 4
                         : (OP == OP_UNIFORM && R == 2 && AUX == (int)BWD_MINMAX) ? 3
                         : (OP == OP_UNIFORM && R == 8 && AUX != (int)BWD_OFF) ? 2   // 1024-element rows with a gradient: cap at 128 regs
                                                                               : 0;

// PACK: 0 = uint8 levels at P.idx8; 1 / 2 / 4 / 8 = P.idx8 receives the levels as packed codes of that width
// (store_levels; VEC only, every row starting on a byte of the packed stream)
template <int OP, int AUX, int R, bool VEC, bool ACC_A = false, int PACK = 0>
__global__ void __launch_bounds__(kWarpCtaThreads, kMinCtas<OP, AUX, R>) warp_rows_kernel(const __grid_constant__ Params P) {
    __shared__ float s_k[OP == OP_NONUNIFORM ? 256 : 1];
    __shared__ float s_t[OP == OP_NONUNIFORM ? 256 : 1];
    Centroids cen{s_k, s_t, P.num_points};
    LaneTable<OP, AUX> rt;
    const int lane = threadIdx.x & 31;
    if constexpr (OP == OP_NONUNIFORM) {
        centroid_setup(s_k, s_t, P.points, P.num_points, P.rule);
        __syncthreads();
        if constexpr (AUX <= 32) rt.load(cen, lane);
    }
    // with one warp per row (kRowPerWarp) the stride only matters past the 2^31 - 1 CTAs a grid can hold
    const int64_t stride = (int64_t)gridDim.x * kWarpsPerCta;
    int64_t row = (int64_t)blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5);
    // rows [0, full_rows) are complete, 16-byte aligned rows of exactly R*128 elements
    const int64_t full_rows = (VEC && P.geo.row_len == R * 128) ? (P.geo.n / P.geo.row_len) : 0;
    if constexpr (VEC) {
        if constexpr (!kRowPerWarp<OP> && R <= 4) {
            if (row < full_rows) {
                float v[4 * R], gv[4 * R];
                warp_load_row<OP, AUX, R, true, true>(P, row, lane, v, gv);
                while (true) {
                    const int64_t next = row + stride;
                    const bool has_next = next < full_rows;
                    float vn[4 * R], gn[4 * R];
                    if (has_next) warp_load_row<OP, AUX, R, true, true>(P, next, lane, vn, gn);
                    warp_compute_row<OP, AUX, R, true, true, false, PACK>(P, cen, rt, row, lane, v, gv);
                    row = next;
                    if (!has_next) break;
#pragma unroll
                    for (int i = 0; i < 4 * R; ++i) { v[i] = vn[i]; gv[i] = gn[i]; }
                }
            }
        } else {
            for (; row < full_rows; row += stride) warp_process_row<OP, AUX, R, true, true, ACC_A, PACK>(P, cen, rt, row, lane);
        }
    }
    for (; row < P.geo.rows; row += stride) warp_process_row<OP, AUX, R, VEC, false, ACC_A, PACK>(P, cen, rt, row, lane);
}

// grid of the one-warp-per-row ops: one CTA per 8 rows
inline int64_t warp_rows_grid(int64_t rows) {
    const int64_t ctas = (rows + kWarpsPerCta - 1) / kWarpsPerCta;
    return ctas < 0x7fffffff ? ctas : 0x7fffffff;
}

}  // namespace qd
