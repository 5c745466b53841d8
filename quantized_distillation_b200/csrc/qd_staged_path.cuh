// qd_staged_path.cuh -- rows of 1025 .. QD_MAX_STAGED_BUCKET floats for the deterministic
// uniform op (forward, every backward mode, fused) and the centroid op: ONE CTA PER ROW, one
// pass over HBM, the row staged in shared memory by the TMA bulk-copy engine.
//
// Pipeline.  The row buffer is a ring of 32 KB chunks, each with its own mbarrier:
//   sweep 1 reduces chunk c (min / max) as soon as its copy has landed, while chunks c+1.. are
//           still in flight;
//   sweep 2 (quantize, gradient, stores) walks the chunks in the same order, and as soon as the
//           CTA is done with chunk c it hands the slot back to the copy engine, which refills it
//           with chunk c of the NEXT row this CTA will process -- so the read of row r+1 overlaps
//           the compute and the writes of row r even when a single row fills the shared memory
//           of the SM.  Short rows (<= kTwoStageMaxRow) additionally keep two whole rows in
//           flight per CTA (STAGES = 2).
// Per row the CTA synchronises once per chunk plus once or twice for the row scalars.
//
// Min/max ("complicated") backward in TWO sweeps.  The reference re-scales the quantized row q
// with its own extremes (quant_functions.py:350-363).  Every float32 op between x and q
// (x-beta, /alpha, *S, round, /S, *alpha, +beta) is monotone non-decreasing for alpha > 0, so
// min(q) = Q(min x) and max(q) = Q(max x) EXACTLY (NaN rows give NaN both ways): beta', alpha'
// follow from the two row scalars of sweep 1 and no sweep over q is needed to find them.  Only two
// elements of the gradient change (first argmax' / argmin' of q), so sweep 2 streams g once, writes
// gout = g, accumulates r_b and the two positions, and thread 0 patches the two elements afterwards.
#pragma once
#include <type_traits>

#include "qd_block_path.cuh"

namespace qd {

constexpr int kTwoStageMaxRow = 3072;  // floats; rows up to here keep two rows in flight per CTA (measured crossover)

struct StagedScratch {
    float mm[2][2][32];  // [exchange parity][min | max][warp]
    int im[2][2][32];    // first positions
    double acc[2][32];   // r_b partials
};

// T threads per CTA, chosen by row length (qd_quant.cu): short rows want MANY small CTAs per SM (cheap
// barriers, many rows in flight), rows that fill the shared memory of an SM want one large CTA (all
// the warps the SM can hold).  Registers are capped at 64 so that 2048 / T CTAs fit.
template <int OP, int BWD, int STAGES, int T>
__global__ void __launch_bounds__(T, T == 64 ? 16 : T == 128 ? 8 : T == 256 ? 4 : T == 512 ? 2 : 1)
staged_rows_kernel(const __grid_constant__ Params P, int stage_floats) {
    static_assert(OP == OP_UNIFORM || OP == OP_NONUNIFORM, "staged path: deterministic uniform / centroid op");
    extern __shared__ __align__(128) float s_dyn[];
    __shared__ __align__(8) uint64_t s_bar[STAGES][kMaxStageChunks];
    __shared__ float s_k[OP == OP_NONUNIFORM ? 256 : 1];
    __shared__ float s_t[OP == OP_NONUNIFORM ? 256 : 1];
    __shared__ StagedScratch sc;
    constexpr int NW = T / 32;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    Centroids cen{s_k, s_t, P.num_points};
    if constexpr (OP == OP_NONUNIFORM) centroid_setup(s_k, s_t, P.points, P.num_points, P.rule);
    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s)
            for (int c = 0; c < kMaxStageChunks; ++c) mbar_init(&s_bar[s][c], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const bool pre = (P.mean != nullptr) || (P.max_element > 0.f);
    const float mean = P.mean ? *P.mean : 0.f;
    const float max_el = P.max_element;
    const uint64_t pol_stream = l2_policy_evict_first();
    const int64_t rows = P.geo.rows, row_len = P.geo.row_len;
    uint32_t phase0 = 0, phase1 = 0;  // bit c = parity the next wait on chunk c of stage 0 / 1 must see
    int xchg = 0;

    // the copy engine's share of row `it` (it-th row of this CTA): chunk c, if that row exists and is
    // 16-byte aligned.  Called by thread 0 only, after every thread is done with the slot.
    auto issue_chunk = [&](int64_t it, int c) {
        const int64_t row = (int64_t)blockIdx.x + it * gridDim.x;
        if (row >= rows) return;
        const int64_t base = row * row_len;
        const int len = (int)min(row_len, P.geo.n - base);
        const float* src = P.x + base;
        if ((reinterpret_cast<uintptr_t>(src) & 15) != 0) return;  // unaligned row: staged by ld.global at consume time
        const int bulk_len = len & ~3;
        const int off = c * kStageChunk;
        if (off >= bulk_len) return;
        float* buf = s_dyn + (STAGES == 2 ? (int)(it & 1) : 0) * stage_floats;
        uint64_t* bar = &s_bar[STAGES == 2 ? (int)(it & 1) : 0][c];
        const uint32_t bytes = (uint32_t)min(kStageChunk, bulk_len - off) * 4u;
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy reads of the slot precede the async write
        mbar_expect_tx(bar, bytes);
        tma_bulk_g2s(buf + off, src + off, bytes, bar);
    };
    if (tid == 0) {
        for (int s = 0; s < STAGES; ++s)
            for (int c = 0; c < kMaxStageChunks; ++c) issue_chunk(s, c);
    }

    for (int64_t it = 0;; ++it) {
        const int64_t row = (int64_t)blockIdx.x + it * gridDim.x;
        if (row >= rows) break;
        const int stage = STAGES == 2 ? (int)(it & 1) : 0;
        float* buf = s_dyn + stage * stage_floats;
        const int64_t base = row * row_len;
        const int len = (int)min(row_len, P.geo.n - base);
        const float* src = P.x + base;
        const bool gvec = (reinterpret_cast<uintptr_t>(src) & 15) == 0;
        const int bulk_len = gvec ? (len & ~3) : 0;
        const int nchunks = (bulk_len + kStageChunk - 1) / kStageChunk;
        const int len4 = len & ~3;  // the shared-memory copy is always 16-byte aligned
        // 128-bit global accesses to the other tensors of this row
        const bool ovec = (((reinterpret_cast<uintptr_t>(P.q + base) | reinterpret_cast<uintptr_t>(P.gout + base) |
                             reinterpret_cast<uintptr_t>(P.g + base)) & 15) == 0) &&
                          ((reinterpret_cast<uintptr_t>(P.idx8 + base) & 3) == 0);

        // ---- sweep 1: min / max as the chunks land ---------------------------------------------
        for (int e = bulk_len + tid; e < len; e += T) buf[e] = ld_stream1(src + e);  // tail / unaligned rows
        float mn = __int_as_float(0x7f800000), mx = __int_as_float(0xff800000);
        uint32_t phase = stage ? phase1 : phase0;
        for (int c = 0; c < nchunks; ++c) {
            mbar_wait(&s_bar[stage][c], (phase >> c) & 1u);
            phase ^= (1u << c);
            const int off = c * kStageChunk;
            const int cl = min(kStageChunk, bulk_len - off);
#pragma unroll 4
            for (int e = tid * 4; e < cl; e += T * 4) {
                float4 t = *reinterpret_cast<const float4*>(buf + off + e);
                if (pre) {
                    t.x = pre_op(t.x, mean, max_el); t.y = pre_op(t.y, mean, max_el);
                    t.z = pre_op(t.z, mean, max_el); t.w = pre_op(t.w, mean, max_el);
                    *reinterpret_cast<float4*>(buf + off + e) = t;
                }
                mn = min_nan(min_nan(mn, t.x), min_nan(t.y, min_nan(t.z, t.w)));
                mx = max_nan(max_nan(mx, t.x), max_nan(t.y, max_nan(t.z, t.w)));
            }
        }
        if (stage) phase1 = phase; else phase0 = phase;
        for (int e = bulk_len + tid; e < len; e += T) {  // same thread that staged the element
            float t = buf[e];
            if (pre) { t = pre_op(t, mean, max_el); buf[e] = t; }
            mn = min_nan(mn, t);
            mx = max_nan(mx, t);
        }
        {
            mn = warp_min(mn);
            mx = warp_max(mx);
            const int par = xchg++ & 1;
            if (lane == 0) { sc.mm[par][0][warp] = mn; sc.mm[par][1][warp] = mx; }
            __syncthreads();  // also: the whole row (incl. pre-op rewrites and the tail) is visible to everyone
            mn = warp_min(sc.mm[par][0][lane & (NW - 1)]);
            mx = warp_max(sc.mm[par][1][lane & (NW - 1)]);
        }
        RowState rs;
        rs.mean = mean;
        rs.beta = mn;
        rs.alpha = make_alpha(mn, mx);
        if (P.alpha != nullptr && tid == 0) { P.alpha[row] = rs.alpha; P.beta[row] = rs.beta; }
        if (P.argmin != nullptr) {  // first occurrence of the extremes (idx_min_rows / idx_max_rows of the reference)
            int imin = 0x7fffffff, imax = 0x7fffffff;
            for (int e = tid; e < len; e += T) {
                const float t = buf[e];
                if (t == mn) imin = min(imin, e);
                if (t == mx) imax = min(imax, e);
            }
            imin = warp_min_int(imin);
            imax = warp_min_int(imax);
            const int par = xchg++ & 1;
            if (lane == 0) { sc.im[par][0][warp] = imin; sc.im[par][1][warp] = imax; }
            __syncthreads();
            imin = warp_min_int(sc.im[par][0][lane & (NW - 1)]);
            imax = warp_min_int(sc.im[par][1][lane & (NW - 1)]);
            if (tid == 0) {
                P.argmin[row] = (imin == 0x7fffffff) ? 0 : imin;
                P.argmax[row] = (imax == 0x7fffffff) ? 0 : imax;
            }
        }

        // ---- sweep 2, chunk by chunk; a finished chunk slot goes back to the copy engine --------
        // (rows that were not bulk-copied have no chunk barriers: they run as one chunk)
        const int sweep_chunks = max(nchunks, 1);
        auto chunk_range = [&](int c, int& lo, int& hi) {
            lo = c * kStageChunk;
            hi = (c == sweep_chunks - 1) ? len4 : min(len4, lo + kStageChunk);
        };
        // the row that inherits this stage may have MORE chunks than this one (rows that are not 16-byte
        // aligned run as a single chunk): the last release also covers every higher chunk index
        auto release = [&](int c) {
            if (tid == 0) {
                issue_chunk(it + STAGES, c);
                if (c == sweep_chunks - 1)
                    for (int c2 = c + 1; c2 < kMaxStageChunks; ++c2) issue_chunk(it + STAGES, c2);
            }
        };
        auto chunk_done = [&](int c) {
            __syncthreads();  // every thread is done reading chunk c of this stage
            release(c);
        };

        if constexpr (OP == OP_UNIFORM) {
            const UniformFast uf = make_uniform_fast(rs.alpha, P.S);
            float qlo = 0.f, qhi = 0.f, rb = 0.f;
            double acc = 0.0;
            int imin2 = 0x7fffffff, imax2 = 0x7fffffff;
            RowDivider div2(1.0f);
            if constexpr (BWD == BWD_MINMAX) {
                float lv;
                qlo = uniform_quantize_auto(mn, rs, uf, P.S, P.rS, P.half_minus_band, lv);  // = min q, see header
                qhi = uniform_quantize_auto(mx, rs, uf, P.S, P.rS, P.half_minus_band, lv);  // = max q
                rs.beta2 = qlo;
                rs.alpha2 = make_alpha(qlo, qhi);
                div2 = RowDivider(rs.alpha2);
            }
            // FASTDIV: the row's alpha' lets both divisions of the min/max term use the hoisted reciprocal
            // (row-uniform, so the test is made once per row instead of twice per element)
            auto sweep = [&](auto fast_tag) {
                constexpr bool FASTDIV = decltype(fast_tag)::value;
                auto term = [&](float xv, float qv, float gv) -> float {
                    const float qh = FASTDIV ? div2.fast(__fsub_rn(qv, rs.beta2)) : RowDivider::slow_div(__fsub_rn(qv, rs.beta2), rs.alpha2);
                    const float xs = FASTDIV ? div2.fast(__fsub_rn(xv, rs.beta2)) : RowDivider::slow_div(__fsub_rn(xv, rs.beta2), rs.alpha2);
                    return __fmul_rn(gv, __fsub_rn(qh, xs));   // v_j = g_j (q_hat_j - x_hat_j)  (quant_functions.py:400)
                };
                for (int c = 0; c < sweep_chunks; ++c) {
                    int lo, hi;
                    chunk_range(c, lo, hi);
#pragma unroll 2
                    for (int e = lo + tid * 4; e < hi; e += T * 4) {
                        const float4 t = *reinterpret_cast<const float4*>(buf + e);
                        float4 gv = make_float4(0.f, 0.f, 0.f, 0.f);
                        if constexpr (BWD != BWD_OFF) {
                            gv = ovec ? ld_hint4(P.g + base + e, pol_stream)
                                      : make_float4(P.g[base + e], P.g[base + e + 1], P.g[base + e + 2], P.g[base + e + 3]);
                        }
                        float lv[4];
                        float4 qo = uniform_quantize_auto4(t, rs.alpha, rs.beta, uf, P.S, P.rS, P.half_minus_band, lv);
                        if constexpr (BWD == BWD_TRUNC) {
                            gv.x = (fabsf(t.x) > 1.0f) ? 0.f : gv.x; gv.y = (fabsf(t.y) > 1.0f) ? 0.f : gv.y;
                            gv.z = (fabsf(t.z) > 1.0f) ? 0.f : gv.z; gv.w = (fabsf(t.w) > 1.0f) ? 0.f : gv.w;
                        }
                        if constexpr (BWD == BWD_MINMAX) {
                            if (qo.x == qlo) imin2 = min(imin2, e);
                            if (qo.y == qlo) imin2 = min(imin2, e + 1);
                            if (qo.z == qlo) imin2 = min(imin2, e + 2);
                            if (qo.w == qlo) imin2 = min(imin2, e + 3);
                            if (qo.x == qhi) imax2 = min(imax2, e);
                            if (qo.y == qhi) imax2 = min(imax2, e + 1);
                            if (qo.z == qhi) imax2 = min(imax2, e + 2);
                            if (qo.w == qhi) imax2 = min(imax2, e + 3);
                            // four float32 terms are added in float32 (three roundings of ~6e-8 relative, far inside the
                            // 1e-6 budget of the float32-vs-float64 summation order), then the group joins the float64 sum
                            const float v4 = __fadd_rn(__fadd_rn(term(t.x, qo.x, gv.x), term(t.y, qo.y, gv.y)),
                                                       __fadd_rn(term(t.z, qo.z, gv.z), term(t.w, qo.w, gv.w)));
                            acc += (double)v4;
                        }
                        if constexpr (BWD != BWD_OFF) {
                            if (ovec) st_hint4(P.gout + base + e, gv, pol_stream);
                            else { P.gout[base + e] = gv.x; P.gout[base + e + 1] = gv.y; P.gout[base + e + 2] = gv.z; P.gout[base + e + 3] = gv.w; }
                        }
                        if (P.q != nullptr) {
                            if (pre) { qo.x = __fadd_rn(qo.x, mean); qo.y = __fadd_rn(qo.y, mean); qo.z = __fadd_rn(qo.z, mean); qo.w = __fadd_rn(qo.w, mean); }
                            if (ovec) st_hint4(P.q + base + e, qo, pol_stream);
                            else { P.q[base + e] = qo.x; P.q[base + e + 1] = qo.y; P.q[base + e + 2] = qo.z; P.q[base + e + 3] = qo.w; }
                        }
                        if (P.idx8 != nullptr) {
                            if (ovec) *reinterpret_cast<uint32_t*>(P.idx8 + base + e) =
                                    (uint32_t)(int)lv[0] | ((uint32_t)(int)lv[1] << 8) | ((uint32_t)(int)lv[2] << 16) | ((uint32_t)(int)lv[3] << 24);
                            else for (int j = 0; j < 4; ++j) P.idx8[base + e + j] = (uint8_t)(int)lv[j];
                        }
                    }
                    if (c == sweep_chunks - 1) {
                        for (int e = len4 + tid; e < len; e += T) {  // scalar tail of the row
                            const float t = buf[e];
                            float lvl;
                            const float qv = uniform_quantize_auto(t, rs, uf, P.S, P.rS, P.half_minus_band, lvl);
                            if constexpr (BWD != BWD_OFF) {
                                float gv = P.g[base + e];
                                if constexpr (BWD == BWD_TRUNC) gv = (fabsf(t) > 1.0f) ? 0.f : gv;
                                if constexpr (BWD == BWD_MINMAX) {
                                    if (qv == qlo) imin2 = min(imin2, e);
                                    if (qv == qhi) imax2 = min(imax2, e);
                                    acc += (double)term(t, qv, gv);
                                }
                                P.gout[base + e] = gv;
                            }
                            if (P.q != nullptr) P.q[base + e] = pre ? __fadd_rn(qv, mean) : qv;
                            if (P.idx8 != nullptr) P.idx8[base + e] = (uint8_t)(int)lvl;
                        }
                    }
                    if (BWD != BWD_MINMAX || c + 1 < sweep_chunks) chunk_done(c);
                }
            };
            if (BWD == BWD_MINMAX && div2.ok) sweep(std::true_type{});
            else sweep(std::false_type{});
            if constexpr (BWD == BWD_MINMAX) {
                // r_b and the two positions: fixed reduction tree (lanes, then warps in order) -> deterministic
                acc = warp_sum(acc);
                imin2 = warp_min_int(imin2);
                imax2 = warp_min_int(imax2);
                const int par = xchg++ & 1;
                if (lane == 0) { sc.acc[par][warp] = acc; sc.im[par][0][warp] = imin2; sc.im[par][1][warp] = imax2; }
                __syncthreads();  // = chunk_done of the last chunk; also orders the gout stores before the patch below
                release(sweep_chunks - 1);
                if (warp == 0) {
                    const double tot = warp_sum(lane < NW ? sc.acc[par][lane] : 0.0);
                    imin2 = warp_min_int(sc.im[par][0][lane & (NW - 1)]);
                    imax2 = warp_min_int(sc.im[par][1][lane & (NW - 1)]);
                    rb = (float)tot;
                    if (lane == 0 && imin2 != imax2) {  // +r at argmax', -r at argmin' (quant_functions.py:380-393)
                        float* pmax = P.gout + base + imax2;
                        float* pmin = P.gout + base + imin2;
                        *pmax = __fadd_rn(__ldcg(pmax), rb);
                        *pmin = __fadd_rn(__ldcg(pmin), -rb);
                    }
                }
            }
        } else {  // OP_NONUNIFORM
            const RowDivider div(rs.alpha);
            const unsigned thr_bits = __float_as_uint(div.thr()) - 1u;
            // KP: size class of the lane table (compile time inside the sweep, chosen once per launch)
            auto sweep = [&](auto kp_tag) {
                constexpr int KP = decltype(kp_tag)::value;
                constexpr bool LANES = KP <= 32;
                LaneSearch<LANES ? KP : 1> ls;
                float q_lane = 0.f;
                if constexpr (LANES) {
                    ls.load(cen, lane);
                    q_lane = ls.row_table(rs.alpha, rs.beta, pre, mean);
                }
                for (int c = 0; c < sweep_chunks; ++c) {
                    int lo, hi;
                    chunk_range(c, lo, hi);
                    // warp-uniform trip count (the lane search shuffles): a warp owns 128 consecutive floats per step
                    for (int e0 = lo + warp * 128; e0 < hi; e0 += T * 4) {
                        const int e = e0 + lane * 4;
                        const bool act = e < hi;
                        const float4 t = act ? *reinterpret_cast<const float4*>(buf + e) : make_float4(0.f, 0.f, 0.f, 0.f);
                        const float a[4] = {__fsub_rn(t.x, rs.beta), __fsub_rn(t.y, rs.beta), __fsub_rn(t.z, rs.beta), __fsub_rn(t.w, rs.beta)};
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
                        float qq[4];
                        int ii[4];
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            if constexpr (LANES) {
                                ii[j] = ls.index(xh[j]);
                                qq[j] = LaneSearch<LANES ? KP : 1>::value(q_lane, ii[j]);
                            } else {
                                float kval;
                                ii[j] = smem_index<256>(cen.k, cen.t, xh[j], kval);
                                qq[j] = from_unit(kval, rs.alpha, rs.beta);
                                if (pre) qq[j] = __fadd_rn(qq[j], mean);
                            }
                        }
                        if (act) {
                            if (P.q != nullptr) {
                                if (ovec) st_hint4(P.q + base + e, make_float4(qq[0], qq[1], qq[2], qq[3]), pol_stream);
                                else { P.q[base + e] = qq[0]; P.q[base + e + 1] = qq[1]; P.q[base + e + 2] = qq[2]; P.q[base + e + 3] = qq[3]; }
                            }
                            if (P.idx8 != nullptr) {
                                if (ovec) *reinterpret_cast<uint32_t*>(P.idx8 + base + e) =
                                        (uint32_t)ii[0] | ((uint32_t)ii[1] << 8) | ((uint32_t)ii[2] << 16) | ((uint32_t)ii[3] << 24);
                                else { P.idx8[base + e] = (uint8_t)ii[0]; P.idx8[base + e + 1] = (uint8_t)ii[1]; P.idx8[base + e + 2] = (uint8_t)ii[2]; P.idx8[base + e + 3] = (uint8_t)ii[3]; }
                            }
                            if (P.idx64 != nullptr) { P.idx64[base + e] = ii[0]; P.idx64[base + e + 1] = ii[1]; P.idx64[base + e + 2] = ii[2]; P.idx64[base + e + 3] = ii[3]; }
                        }
                    }
                    if (c == sweep_chunks - 1) {
                        for (int e = len4 + tid; e < len; e += T) {  // scalar tail: table search in shared memory
                            const float xh = div.exact(__fsub_rn(buf[e], rs.beta));
                            float kval;
                            const int id = smem_index<256>(cen.k, cen.t, xh, kval);
                            float qv = from_unit(kval, rs.alpha, rs.beta);
                            if (pre) qv = __fadd_rn(qv, mean);
                            if (P.q != nullptr) P.q[base + e] = qv;
                            if (P.idx8 != nullptr) P.idx8[base + e] = (uint8_t)id;
                            if (P.idx64 != nullptr) P.idx64[base + e] = id;
                        }
                    }
                    chunk_done(c);
                }
            };
            const int K = P.num_points;
            if (K <= 4) sweep(std::integral_constant<int, 4>{});
            else if (K <= 8) sweep(std::integral_constant<int, 8>{});
            else if (K <= 16) sweep(std::integral_constant<int, 16>{});
            else if (K <= 32) sweep(std::integral_constant<int, 32>{});
            else sweep(std::integral_constant<int, 256>{});
        }
    }
}

}  // namespace qd
