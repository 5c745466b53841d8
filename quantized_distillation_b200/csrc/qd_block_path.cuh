// qd_block_path.cuh -- the round-1 kernels for rows of 1025 .. QD_MAX_STAGED_BUCKET elements, plus the TMA /
// mbarrier primitives and CTA reductions the staged ring (qd_staged_path.cuh) builds on.
//
// Since round 2 the deterministic uniform op (forward, every backward mode) and the centroid op run on the
// staged chunk ring; this kernel keeps the ops the ring does not implement -- per-row statistics, x_hat in the
// padded layout, stochastic rounding -- in two variants, and the min/max backward on rows of 1025 ..
// kWarp2MinmaxMaxRow floats in the first:
//
// WARP TWO-PASS (GROUP = 32, rows up to 2 * kWarpTwoPassMaxRow floats): a warp streams its row once for
// min/max (tagged L2::evict_last) and again (L2 hit) for the element-wise pass; no block barrier anywhere,
// sixteen rows in flight per CTA.
//
// WHOLE-ROW STAGING (GROUP = 512, longer rows): the row is staged in shared memory by the TMA bulk-copy engine
// (cp.async.bulk.shared::cluster.global with mbarrier complete_tx; SASS UBLKCP): one elected thread enqueues the
// row in 32 KB chunks, each chunk signalling its own mbarrier, and the 512 threads reduce chunk c while chunks
// c+1.. are still in flight.  Rows whose global address is not 16-byte aligned fall back to a cooperative
// ld.global -> st.shared copy.  Shared memory is sized to the row (dynamic).
//
// The min/max backward here uses the same two-sweep formulation as the ring (analytic extremes of q, the two
// changed elements patched after the sweep).  All element loops are 128-bit with a scalar tail.
#pragma once
#include "qd_rowops.cuh"

namespace qd {

constexpr int kBlockCtaThreads = 512;
constexpr int kStageChunk = 8192;  // floats per TMA bulk copy (32 KB)
constexpr int kMaxStageChunks = (QD_MAX_STAGED_BUCKET + kStageChunk - 1) / kStageChunk;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// Bounded wait: a bulk copy that never completes (a bad pointer from the caller) must fail the
// launch with an error, not hang the GPU -- after ~2^26 polls the kernel traps.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    for (uint32_t spins = 0;; ++spins) {
        uint32_t done;
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(addr), "r"(parity)
            : "memory");
        if (done) return;
        if (spins > (1u << 26)) __trap();
    }
}
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// CTA-wide reductions through a small shared scratch (16 warps)
template <bool IS_MIN>
__device__ __forceinline__ float cta_minmax(float v, float* scratch) {
    v = IS_MIN ? warp_min(v) : warp_max(v);
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();
    if (lane == 0) scratch[w] = v;
    __syncthreads();
    float r = scratch[lane < (blockDim.x >> 5) ? lane : 0];
    return IS_MIN ? warp_min(r) : warp_max(r);
}
__device__ __forceinline__ int cta_min_int(int v, int* scratch) {
    v = warp_min_int(v);
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();
    if (lane == 0) scratch[w] = v;
    __syncthreads();
    int r = scratch[lane < (blockDim.x >> 5) ? lane : 0];
    return warp_min_int(r);
}
__device__ __forceinline__ double cta_sum(double v, double* scratch) {
    v = warp_sum(v);
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();
    if (lane == 0) scratch[w] = v;
    __syncthreads();
    double r = (lane < (blockDim.x >> 5)) ? scratch[lane] : 0.0;
    return warp_sum(r);  // fixed tree: deterministic
}

// Round-1 measurement (tools/block_bench.py, 64 Mi floats): warp-per-row two-pass won up to 2048-4096 floats per
// row, the whole-row staging above that, up to the 49152-float shared-memory limit.
constexpr int kWarpTwoPassMaxRow = 2048;  // floats; rows up to here: one WARP per row, two passes (second from L1/L2)
constexpr int kWarp2MinmaxMaxRow = 2048;  // floats; the min/max backward takes the two-pass variant up to here (qd_quant.cu)

// GROUP = 32: a warp owns the row (no block barriers at all, dozens of rows in flight per SM);
// GROUP = kBlockCtaThreads: the whole CTA owns the row.
template <int GROUP, bool IS_MIN>
__device__ __forceinline__ float grp_minmax(float v, float* scratch) {
    if constexpr (GROUP == 32) return IS_MIN ? warp_min(v) : warp_max(v);
    else return cta_minmax<IS_MIN>(v, scratch);
}
template <int GROUP>
__device__ __forceinline__ int grp_min_int(int v, int* scratch) {
    if constexpr (GROUP == 32) return warp_min_int(v);
    else return cta_min_int(v, scratch);
}
template <int GROUP>
__device__ __forceinline__ double grp_sum(double v, double* scratch) {
    if constexpr (GROUP == 32) return warp_sum(v);
    else return cta_sum(v, scratch);
}

// Calls f4(e, float4) on aligned groups of four elements and f1(e, float) on the tail (or on
// every element when the global row is not 16-byte aligned and not staged).
template <bool STAGED, int GROUP, class F4, class F1>
__device__ __forceinline__ void for_each_in_row(const float* s_row, const float* src, int len, bool gvec, bool pre,
                                                float mean, float max_el, F4 f4, F1 f1) {
    const int gtid = (GROUP == 32) ? (threadIdx.x & 31) : threadIdx.x;
    const int len4 = (STAGED || gvec) ? (len & ~3) : 0;
#pragma unroll 2
    for (int e = gtid * 4; e < len4; e += GROUP * 4) {
        float4 t = STAGED ? *reinterpret_cast<const float4*>(s_row + e) : *reinterpret_cast<const float4*>(src + e);
        if (!STAGED && pre) {
            t.x = pre_op(t.x, mean, max_el); t.y = pre_op(t.y, mean, max_el);
            t.z = pre_op(t.z, mean, max_el); t.w = pre_op(t.w, mean, max_el);
        }
        f4(e, t);
    }
    for (int e = len4 + gtid; e < len; e += GROUP) {
        float t = STAGED ? s_row[e] : src[e];
        if (!STAGED && pre) t = pre_op(t, mean, max_el);
        f1(e, t);
    }
}

template <int OP, int BWD, bool STAGED, int GROUP>
__global__ void __launch_bounds__(kBlockCtaThreads) block_rows_kernel(const __grid_constant__ Params P) {
    static_assert(!(STAGED && GROUP == 32), "staging is a CTA-wide operation");
    static_assert(OP == OP_STATS || OP == OP_SCALE || (OP == OP_UNIFORM && (BWD == BWD_OFF || (BWD == BWD_MINMAX && GROUP == 32))),
                  "block path: stats, scale, uniform forward (stochastic rounding), min/max backward warp two-pass");
    extern __shared__ __align__(128) float s_row[];
    __shared__ __align__(8) uint64_t s_bar[kMaxStageChunks];
    __shared__ double s_scratch[kBlockCtaThreads / 32];

    if (STAGED && threadIdx.x == 0) {
        for (int c = 0; c < kMaxStageChunks; ++c) mbar_init(&s_bar[c], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const int tid = (GROUP == 32) ? (threadIdx.x & 31) : threadIdx.x;
    const bool pre = (P.mean != nullptr) || (P.max_element > 0.f);
    const float mean = P.mean ? *P.mean : 0.f;
    const float max_el = P.max_element;
    uint32_t phase_bits = 0;  // bit c = parity the next wait on s_bar[c] must see
    const uint64_t pol_keep = l2_policy_evict_last(), pol_stream = l2_policy_evict_first();
    constexpr int kGroups = kBlockCtaThreads / GROUP;  // rows in flight per CTA

    for (int64_t row = (int64_t)blockIdx.x * kGroups + (GROUP == 32 ? (threadIdx.x >> 5) : 0); row < P.geo.rows;
         row += (int64_t)gridDim.x * kGroups) {
        const int64_t base = row * P.geo.row_len;
        const int len = (int)min(P.geo.row_len, P.geo.n - base);
        const float* src = P.x + base;
        const bool gvec = ((reinterpret_cast<uintptr_t>(src) & 15) == 0);
        // 128-bit stores need every output row to be 16-byte aligned too
        const bool ovec = (((reinterpret_cast<uintptr_t>(P.q + base) | reinterpret_cast<uintptr_t>(P.gout + base) |
                             reinterpret_cast<uintptr_t>(P.g + base) | reinterpret_cast<uintptr_t>(P.xhat + base)) & 15) == 0) &&
                          ((reinterpret_cast<uintptr_t>(P.idx8 + base) & 3) == 0);

        float mn = __int_as_float(0x7f800000), mx = __int_as_float(0xff800000);
        if constexpr (STAGED) {
            const int bulk_len = gvec ? (len & ~3) : 0;  // multiple of 16 bytes
            const int nchunks = (bulk_len + kStageChunk - 1) / kStageChunk;
            if (tid == 0 && nchunks > 0) {
                // generic-proxy reads of the previous row are complete (barrier at loop end);
                // order them before the async-proxy writes that follow
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                for (int c = 0; c < nchunks; ++c) {
                    const int off = c * kStageChunk;
                    const uint32_t bytes = (uint32_t)min(kStageChunk, bulk_len - off) * 4u;
                    mbar_expect_tx(&s_bar[c], bytes);
                    tma_bulk_g2s(s_row + off, src + off, bytes, &s_bar[c]);
                }
            }
            for (int e = bulk_len + tid; e < len; e += kBlockCtaThreads) s_row[e] = ld_stream1(src + e);
            // min / max, chunk by chunk as the copies land
            for (int c = 0; c < nchunks; ++c) {
                mbar_wait(&s_bar[c], (phase_bits >> c) & 1u);
                phase_bits ^= (1u << c);
                const int off = c * kStageChunk;
                const int cl = min(kStageChunk, bulk_len - off);
                for (int e = tid * 4; e < cl; e += kBlockCtaThreads * 4) {
                    float4 t = *reinterpret_cast<const float4*>(s_row + off + e);
                    if (pre) {
                        t.x = pre_op(t.x, mean, max_el); t.y = pre_op(t.y, mean, max_el);
                        t.z = pre_op(t.z, mean, max_el); t.w = pre_op(t.w, mean, max_el);
                        *reinterpret_cast<float4*>(s_row + off + e) = t;
                    }
                    mn = min_nan(min_nan(mn, t.x), min_nan(t.y, min_nan(t.z, t.w)));
                    mx = max_nan(max_nan(mx, t.x), max_nan(t.y, max_nan(t.z, t.w)));
                }
            }
            __syncthreads();  // scalar-staged tail visible
            for (int e = bulk_len + tid; e < len; e += kBlockCtaThreads) {
                float t = s_row[e];
                if (pre) { t = pre_op(t, mean, max_el); s_row[e] = t; }
                mn = min_nan(mn, t);
                mx = max_nan(mx, t);
            }
        } else {
            // first pass over the row from HBM (it stays in L2 for the passes below)
            const int len4 = gvec ? (len & ~3) : 0;
#pragma unroll 4
            for (int e = tid * 4; e < len4; e += GROUP * 4) {
                float4 t = ld_hint4(src + e, pol_keep);          // keep the row in L2 for the passes below
                if (pre) {
                    t.x = pre_op(t.x, mean, max_el); t.y = pre_op(t.y, mean, max_el);
                    t.z = pre_op(t.z, mean, max_el); t.w = pre_op(t.w, mean, max_el);
                }
                mn = min_nan(min_nan(mn, t.x), min_nan(t.y, min_nan(t.z, t.w)));
                mx = max_nan(max_nan(mx, t.x), max_nan(t.y, max_nan(t.z, t.w)));
            }
            for (int e = len4 + tid; e < len; e += GROUP) {
                float t = ld_stream1(src + e);
                if (pre) t = pre_op(t, mean, max_el);
                mn = min_nan(mn, t);
                mx = max_nan(mx, t);
            }
        }
        mn = grp_minmax<GROUP, true>(mn, reinterpret_cast<float*>(s_scratch));
        mx = grp_minmax<GROUP, false>(mx, reinterpret_cast<float*>(s_scratch));
        RowState rs;
        rs.mean = mean;
        rs.beta = mn;
        rs.alpha = make_alpha(mn, mx);
        if (P.alpha != nullptr && tid == 0) { P.alpha[row] = rs.alpha; P.beta[row] = rs.beta; }
        if (P.argmin != nullptr) {
            int imin = 0x7fffffff, imax = 0x7fffffff;
            auto scan1 = [&](int e, float t) {
                if (t == mn) imin = min(imin, e);
                if (t == mx) imax = min(imax, e);
            };
            for_each_in_row<STAGED, GROUP>(s_row, src, len, gvec, pre, mean, max_el,
                                    [&](int e, float4 t) { scan1(e, t.x); scan1(e + 1, t.y); scan1(e + 2, t.z); scan1(e + 3, t.w); },
                                    scan1);
            imin = grp_min_int<GROUP>(imin, reinterpret_cast<int*>(s_scratch));
            imax = grp_min_int<GROUP>(imax, reinterpret_cast<int*>(s_scratch));
            if (tid == 0) {
                P.argmin[row] = (imin == 0x7fffffff) ? 0 : imin;
                P.argmax[row] = (imax == 0x7fffffff) ? 0 : imax;
            }
        }

        // ---- element-wise pass ---------------------------------------------------
        if constexpr (OP == OP_SCALE) {
            const int plen = (int)P.geo.row_len;  // padded layout: the tail repeats x_hat of the last element
            float lastv = STAGED ? s_row[len - 1] : src[len - 1];
            if (!STAGED && pre) lastv = pre_op(lastv, mean, max_el);
            const float last = to_unit(lastv, rs.beta, rs.alpha);
            float* dst = P.xhat + base;
            for_each_in_row<STAGED, GROUP>(s_row, src, len, gvec, pre, mean, max_el,
                                    [&](int e, float4 t) {
                                        float4 o = make_float4(to_unit(t.x, rs.beta, rs.alpha), to_unit(t.y, rs.beta, rs.alpha),
                                                               to_unit(t.z, rs.beta, rs.alpha), to_unit(t.w, rs.beta, rs.alpha));
                                        if (ovec) st_stream4(dst + e, o);
                                        else { dst[e] = o.x; dst[e + 1] = o.y; dst[e + 2] = o.z; dst[e + 3] = o.w; }
                                    },
                                    [&](int e, float t) { dst[e] = to_unit(t, rs.beta, rs.alpha); });
            for (int e = len + tid; e < plen; e += GROUP) dst[e] = last;
        } else if constexpr (OP == OP_UNIFORM) {
            float rb = 0.f;
            int imin2 = 0, imax2 = 0;
            const UniformFast uf = make_uniform_fast(rs.alpha, P.S);
            auto quant = [&](float xv, int64_t ge, float& lvl) -> float {
                if (P.stochastic) {
                    Philox rng(P.seed);
                    uint4 rnd = rng(P.offset + (uint64_t)(ge >> 2));
                    uint32_t w = (ge & 3) == 0 ? rnd.x : (ge & 3) == 1 ? rnd.y : (ge & 3) == 2 ? rnd.z : rnd.w;
                    return uniform_quantize_stochastic(xv, rs, P.S, u01(w), lvl);
                }
                return uniform_quantize_auto(xv, rs, uf, P.S, P.rS, P.half_minus_band, lvl);
            };
            float qlo = 0.f, qhi = 0.f;
            double acc = 0.0;
            RowDivider div2(1.0f);
            if constexpr (BWD == BWD_MINMAX) {
                // second scaling of the quantized row (quant_functions.py:350-363): q is a monotone function
                // of x, so min q = Q(min x), max q = Q(max x) exactly (qd_staged_path.cuh) -- no sweep over q
                float lvl;
                qlo = quant(mn, 0, lvl);
                qhi = quant(mx, 0, lvl);
                rs.beta2 = qlo;
                rs.alpha2 = make_alpha(qlo, qhi);
                div2 = RowDivider(rs.alpha2);
                imin2 = 0x7fffffff; imax2 = 0x7fffffff;
            }
            // gout = g here; the two elements the min/max backward changes are patched after the sweep
            auto fix = [&](int e, float xv, float qv, float gv) -> float {
                if constexpr (BWD == BWD_MINMAX) {
                    if (qv == qlo) imin2 = min(imin2, e);
                    if (qv == qhi) imax2 = min(imax2, e);
                    acc += (double)minmax_term(xv, qv, gv, rs.beta2, div2);
                }
                return gv;
            };
            for_each_in_row<STAGED, GROUP>(
                s_row, src, len, gvec, pre, mean, max_el,
                [&](int e, float4 t) {
                    float lv[4];
                    float4 qo;
                    if (P.stochastic)
                        qo = make_float4(quant(t.x, base + e, lv[0]), quant(t.y, base + e + 1, lv[1]),
                                         quant(t.z, base + e + 2, lv[2]), quant(t.w, base + e + 3, lv[3]));
                    else
                        qo = uniform_quantize_auto4(t, rs.alpha, rs.beta, uf, P.S, P.rS, P.half_minus_band, lv);
                    if constexpr (BWD != BWD_OFF) {
                        float4 gv = ovec ? *reinterpret_cast<const float4*>(P.g + base + e)
                                         : make_float4(P.g[base + e], P.g[base + e + 1], P.g[base + e + 2], P.g[base + e + 3]);
                        gv.x = fix(e, t.x, qo.x, gv.x); gv.y = fix(e + 1, t.y, qo.y, gv.y);
                        gv.z = fix(e + 2, t.z, qo.z, gv.z); gv.w = fix(e + 3, t.w, qo.w, gv.w);
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
                },
                [&](int e, float t) {
                    float lvl;
                    float qv = quant(t, base + e, lvl);
                    if constexpr (BWD != BWD_OFF) P.gout[base + e] = fix(e, t, qv, P.g[base + e]);
                    if (P.q != nullptr) P.q[base + e] = pre ? __fadd_rn(qv, mean) : qv;
                    if (P.idx8 != nullptr) P.idx8[base + e] = (uint8_t)(int)lvl;
                });
            if constexpr (BWD == BWD_MINMAX) {
                imin2 = grp_min_int<GROUP>(imin2, reinterpret_cast<int*>(s_scratch));
                imax2 = grp_min_int<GROUP>(imax2, reinterpret_cast<int*>(s_scratch));
                rb = (float)grp_sum<GROUP>(acc, s_scratch);
                __syncwarp();   // the row's gout stores are ordered before the patch
                if (tid == 0 && imin2 != imax2) {  // +r at argmax', -r at argmin' (quant_functions.py:380-393)
                    float* pmax = P.gout + base + imax2;
                    float* pmin = P.gout + base + imin2;
                    *pmax = __fadd_rn(__ldcg(pmax), rb);
                    *pmin = __fadd_rn(__ldcg(pmin), -rb);
                }
            }
        }
        if constexpr (GROUP != 32) __syncthreads();  // everyone is done with the row (and s_row) before the next one
    }
}

}  // namespace qd
