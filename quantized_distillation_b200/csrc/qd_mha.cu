// qd_mha.cu -- the core of onmt's Transformer sublayers (onmt/modules/MultiHeadedAttn.py:44-110 between the three
// projections and the residual, and onmt/modules/UtilClass.py:24-46, onmt's own LayerNorm), forward and backward.  The
// Linears (linear_keys / linear_values / linear_query, w_1 / w_2) stay GEMMs outside.
//
// Attention.  q [B, Lq, D], k and v [B, Lk, D], D = h*dh: the projections' outputs in their own layout; head hd of
// row (b, t) is q[(b*Lq + t)*D + hd*dh + j], so nothing is transposed on the way in or out.  probs and the backward's
// workspace are [B, h, Lq, Lk] (bh = b*h + hd), keep [B*h, Lq, Lk], top [B, Lq, Lk], out [B, Lq, D].
//
// Forward (qd_mha_fwd): one 256-thread CTA per (b, head, tile of up to kMhTile query rows), three phases:
//   1. scores (qd_attn_tile.cuh's tile_dots): warp w owns keys s = w + 8k, lane l the elements j = l + 32i; a lane-strided float32 sum and a
//      butterfly over the warp, then x = sum / sqrt(dh), or -inf where the mask is set.  The scores go to probs.
//   2. softmax: warp t owns row t; max, sum of expf(x - max) (lane-strided, butterfly), then p = expf(x - max) / sum in
//      place; head 0 copies its row to top.  An all-masked row is -inf - -inf = NaN throughout, as torch's softmax.
//   3. values: thread e owns (row t, element j) = (e / dh, e % dh) and sums p'_s v_s[j] over s in order, with
//      p' = p * keep * scale under dropout.
// Backward: qd_mha_bwd_rows runs the same phases on grad_out (G = (grad_out . v_s) keep scale + [head 0] grad_top, then
// dS = p (G - sum_s p G) / sqrt(dh), zero where masked, into the workspace, then grad_q = sum_s dS k_s); qd_mha_bwd_keys
// gives each CTA kMhKChunk keys of one (b, head) and sums p'_{t,s} grad_out_t and dS_{t,s} q_t over t in order.
//
// Layer norm (qd_onmt_layernorm_fwd / _bwd): one warp per row of width d, z = x (+ residual), lane-strided sums and a
// butterfly.  The backward recomputes z, the mean and the std in the forward's order (the same bits), writes grad_x,
// and sums dy * xhat and dy over its chunk of kLnChunk rows per column into a workspace; a second launch sums the
// chunks in order.
//
// Which thread owns which element, and every summation order, depend only on (Lk, dh) and d: a row gives the same bits
// alone or in any batch; all loads are scalar, so the alignment of a view changes nothing either.
#include <cmath>

#include "qd_attn_tile.cuh"
#include "qd_launch.h"

using namespace qd;

namespace {

constexpr int kMhThreads = 256;
constexpr int kMhWarps = kMhThreads / 32;
constexpr int kMhTile = 8;           // query rows of one (b, head) per CTA (phase 2 gives each a warp)
constexpr int kMhKChunk = 8;         // keys per CTA of the key-side gradients
constexpr int kLnChunk = 32;         // rows per CTA of the layer norm's backward (one partial per chunk and column)
static_assert(kMhTile <= kMhWarps, "phase 2 gives each row of a tile its own warp");

struct MhArgs {
    const float* q;           // [B, Lq, D]
    const float* k;           // [B, Lk, D]
    const float* v;           // [B, Lk, D]
    const uint8_t* mask;      // [B, Lq, Lk] through (mB, mQ, mK), or NULL
    const uint8_t* keep;      // [B*h, Lq, Lk] or NULL
    const float* grad_out;    // [B, Lq, D]
    const float* grad_top;    // [B, Lq, Lk] or NULL
    float* probs;             // [B, h, Lq, Lk]
    float* top;               // [B, Lq, Lk]
    float* out;               // [B, Lq, D]
    float* ds;                // workspace [B, h, Lq, Lk]
    float* grad_q;
    float* grad_k;
    float* grad_v;
    int64_t B, Lq, Lk, h, dh, D, mB, mQ, mK;
    float scale, rdh;         // dropout's 1/(1-p); sqrt(dh) rounded to float32
};

__device__ __forceinline__ bool masked(const MhArgs& a, int64_t b, int64_t t, int64_t s) {
    return a.mask != nullptr && a.mask[b * a.mB + t * a.mQ + s * a.mK] != 0;
}

// p * keep * scale, the reference's dropout (p * 0 keeps a NaN of an all-masked row, as torch does)
__device__ __forceinline__ float dropped(const MhArgs& a, float p, int64_t idx) {
    return a.keep == nullptr ? p : __fmul_rn(__fmul_rn(p, (float)a.keep[idx]), a.scale);
}

__global__ void __launch_bounds__(kMhThreads) mha_fwd_kernel(MhArgs a) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int64_t bh = blockIdx.x; bh < a.B * a.h; bh += gridDim.x)
    for (int64_t t0 = (int64_t)blockIdx.y * kMhTile; t0 < a.Lq; t0 += (int64_t)gridDim.y * kMhTile) {
        const int64_t b = bh / a.h, hd = bh - b * a.h;
        const int nt = (int)min((int64_t)kMhTile, a.Lq - t0);
        const int64_t row = b * a.Lq + t0, col = hd * a.dh;
        float* P = a.probs + (bh * a.Lq + t0) * a.Lk;
        attn::tile_dots<kMhTile, kMhWarps, 2>(a.q + row * a.D + col, a.D, a.k + b * a.Lk * a.D + col, a.D, a.Lk, a.dh, nt,
                                              [&](int t, int64_t s, float d) {
                                                  P[t * a.Lk + s] = masked(a, b, t0 + t, s) ? -INFINITY : __fdiv_rn(d, a.rdh);
                                              });
        __syncthreads();
        if (warp < nt) {
            float* p = P + warp * a.Lk;
            // attn::softmax_row with a store that also writes top schedules this kernel differently, and measured
            // slower at Lk = 100, so the row is written out here
            float m = -INFINITY;
            for (int64_t s = lane; s < a.Lk; s += 32) m = fmaxf(m, p[s]);
            m = attn::warp_fmax(m);
            float l = 0.f;
            for (int64_t s = lane; s < a.Lk; s += 32) l = __fadd_rn(l, expf(__fsub_rn(p[s], m)));
            l = attn::warp_sum(l);
            float* top = hd == 0 ? a.top + (row + warp) * a.Lk : nullptr;
            for (int64_t s = lane; s < a.Lk; s += 32) {
                const float y = __fdiv_rn(expf(__fsub_rn(p[s], m)), l);
                p[s] = y;
                if (top != nullptr) top[s] = y;
            }
        }
        __syncthreads();
        const float* vb = a.v + b * a.Lk * a.D + col;
        const int64_t pk = (bh * a.Lq + t0) * a.Lk;
        for (int64_t e = threadIdx.x; e < nt * a.dh; e += kMhThreads) {
            const int64_t t = e / a.dh, j = e - t * a.dh;
            float acc = 0.f;
#pragma unroll 4
            for (int64_t s = 0; s < a.Lk; ++s)
                acc = __fadd_rn(acc, __fmul_rn(dropped(a, P[t * a.Lk + s], pk + t * a.Lk + s), __ldg(vb + s * a.D + j)));
            a.out[(row + t) * a.D + col + j] = acc;
        }
    }
}

__global__ void __launch_bounds__(kMhThreads) mha_bwd_rows_kernel(MhArgs a) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int64_t bh = blockIdx.x; bh < a.B * a.h; bh += gridDim.x)
    for (int64_t t0 = (int64_t)blockIdx.y * kMhTile; t0 < a.Lq; t0 += (int64_t)gridDim.y * kMhTile) {
        const int64_t b = bh / a.h, hd = bh - b * a.h;
        const int nt = (int)min((int64_t)kMhTile, a.Lq - t0);
        const int64_t row = b * a.Lq + t0, col = hd * a.dh, pk = (bh * a.Lq + t0) * a.Lk;
        float* W = a.ds + pk;
        const float* gt = (hd == 0 && a.grad_top != nullptr) ? a.grad_top + row * a.Lk : nullptr;
        attn::tile_dots<kMhTile, kMhWarps, 2>(a.grad_out + row * a.D + col, a.D, a.v + b * a.Lk * a.D + col, a.D, a.Lk, a.dh,
                                              nt, [&](int t, int64_t s, float d) { W[t * a.Lk + s] = d; });
        __syncthreads();
        if (warp < nt) {
            const float* p = a.probs + pk + warp * a.Lk;
            float* w = W + warp * a.Lk;
            float d = 0.f;
            for (int64_t s = lane; s < a.Lk; s += 32) {
                float g = dropped(a, w[s], pk + warp * a.Lk + s);
                if (gt != nullptr) g = __fadd_rn(g, __ldg(gt + warp * a.Lk + s));
                w[s] = g;
                d = __fadd_rn(d, __fmul_rn(__ldg(p + s), g));
            }
            d = attn::warp_sum(d);
            for (int64_t s = lane; s < a.Lk; s += 32)
                w[s] = masked(a, b, t0 + warp, s) ? 0.f : __fdiv_rn(__fmul_rn(__ldg(p + s), __fsub_rn(w[s], d)), a.rdh);
        }
        __syncthreads();
        const float* kb = a.k + b * a.Lk * a.D + col;
        for (int64_t e = threadIdx.x; e < nt * a.dh; e += kMhThreads) {
            const int64_t t = e / a.dh, j = e - t * a.dh;
            float acc = 0.f;
#pragma unroll 4
            for (int64_t s = 0; s < a.Lk; ++s) acc = __fadd_rn(acc, __fmul_rn(W[t * a.Lk + s], __ldg(kb + s * a.D + j)));
            a.grad_q[(row + t) * a.D + col + j] = acc;
        }
    }
}

__global__ void __launch_bounds__(kMhThreads) mha_bwd_keys_kernel(MhArgs a) {
    for (int64_t bh = blockIdx.x; bh < a.B * a.h; bh += gridDim.x)
    for (int64_t s0 = (int64_t)blockIdx.y * kMhKChunk; s0 < a.Lk; s0 += (int64_t)gridDim.y * kMhKChunk) {
        const int64_t b = bh / a.h, hd = bh - b * a.h;
        const int ns = (int)min((int64_t)kMhKChunk, a.Lk - s0);
        const int64_t col = hd * a.dh;
        for (int64_t e = threadIdx.x; e < ns * a.dh; e += kMhThreads) {
            const int64_t s = s0 + e / a.dh, j = e - (e / a.dh) * a.dh;
            float gv = 0.f, gk = 0.f;
            for (int64_t t = 0; t < a.Lq; ++t) {
                const int64_t pi = (bh * a.Lq + t) * a.Lk + s, ri = (b * a.Lq + t) * a.D + col + j;
                gv = __fadd_rn(gv, __fmul_rn(dropped(a, __ldg(a.probs + pi), pi), __ldg(a.grad_out + ri)));
                gk = __fadd_rn(gk, __fmul_rn(__ldg(a.ds + pi), __ldg(a.q + ri)));
            }
            const int64_t o = (b * a.Lk + s) * a.D + col + j;
            a.grad_v[o] = gv;
            a.grad_k[o] = gk;
        }
    }
}

struct LnArgs {
    const float* x;           // [rows, d]
    const float* res;         // [rows, d] or NULL
    const float* a2;          // [d]
    const float* b2;          // [d]
    const float* grad_y;      // [rows, d]
    float* y;
    float* grad_x;
    float* partial;           // workspace [2, chunks, d]
    float* grad_a2;
    float* grad_b2;
    int64_t rows, d, chunks;
    float eps;
};

__device__ __forceinline__ float ln_z(const LnArgs& a, int64_t i) {
    const float x = __ldg(a.x + i);
    return a.res == nullptr ? x : __fadd_rn(x, __ldg(a.res + i));
}

// mean, std (unbiased) and std + eps of row r (d >= 2), in one fixed order
__device__ __forceinline__ void ln_stats(const LnArgs& a, int64_t r, float& mu, float& sd, float& den) {
    const int lane = threadIdx.x & 31;
    const int64_t base = r * a.d;
    float s = 0.f;
    for (int64_t j = lane; j < a.d; j += 32) s = __fadd_rn(s, ln_z(a, base + j));
    mu = __fdiv_rn(attn::warp_sum(s), (float)a.d);
    float q = 0.f;
    for (int64_t j = lane; j < a.d; j += 32) {
        const float c = __fsub_rn(ln_z(a, base + j), mu);
        q = __fadd_rn(q, __fmul_rn(c, c));
    }
    sd = __fsqrt_rn(__fdiv_rn(attn::warp_sum(q), (float)(a.d - 1)));
    den = __fadd_rn(sd, a.eps);
}

__global__ void __launch_bounds__(kMhThreads) ln_fwd_kernel(LnArgs a) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int64_t r = (int64_t)blockIdx.x * kMhWarps + warp; r < a.rows; r += (int64_t)gridDim.x * kMhWarps) {
        const int64_t base = r * a.d;
        if (a.d == 1) {
            if (lane == 0) a.y[base] = ln_z(a, base);
            continue;
        }
        float mu, sd, den;
        ln_stats(a, r, mu, sd, den);
        for (int64_t j = lane; j < a.d; j += 32) {
            const float xh = __fdiv_rn(__fsub_rn(ln_z(a, base + j), mu), den);
            a.y[base + j] = __fadd_rn(__fmul_rn(xh, __ldg(a.a2 + j)), __ldg(a.b2 + j));
        }
    }
}

// grad_z = (g - mean g) / den + k c with g = dy a2, c = z - mu, k = -(sum g c / den^2) / ((d - 1) sd)
__global__ void __launch_bounds__(kMhThreads) ln_bwd_kernel(LnArgs a) {
    __shared__ float s_mu[kLnChunk], s_den[kLnChunk];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int64_t c0 = blockIdx.x; c0 < a.chunks; c0 += gridDim.x) {
        const int64_t r0 = c0 * kLnChunk;
        const int nr = (int)min((int64_t)kLnChunk, a.rows - r0);
        for (int i = warp; i < nr; i += kMhWarps) {
            const int64_t r = r0 + i, base = r * a.d;
            if (a.d == 1) {
                if (lane == 0) a.grad_x[base] = __ldg(a.grad_y + base);
                continue;
            }
            float mu, sd, den;
            ln_stats(a, r, mu, sd, den);
            float sg = 0.f, sgc = 0.f;
            for (int64_t j = lane; j < a.d; j += 32) {
                const float g = __fmul_rn(__ldg(a.grad_y + base + j), __ldg(a.a2 + j));
                sg = __fadd_rn(sg, g);
                sgc = __fadd_rn(sgc, __fmul_rn(g, __fsub_rn(ln_z(a, base + j), mu)));
            }
            const float mg = __fdiv_rn(attn::warp_sum(sg), (float)a.d);
            const float kc = -__fdiv_rn(__fdiv_rn(attn::warp_sum(sgc), __fmul_rn(den, den)), __fmul_rn((float)(a.d - 1), sd));
            for (int64_t j = lane; j < a.d; j += 32) {
                const float g = __fmul_rn(__ldg(a.grad_y + base + j), __ldg(a.a2 + j));
                const float c = __fsub_rn(ln_z(a, base + j), mu);
                a.grad_x[base + j] = __fadd_rn(__fdiv_rn(__fsub_rn(g, mg), den), __fmul_rn(kc, c));
            }
            if (lane == 0) s_mu[i] = mu, s_den[i] = den;
        }
        __syncthreads();
        if (a.d > 1) {
            for (int64_t j = threadIdx.x; j < a.d; j += kMhThreads) {
                float pa = 0.f, pb = 0.f;
                for (int i = 0; i < nr; ++i) {
                    const int64_t o = (r0 + i) * a.d + j;
                    const float dy = __ldg(a.grad_y + o);
                    pa = __fadd_rn(pa, __fmul_rn(dy, __fdiv_rn(__fsub_rn(ln_z(a, o), s_mu[i]), s_den[i])));
                    pb = __fadd_rn(pb, dy);
                }
                a.partial[c0 * a.d + j] = pa;
                a.partial[(a.chunks + c0) * a.d + j] = pb;
            }
        }
        __syncthreads();
    }
}

// grad_a2[j] (o = j) and grad_b2[j] (o = d + j): the sum of the chunks' partials, chunk 0 first
__global__ void __launch_bounds__(kMhThreads) ln_param_kernel(LnArgs a) {
    const int64_t stride = (int64_t)gridDim.x * kMhThreads;
    for (int64_t o = (int64_t)blockIdx.x * kMhThreads + threadIdx.x; o < 2 * a.d; o += stride) {
        const int64_t half = o / a.d, j = o - half * a.d;
        float s = 0.f;
        if (a.d > 1) {
            const float* p = a.partial + half * a.chunks * a.d + j;
            for (int64_t c = 0; c < a.chunks; ++c) s = __fadd_rn(s, p[c * a.d]);
        }
        (half == 0 ? a.grad_a2 : a.grad_b2)[j] = s;
    }
}

// checks of the sizes and the mask both attention calls share; fills the sizes of a and the mask's byte span
int check_mha(const float* q, const float* k, const float* v, const uint8_t* mask, int64_t mB, int64_t mQ, int64_t mK,
              int64_t B, int64_t Lq, int64_t Lk, int64_t heads, int64_t dh, MhArgs* a, size_t* mask_span) {
    if (B < 1 || Lq < 1 || Lk < 1 || heads < 1 || dh < 1)
        return fail(QD_ERR_INVALID_ARG, "B, Lq, Lk, heads and dh must be >= 1 (B=%lld Lq=%lld Lk=%lld heads=%lld dh=%lld)",
                    (long long)B, (long long)Lq, (long long)Lk, (long long)heads, (long long)dh);
    const int64_t lim = INT64_MAX / 16;
    const int64_t L = Lq > Lk ? Lq : Lk;
    if (heads > lim / dh || B > lim / (heads * dh) || L > lim / (B * heads * dh) || Lk > lim / (B * heads * Lq))
        return fail(QD_ERR_INVALID_ARG, "B * L * heads * dh or B * heads * Lq * Lk overflows 64-bit indexing");
    *mask_span = 0;
    if (mask != nullptr) {
        if (mB < 0 || mQ < 0 || mK < 0) return fail(QD_ERR_INVALID_ARG, "mask strides must be >= 0");
        if ((B > 1 && mB > lim / (B - 1)) || (Lq > 1 && mQ > lim / (Lq - 1)) || (Lk > 1 && mK > lim / (Lk - 1)))
            return fail(QD_ERR_INVALID_ARG, "the mask's extent overflows 64-bit indexing");
        *mask_span = (size_t)((B - 1) * mB + (Lq - 1) * mQ + (Lk - 1) * mK + 1);
    }
    if (q == nullptr || k == nullptr || v == nullptr) return fail(QD_ERR_INVALID_ARG, "NULL q, k or v");
    a->q = q, a->k = k, a->v = v, a->mask = mask, a->mB = mB, a->mQ = mQ, a->mK = mK;
    a->B = B, a->Lq = Lq, a->Lk = Lk, a->h = heads, a->dh = dh, a->D = heads * dh;
    a->rdh = (float)std::sqrt((double)dh);
    return QD_OK;
}

int check_ln(const float* x, const float* a2, int64_t rows, int64_t d, float eps, LnArgs* a) {
    if (rows < 0 || d < 1) return fail(QD_ERR_INVALID_ARG, "rows must be >= 0 and d >= 1 (rows=%lld d=%lld)", (long long)rows, (long long)d);
    if (rows > INT64_MAX / 16 / d) return fail(QD_ERR_INVALID_ARG, "rows * d overflows 64-bit indexing");
    if (!std::isfinite(eps)) return fail(QD_ERR_INVALID_ARG, "eps must be finite");
    if (x == nullptr || a2 == nullptr) return fail(QD_ERR_INVALID_ARG, "NULL x or a_2");
    a->x = x, a->a2 = a2, a->rows = rows, a->d = d, a->eps = eps;
    a->chunks = (rows + kLnChunk - 1) / kLnChunk;
    return QD_OK;
}

}  // namespace

extern "C" size_t qd_mha_workspace_bytes(int64_t B, int64_t heads, int64_t Lq, int64_t Lk) {
    return B > 0 && heads > 0 && Lq > 0 && Lk > 0 ? (size_t)B * (size_t)heads * (size_t)Lq * (size_t)Lk * sizeof(float) : 0;
}

extern "C" int qd_mha_fwd(const float* q, const float* k, const float* v, const uint8_t* mask, int64_t mask_batch_stride,
                          int64_t mask_query_stride, int64_t mask_key_stride, const uint8_t* keep, float keep_scale,
                          int64_t B, int64_t Lq, int64_t Lk, int64_t heads, int64_t dh, float* out, float* probs,
                          float* top, qd_stream_t stream) {
    MhArgs a{};
    size_t mspan;
    int rc = check_mha(q, k, v, mask, mask_batch_stride, mask_query_stride, mask_key_stride, B, Lq, Lk, heads, dh, &a, &mspan);
    if (rc) return rc;
    if (keep != nullptr && !std::isfinite(keep_scale)) return fail(QD_ERR_INVALID_ARG, "keep_scale must be finite");
    if (out == nullptr || probs == nullptr || top == nullptr) return fail(QD_ERR_INVALID_ARG, "NULL out, probs or top");
    if (misaligned(q, 4) || misaligned(k, 4) || misaligned(v, 4) || misaligned(out, 4) || misaligned(probs, 4) || misaligned(top, 4))
        return fail(QD_ERR_INVALID_ARG, "float arrays must be 4-byte aligned");
    const size_t qb = (size_t)(B * Lq * a.D) * sizeof(float), kb = (size_t)(B * Lk * a.D) * sizeof(float);
    const size_t pn = (size_t)(B * heads * Lq * Lk), tb = (size_t)(B * Lq * Lk) * sizeof(float);
    rc = check_disjoint({{q, qb}, {k, kb}, {v, kb}, {mask, mspan}, {keep, pn}}, {{out, qb}, {probs, pn * sizeof(float)}, {top, tb}});
    if (rc) return rc;
    a.keep = keep, a.scale = keep_scale, a.out = out, a.probs = probs, a.top = top;
    // blockIdx.x walks the (b, head) pairs, blockIdx.y the tiles (or key chunks) of one; both loop past the grid
    mha_fwd_kernel<<<grid_2d(B * heads, (Lq + kMhTile - 1) / kMhTile), kMhThreads, 0, as_stream(stream)>>>(a);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

extern "C" int qd_mha_bwd(const float* grad_out, const float* grad_top, const float* q, const float* k, const float* v,
                          const float* probs, const uint8_t* mask, int64_t mask_batch_stride, int64_t mask_query_stride,
                          int64_t mask_key_stride, const uint8_t* keep, float keep_scale, int64_t B, int64_t Lq,
                          int64_t Lk, int64_t heads, int64_t dh, float* grad_q, float* grad_k, float* grad_v,
                          void* workspace, size_t workspace_bytes, qd_stream_t stream) {
    MhArgs a{};
    size_t mspan;
    int rc = check_mha(q, k, v, mask, mask_batch_stride, mask_query_stride, mask_key_stride, B, Lq, Lk, heads, dh, &a, &mspan);
    if (rc) return rc;
    if (keep != nullptr && !std::isfinite(keep_scale)) return fail(QD_ERR_INVALID_ARG, "keep_scale must be finite");
    if (grad_out == nullptr || probs == nullptr || grad_q == nullptr || grad_k == nullptr || grad_v == nullptr)
        return fail(QD_ERR_INVALID_ARG, "NULL grad_out, probs, grad_q, grad_k or grad_v");
    if (misaligned(grad_out, 4) || misaligned(grad_top, 4) || misaligned(q, 4) || misaligned(k, 4) || misaligned(v, 4) ||
        misaligned(probs, 4) || misaligned(grad_q, 4) || misaligned(grad_k, 4) || misaligned(grad_v, 4))
        return fail(QD_ERR_INVALID_ARG, "float arrays must be 4-byte aligned");
    const size_t need = qd_mha_workspace_bytes(B, heads, Lq, Lk);
    rc = check_workspace(workspace, workspace_bytes, need, 4, "qd_mha_workspace_bytes(B, heads, Lq, Lk)");
    if (rc) return rc;
    const size_t qb = (size_t)(B * Lq * a.D) * sizeof(float), kb = (size_t)(B * Lk * a.D) * sizeof(float);
    const size_t pn = (size_t)(B * heads * Lq * Lk), tb = (size_t)(B * Lq * Lk) * sizeof(float);
    rc = check_disjoint({{grad_out, qb}, {grad_top, tb}, {q, qb}, {k, kb}, {v, kb}, {probs, pn * sizeof(float)}, {mask, mspan}, {keep, pn}},
                        {{grad_q, qb}, {grad_k, kb}, {grad_v, kb}, {workspace, need}});
    if (rc) return rc;
    a.grad_out = grad_out, a.grad_top = grad_top, a.probs = const_cast<float*>(probs), a.keep = keep, a.scale = keep_scale;
    a.ds = static_cast<float*>(workspace), a.grad_q = grad_q, a.grad_k = grad_k, a.grad_v = grad_v;
    cudaStream_t st = as_stream(stream);
    mha_bwd_rows_kernel<<<grid_2d(B * heads, (Lq + kMhTile - 1) / kMhTile), kMhThreads, 0, st>>>(a);
    mha_bwd_keys_kernel<<<grid_2d(B * heads, (Lk + kMhKChunk - 1) / kMhKChunk), kMhThreads, 0, st>>>(a);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

extern "C" size_t qd_onmt_layernorm_workspace_bytes(int64_t rows, int64_t d) {
    return rows > 0 && d > 1 ? (size_t)2 * (size_t)((rows + kLnChunk - 1) / kLnChunk) * (size_t)d * sizeof(float) : 0;
}

extern "C" int qd_onmt_layernorm_fwd(const float* x, const float* residual, const float* a_2, const float* b_2,
                                     int64_t rows, int64_t d, float eps, float* y, qd_stream_t stream) {
    LnArgs a{};
    int rc = check_ln(x, a_2, rows, d, eps, &a);
    if (rc) return rc;
    if (b_2 == nullptr || y == nullptr) return fail(QD_ERR_INVALID_ARG, "NULL b_2 or y");
    if (misaligned(x, 4) || misaligned(residual, 4) || misaligned(a_2, 4) || misaligned(b_2, 4) || misaligned(y, 4))
        return fail(QD_ERR_INVALID_ARG, "float arrays must be 4-byte aligned");
    const size_t xb = (size_t)(rows * d) * sizeof(float), pb = (size_t)d * sizeof(float);
    rc = check_disjoint({{x, xb}, {residual, xb}, {a_2, pb}, {b_2, pb}}, {{y, xb}});
    if (rc) return rc;
    if (rows == 0) return QD_OK;
    a.res = residual, a.b2 = b_2, a.y = y;
    ln_fwd_kernel<<<clamp_grid((rows + kMhWarps - 1) / kMhWarps), kMhThreads, 0, as_stream(stream)>>>(a);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

extern "C" int qd_onmt_layernorm_bwd(const float* grad_y, const float* x, const float* residual, const float* a_2,
                                     int64_t rows, int64_t d, float eps, float* grad_x,
                                     float* grad_a_2, float* grad_b_2, void* workspace, size_t workspace_bytes,
                                     qd_stream_t stream) {
    LnArgs a{};
    int rc = check_ln(x, a_2, rows, d, eps, &a);
    if (rc) return rc;
    if (grad_y == nullptr || grad_x == nullptr || grad_a_2 == nullptr || grad_b_2 == nullptr)
        return fail(QD_ERR_INVALID_ARG, "NULL grad_y, grad_x, grad_a_2 or grad_b_2");
    if (misaligned(grad_y, 4) || misaligned(x, 4) || misaligned(residual, 4) || misaligned(a_2, 4) || misaligned(grad_x, 4) ||
        misaligned(grad_a_2, 4) || misaligned(grad_b_2, 4))
        return fail(QD_ERR_INVALID_ARG, "float arrays must be 4-byte aligned");
    const size_t need = qd_onmt_layernorm_workspace_bytes(rows, d);
    if (need > 0 || workspace != nullptr) {   // d = 1 or rows = 0 takes a NULL workspace, but no misaligned one
        rc = check_workspace(workspace, workspace_bytes, need, 4, "qd_onmt_layernorm_workspace_bytes(rows, d)");
        if (rc) return rc;
    }
    const size_t xb = (size_t)(rows * d) * sizeof(float), pb = (size_t)d * sizeof(float);
    rc = check_disjoint({{grad_y, xb}, {x, xb}, {residual, xb}, {a_2, pb}},
                        {{grad_x, xb}, {grad_a_2, pb}, {grad_b_2, pb}, {workspace, need}});
    if (rc) return rc;
    a.res = residual, a.grad_y = grad_y, a.grad_x = grad_x, a.grad_a2 = grad_a_2, a.grad_b2 = grad_b_2;
    a.partial = static_cast<float*>(workspace);
    cudaStream_t st = as_stream(stream);
    if (rows > 0) ln_bwd_kernel<<<clamp_grid(a.chunks), kMhThreads, 0, st>>>(a);
    ln_param_kernel<<<clamp_grid((2 * d + kMhThreads - 1) / kMhThreads), kMhThreads, 0, st>>>(a);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}
