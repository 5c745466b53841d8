// qd_attention.cu -- the core of onmt's GlobalAttention for the "dot" and "general" scores
// (onmt/modules/GlobalAttention.py:108-188): score -> softmax over the source -> weighted context -> [c | input].  The
// query projection linear_in and the output linear_out + tanh stay GEMMs outside.
//
// Rows: batch entry n has T query rows; q and input are n-major ([N, T, H], row n*T + t), align and concat are t-major
// ([T, N, .], row t*N + n), the order the reference returns them.  Row (n, t) attends to the context slab of n, read at
// context + n*sN + s*sS + h: the contiguous [N, S, H] and the transposed view of a contiguous [S, N, H] alike.
//
// Forward (qd_attn_fwd): one 256-thread CTA per tile of up to kAtTile rows of one n, three phases:
//   1. scores (qd_attn_tile.cuh's tile_dots): warp w owns the source positions s = w + 8k, lane l the elements
//      h = l + 32j; per row a lane-strided float32 sum and a butterfly over the warp.  The raw scores go to align.
//   2. softmax (softmax_row): warp t owns row t of the tile; max, then sum of expf(x - max) (lane-strided, butterfly),
//      then align = expf(x - max) / sum in place.
//   3. context: thread j owns h = j + 256k and sums align_s * h_s over s in order; it writes c and copies input beside.
// The slab is read from HBM once per tile in phase 1; phase 3 reads it again from L2 (at most S*H*4 bytes per tile).
//
// Backward: qd_attn_bwd_rows runs the same three phases on grad_concat (ga = gc . h_s + grad_align, then
// gs = align (ga - sum_s align ga) into the workspace, then grad_q = sum_s gs h_s); qd_attn_bwd_context gives each CTA
// kAtSChunk source positions of one n and sums a_{r,s} gc_r + gs_{r,s} q_r over that n's rows in the order t = 0..T-1.
//
// Which thread owns which element, and every summation order, depend only on (S, H): a row's forward bits are the
// same alone or in any batch; all loads are scalar, so the alignment of a view changes nothing either.
#include <cmath>

#include "qd_attn_tile.cuh"
#include "qd_launch.h"

using namespace qd;

namespace {

constexpr int kAtThreads = 256;
constexpr int kAtWarps = kAtThreads / 32;
constexpr int kAtTile = 8;          // query rows of one batch entry per CTA (phase 2 gives each a warp)
constexpr int kAtSChunk = 8;        // source positions per CTA of the context gradient
static_assert(kAtTile <= kAtWarps, "phase 2 gives each row of a tile its own warp");

// out[t*os + h] = sum_s p[t*ps + s] h_s[h] for the nt rows of a tile, s in order
__device__ __forceinline__ void tile_weighted_sum(const float* __restrict__ ctx, int64_t sS, int64_t S, int64_t H,
                                                  const float* p, int64_t ps, int nt, float* __restrict__ out, int64_t os) {
    for (int64_t h = threadIdx.x; h < H; h += kAtThreads) {
        float acc[kAtTile];
#pragma unroll
        for (int t = 0; t < kAtTile; ++t) acc[t] = 0.f;
#pragma unroll 4
        for (int64_t s = 0; s < S; ++s) {
            const float x = __ldg(ctx + s * sS + h);
#pragma unroll
            for (int t = 0; t < kAtTile; ++t)
                if (t < nt) acc[t] = __fadd_rn(acc[t], __fmul_rn(p[t * ps + s], x));
        }
#pragma unroll
        for (int t = 0; t < kAtTile; ++t)
            if (t < nt) out[t * os + h] = acc[t];
    }
}

struct AtShape {
    const float* ctx;
    int64_t sN, sS, N, T, S, H;
};

struct AtFwdArgs {
    AtShape g;
    const float* q;       // [N, T, H]
    const float* input;   // [N, T, H]
    float* align;         // [T, N, S]
    float* concat;        // [T, N, 2H]
};

__global__ void __launch_bounds__(kAtThreads) attn_fwd_kernel(AtFwdArgs a) {
    const AtShape g = a.g;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int64_t n = blockIdx.x; n < g.N; n += gridDim.x)
    for (int64_t t0 = (int64_t)blockIdx.y * kAtTile; t0 < g.T; t0 += (int64_t)gridDim.y * kAtTile) {
        const int nt = (int)min((int64_t)kAtTile, g.T - t0);
        const float* ctx = g.ctx + n * g.sN;
        const int64_t in_row = (n * g.T + t0) * g.H, out_row = t0 * g.N + n;
        float* al = a.align + out_row * g.S;
        const int64_t as = g.N * g.S;
        attn::tile_dots<kAtTile, kAtWarps, 4>(a.q + in_row, g.H, ctx, g.sS, g.S, g.H, nt,
                                              [&](int t, int64_t s, float d) { al[t * as + s] = d; });
        __syncthreads();
        if (warp < nt) {
            float* row = al + warp * as;
            attn::softmax_row(row, g.S, lane, [&](int64_t s, float y) { row[s] = y; });
        }
        __syncthreads();
        float* cc = a.concat + out_row * 2 * g.H;
        const int64_t cs = g.N * 2 * g.H;
        tile_weighted_sum(ctx, g.sS, g.S, g.H, al, as, nt, cc, cs);
        for (int64_t h = threadIdx.x; h < g.H; h += kAtThreads)
            for (int t = 0; t < nt; ++t) cc[t * cs + g.H + h] = __ldg(a.input + in_row + t * g.H + h);
    }
}

struct AtBwdArgs {
    AtShape g;
    const float* grad_concat;   // [T, N, 2H]
    const float* grad_align;    // [T, N, S] or NULL
    const float* align;         // [T, N, S]
    const float* q;             // [N, T, H]
    float* gs;                  // workspace [T, N, S]
    float* grad_q;              // [N, T, H]
    float* grad_ctx;            // the context's layout
};

__global__ void __launch_bounds__(kAtThreads) attn_bwd_rows_kernel(AtBwdArgs a) {
    const AtShape g = a.g;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int64_t n = blockIdx.x; n < g.N; n += gridDim.x)
    for (int64_t t0 = (int64_t)blockIdx.y * kAtTile; t0 < g.T; t0 += (int64_t)gridDim.y * kAtTile) {
        const int nt = (int)min((int64_t)kAtTile, g.T - t0);
        const float* ctx = g.ctx + n * g.sN;
        const int64_t in_row = (n * g.T + t0) * g.H, out_row = t0 * g.N + n;
        const int64_t as = g.N * g.S;
        float* gs = a.gs + out_row * g.S;
        const float* ga = a.grad_align != nullptr ? a.grad_align + out_row * g.S : nullptr;
        attn::tile_dots<kAtTile, kAtWarps, 4>(a.grad_concat + out_row * 2 * g.H, g.N * 2 * g.H, ctx, g.sS, g.S, g.H, nt,
                                              [&](int t, int64_t s, float d) {
                                                  if (ga != nullptr) d = __fadd_rn(d, __ldg(ga + t * as + s));
                                                  gs[t * as + s] = d;
                                              });
        __syncthreads();
        if (warp < nt) attn::softmax_row_bwd(a.align + out_row * g.S + warp * as, gs + warp * as, g.S, lane);
        __syncthreads();
        tile_weighted_sum(ctx, g.sS, g.S, g.H, gs, as, nt, a.grad_q + in_row, g.H);
    }
}

__global__ void __launch_bounds__(kAtThreads) attn_bwd_context_kernel(AtBwdArgs a) {
    const AtShape g = a.g;
    for (int64_t n = blockIdx.x; n < g.N; n += gridDim.x)
    for (int64_t s0 = (int64_t)blockIdx.y * kAtSChunk; s0 < g.S; s0 += (int64_t)gridDim.y * kAtSChunk) {
        const int ns = (int)min((int64_t)kAtSChunk, g.S - s0);
        for (int64_t h = threadIdx.x; h < g.H; h += kAtThreads) {
            float acc[kAtSChunk];
#pragma unroll
            for (int j = 0; j < kAtSChunk; ++j) acc[j] = 0.f;
            for (int64_t t = 0; t < g.T; ++t) {
                const int64_t r = t * g.N + n;
                const float gc = __ldg(a.grad_concat + r * 2 * g.H + h), qv = __ldg(a.q + (n * g.T + t) * g.H + h);
                const float* al = a.align + r * g.S + s0;
                const float* gs = a.gs + r * g.S + s0;
#pragma unroll
                for (int j = 0; j < kAtSChunk; ++j)
                    if (j < ns) acc[j] = __fadd_rn(acc[j], __fadd_rn(__fmul_rn(__ldg(al + j), gc), __fmul_rn(__ldg(gs + j), qv)));
            }
#pragma unroll
            for (int j = 0; j < kAtSChunk; ++j)
                if (j < ns) a.grad_ctx[n * g.sN + (s0 + j) * g.sS + h] = acc[j];
        }
    }
}

// ---- "mlp" (Bahdanau) attention: score[n, t, s] = sum_h v_h tanhf(wq[n, t, h] + uh[n, s, h]) ----
struct MlpScore {
    const float* wq;            // [N, T, H]
    const float* uh;            // read at uh[n*uN + s*uS + h]
    int64_t uN, uS;
    const float* v;             // [H]
};

struct MlpFwdArgs {
    AtShape g;                  // the context
    MlpScore m;
    const float* input;         // [N, T, H]
    float* align;               // [T, N, S]
    float* concat;              // [T, N, 2H]
};

struct MlpBwdArgs {
    AtShape g;
    MlpScore m;
    const float* grad_concat;   // [T, N, 2H]
    const float* grad_align;    // [T, N, S] or NULL
    const float* align;         // [T, N, S]
    float* gs;                  // workspace [T, N, S]
    float* gv_part;             // workspace [N, chunks, H]: the grad_v partial of (n, source chunk)
    int64_t chunks;             // ceil(S / kAtSChunk)
    float* grad_wq;             // [N, T, H]
    float* grad_uh;             // uh's layout
    float* grad_v;              // [H]
    float* grad_ctx;            // the context's layout
};

// d score / d (wq + uh) of one term, scaled by gs: gs v_h (1 - e^2), the same expression in both backward kernels
__device__ __forceinline__ float mlp_term(float gs, float vh, float e) {
    return __fmul_rn(gs, __fmul_rn(vh, __fsub_rn(1.f, __fmul_rn(e, e))));
}

// tile_dots's order with the mlp score: warp w owns the source positions s = w + 8k, lane l the elements h = l + 32j;
// per row a lane-strided float32 sum of v_h tanhf(wq_t[h] + uh_s[h]) and a butterfly over the warp
template <class F>
__device__ __forceinline__ void tile_mlp_scores(const float* __restrict__ wq, const float* __restrict__ uh, int64_t uS,
                                                const float* __restrict__ v, int64_t S, int64_t H, int nt, F&& fin) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int64_t s = warp; s < S; s += kAtWarps) {
        const float* us = uh + s * uS;
        float acc[kAtTile];
#pragma unroll
        for (int t = 0; t < kAtTile; ++t) acc[t] = 0.f;
#pragma unroll 2
        for (int64_t h = lane; h < H; h += 32) {
            const float x = __ldg(us + h), vh = __ldg(v + h);
#pragma unroll
            for (int t = 0; t < kAtTile; ++t) {
                if (t >= nt) break;
                acc[t] = __fadd_rn(acc[t], __fmul_rn(vh, tanhf(__fadd_rn(__ldg(wq + t * H + h), x))));
            }
        }
#pragma unroll
        for (int t = 0; t < kAtTile; ++t) {
            if (t >= nt) break;
            const float d = attn::warp_sum(acc[t]);
            if (lane == 0) fin(t, s, d);
        }
    }
}

__global__ void __launch_bounds__(kAtThreads) attn_mlp_fwd_kernel(MlpFwdArgs a) {
    const AtShape g = a.g;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int64_t n = blockIdx.x; n < g.N; n += gridDim.x)
    for (int64_t t0 = (int64_t)blockIdx.y * kAtTile; t0 < g.T; t0 += (int64_t)gridDim.y * kAtTile) {
        const int nt = (int)min((int64_t)kAtTile, g.T - t0);
        const float* ctx = g.ctx + n * g.sN;
        const int64_t in_row = (n * g.T + t0) * g.H, out_row = t0 * g.N + n;
        float* al = a.align + out_row * g.S;
        const int64_t as = g.N * g.S;
        tile_mlp_scores(a.m.wq + in_row, a.m.uh + n * a.m.uN, a.m.uS, a.m.v, g.S, g.H, nt,
                        [&](int t, int64_t s, float d) { al[t * as + s] = d; });
        __syncthreads();
        if (warp < nt) {
            float* row = al + warp * as;
            attn::softmax_row(row, g.S, lane, [&](int64_t s, float y) { row[s] = y; });
        }
        __syncthreads();
        float* cc = a.concat + out_row * 2 * g.H;
        const int64_t cs = g.N * 2 * g.H;
        tile_weighted_sum(ctx, g.sS, g.S, g.H, al, as, nt, cc, cs);
        for (int64_t h = threadIdx.x; h < g.H; h += kAtThreads)
            for (int t = 0; t < nt; ++t) cc[t * cs + g.H + h] = __ldg(a.input + in_row + t * g.H + h);
    }
}

// Per tile of rows: gs as attn_bwd_rows_kernel's phases 1-2, then grad_wq[t, h] = sum_s mlp_term, s in order
__global__ void __launch_bounds__(kAtThreads) attn_mlp_bwd_rows_kernel(MlpBwdArgs a) {
    const AtShape g = a.g;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int64_t n = blockIdx.x; n < g.N; n += gridDim.x)
    for (int64_t t0 = (int64_t)blockIdx.y * kAtTile; t0 < g.T; t0 += (int64_t)gridDim.y * kAtTile) {
        const int nt = (int)min((int64_t)kAtTile, g.T - t0);
        const float* ctx = g.ctx + n * g.sN;
        const float* uh = a.m.uh + n * a.m.uN;
        const int64_t in_row = (n * g.T + t0) * g.H, out_row = t0 * g.N + n;
        const int64_t as = g.N * g.S;
        float* gs = a.gs + out_row * g.S;
        const float* ga = a.grad_align != nullptr ? a.grad_align + out_row * g.S : nullptr;
        attn::tile_dots<kAtTile, kAtWarps, 4>(a.grad_concat + out_row * 2 * g.H, g.N * 2 * g.H, ctx, g.sS, g.S, g.H, nt,
                                              [&](int t, int64_t s, float d) {
                                                  if (ga != nullptr) d = __fadd_rn(d, __ldg(ga + t * as + s));
                                                  gs[t * as + s] = d;
                                              });
        __syncthreads();
        if (warp < nt) attn::softmax_row_bwd(a.align + out_row * g.S + warp * as, gs + warp * as, g.S, lane);
        __syncthreads();
        for (int64_t h = threadIdx.x; h < g.H; h += kAtThreads) {
            const float vh = __ldg(a.m.v + h);
            float w[kAtTile], acc[kAtTile];
#pragma unroll
            for (int t = 0; t < kAtTile; ++t) {
                w[t] = t < nt ? __ldg(a.m.wq + in_row + t * g.H + h) : 0.f;
                acc[t] = 0.f;
            }
            for (int64_t s = 0; s < g.S; ++s) {
                const float x = __ldg(uh + s * a.m.uS + h);
#pragma unroll
                for (int t = 0; t < kAtTile; ++t) {
                    if (t >= nt) break;
                    acc[t] = __fadd_rn(acc[t], mlp_term(gs[t * as + s], vh, tanhf(__fadd_rn(w[t], x))));
                }
            }
#pragma unroll
            for (int t = 0; t < kAtTile; ++t)
                if (t < nt) a.grad_wq[in_row + t * g.H + h] = acc[t];
        }
    }
}

// Per kAtSChunk source positions of one n, over that n's rows in t order: grad_uh[s, h] = sum_t mlp_term,
// grad_context[s, h] = sum_t align_{t,s} gc_t[h], and the grad_v partial sum_t sum_s gs e (s in order within t)
__global__ void __launch_bounds__(kAtThreads) attn_mlp_bwd_source_kernel(MlpBwdArgs a) {
    const AtShape g = a.g;
    for (int64_t n = blockIdx.x; n < g.N; n += gridDim.x)
    for (int64_t s0 = (int64_t)blockIdx.y * kAtSChunk; s0 < g.S; s0 += (int64_t)gridDim.y * kAtSChunk) {
        const int ns = (int)min((int64_t)kAtSChunk, g.S - s0);
        const float* uh = a.m.uh + n * a.m.uN + s0 * a.m.uS;
        float* part = a.gv_part + (n * a.chunks + s0 / kAtSChunk) * g.H;
        for (int64_t h = threadIdx.x; h < g.H; h += kAtThreads) {
            const float vh = __ldg(a.m.v + h);
            float x[kAtSChunk], au[kAtSChunk], ac[kAtSChunk], pv = 0.f;
#pragma unroll
            for (int j = 0; j < kAtSChunk; ++j) {
                x[j] = j < ns ? __ldg(uh + j * a.m.uS + h) : 0.f;
                au[j] = ac[j] = 0.f;
            }
            for (int64_t t = 0; t < g.T; ++t) {
                const int64_t r = t * g.N + n;
                const float gc = __ldg(a.grad_concat + r * 2 * g.H + h), w = __ldg(a.m.wq + (n * g.T + t) * g.H + h);
                const float* al = a.align + r * g.S + s0;
                const float* gs = a.gs + r * g.S + s0;
#pragma unroll
                for (int j = 0; j < kAtSChunk; ++j) {
                    if (j < ns) {
                        const float e = tanhf(__fadd_rn(w, x[j])), gsv = __ldg(gs + j);
                        au[j] = __fadd_rn(au[j], mlp_term(gsv, vh, e));
                        ac[j] = __fadd_rn(ac[j], __fmul_rn(__ldg(al + j), gc));
                        pv = __fadd_rn(pv, __fmul_rn(gsv, e));
                    }
                }
            }
#pragma unroll
            for (int j = 0; j < kAtSChunk; ++j) {
                if (j < ns) {
                    a.grad_uh[n * a.m.uN + (s0 + j) * a.m.uS + h] = au[j];
                    a.grad_ctx[n * g.sN + (s0 + j) * g.sS + h] = ac[j];
                }
            }
            part[h] = pv;
        }
    }
}

// grad_v[h]: the sum of the (n, chunk) partials, n-major, chunk 0 first
__global__ void __launch_bounds__(kAtThreads) attn_mlp_grad_v_kernel(MlpBwdArgs a) {
    const int64_t rows = a.g.N * a.chunks, H = a.g.H;
    for (int64_t h = (int64_t)blockIdx.x * kAtThreads + threadIdx.x; h < H; h += (int64_t)gridDim.x * kAtThreads) {
        const float* p = a.gv_part + h;
        float s = 0.f;
#pragma unroll 8
        for (int64_t r = 0; r < rows; ++r) s = __fadd_rn(s, __ldg(p + r * H));
        a.grad_v[h] = s;
    }
}

// checks of the sizes and the context layout both calls share; R = N*T.  span: bytes from context to its last element
// (`what` names the tensor read through those strides in the messages)
int check_shape(const float* ctx, int64_t sN, int64_t sS, int64_t N, int64_t T, int64_t S, int64_t H, int64_t* R,
                size_t* span, const char* what = "context") {
    if (N < 0 || T < 0 || S < 0 || H < 0) return fail(QD_ERR_INVALID_ARG, "sizes must be >= 0 (N=%lld T=%lld S=%lld H=%lld)",
                                                      (long long)N, (long long)T, (long long)S, (long long)H);
    if (T > 0 && N > INT64_MAX / T) return fail(QD_ERR_INVALID_ARG, "N * T overflows 64-bit indexing");
    *R = N * T;
    *span = 0;
    if (*R == 0) return QD_OK;
    if (S == 0 || H == 0) return fail(QD_ERR_INVALID_ARG, "S and H must be >= 1 when there are rows (S=%lld H=%lld)",
                                      (long long)S, (long long)H);
    if (sN < 0 || sS < 0) return fail(QD_ERR_INVALID_ARG, "%s strides must be >= 0", what);
    const int64_t lim = INT64_MAX / 8;
    if (*R > lim / S || *R > lim / (2 * H)) return fail(QD_ERR_INVALID_ARG, "rows * S or rows * 2H overflows 64-bit indexing");
    if ((N > 1 && sN > (lim - H) / (N - 1)) || (S > 1 && sS > (lim - H) / (S - 1)) ||
        (N - 1) * sN > lim - H - (S - 1) * sS)
        return fail(QD_ERR_INVALID_ARG, "the %s's extent overflows 64-bit indexing", what);
    // the (batch, source) rows of H elements must not overlap: the smaller stride covers a row, the larger its run
    int64_t lo = sS, clo = S, hi = sN, chi = N;
    if (sN < sS || (sN == sS && N < S)) lo = sN, clo = N, hi = sS, chi = S;
    if ((clo > 1 && lo < H) || (chi > 1 && hi < (clo - 1) * lo + H))
        return fail(QD_ERR_INVALID_ARG, "%s strides (batch %lld, source %lld) make rows of %lld elements overlap",
                    what, (long long)sN, (long long)sS, (long long)H);
    if (ctx == nullptr) return fail(QD_ERR_INVALID_ARG, "NULL %s", what);
    *span = (size_t)((N - 1) * sN + (S - 1) * sS + H) * sizeof(float);
    return QD_OK;
}

}  // namespace

extern "C" size_t qd_attn_workspace_bytes(int64_t rows, int64_t S) {
    return rows > 0 && S > 0 ? (size_t)rows * (size_t)S * sizeof(float) : 0;
}

extern "C" int qd_attn_fwd(int kind, const float* q, const float* input, const float* context, int64_t ctx_batch_stride,
                           int64_t ctx_src_stride, int64_t N, int64_t T, int64_t S, int64_t H, float* align, float* concat,
                           qd_stream_t stream) {
    if (kind != QD_ATTN_DOT && kind != QD_ATTN_GENERAL) return fail(QD_ERR_INVALID_ARG, "kind must be QD_ATTN_DOT or QD_ATTN_GENERAL");
    if (kind == QD_ATTN_DOT && q != nullptr && q != input) return fail(QD_ERR_INVALID_ARG, "dot attention reads its query from input: q must be NULL");
    int64_t R;
    size_t span;
    int rc = check_shape(context, ctx_batch_stride, ctx_src_stride, N, T, S, H, &R, &span);
    if (rc) return rc;
    if (R == 0) return QD_OK;
    if (kind == QD_ATTN_DOT) q = input;
    if (q == nullptr || input == nullptr || align == nullptr || concat == nullptr) return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if (misaligned(q, 4) || misaligned(input, 4) || misaligned(context, 4) || misaligned(align, 4) || misaligned(concat, 4))
        return fail(QD_ERR_INVALID_ARG, "float arrays must be 4-byte aligned");
    const size_t row_bytes = (size_t)(R * H) * sizeof(float), al_bytes = (size_t)(R * S) * sizeof(float);
    rc = check_disjoint({{q, row_bytes}, {input, row_bytes}, {context, span}}, {{align, al_bytes}, {concat, 2 * row_bytes}});
    if (rc) return rc;
    AtFwdArgs a{};
    a.g = AtShape{context, ctx_batch_stride, ctx_src_stride, N, T, S, H};
    a.q = q, a.input = input, a.align = align, a.concat = concat;
    // blockIdx.x walks the batch entries, blockIdx.y the tiles (or source chunks) of one; both loop past the grid
    attn_fwd_kernel<<<grid_2d(N, (T + kAtTile - 1) / kAtTile), kAtThreads, 0, as_stream(stream)>>>(a);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

extern "C" int qd_attn_bwd(const float* grad_concat, const float* grad_align, const float* align, const float* q,
                           const float* context, int64_t ctx_batch_stride, int64_t ctx_src_stride, int64_t N, int64_t T,
                           int64_t S, int64_t H, float* grad_q, float* grad_context, void* workspace, size_t workspace_bytes,
                           qd_stream_t stream) {
    int64_t R;
    size_t span;
    int rc = check_shape(context, ctx_batch_stride, ctx_src_stride, N, T, S, H, &R, &span);
    if (rc) return rc;
    if (R == 0) return QD_OK;
    if (grad_concat == nullptr || align == nullptr || q == nullptr || grad_q == nullptr || grad_context == nullptr)
        return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if (misaligned(grad_concat, 4) || misaligned(grad_align, 4) || misaligned(align, 4) || misaligned(q, 4) ||
        misaligned(context, 4) || misaligned(grad_q, 4) || misaligned(grad_context, 4))
        return fail(QD_ERR_INVALID_ARG, "float arrays must be 4-byte aligned");
    const size_t need = qd_attn_workspace_bytes(R, S);
    rc = check_workspace(workspace, workspace_bytes, need, 4, "qd_attn_workspace_bytes(N * T, S)");
    if (rc) return rc;
    const size_t row_bytes = (size_t)(R * H) * sizeof(float), al_bytes = (size_t)(R * S) * sizeof(float);
    rc = check_disjoint({{grad_concat, 2 * row_bytes}, {grad_align, al_bytes}, {align, al_bytes}, {q, row_bytes}, {context, span}},
                        {{grad_q, row_bytes}, {grad_context, span}, {workspace, need}});
    if (rc) return rc;
    AtBwdArgs a{};
    a.g = AtShape{context, ctx_batch_stride, ctx_src_stride, N, T, S, H};
    a.grad_concat = grad_concat, a.grad_align = grad_align, a.align = align, a.q = q;
    a.gs = static_cast<float*>(workspace), a.grad_q = grad_q, a.grad_ctx = grad_context;
    cudaStream_t st = as_stream(stream);
    attn_bwd_rows_kernel<<<grid_2d(N, (T + kAtTile - 1) / kAtTile), kAtThreads, 0, st>>>(a);
    attn_bwd_context_kernel<<<grid_2d(N, (S + kAtSChunk - 1) / kAtSChunk), kAtThreads, 0, st>>>(a);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

extern "C" size_t qd_attn_mlp_workspace_bytes(int64_t N, int64_t T, int64_t S, int64_t H) {
    if (N <= 0 || T <= 0 || S <= 0 || H <= 0) return 0;
    const uint64_t chunks = (uint64_t)((S + kAtSChunk - 1) / kAtSChunk);
    uint64_t rs, part, total;
    if (__builtin_mul_overflow((uint64_t)N, (uint64_t)T, &rs) || __builtin_mul_overflow(rs, (uint64_t)S, &rs) ||
        __builtin_mul_overflow((uint64_t)N, chunks, &part) || __builtin_mul_overflow(part, (uint64_t)H, &part) ||
        __builtin_add_overflow(rs, part, &total) || total > SIZE_MAX / sizeof(float))
        return 0;                     // past what the calls accept: they refuse such sizes before the workspace
    return (size_t)total * sizeof(float);
}

extern "C" int qd_attn_mlp_fwd(const float* wq, const float* uh, int64_t uh_batch_stride, int64_t uh_src_stride,
                               const float* v, const float* input, const float* context, int64_t ctx_batch_stride,
                               int64_t ctx_src_stride, int64_t N, int64_t T, int64_t S, int64_t H, float* align,
                               float* concat, qd_stream_t stream) {
    int64_t R;
    size_t span, uspan;
    int rc = check_shape(context, ctx_batch_stride, ctx_src_stride, N, T, S, H, &R, &span);
    if (rc) return rc;
    rc = check_shape(uh, uh_batch_stride, uh_src_stride, N, T, S, H, &R, &uspan, "uh");
    if (rc) return rc;
    if (R == 0) return QD_OK;
    if (wq == nullptr || v == nullptr || input == nullptr || align == nullptr || concat == nullptr)
        return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if (misaligned(wq, 4) || misaligned(uh, 4) || misaligned(v, 4) || misaligned(input, 4) || misaligned(context, 4) ||
        misaligned(align, 4) || misaligned(concat, 4))
        return fail(QD_ERR_INVALID_ARG, "float arrays must be 4-byte aligned");
    const size_t row_bytes = (size_t)(R * H) * sizeof(float), al_bytes = (size_t)(R * S) * sizeof(float);
    const size_t v_bytes = (size_t)H * sizeof(float);
    rc = check_disjoint({{wq, row_bytes}, {uh, uspan}, {v, v_bytes}, {input, row_bytes}, {context, span}},
                        {{align, al_bytes}, {concat, 2 * row_bytes}});
    if (rc) return rc;
    MlpFwdArgs a{};
    a.g = AtShape{context, ctx_batch_stride, ctx_src_stride, N, T, S, H};
    a.m = MlpScore{wq, uh, uh_batch_stride, uh_src_stride, v};
    a.input = input;
    a.align = align, a.concat = concat;
    attn_mlp_fwd_kernel<<<grid_2d(N, (T + kAtTile - 1) / kAtTile), kAtThreads, 0, as_stream(stream)>>>(a);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

extern "C" int qd_attn_mlp_bwd(const float* grad_concat, const float* grad_align, const float* align, const float* wq,
                               const float* uh, int64_t uh_batch_stride, int64_t uh_src_stride, const float* v,
                               const float* context, int64_t ctx_batch_stride, int64_t ctx_src_stride, int64_t N,
                               int64_t T, int64_t S, int64_t H, float* grad_wq, float* grad_uh, float* grad_v,
                               float* grad_context, void* workspace, size_t workspace_bytes, qd_stream_t stream) {
    int64_t R;
    size_t span, uspan;
    int rc = check_shape(context, ctx_batch_stride, ctx_src_stride, N, T, S, H, &R, &span);
    if (rc) return rc;
    rc = check_shape(uh, uh_batch_stride, uh_src_stride, N, T, S, H, &R, &uspan, "uh");
    if (rc) return rc;
    if (R == 0) return QD_OK;
    if (grad_concat == nullptr || align == nullptr || wq == nullptr || v == nullptr || grad_wq == nullptr ||
        grad_uh == nullptr || grad_v == nullptr || grad_context == nullptr)
        return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if (misaligned(grad_concat, 4) || misaligned(grad_align, 4) || misaligned(align, 4) || misaligned(wq, 4) ||
        misaligned(uh, 4) || misaligned(v, 4) || misaligned(context, 4) || misaligned(grad_wq, 4) ||
        misaligned(grad_uh, 4) || misaligned(grad_v, 4) || misaligned(grad_context, 4))
        return fail(QD_ERR_INVALID_ARG, "float arrays must be 4-byte aligned");
    const size_t need = qd_attn_mlp_workspace_bytes(N, T, S, H);
    rc = check_workspace(workspace, workspace_bytes, need, 4, "qd_attn_mlp_workspace_bytes(N, T, S, H)");
    if (rc) return rc;
    const size_t row_bytes = (size_t)(R * H) * sizeof(float), al_bytes = (size_t)(R * S) * sizeof(float);
    const size_t v_bytes = (size_t)H * sizeof(float);
    rc = check_disjoint({{grad_concat, 2 * row_bytes}, {grad_align, al_bytes}, {align, al_bytes}, {wq, row_bytes},
                         {uh, uspan}, {v, v_bytes}, {context, span}},
                        {{grad_wq, row_bytes}, {grad_uh, uspan}, {grad_v, v_bytes}, {grad_context, span}, {workspace, need}});
    if (rc) return rc;
    MlpBwdArgs a{};
    a.g = AtShape{context, ctx_batch_stride, ctx_src_stride, N, T, S, H};
    a.m = MlpScore{wq, uh, uh_batch_stride, uh_src_stride, v};
    a.grad_concat = grad_concat, a.grad_align = grad_align, a.align = align;
    a.gs = static_cast<float*>(workspace), a.gv_part = a.gs + R * S, a.chunks = (S + kAtSChunk - 1) / kAtSChunk;
    a.grad_wq = grad_wq, a.grad_uh = grad_uh, a.grad_v = grad_v, a.grad_ctx = grad_context;
    cudaStream_t st = as_stream(stream);
    attn_mlp_bwd_rows_kernel<<<grid_2d(N, (T + kAtTile - 1) / kAtTile), kAtThreads, 0, st>>>(a);
    attn_mlp_bwd_source_kernel<<<grid_2d(N, a.chunks), kAtThreads, 0, st>>>(a);
    attn_mlp_grad_v_kernel<<<clamp_grid((H + kAtThreads - 1) / kAtThreads), kAtThreads, 0, st>>>(a);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}
