// qd_sru.cu -- the SRU recurrence of onmt's SRU layers (onmt/modules/SRU.py:71-347, sru_fwd / sru_bwd /
// sru_bi_fwd / sru_bi_bwd), forward and backward.  The projection u = x_2d.mm(weight) stays a GEMM outside.
//
// Columns: col = b*(dir*d) + j walks [batch, dir*d]; u is [len, batch, dir*d, k] (the k values of a column adjacent),
// x, h, c, grad_h, grad_x are [len, batch, dir*d], init, mask_h, grad_last, grad_init are [batch, dir*d].  A
// bidirectional column with j >= d runs backwards in time.  One thread owns one column and runs its serial loop over
// time with the reference's float32 expressions in the reference's order (compiled -fmad=false: no contraction), so
// a column's bits depend on nothing but its own inputs: not on batch, CTA shape or launch.
//
// Each step's loads are issued kSruAhead steps before its math, from a ring of registers: with one thread per column
// a step's load latency is otherwise paid once per step, and at the NMT shapes (32,000 to 64,000 columns) too few
// loads are in flight to cover it.
//
// Backward: sru_bwd_kernel writes grad_u, grad_x, grad_init and the per-(batch, column) bias partials into the
// workspace, [2, batch, dir*d] as the reference's grad_bias; sru_bias_kernel sums them over the batch in b order.
#include <cmath>

#include "qd_launch.h"

using namespace qd;

namespace {

constexpr int kSruThreads = 128;
constexpr int kSruAhead = 4;        // steps whose loads are in flight ahead of the math

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ float reluf_(float x) { return (x > 0.f) ? x : 0.f; }
__device__ __forceinline__ float act_(int activation, float x) {
    return (activation == 1) ? tanhf(x) : ((activation == 2) ? reluf_(x) : x);
}

struct SruArgs {
    const float* u;
    const float* x;          // [len, batch, dir*d] when k = 3, NULL when k = 4
    const float* bias;       // [2 * dir*d]
    const float* init;       // [batch, dir*d] or NULL (zeros)
    const float* mask_h;     // [batch, dir*d] or NULL (ones)
    const float* c;          // backward: the forward's c
    const float* grad_h;
    const float* grad_last;  // [batch, dir*d] or NULL (zeros)
    float* h;
    float* cout;
    float* grad_u;
    float* grad_x;
    float* grad_init;        // or NULL
    float* partial;          // workspace [2, batch, dir*d]
    float* grad_bias;        // [2 * dir*d]
    int64_t len, ncols, dcols, d;
    int bidir, activation;
};

// u0, u1, u2 and the highway value of one step: u[..., 3] for k = 4, x for k = 3
template <int K, bool V4>
__device__ __forceinline__ void load_u(const SruArgs& a, int64_t tc, float& u0, float& u1, float& u2, float& xv) {
    const float* up = a.u + tc * K;
    if constexpr (V4) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(up));
        u0 = v.x, u1 = v.y, u2 = v.z, xv = v.w;
    } else {
        u0 = __ldg(up), u1 = __ldg(up + 1), u2 = __ldg(up + 2);
        xv = (K == 3) ? __ldg(a.x + tc) : __ldg(up + 3);
    }
}

template <int K, bool V4>
__global__ void __launch_bounds__(kSruThreads) sru_fwd_kernel(SruArgs a) {
    const int64_t stride = (int64_t)gridDim.x * kSruThreads;
    for (int64_t col = (int64_t)blockIdx.x * kSruThreads + threadIdx.x; col < a.ncols; col += stride) {
        const int64_t j = col % a.dcols;
        const bool flip = a.bidir && j >= a.d;
        const float bias1 = __ldg(a.bias + j), bias2 = __ldg(a.bias + j + a.dcols);
        const float mask = (a.mask_h == nullptr) ? 1.f : __ldg(a.mask_h + col);
        float cur = (a.init == nullptr) ? 0.f : __ldg(a.init + col);
        // step i is time t = flip ? len-1-i : i; (t*ncols + col) advances by dt per step
        const int64_t dt = flip ? -a.ncols : a.ncols;
        const int64_t tc0 = (flip ? (a.len - 1) * a.ncols : 0) + col;
        float r0[kSruAhead], r1[kSruAhead], r2[kSruAhead], rx[kSruAhead];
#pragma unroll
        for (int s = 0; s < kSruAhead; ++s)
            if (s < a.len) load_u<K, V4>(a, tc0 + s * dt, r0[s], r1[s], r2[s], rx[s]);
        for (int64_t i0 = 0; i0 < a.len; i0 += kSruAhead) {
#pragma unroll
            for (int s = 0; s < kSruAhead; ++s) {
                const int64_t i = i0 + s;
                if (i < a.len) {
                    const float u0 = r0[s], u1 = r1[s], u2 = r2[s], xv = rx[s];
                    const int64_t tc = tc0 + i * dt;
                    if (i + kSruAhead < a.len) load_u<K, V4>(a, tc + kSruAhead * dt, r0[s], r1[s], r2[s], rx[s]);
                    const float g1 = sigmoidf_(u1 + bias1);
                    const float g2 = sigmoidf_(u2 + bias2);
                    cur = (cur - u0) * g1 + u0;
                    a.cout[tc] = cur;
                    const float val = act_(a.activation, cur);
                    a.h[tc] = (val * mask - xv) * g2 + xv;
                }
            }
        }
    }
}

// (kSruThreads, 1): without the minimum, ptxas spills the vector variant at 96 registers
template <int K, bool V4>
__global__ void __launch_bounds__(kSruThreads, 1) sru_bwd_kernel(SruArgs a) {
    const int64_t stride = (int64_t)gridDim.x * kSruThreads;
    for (int64_t col = (int64_t)blockIdx.x * kSruThreads + threadIdx.x; col < a.ncols; col += stride) {
        const int64_t j = col % a.dcols;
        const bool flip = a.bidir && j >= a.d;
        const float bias1 = __ldg(a.bias + j), bias2 = __ldg(a.bias + j + a.dcols);
        const float mask = (a.mask_h == nullptr) ? 1.f : __ldg(a.mask_h + col);
        const float init = (a.init == nullptr) ? 0.f : __ldg(a.init + col);
        float gbias1 = 0.f, gbias2 = 0.f;
        float cur = (a.grad_last == nullptr) ? 0.f : __ldg(a.grad_last + col);
        // step i runs the forward's steps backwards: time t = flip ? i : len-1-i, its predecessor t - dt
        const int64_t dt = flip ? a.ncols : -a.ncols;
        const int64_t tc0 = (flip ? 0 : (a.len - 1) * a.ncols) + col;
        float r0[kSruAhead], r1[kSruAhead], r2[kSruAhead], rx[kSruAhead], rg[kSruAhead], rp[kSruAhead];
#pragma unroll
        for (int s = 0; s < kSruAhead; ++s) {
            if (s < a.len) {
                const int64_t tc = tc0 + s * dt;
                load_u<K, V4>(a, tc, r0[s], r1[s], r2[s], rx[s]);
                rg[s] = __ldg(a.grad_h + tc);
                rp[s] = (s + 1 < a.len) ? __ldg(a.c + tc + dt) : init;
            }
        }
        float c_here = __ldg(a.c + tc0);
        for (int64_t i0 = 0; i0 < a.len; i0 += kSruAhead) {
#pragma unroll
            for (int s = 0; s < kSruAhead; ++s) {
                const int64_t i = i0 + s;
                if (i < a.len) {
                    const float u_val = r0[s], u1 = r1[s], u2 = r2[s], x_val = rx[s], gh_val = rg[s];
                    const float prev_c_val = rp[s];
                    const int64_t tc = tc0 + i * dt;
                    if (i + kSruAhead < a.len) {
                        const int64_t tn = tc + kSruAhead * dt;
                        load_u<K, V4>(a, tn, r0[s], r1[s], r2[s], rx[s]);
                        rg[s] = __ldg(a.grad_h + tn);
                        rp[s] = (i + kSruAhead + 1 < a.len) ? __ldg(a.c + tn + dt) : init;
                    }
                    const float g1 = sigmoidf_(u1 + bias1);
                    const float g2 = sigmoidf_(u2 + bias2);
                    const float c_val = act_(a.activation, c_here);
                    const float gx = gh_val * (1 - g2);
                    const float gg2 = gh_val * (c_val * mask - x_val) * (g2 * (1 - g2));
                    gbias2 += gg2;
                    const float tmp = (a.activation == 1) ? (g2 * (1 - c_val * c_val))
                                                          : (((a.activation == 0) || (c_val > 0)) ? g2 : 0.f);
                    const float gc = gh_val * mask * tmp + cur;
                    const float gu0 = gc * (1 - g1);
                    const float gg1 = gc * (prev_c_val - u_val) * (g1 * (1 - g1));
                    gbias1 += gg1;
                    cur = gc * g1;
                    c_here = prev_c_val;
                    float* gup = a.grad_u + tc * K;
                    if constexpr (V4) {
                        *reinterpret_cast<float4*>(gup) = make_float4(gu0, gg1, gg2, gx);
                    } else {
                        gup[0] = gu0, gup[1] = gg1, gup[2] = gg2;
                        if (K == 3) a.grad_x[tc] = gx; else gup[3] = gx;
                    }
                }
            }
        }
        a.partial[col] = gbias1;
        a.partial[col + a.ncols] = gbias2;
        if (a.grad_init != nullptr) a.grad_init[col] = cur;
    }
}

// grad_bias[half*dcols + j] = sum over b = 0..batch-1, in order, of partial[half][b][j]
__global__ void __launch_bounds__(kSruThreads) sru_bias_kernel(SruArgs a) {
    const int64_t stride = (int64_t)gridDim.x * kSruThreads, batch = a.ncols / a.dcols;
    for (int64_t o = (int64_t)blockIdx.x * kSruThreads + threadIdx.x; o < 2 * a.dcols; o += stride) {
        const int64_t half = o / a.dcols, j = o - half * a.dcols;
        const float* p = a.partial + half * a.ncols + j;
        float s = 0.f;
        for (int64_t b = 0; b < batch; ++b) s = s + p[b * a.dcols];
        a.grad_bias[o] = s;
    }
}

// checks both calls share; on success fills the sizes of a
int check_common(const float* u, const float* x, const float* bias, int64_t len, int64_t batch, int64_t d, int k,
                 int bidirectional, int activation, SruArgs* a) {
    if (len <= 0 || batch <= 0 || d <= 0)
        return fail(QD_ERR_INVALID_ARG, "len, batch and d must be >= 1 (len=%lld batch=%lld d=%lld)", (long long)len,
                    (long long)batch, (long long)d);
    if (k != 3 && k != 4) return fail(QD_ERR_INVALID_ARG, "k must be 3 or 4 (k=%d)", k);
    if (bidirectional != 0 && bidirectional != 1) return fail(QD_ERR_INVALID_ARG, "bidirectional must be 0 or 1");
    if (activation < 0 || activation > 2) return fail(QD_ERR_INVALID_ARG, "activation must be 0, 1 or 2 (%d)", activation);
    const int64_t lim = INT64_MAX / 16, dir = bidirectional ? 2 : 1;
    if (d > lim / dir || batch > lim / (dir * d) || len > lim / (batch * dir * d * k))
        return fail(QD_ERR_INVALID_ARG, "len * batch * dir * d * k overflows 64-bit indexing");
    if (u == nullptr || bias == nullptr) return fail(QD_ERR_INVALID_ARG, "NULL u or bias");
    if (k == 3 && x == nullptr) return fail(QD_ERR_INVALID_ARG, "k = 3 reads the highway input x: x must not be NULL");
    if (k == 4 && x != nullptr) return fail(QD_ERR_INVALID_ARG, "k = 4 reads the highway input from u: x must be NULL");
    a->len = len, a->dcols = dir * d, a->ncols = batch * dir * d, a->d = d;
    a->bidir = bidirectional, a->activation = activation;
    return QD_OK;
}

unsigned grid_of(int64_t n) { return clamp_grid((n + kSruThreads - 1) / kSruThreads); }

template <class F>
void with_k(int k, bool v4, F&& f) {
    if (k == 3) f(std::integral_constant<int, 3>{}, std::false_type{});
    else if (v4) f(std::integral_constant<int, 4>{}, std::true_type{});
    else f(std::integral_constant<int, 4>{}, std::false_type{});
}

}  // namespace

extern "C" size_t qd_sru_workspace_bytes(int64_t batch, int64_t d, int bidirectional) {
    return batch > 0 && d > 0 ? (size_t)2 * (size_t)batch * (size_t)(bidirectional ? 2 : 1) * (size_t)d * sizeof(float) : 0;
}

extern "C" int qd_sru_fwd(const float* u, const float* x, const float* bias, const float* init, const float* mask_h,
                          int64_t len, int64_t batch, int64_t d, int k, int bidirectional, int activation, float* h,
                          float* c, qd_stream_t stream) {
    SruArgs a{};
    int rc = check_common(u, x, bias, len, batch, d, k, bidirectional, activation, &a);
    if (rc) return rc;
    if (h == nullptr || c == nullptr) return fail(QD_ERR_INVALID_ARG, "NULL h or c");
    if (misaligned(u, 4) || misaligned(x, 4) || misaligned(bias, 4) || misaligned(init, 4) || misaligned(mask_h, 4) ||
        misaligned(h, 4) || misaligned(c, 4))
        return fail(QD_ERR_INVALID_ARG, "float arrays must be 4-byte aligned");
    const size_t seq = (size_t)(len * a.ncols) * sizeof(float), col = (size_t)a.ncols * sizeof(float);
    rc = check_disjoint({{u, seq * k}, {x, seq}, {bias, 2 * (size_t)a.dcols * sizeof(float)}, {init, col}, {mask_h, col}},
                        {{h, seq}, {c, seq}});
    if (rc) return rc;
    a.u = u, a.x = x, a.bias = bias, a.init = init, a.mask_h = mask_h, a.h = h, a.cout = c;
    cudaStream_t st = as_stream(stream);
    with_k(k, aligned16(u), [&](auto K, auto V4) {
        sru_fwd_kernel<decltype(K)::value, decltype(V4)::value><<<grid_of(a.ncols), kSruThreads, 0, st>>>(a);
    });
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

extern "C" int qd_sru_bwd(const float* u, const float* x, const float* bias, const float* init, const float* mask_h,
                          const float* c, const float* grad_h, const float* grad_last, int64_t len, int64_t batch,
                          int64_t d, int k, int bidirectional, int activation, float* grad_u, float* grad_x,
                          float* grad_bias, float* grad_init, void* workspace, size_t workspace_bytes,
                          qd_stream_t stream) {
    SruArgs a{};
    int rc = check_common(u, x, bias, len, batch, d, k, bidirectional, activation, &a);
    if (rc) return rc;
    if (c == nullptr || grad_h == nullptr || grad_u == nullptr || grad_bias == nullptr)
        return fail(QD_ERR_INVALID_ARG, "NULL c, grad_h, grad_u or grad_bias");
    if (k == 3 && grad_x == nullptr) return fail(QD_ERR_INVALID_ARG, "k = 3 writes grad_x: it must not be NULL");
    if (k == 4 && grad_x != nullptr) return fail(QD_ERR_INVALID_ARG, "k = 4 has no grad_x: it must be NULL");
    if (misaligned(u, 4) || misaligned(x, 4) || misaligned(bias, 4) || misaligned(init, 4) || misaligned(mask_h, 4) ||
        misaligned(c, 4) || misaligned(grad_h, 4) || misaligned(grad_last, 4) || misaligned(grad_u, 4) ||
        misaligned(grad_x, 4) || misaligned(grad_bias, 4) || misaligned(grad_init, 4))
        return fail(QD_ERR_INVALID_ARG, "float arrays must be 4-byte aligned");
    const size_t need = qd_sru_workspace_bytes(batch, d, bidirectional);
    rc = check_workspace(workspace, workspace_bytes, need, 4, "qd_sru_workspace_bytes(batch, d, bidirectional)");
    if (rc) return rc;
    const size_t seq = (size_t)(len * a.ncols) * sizeof(float), col = (size_t)a.ncols * sizeof(float);
    const size_t nb = 2 * (size_t)a.dcols * sizeof(float);
    rc = check_disjoint({{u, seq * k}, {x, seq}, {bias, nb}, {init, col}, {mask_h, col}, {c, seq}, {grad_h, seq}, {grad_last, col}},
                        {{grad_u, seq * k}, {grad_x, seq}, {grad_bias, nb}, {grad_init, col}, {workspace, need}});
    if (rc) return rc;
    a.u = u, a.x = x, a.bias = bias, a.init = init, a.mask_h = mask_h, a.c = c, a.grad_h = grad_h;
    a.grad_last = grad_last, a.grad_u = grad_u, a.grad_x = grad_x, a.grad_init = grad_init;
    a.partial = static_cast<float*>(workspace), a.grad_bias = grad_bias;
    cudaStream_t st = as_stream(stream);
    with_k(k, aligned16(u) && aligned16(grad_u), [&](auto K, auto V4) {
        sru_bwd_kernel<decltype(K)::value, decltype(V4)::value><<<grid_of(a.ncols), kSruThreads, 0, st>>>(a);
    });
    sru_bias_kernel<<<grid_of(2 * a.dcols), kSruThreads, 0, st>>>(a);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}
