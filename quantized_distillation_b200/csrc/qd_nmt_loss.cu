// qd_nmt_loss.cu -- the loss of the NMT loop over the target vocabulary (onmt/Loss.py:97-120, NMTLossCompute), fused:
// NLL of the generator's log-softmax at the target, plus w times the KL divergence to the teacher's softmax, the sum
// over non-padding rows, the word and correct-word counts, and the gradient to the student logits.
//
// Forward (qd_nmt_loss_fwd): one CTA per row reads the student row and, with a teacher, the teacher row once.  Each
// thread keeps online (max, sum) pairs for both rows and the cross term A = sum_c e^{z_t - m_t} (z_t - z_s), the sums in
// float64 over IEEE expf terms, and the first-occurrence argmax of the student row; a fixed-shape tree folds the
// threads.  Thread t owns the groups of four columns 4k .. 4k+3 with k = t mod kNlThreads, whatever the row's
// alignment (a 16-byte aligned row loads each group as one float4, any other row loads it element by element), so a
// row's results depend only on V: the same bits alone or at any position of any batch.  The row's loss partial (float64)
// and its kind go to the workspace; one CTA then folds them in a fixed order into the float32 loss and the int64 counts.
//
// Backward (qd_nmt_loss_bwd): one CTA per row reads both rows again, with the row's lse from the forward, and writes
// g * (exp(z_s - lse_s) - w exp(z_t - lse_t) - (1 - w)[c = y]) once.  g is read on the device.
#include <cmath>

#include "qd_launch.h"
#include "qd_lse.cuh"

using namespace qd;

namespace {

constexpr int kNlThreads = kLseThreads;   // per row, forward and backward; the lse walk of qd_lse.cuh
constexpr int kNlReduceThreads = 512;

enum RowKind : int { kRowPad = 0, kRowWord = 1, kRowCorrect = 2, kRowInvalid = 3 };

struct RowPartial {                  // one per row in the workspace
    double loss;
    int kind;
    int pad_;
};

struct NlArgs {
    const float* zs;                 // [R, V]
    const float* zt;                 // [R, V] or NULL
    const int64_t* target;           // [R]
    float* row_lse;                  // [R][2]: lse_s, lse_t
    RowPartial* part;                // [R]
    int64_t R, V, padding_idx;
    double w;
};

// a * f for a rescale factor f in [0, 1]; an infinite cross term stays infinite (inf * 0 would be NaN)
__device__ __forceinline__ double scale_a(double a, double f) { return isinf(a) ? a : a * f; }

struct Online {                      // one thread's state over its columns
    LseAcc s;                        // the student's (max, sum)
    float mt = -INFINITY, best = -INFINITY;
    double st = 0.0, a = 0.0;
    int64_t arg = -1;
};

template <bool TEACHER>
__device__ __forceinline__ void absorb(Online& o, const float (&s)[4], const float (&t)[4], int64_t c) {
    lse_absorb(o.s, s);
    if (TEACHER) {
        float gt = fmaxf(fmaxf(t[0], t[1]), fmaxf(t[2], t[3]));
        if (gt > o.mt) {
            const double f = lse_rescale(o.mt, gt);
            o.st *= f;
            o.a = scale_a(o.a, f);
            o.mt = gt;
        }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        if (o.arg < 0 || s[j] > o.best) {
            o.best = s[j];
            o.arg = c + j;
        }
        // a teacher -inf adds 0 (never 0 * inf); a finite teacher logit against a student -inf is a positive teacher
        // probability against a zero one: the KL is +inf, even where the float32 exponential underflows
        if (TEACHER && t[j] != -INFINITY) {
            const float e = expf(__fsub_rn(t[j], o.mt));
            o.st += (double)e;
            if (s[j] == -INFINITY) o.a = INFINITY;
            else o.a += (double)e * ((double)t[j] - (double)s[j]);
        }
    }
}

// o <- o combined with p; an argmax tie keeps the lower column
template <bool TEACHER>
__device__ __forceinline__ void combine(Online& o, const Online& p) {
    lse_combine(o.s, p.s);
    if (TEACHER) {
        const float mt = fmaxf(o.mt, p.mt);
        const double fo = lse_rescale(o.mt, mt), fp = lse_rescale(p.mt, mt);
        o.st = o.st * fo + p.st * fp;
        o.a = scale_a(o.a, fo) + scale_a(p.a, fp);
        o.mt = mt;
    }
    if (p.arg >= 0 && (o.arg < 0 || p.best > o.best || (p.best == o.best && p.arg < o.arg))) {
        o.best = p.best;
        o.arg = p.arg;
    }
}

template <bool TEACHER>
__global__ void __launch_bounds__(kNlThreads) nmt_loss_fwd_kernel(NlArgs a) {
    __shared__ Online s_o[kNlThreads];
    for (int64_t r = blockIdx.x; r < a.R; r += gridDim.x) {
        const float* zs = a.zs + r * a.V;
        const float* zt = TEACHER ? a.zt + r * a.V : nullptr;
        const bool vs = aligned16_dev(zs), vt = TEACHER && aligned16_dev(zt);
        Online o;
        const int64_t groups = (a.V + 3) / 4;
        int64_t k = threadIdx.x;
        // two groups in flight per thread
        for (; k + kNlThreads < groups; k += 2 * kNlThreads) {
            float s0[4], s1[4], t0[4], t1[4];
            load_group(zs, vs, 4 * k, a.V, s0);
            load_group(zs, vs, 4 * (k + kNlThreads), a.V, s1);
            if (TEACHER) {
                load_group(zt, vt, 4 * k, a.V, t0);
                load_group(zt, vt, 4 * (k + kNlThreads), a.V, t1);
            }
            absorb<TEACHER>(o, s0, t0, 4 * k);
            absorb<TEACHER>(o, s1, t1, 4 * (k + kNlThreads));
        }
        if (k < groups) {
            float s0[4], t0[4];
            load_group(zs, vs, 4 * k, a.V, s0);
            if (TEACHER) load_group(zt, vt, 4 * k, a.V, t0);
            absorb<TEACHER>(o, s0, t0, 4 * k);
        }
        s_o[threadIdx.x] = o;
        __syncthreads();
        for (int h = kNlThreads / 2; h > 0; h >>= 1) {
            if ((int)threadIdx.x < h) {
                Online lo = s_o[threadIdx.x];
                combine<TEACHER>(lo, s_o[threadIdx.x + h]);
                s_o[threadIdx.x] = lo;
            }
            __syncthreads();
        }
        if (threadIdx.x == 0) {
            const Online f = s_o[0];
            const double lse_s = lse_value(f.s);
            const double lse_t = TEACHER ? (double)f.mt + log(f.st) : 0.0;
            a.row_lse[2 * r] = (float)lse_s;
            a.row_lse[2 * r + 1] = (float)lse_t;
            const int64_t y = __ldg(a.target + r);
            RowPartial p{0.0, kRowPad, 0};
            if (a.padding_idx >= 0 && y == a.padding_idx) {
            } else if (y < 0 || y >= a.V) {
                p.loss = __longlong_as_double(0x7ff8000000000000LL);
                p.kind = kRowInvalid;
            } else {
                const double nll = lse_s - (double)__ldg(zs + y);
                p.loss = nll;
                if (TEACHER) p.loss = (1.0 - a.w) * nll + a.w * (f.a / f.st - lse_t + lse_s);
                p.kind = f.arg == y ? kRowCorrect : kRowWord;
            }
            a.part[r] = p;
        }
        __syncthreads();                 // s_o is reused by the next row
    }
}

// one CTA: loss = (float)(sum of the row partials), counts = {n_words, n_correct, n_invalid}, rows folded in a fixed order
__global__ void __launch_bounds__(kNlReduceThreads) nmt_loss_reduce_kernel(const RowPartial* part, int64_t R, float* loss,
                                                                         long long* counts) {
    __shared__ double s_l[kNlReduceThreads];
    __shared__ long long s_c[3][kNlReduceThreads];
    double l = 0.0;
    long long c[3] = {0, 0, 0};
    for (int64_t r = threadIdx.x; r < R; r += kNlReduceThreads) {
        const RowPartial p = part[r];
        l += p.loss;
        c[0] += p.kind == kRowWord || p.kind == kRowCorrect;
        c[1] += p.kind == kRowCorrect;
        c[2] += p.kind == kRowInvalid;
    }
    s_l[threadIdx.x] = l;
    for (int j = 0; j < 3; ++j) s_c[j][threadIdx.x] = c[j];
    __syncthreads();
    for (int h = kNlReduceThreads / 2; h > 0; h >>= 1) {
        if ((int)threadIdx.x < h) {
            s_l[threadIdx.x] += s_l[threadIdx.x + h];
            for (int j = 0; j < 3; ++j) s_c[j][threadIdx.x] += s_c[j][threadIdx.x + h];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        *loss = (float)s_l[0];
        for (int j = 0; j < 3; ++j) counts[j] = s_c[j][0];
    }
}

struct NlBwdArgs {
    const float* zs;
    const float* zt;
    const int64_t* target;
    const float* row_lse;
    const float* grad_loss;
    float* grad;
    int64_t R, V, padding_idx;
    float w;
};

template <bool TEACHER>
__global__ void __launch_bounds__(kNlThreads) nmt_loss_bwd_kernel(NlBwdArgs a) {
    const float g = __ldg(a.grad_loss);
    const float one_minus_w = __fsub_rn(1.f, a.w);
    for (int64_t r = blockIdx.x; r < a.R; r += gridDim.x) {
        const float* zs = a.zs + r * a.V;
        const float* zt = TEACHER ? a.zt + r * a.V : nullptr;
        float* out = a.grad + r * a.V;
        const int64_t y = __ldg(a.target + r);
        const bool pad = a.padding_idx >= 0 && y == a.padding_idx, invalid = !pad && (y < 0 || y >= a.V);
        const float lse_s = __ldg(a.row_lse + 2 * r), lse_t = __ldg(a.row_lse + 2 * r + 1);
        const bool vs = aligned16_dev(zs), vt = TEACHER && aligned16_dev(zt), vo = aligned16_dev(out);
        for (int64_t k = threadIdx.x; 4 * k < a.V; k += kNlThreads) {
            const int64_t c = 4 * k;
            float o[4];
            if (pad || invalid) {
                const float fill = pad ? 0.f : __int_as_float(0x7fc00000);
                o[0] = o[1] = o[2] = o[3] = fill;
            } else {
                float s[4], t[4];
                load_group(zs, vs, c, a.V, s);
                if (TEACHER) load_group(zt, vt, c, a.V, t);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    float d = expf(__fsub_rn(s[j], lse_s));
                    if (TEACHER) d = __fsub_rn(d, __fmul_rn(a.w, expf(__fsub_rn(t[j], lse_t))));
                    if (c + j == y) d = __fsub_rn(d, one_minus_w);
                    o[j] = __fmul_rn(g, d);
                }
            }
            if (vo && c + 4 <= a.V) {
                *reinterpret_cast<float4*>(out + c) = make_float4(o[0], o[1], o[2], o[3]);
            } else {
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (c + j < a.V) out[c + j] = o[j];
            }
        }
    }
}

bool overlap(const void* a, size_t na, const void* b, size_t nb) {
    const uintptr_t pa = reinterpret_cast<uintptr_t>(a), pb = reinterpret_cast<uintptr_t>(b);
    return a != nullptr && b != nullptr && na > 0 && nb > 0 && pa < pb + nb && pb < pa + na;
}

// the checks both calls share
int check_common(const float* logits, const int64_t* target, int64_t R, int64_t V, int64_t padding_idx, float w) {
    if (R < 0 || V < 1) return fail(QD_ERR_INVALID_ARG, "rows must be >= 0 and V >= 1 (rows=%lld V=%lld)", (long long)R, (long long)V);
    if (R > 0 && (logits == nullptr || target == nullptr)) return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if (R > INT64_MAX / 4 / V) return fail(QD_ERR_INVALID_ARG, "rows * V overflows 64-bit indexing");
    if (padding_idx < -1 || padding_idx >= V) return fail(QD_ERR_INVALID_ARG, "padding_idx must be -1 (none) or in [0, V)");
    if (!(w >= 0.f && w <= 1.f)) return fail(QD_ERR_INVALID_ARG, "weight_teacher_loss must be in [0, 1]");
    if ((reinterpret_cast<uintptr_t>(logits) & 3) || (reinterpret_cast<uintptr_t>(target) & 7))
        return fail(QD_ERR_INVALID_ARG, "logits must be 4-byte and target 8-byte aligned");
    return QD_OK;
}

constexpr int kNlMaxGrid = 1 << 20;   // rows beyond it loop inside the CTAs

}  // namespace

extern "C" size_t qd_nmt_loss_workspace_bytes(int64_t rows) { return rows > 0 ? (size_t)rows * sizeof(RowPartial) : 0; }

extern "C" int qd_nmt_loss_fwd(const float* logits, const float* teacher_logits, const int64_t* target, int64_t rows, int64_t V,
                               int64_t padding_idx, float w, float* row_lse, float* loss, int64_t* counts, void* workspace,
                               size_t workspace_bytes, qd_stream_t stream) {
    int rc = check_common(logits, target, rows, V, padding_idx, w);
    if (rc) return rc;
    if (loss == nullptr || counts == nullptr || (rows > 0 && row_lse == nullptr)) return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if ((reinterpret_cast<uintptr_t>(teacher_logits) & 3) || (reinterpret_cast<uintptr_t>(row_lse) & 3) ||
        (reinterpret_cast<uintptr_t>(loss) & 3) || (reinterpret_cast<uintptr_t>(counts) & 7))
        return fail(QD_ERR_INVALID_ARG, "misaligned output (teacher_logits, row_lse, loss 4 bytes, counts 8 bytes)");
    const size_t need = qd_nmt_loss_workspace_bytes(rows);
    if (need > 0 && (workspace == nullptr || workspace_bytes < need || (reinterpret_cast<uintptr_t>(workspace) & 15)))
        return fail(QD_ERR_WORKSPACE, "workspace must be 16-byte aligned and hold qd_nmt_loss_workspace_bytes(%lld) = %zu bytes",
                    (long long)rows, need);
    const size_t in_bytes = (size_t)(rows * V) * sizeof(float);
    const void* outs[4] = {row_lse, loss, counts, workspace};
    const size_t out_bytes[4] = {(size_t)rows * 2 * sizeof(float), sizeof(float), 3 * sizeof(int64_t), need};
    for (int i = 0; i < 4; ++i) {
        if (overlap(outs[i], out_bytes[i], logits, in_bytes) || overlap(outs[i], out_bytes[i], teacher_logits, in_bytes) ||
            overlap(outs[i], out_bytes[i], target, (size_t)rows * sizeof(int64_t)))
            return fail(QD_ERR_INVALID_ARG, "outputs must not overlap the inputs");
        for (int j = 0; j < i; ++j)
            if (overlap(outs[i], out_bytes[i], outs[j], out_bytes[j])) return fail(QD_ERR_INVALID_ARG, "outputs must not overlap each other");
    }
    NlArgs a{};
    a.zs = logits, a.zt = teacher_logits, a.target = target, a.row_lse = row_lse;
    a.part = static_cast<RowPartial*>(workspace);
    a.R = rows, a.V = V, a.padding_idx = padding_idx;
    a.w = teacher_logits != nullptr ? (double)w : 0.0;
    cudaStream_t st = as_stream(stream);
    if (rows > 0) {
        const unsigned grid = (unsigned)(rows < kNlMaxGrid ? rows : kNlMaxGrid);
        if (teacher_logits != nullptr) nmt_loss_fwd_kernel<true><<<grid, kNlThreads, 0, st>>>(a);
        else nmt_loss_fwd_kernel<false><<<grid, kNlThreads, 0, st>>>(a);
    }
    nmt_loss_reduce_kernel<<<1, kNlReduceThreads, 0, st>>>(a.part, rows, loss, reinterpret_cast<long long*>(counts));
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

extern "C" int qd_nmt_loss_bwd(const float* logits, const float* teacher_logits, const int64_t* target, const float* row_lse,
                               const float* grad_loss, int64_t rows, int64_t V, int64_t padding_idx, float w, float* grad_logits,
                               qd_stream_t stream) {
    int rc = check_common(logits, target, rows, V, padding_idx, w);
    if (rc) return rc;
    if (rows == 0) return QD_OK;
    if (row_lse == nullptr || grad_loss == nullptr || grad_logits == nullptr) return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if ((reinterpret_cast<uintptr_t>(teacher_logits) & 3) || (reinterpret_cast<uintptr_t>(row_lse) & 3) ||
        (reinterpret_cast<uintptr_t>(grad_loss) & 3) || (reinterpret_cast<uintptr_t>(grad_logits) & 3))
        return fail(QD_ERR_INVALID_ARG, "float arguments must be 4-byte aligned");
    const size_t bytes = (size_t)(rows * V) * sizeof(float);
    if (overlap(grad_logits, bytes, logits, bytes) || overlap(grad_logits, bytes, teacher_logits, bytes) ||
        overlap(grad_logits, bytes, target, (size_t)rows * sizeof(int64_t)) ||
        overlap(grad_logits, bytes, row_lse, (size_t)rows * 2 * sizeof(float)) || overlap(grad_logits, bytes, grad_loss, sizeof(float)))
        return fail(QD_ERR_INVALID_ARG, "grad_logits must not overlap the inputs");
    NlBwdArgs a{};
    a.zs = logits, a.zt = teacher_logits, a.target = target, a.row_lse = row_lse, a.grad_loss = grad_loss, a.grad = grad_logits;
    a.R = rows, a.V = V, a.padding_idx = padding_idx;
    a.w = teacher_logits != nullptr ? w : 0.f;
    const unsigned grid = (unsigned)(rows < kNlMaxGrid ? rows : kNlMaxGrid);
    cudaStream_t st = as_stream(stream);
    if (teacher_logits != nullptr) nmt_loss_bwd_kernel<true><<<grid, kNlThreads, 0, st>>>(a);
    else nmt_loss_bwd_kernel<false><<<grid, kNlThreads, 0, st>>>(a);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}
