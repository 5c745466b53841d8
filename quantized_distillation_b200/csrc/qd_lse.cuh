// qd_lse.cuh -- the log-sum-exp of a vocabulary row, shared by the NMT loss (qd_nmt_loss.cu) and the beam search step
// (qd_beam.cu), so that a row's log-probabilities are the same bits in training and in translation.
//
// A row is walked by kLseThreads threads: thread t owns the groups of four columns 4k .. 4k+3 with k = t mod
// kLseThreads and absorbs them in increasing k; the threads' (max, sum) pairs are then folded by the tree
// lo[t] <- lse_combine(lo[t], lo[t + h]) for h = kLseThreads/2 .. 1.  The sum is float64 over IEEE expf terms, and
// lse = (double)max + log(sum).  Any kernel that walks and folds a row this way gets the same lse bits.
#pragma once

#include <cmath>
#include <cstdint>

namespace qd {

constexpr int kLseThreads = 256;

__device__ __forceinline__ bool aligned16_dev(const float* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// group k (columns 4k .. 4k+3) of a row; columns at or past V read as -inf and are never loaded
__device__ __forceinline__ void load_group(const float* row, bool vec, int64_t c, int64_t V, float (&v)[4]) {
    if (vec && c + 4 <= V) {
        const float4 q = __ldg(reinterpret_cast<const float4*>(row + c));
        v[0] = q.x, v[1] = q.y, v[2] = q.z, v[3] = q.w;
    } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = c + j < V ? __ldg(row + c + j) : -INFINITY;
    }
}

// the factor that rescales a sum taken against max m to the max m_new >= m; the sum is 0 while m is -inf
__device__ __forceinline__ double lse_rescale(float m, float m_new) {
    return m == -INFINITY ? 0.0 : exp((double)m - (double)m_new);
}

struct LseAcc {                      // online (max, sum of exp(x - max)) over a thread's columns
    float m = -INFINITY;
    double s = 0.0;
};

__device__ __forceinline__ void lse_absorb(LseAcc& o, const float (&x)[4]) {
    const float gm = fmaxf(fmaxf(x[0], x[1]), fmaxf(x[2], x[3]));
    if (gm > o.m) {
        o.s *= lse_rescale(o.m, gm);
        o.m = gm;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j)      // -inf (and the columns past V) add exactly 0; NaN propagates into the sum
        if (x[j] != -INFINITY) o.s += (double)expf(__fsub_rn(x[j], o.m));
}

__device__ __forceinline__ void lse_combine(LseAcc& o, const LseAcc& p) {
    const float m = fmaxf(o.m, p.m);
    o.s = o.s * lse_rescale(o.m, m) + p.s * lse_rescale(p.m, m);
    o.m = m;
}

// -inf for a row that is all -inf, NaN for a row holding NaN
__device__ __forceinline__ double lse_value(const LseAcc& o) { return (double)o.m + log(o.s); }

}  // namespace qd
