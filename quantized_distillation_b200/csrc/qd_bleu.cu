// qd_bleu.cu -- multi-bleu.perl's corpus statistics (perl_scripts/multi-bleu.perl:60-120) on int32 word ids.
//
// bleu_stats_kernel: one warp per sentence.  Lanes stride over the hypothesis positions i; for each i one pass over
// the hypothesis gives the longest match (up to 4 words) of i's suffix at an earlier position (so whether i starts the
// first occurrence of its n-grams) and at i or later (count_hyp), and one pass per reference gives count_ref.  A
// position that starts the first occurrence of its n-gram adds min(count_hyp, max_r count_ref), which is the clipped
// count of every distinct n-gram once.  Words are compared directly: no hashing, so no collision can change a count.
// A sentence whose words (hypothesis and references) fit in its warp's kStageWords of shared memory is staged there;
// a longer one is read from global memory by the same code.
//
// bleu_fold_kernel: one CTA sums the per-sentence rows column by column.  Integer sums: exact, and the order is fixed.
//
// No atomics, no host synchronisation, no allocation: the same integers on any stream, in any batch, eager or replayed
// from a CUDA graph.
#include "qd_launch.h"

using namespace qd;

namespace {

constexpr int kStatsWarps = 4;
constexpr int kStageWords = 2048;            // per warp: 8 KB, 32 KB per CTA
constexpr int kFoldThreads = 256;
constexpr int64_t kNoReference = 9999;       // multi-bleu's ($closest_diff, $closest_length) start

struct StatsArgs {
    const int32_t* hyp_words;
    const int64_t* hyp_offsets;
    const int32_t* ref_words;
    const int64_t* ref_offsets;
    const int64_t* ref_first;
    const int64_t* ref_count;
    int64_t* stats;
    int64_t n_hyp_words, n_sent, n_ref_words, n_refs;
};

__device__ __forceinline__ int64_t clamp64(int64_t v, int64_t lo, int64_t hi) { return v < lo ? lo : v > hi ? hi : v; }

// words a[0 .. lim) equal to b[0 .. lim), counted from the start (lim <= 4)
__device__ __forceinline__ int match(const int32_t* a, const int32_t* b, int lim) {
    int m = 0;
    while (m < lim && a[m] == b[m]) ++m;
    return m;
}

__device__ __forceinline__ int64_t warp_sum(int64_t v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
    return v;
}

__global__ void __launch_bounds__(kStatsWarps * 32) bleu_stats_kernel(StatsArgs a) {
    __shared__ int32_t s_words[kStatsWarps][kStageWords];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int64_t s = (int64_t)blockIdx.x * kStatsWarps + warp; s < a.n_sent; s += (int64_t)gridDim.x * kStatsWarps) {
        const int64_t h0 = clamp64(a.hyp_offsets[s], 0, a.n_hyp_words);
        const int64_t L = clamp64(a.hyp_offsets[s + 1], h0, a.n_hyp_words) - h0;
        int64_t rf = a.ref_first[s], rc = a.ref_count[s];
        if (rf < 0 || rc < 0 || rf > a.n_refs || rc > a.n_refs - rf) rc = 0;       // an out-of-range span: no reference
        // closest reference length (multi-bleu.perl:68-79) and the words to stage; every lane computes the same
        int64_t closest_diff = kNoReference, closest_len = kNoReference, ref_words = 0;
        for (int64_t r = rf; r < rf + rc; ++r) {
            const int64_t r0 = clamp64(a.ref_offsets[r], 0, a.n_ref_words);
            const int64_t len = clamp64(a.ref_offsets[r + 1], r0, a.n_ref_words) - r0;
            const int64_t diff = len > L ? len - L : L - len;
            if (diff < closest_diff) closest_diff = diff, closest_len = len;
            else if (diff == closest_diff && len < closest_len) closest_len = len;
            ref_words += len;
        }
        const bool staged = L + ref_words <= kStageWords;
        const int32_t* hyp = a.hyp_words + h0;
        if (staged) {
            int32_t* st = s_words[warp];
            for (int64_t i = lane; i < L; i += 32) st[i] = hyp[i];
            int64_t at = L;
            for (int64_t r = rf; r < rf + rc; ++r) {
                const int64_t r0 = clamp64(a.ref_offsets[r], 0, a.n_ref_words);
                const int64_t len = clamp64(a.ref_offsets[r + 1], r0, a.n_ref_words) - r0;
                for (int64_t i = lane; i < len; i += 32) st[at + i] = a.ref_words[r0 + i];
                at += len;
            }
            __syncwarp();
            hyp = st;
        }
        int64_t correct[4] = {0, 0, 0, 0};
        for (int64_t i = lane; i < L; i += 32) {
            const int lim = L - i < 4 ? (int)(L - i) : 4;         // n-grams of length 1 .. lim start at i
            int seen = 0;                                         // longest match at an earlier position
            for (int64_t j = 0; j < i && seen < lim; ++j) {
                const int m = match(hyp + j, hyp + i, lim);
                seen = m > seen ? m : seen;
            }
            if (seen == lim) continue;                            // every n-gram at i occurred before
            int cnt_h[4] = {0, 0, 0, 0}, cnt_r[4] = {0, 0, 0, 0};
            for (int64_t j = i; j < L; ++j) {
                const int m = match(hyp + j, hyp + i, L - j < lim ? (int)(L - j) : lim);
#pragma unroll
                for (int n = 0; n < 4; ++n) cnt_h[n] += m > n;
            }
            const int32_t* ref = hyp + L;                         // staged references follow the hypothesis
            for (int64_t r = rf; r < rf + rc; ++r) {
                const int64_t r0 = clamp64(a.ref_offsets[r], 0, a.n_ref_words);
                const int64_t len = clamp64(a.ref_offsets[r + 1], r0, a.n_ref_words) - r0;
                if (!staged) ref = a.ref_words + r0;
                int c[4] = {0, 0, 0, 0};
                for (int64_t p = 0; p < len; ++p) {
                    const int m = match(ref + p, hyp + i, len - p < lim ? (int)(len - p) : lim);
#pragma unroll
                    for (int n = 0; n < 4; ++n) c[n] += m > n;
                }
#pragma unroll
                for (int n = 0; n < 4; ++n) cnt_r[n] = c[n] > cnt_r[n] ? c[n] : cnt_r[n];
                if (staged) ref += len;
            }
#pragma unroll
            for (int n = 0; n < 4; ++n)
                if (n >= seen && n < lim) correct[n] += cnt_h[n] < cnt_r[n] ? cnt_h[n] : cnt_r[n];
        }
        int64_t v = lane == 0 ? L : lane == 1 ? closest_len : L - (lane - 6) > 0 ? L - (lane - 6) : 0;  // total[n] = L-n+1
#pragma unroll
        for (int n = 0; n < 4; ++n) {
            const int64_t c = warp_sum(correct[n]);
            if (lane == n + 2) v = c;
        }
        if (lane < QD_BLEU_STATS) a.stats[s * QD_BLEU_STATS + lane] = v;
        __syncwarp();                                             // the staged words are reused by the next sentence
    }
}

__global__ void __launch_bounds__(kFoldThreads) bleu_fold_kernel(const int64_t* stats, int64_t n, int64_t* totals) {
    __shared__ int64_t s_part[kFoldThreads / 32][QD_BLEU_STATS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int64_t acc[QD_BLEU_STATS];
#pragma unroll
    for (int c = 0; c < QD_BLEU_STATS; ++c) acc[c] = 0;
    for (int64_t s = threadIdx.x; s < n; s += kFoldThreads)
#pragma unroll
        for (int c = 0; c < QD_BLEU_STATS; ++c) acc[c] += stats[s * QD_BLEU_STATS + c];
#pragma unroll
    for (int c = 0; c < QD_BLEU_STATS; ++c) {
        const int64_t v = warp_sum(acc[c]);
        if (lane == 0) s_part[warp][c] = v;
    }
    __syncthreads();
    if ((int)threadIdx.x < QD_BLEU_STATS) {
        int64_t v = 0;
        for (int w = 0; w < kFoldThreads / 32; ++w) v += s_part[w][threadIdx.x];
        totals[threadIdx.x] = v;
    }
}

}  // namespace

extern "C" int qd_bleu_stats(const int32_t* hyp_words, int64_t n_hyp_words, const int64_t* hyp_offsets, int64_t n_sent,
                             const int32_t* ref_words, int64_t n_ref_words, const int64_t* ref_offsets, int64_t n_refs,
                             const int64_t* ref_first, const int64_t* ref_count, int64_t* stats, qd_stream_t stream) {
    if (n_sent < 0 || n_hyp_words < 0 || n_ref_words < 0 || n_refs < 0)
        return fail(QD_ERR_INVALID_ARG, "counts must be >= 0 (n_sent=%lld n_hyp_words=%lld n_ref_words=%lld n_refs=%lld)",
                    (long long)n_sent, (long long)n_hyp_words, (long long)n_ref_words, (long long)n_refs);
    const int64_t lim = INT64_MAX / 16;
    if (n_sent > lim || n_hyp_words > lim || n_ref_words > lim || n_refs > lim)
        return fail(QD_ERR_INVALID_ARG, "counts past 64-bit indexing");
    if (n_sent == 0) return QD_OK;
    if (hyp_offsets == nullptr || ref_offsets == nullptr || ref_first == nullptr || ref_count == nullptr || stats == nullptr ||
        (n_hyp_words > 0 && hyp_words == nullptr) || (n_ref_words > 0 && ref_words == nullptr))
        return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if (misaligned(hyp_words, 4) || misaligned(ref_words, 4) || misaligned(hyp_offsets, 8) || misaligned(ref_offsets, 8) ||
        misaligned(ref_first, 8) || misaligned(ref_count, 8) || misaligned(stats, 8))
        return fail(QD_ERR_INVALID_ARG, "misaligned argument (word arrays 4 bytes, offsets, spans and stats 8 bytes)");
    const int rc = check_disjoint({{hyp_words, (size_t)n_hyp_words * 4}, {hyp_offsets, (size_t)(n_sent + 1) * 8},
                                   {ref_words, (size_t)n_ref_words * 4}, {ref_offsets, (size_t)(n_refs + 1) * 8},
                                   {ref_first, (size_t)n_sent * 8}, {ref_count, (size_t)n_sent * 8}},
                                  {{stats, (size_t)n_sent * QD_BLEU_STATS * 8}});
    if (rc) return rc;
    StatsArgs sa{};
    sa.hyp_words = hyp_words, sa.hyp_offsets = hyp_offsets, sa.ref_words = ref_words, sa.ref_offsets = ref_offsets;
    sa.ref_first = ref_first, sa.ref_count = ref_count, sa.stats = stats;
    sa.n_hyp_words = n_hyp_words, sa.n_sent = n_sent, sa.n_ref_words = n_ref_words, sa.n_refs = n_refs;
    const int64_t blocks = (n_sent + kStatsWarps - 1) / kStatsWarps;
    bleu_stats_kernel<<<clamp_grid(blocks), kStatsWarps * 32, 0, as_stream(stream)>>>(sa);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

extern "C" int qd_bleu_fold(const int64_t* stats, int64_t n_sent, int64_t* totals, qd_stream_t stream) {
    if (n_sent < 0) return fail(QD_ERR_INVALID_ARG, "n_sent must be >= 0 (n_sent=%lld)", (long long)n_sent);
    if (n_sent > INT64_MAX / 16 / QD_BLEU_STATS) return fail(QD_ERR_INVALID_ARG, "n_sent past 64-bit indexing");
    if (totals == nullptr || (n_sent > 0 && stats == nullptr)) return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if (misaligned(stats, 8) || misaligned(totals, 8)) return fail(QD_ERR_INVALID_ARG, "misaligned argument (8 bytes)");
    const int rc = check_disjoint({{stats, (size_t)n_sent * QD_BLEU_STATS * 8}}, {{totals, QD_BLEU_STATS * 8}});
    if (rc) return rc;
    bleu_fold_kernel<<<1, kFoldThreads, 0, as_stream(stream)>>>(stats, n_sent, totals);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}
