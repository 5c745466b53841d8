// qd_beam.cu -- one step of B onmt beam searches at once (onmt/Beam.py:55-106, Beam.advance), on the [K*B, V] scores
// of the decoder batch in onmt's beam-major row order r = k*B + b.
//
// The K selected entries of a sentence are the top K of its K*V keys, compared on the exact float32 key (NaN above
// every number, -0 equal to +0) with ties to the lower flat index k*V + j.  Rounding in x - lse and in + scores[k] is
// monotone but not strict, so two different logits can give equal keys; the candidates of a row are therefore chosen
// on the key itself, never on the logit.
//
// beam_row_kernel: one CTA per row.  With normalize, the row's lse first, by the walk and fold of qd_lse.cuh (the bits
// of qd_nmt_loss_fwd's lse_s); then a second pass over the row (mostly from L2) where each thread keeps the best KC
// (key, column) pairs of its columns in registers, sorted, behind a threshold.  Each warp pops its K best by K rounds
// of a warp maximum, warp 0 merges the warps' lists the same way, and the row's K best go to the workspace with their
// keys recomputed from the logit (the comparisons run on an order-preserving integer image of the key).  A row whose
// last token is EOS is never read: its K candidates are (-1e20, columns 0 .. K-1).
//
// beam_merge_kernel: one warp per sentence merges the K sorted lists of its K rows (lane k holds row k's head) by K
// rounds of a warp maximum, writes the new scores, tokens and back pointers and updates the finished counters.
//
// No atomics, no host synchronisation, no allocation: a step gives the same bits on any stream, in any batch, eager
// or replayed from a CUDA graph.
#include <cmath>

#include "qd_launch.h"
#include "qd_lse.cuh"

using namespace qd;

namespace {

constexpr int kRowThreads = kLseThreads;     // a row's lse must be walked exactly as the NMT loss walks it
constexpr int kRowWarps = kRowThreads / 32;
constexpr int kMergeWarps = 4;
constexpr int kBeamMaxGrid = 1 << 20;        // rows or sentences beyond it loop inside the CTAs
constexpr float kEosRowKey = -1e20f;         // Beam.py:75, beamLk[i] = -1e20 on a float32 tensor

struct Cand {                                // workspace: [K*B rows][K], each row's K best, best first
    float key;
    uint32_t col;
};

// an order-preserving image of a key: larger is better, NaN above +inf, -0 equal to +0
__device__ __forceinline__ uint32_t key_order(float f) {
    if (f != f) return 0xFFFFFFFFu;
    const uint32_t u = __float_as_uint(f == 0.f ? 0.f : f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// (key, column) as one integer, larger is better: a key tie goes to the lower column.  0 is below every candidate.
__device__ __forceinline__ unsigned long long row_pack(float key, uint32_t col) {
    return ((unsigned long long)key_order(key) << 32) | (0xFFFFFFFFu - col);
}

__device__ __forceinline__ unsigned long long warp_max(unsigned long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long w = __shfl_xor_sync(0xFFFFFFFFu, v, o);
        v = w > v ? w : v;
    }
    return v;
}

struct RowArgs {
    const float* out;                        // [K*B, V]
    const float* scores;                     // [K*B]
    const int64_t* last_tokens;              // [K*B]
    Cand* cand;                              // [K*B][K]
    int64_t B, V, eos;
    int K, first;
};

// the key of column c of a row, exactly as Beam.advance forms it
template <bool NORMALIZE>
__device__ __forceinline__ float beam_key(float x, float lse, float score, bool first) {
    const float lp = NORMALIZE ? __fsub_rn(x, lse) : x;
    return first ? lp : __fadd_rn(lp, score);
}

template <int KC, bool NORMALIZE>
__global__ void __launch_bounds__(kRowThreads) beam_row_kernel(RowArgs a) {
    __shared__ LseAcc s_l[kRowThreads];
    __shared__ unsigned long long s_w[kRowWarps][KC];
    __shared__ float s_lse;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int K = a.K;
    const bool first = a.first != 0;
    const int64_t rows = first ? a.B : (int64_t)K * a.B;    // the first step reads beam 0 only (Beam.py:77)
    for (int64_t r = blockIdx.x; r < rows; r += gridDim.x) {
        Cand* cand = a.cand + r * K;
        if (!first && __ldg(a.last_tokens + r) == a.eos) {   // EOS has no children (Beam.py:72-75)
            if ((int)threadIdx.x < K) cand[threadIdx.x] = Cand{kEosRowKey, (uint32_t)threadIdx.x};
            continue;
        }
        const float* row = a.out + r * a.V;
        const bool vec = aligned16_dev(row);
        const int64_t groups = (a.V + 3) / 4;
        float lse = 0.f;
        if (NORMALIZE) {
            LseAcc o;
            for (int64_t k = threadIdx.x; k < groups; k += kRowThreads) {
                float v[4];
                load_group(row, vec, 4 * k, a.V, v);
                lse_absorb(o, v);
            }
            s_l[threadIdx.x] = o;
            __syncthreads();
            for (int h = kRowThreads / 2; h > 0; h >>= 1) {
                if ((int)threadIdx.x < h) {
                    LseAcc lo = s_l[threadIdx.x];
                    lse_combine(lo, s_l[threadIdx.x + h]);
                    s_l[threadIdx.x] = lo;
                }
                __syncthreads();
            }
            if (threadIdx.x == 0) s_lse = (float)lse_value(s_l[0]);
            __syncthreads();
            lse = s_lse;
        }
        const float score = first ? 0.f : __ldg(a.scores + r);

        // this thread's best KC >= K, best first; its columns come in increasing order, so an equal key never
        // displaces.  A newcomer must beat best[KC-1] (a static index: best[] stays in registers).
        unsigned long long best[KC];
#pragma unroll
        for (int i = 0; i < KC; ++i) best[i] = 0;
        for (int64_t k = threadIdx.x; k < groups; k += kRowThreads) {
            float v[4];
            load_group(row, vec, 4 * k, a.V, v);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int64_t c = 4 * k + j;
                if (c >= a.V) break;
                const unsigned long long p = row_pack(beam_key<NORMALIZE>(v[j], lse, score, first), (uint32_t)c);
                if (p > best[KC - 1]) {
#pragma unroll
                    for (int i = KC - 1; i > 0; --i) {
                        if (p > best[i - 1]) best[i] = best[i - 1];
                        else if (p > best[i]) best[i] = p;
                    }
                    if (p > best[0]) best[0] = p;
                }
            }
        }
        // each warp's K best, best first
        for (int i = 0; i < K; ++i) {
            const unsigned long long m = warp_max(best[0]);
            if (lane == 0) s_w[warp][i] = m;
            if (m != 0 && best[0] == m) {
#pragma unroll
                for (int t = 0; t < KC - 1; ++t) best[t] = best[t + 1];
                best[KC - 1] = 0;
            }
        }
        __syncthreads();
        if (warp == 0) {
            int p = 0;
            unsigned long long mine = 0;
            for (int i = 0; i < K; ++i) {
                const unsigned long long head = lane < kRowWarps && p < K ? s_w[lane][p] : 0;
                const unsigned long long m = warp_max(head);
                if (m != 0 && head == m) ++p;
                if (lane == i) mine = m;
            }
            if (lane < K) {
                const uint32_t col = 0xFFFFFFFFu - (uint32_t)mine;
                cand[lane] = Cand{beam_key<NORMALIZE>(__ldg(row + col), lse, score, first), col};
            }
        }
        __syncthreads();                                     // s_l, s_w and s_lse are reused by the next row
    }
}

struct MergeArgs {
    const Cand* cand;
    float* scores;
    int64_t* origin;
    int64_t* flat_origin;
    int64_t* tokens;
    int32_t* n_finished;
    uint8_t* eos_top;
    int64_t B, eos;
    int K, first;
};

__global__ void __launch_bounds__(kMergeWarps * 32) beam_merge_kernel(MergeArgs a) {
    const int lane = threadIdx.x & 31;
    const int K = a.K, rows = a.first ? 1 : a.K;
    for (int64_t b = (int64_t)blockIdx.x * kMergeWarps + (threadIdx.x >> 5); b < a.B; b += (int64_t)gridDim.x * kMergeWarps) {
        const Cand* mine = a.cand + ((int64_t)lane * a.B + b) * K;   // lane k walks row k*B + b
        int p = 0;
        Cand head{0.f, 0};
        if (lane < rows) head = mine[0];
        float key = 0.f;
        uint32_t col = 0;
        int from = 0;
        for (int i = 0; i < K; ++i) {
            // a key tie across rows goes to the lower row: its flat index k*V + j is lower whatever j
            const unsigned long long h = lane < rows && p < K ? ((unsigned long long)key_order(head.key) << 32) | (31u - lane) : 0;
            const unsigned long long m = warp_max(h);
            const int w = 31 - (int)(m & 31u);
            const float wk = __shfl_sync(0xFFFFFFFFu, head.key, w);
            const uint32_t wc = __shfl_sync(0xFFFFFFFFu, head.col, w);
            if (lane == i) key = wk, col = wc, from = w;
            if (lane == w && ++p < K) head = mine[p];
        }
        const bool is_eos = lane < K && (int64_t)col == a.eos;
        const unsigned n_eos = __popc(__ballot_sync(0xFFFFFFFFu, is_eos));
        if (lane < K) {
            const int64_t o = (int64_t)lane * a.B + b;
            a.scores[o] = key;
            a.origin[o] = from;
            a.tokens[o] = col;
            a.flat_origin[o] = (int64_t)from * a.B + b;
        }
        if (lane == 0) {
            a.n_finished[b] += (int32_t)n_eos;
            if (is_eos) a.eos_top[b] = 1;                    // lane 0 holds beam 0's token (Beam.py:104-106)
        }
    }
}

bool overlap(const void* a, size_t na, const void* b, size_t nb) {
    const uintptr_t pa = reinterpret_cast<uintptr_t>(a), pb = reinterpret_cast<uintptr_t>(b);
    return a != nullptr && b != nullptr && na > 0 && nb > 0 && pa < pb + nb && pb < pa + na;
}

bool misaligned(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) != 0; }

template <int KC>
void launch_rows(const RowArgs& a, bool normalize, unsigned grid, cudaStream_t st) {
    if (normalize) beam_row_kernel<KC, true><<<grid, kRowThreads, 0, st>>>(a);
    else beam_row_kernel<KC, false><<<grid, kRowThreads, 0, st>>>(a);
}

}  // namespace

extern "C" size_t qd_beam_workspace_bytes(int64_t batch, int beam) {
    if (batch <= 0 || beam < 1 || beam > QD_BEAM_MAX || batch > (int64_t)(SIZE_MAX / sizeof(Cand) / (QD_BEAM_MAX * QD_BEAM_MAX)))
        return 0;
    return (size_t)batch * beam * beam * sizeof(Cand);
}

extern "C" int qd_beam_step(const float* out, int normalize, int64_t batch, int beam, int64_t V, int64_t eos, int first_step,
                            float* scores, const int64_t* last_tokens, int64_t* origin, int64_t* flat_origin, int64_t* tokens,
                            int32_t* n_finished, uint8_t* eos_top, void* workspace, size_t workspace_bytes, qd_stream_t stream) {
    if (beam < 1 || beam > QD_BEAM_MAX) return fail(QD_ERR_INVALID_ARG, "beam must be in [1, %d] (beam=%d)", QD_BEAM_MAX, beam);
    if (batch < 0) return fail(QD_ERR_INVALID_ARG, "batch must be >= 0 (batch=%lld)", (long long)batch);
    if (normalize != 0 && normalize != 1) return fail(QD_ERR_INVALID_ARG, "normalize must be 0 or 1");
    if (V < beam) return fail(QD_ERR_INVALID_ARG, "V must be >= beam: the first step selects beam entries of one row (V=%lld)", (long long)V);
    if (V > (int64_t)UINT32_MAX) return fail(QD_ERR_INVALID_ARG, "V must be below 2^32 (V=%lld)", (long long)V);
    if (eos < 0 || eos >= V) return fail(QD_ERR_INVALID_ARG, "eos must be in [0, V) (eos=%lld)", (long long)eos);
    if (batch > INT64_MAX / beam / V) return fail(QD_ERR_INVALID_ARG, "batch * beam * V overflows 64-bit indexing");
    if (batch == 0) return QD_OK;
    if (out == nullptr || scores == nullptr || last_tokens == nullptr || origin == nullptr || flat_origin == nullptr ||
        tokens == nullptr || n_finished == nullptr || eos_top == nullptr)
        return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if (misaligned(out, 4) || misaligned(scores, 4) || misaligned(last_tokens, 8) || misaligned(origin, 8) ||
        misaligned(flat_origin, 8) || misaligned(tokens, 8) || misaligned(n_finished, 4))
        return fail(QD_ERR_INVALID_ARG, "misaligned argument (out, scores, n_finished 4 bytes; token and origin arrays 8 bytes)");
    const size_t need = qd_beam_workspace_bytes(batch, beam);
    if (workspace == nullptr || workspace_bytes < need || misaligned(workspace, 16))
        return fail(QD_ERR_WORKSPACE, "workspace must be 16-byte aligned and hold qd_beam_workspace_bytes(%lld, %d) = %zu bytes",
                    (long long)batch, beam, need);
    const int64_t R = batch * beam;
    const void* ins[2] = {out, last_tokens};
    const size_t in_bytes[2] = {(size_t)(R * V) * sizeof(float), (size_t)R * sizeof(int64_t)};
    const void* outs[7] = {scores, origin, flat_origin, tokens, n_finished, eos_top, workspace};
    const size_t out_bytes[7] = {(size_t)R * sizeof(float), (size_t)R * sizeof(int64_t), (size_t)R * sizeof(int64_t),
                                 (size_t)R * sizeof(int64_t), (size_t)batch * sizeof(int32_t), (size_t)batch, need};
    for (int i = 0; i < 7; ++i) {
        for (int j = 0; j < 2; ++j)
            if (overlap(outs[i], out_bytes[i], ins[j], in_bytes[j])) return fail(QD_ERR_INVALID_ARG, "outputs must not overlap the inputs");
        for (int j = 0; j < i; ++j)
            if (overlap(outs[i], out_bytes[i], outs[j], out_bytes[j])) return fail(QD_ERR_INVALID_ARG, "outputs must not overlap each other");
    }
    RowArgs ra{};
    ra.out = out, ra.scores = scores, ra.last_tokens = last_tokens, ra.cand = static_cast<Cand*>(workspace);
    ra.B = batch, ra.V = V, ra.eos = eos, ra.K = beam, ra.first = first_step != 0;
    const int64_t rows = first_step ? batch : R;
    const unsigned grid = (unsigned)(rows < kBeamMaxGrid ? rows : kBeamMaxGrid);
    cudaStream_t st = as_stream(stream);
    if (beam == 1) launch_rows<1>(ra, normalize, grid, st);
    else if (beam == 2) launch_rows<2>(ra, normalize, grid, st);
    else if (beam <= 4) launch_rows<4>(ra, normalize, grid, st);
    else if (beam <= 8) launch_rows<8>(ra, normalize, grid, st);
    else launch_rows<16>(ra, normalize, grid, st);
    MergeArgs ma{};
    ma.cand = ra.cand, ma.scores = scores, ma.origin = origin, ma.flat_origin = flat_origin, ma.tokens = tokens;
    ma.n_finished = n_finished, ma.eos_top = eos_top, ma.B = batch, ma.eos = eos, ma.K = beam, ma.first = ra.first;
    const int64_t merge_blocks = (batch + kMergeWarps - 1) / kMergeWarps;
    beam_merge_kernel<<<(unsigned)(merge_blocks < kBeamMaxGrid ? merge_blocks : kBeamMaxGrid), kMergeWarps * 32, 0, st>>>(ma);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}
