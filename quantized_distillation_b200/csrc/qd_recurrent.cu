// qd_recurrent.cu -- LSTM and GRU layers on fixed-width packed weights: one fused cell step (qd_packed_lstm_cell,
// qd_packed_gru_cell) and a layer in one direction over a padded batch or a PackedSequence (qd_packed_lstm_layer,
// qd_packed_gru_layer: one cell launch per step, the step loop shared).
#include <algorithm>
#include <vector>

#include "qd_launch.h"
#include "qd_packed_walk.cuh"

using namespace qd;

// ------------------------------------------------------------------ f2: LSTM cell on packed weights
// Hidden unit j has four rows in each weight, its gates i, f, g, o (rows j, H+j, 2H+j, 3H+j: torch's order), so a warp
// owns one unit and runs the quad walk of qd_packed_linear over those four rows: first over x against W_ih, then over
// h against W_hh.  Each sum is folded with warp_sum's butterfly exactly as qd_packed_linear folds it, so S_ih + b_ih
// is bit for bit qd_packed_linear(x, W_ih, b_ih) and S_hh is qd_packed_linear(h, W_hh, NULL).  Every lane then holds
// every row's sums; lane i keeps row m0+i's four preactivations ((S_ih + b_ih) + S_hh) + b_hh and applies the cell
// update in registers.  The preactivations never reach memory, there are no atomics and no workspace.
//
// A CTA is kPlWarps units x MT rows (blockIdx.y = row tile) and stages each operand's tile once per chunk, so the
// grid covers every (unit slab, row tile) once.
// one packed weight [G*H, K] (G gates per hidden unit: 4 for the LSTM, 3 for the GRU), with the fields the walk reads
struct CellOperand {
    const uint8_t* packed;
    const float* alpha;
    const float* beta;
    const float* points;
    int64_t K;
    int64_t in_bytes;           // ceil(G*H*K*bits/8)
    int64_t L, rows;            // bucket row length and bucket count (geometry_of)
    int64_t step_q, step_r;     // (128*E) / L and (128*E) % L
    int64_t kc;                 // columns per chunk of its activation tile
    int num_points;
    bool quad_aligned;
};

struct PackedLstmArgs {
    CellOperand w[2];           // W_ih (over x), W_hh (over h)
    const float* x;             // x rows, stride ldx
    const float* h;             // h rows 0 .. m_prev-1, stride ldh
    const float* h0;            // h rows m_prev .. m-1, stride H
    const float* c_in;          // [m, H]
    const float* b_ih;          // may be NULL
    const float* b_hh;
    float* h_out;               // stride ldo
    float* c_out;               // [m, H], may be c_in
    float* h_n;                 // rows m_next .. m-1 also written here (stride H); may be NULL
    int64_t ldx, ldh, ldo;
    int64_t m, m_prev, m_next, H;
    float S;                    // uniform: levels - 1; 0: non-uniform
    bool x_vec, h_vec;          // every row of x (of h and h0) 16-byte aligned and I (H) a multiple of 4
};

__device__ __forceinline__ float lstm_sigmoid(float z) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-z))); }

// both operands' unit tables: c/S at the model's levels, or each weight's own points
template <class Args>
__device__ __forceinline__ void load_cell_tables(const Args& a, float (&s_unit)[2][256]) {
    if (a.S != 0.f) {
        load_unit_table<true>(s_unit[0], nullptr, 0, a.S);
        load_unit_table<true>(s_unit[1], nullptr, 0, a.S);
    } else {
        load_unit_table<false>(s_unit[0], a.w[0].points, a.w[0].num_points, 0.f);
        load_unit_table<false>(s_unit[1], a.w[1].points, a.w[1].num_points, 0.f);
    }
}

// acc[r][i]: this lane's share of the sum of weight row orow[r] against x row m0+i, over all of the operand's columns
template <int BITS, int MT, int R, class Row>
__device__ __forceinline__ void gate_sums(const CellOperand& w, const float* s_unit, float4* s_x, Row row, int64_t m0, int64_t m, bool vec,
                                          int lane, const int64_t (&orow)[R], float (&acc)[R][MT]) {
    constexpr int E = 32 / BITS;
    const int kc4 = (int)(w.kc / 4);
    const int64_t kq = w.kc / (4 * E), qpr = (w.K + 4 * E - 1) / (4 * E), chunks = (w.K + w.kc - 1) / w.kc;
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
        for (int i = 0; i < MT; ++i) acc[r][i] = 0.f;
    for (int64_t c = 0; c < chunks; ++c) {
        __syncthreads();                                   // the previous tile (and, first, the unit tables) consumed
        pl_stage<BITS, MT>(s_x, row, m0, m, w.K, w.kc, kc4, vec, c);
        __syncthreads();
        pl_walk<BITS, MT>(w, s_unit, s_x, kc4, kq, qpr, c, lane, orow, acc);
    }
}

template <int BI, int BH, int MT>
__global__ void __launch_bounds__(kPlThreads, 1) packed_lstm_cell_kernel(PackedLstmArgs a) {
    extern __shared__ float4 s_x[];
    __shared__ float s_unit[2][256];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t m0 = (int64_t)blockIdx.y * MT;
    const int64_t j = (int64_t)blockIdx.x * kPlWarps + warp;
    const int64_t ju = j < a.H ? j : a.H - 1;             // units past H repeat unit H-1: computed, never written
    load_cell_tables(a, s_unit);
    int64_t orow[kPlRowsPerWarp];
#pragma unroll
    for (int r = 0; r < kPlRowsPerWarp; ++r) orow[r] = r * a.H + ju;
    float acc[kPlRowsPerWarp][MT];
    float pre[kPlRowsPerWarp];                             // lane i: row m0+i's preactivations
    auto x_row = [&](int64_t i) { return a.x + i * a.ldx; };
    gate_sums<BI, MT>(a.w[0], s_unit[0], s_x, x_row, m0, a.m, a.x_vec, lane, orow, acc);
#pragma unroll
    for (int r = 0; r < kPlRowsPerWarp; ++r) {
        const float b = a.b_ih != nullptr ? __ldg(a.b_ih + orow[r]) : 0.f;
        pre[r] = 0.f;
#pragma unroll
        for (int i = 0; i < MT; ++i) {
            float s = warp_sum(acc[r][i]);
            if (a.b_ih != nullptr) s = __fadd_rn(s, b);
            if (lane == i) pre[r] = s;
        }
    }
    auto h_row = [&](int64_t i) { return i < a.m_prev ? a.h + i * a.ldh : a.h0 + i * a.H; };
    gate_sums<BH, MT>(a.w[1], s_unit[1], s_x, h_row, m0, a.m, a.h_vec, lane, orow, acc);
#pragma unroll
    for (int r = 0; r < kPlRowsPerWarp; ++r) {
        const float b = a.b_hh != nullptr ? __ldg(a.b_hh + orow[r]) : 0.f;
#pragma unroll
        for (int i = 0; i < MT; ++i) {
            float s = __fadd_rn(pre[r], warp_sum(acc[r][i]));
            if (a.b_hh != nullptr) s = __fadd_rn(s, b);
            if (lane == i) pre[r] = s;
        }
    }
    const int64_t row = m0 + lane;
    if (j >= a.H || lane >= MT || row >= a.m) return;
    const float ig = lstm_sigmoid(pre[0]), fg = lstm_sigmoid(pre[1]), gg = tanhf(pre[2]), og = lstm_sigmoid(pre[3]);
    const float c = __fadd_rn(__fmul_rn(fg, a.c_in[row * a.H + j]), __fmul_rn(ig, gg));
    const float h = __fmul_rn(og, tanhf(c));
    a.c_out[row * a.H + j] = c;
    a.h_out[row * a.ldo + j] = h;
    if (a.h_n != nullptr && row >= a.m_next) a.h_n[row * a.H + j] = h;
}

// ------------------------------------------------------------------ f2: GRU cell on packed weights
// Hidden unit j has three rows in each weight, its gates r, z, n (rows j, H+j, 2H+j: torch's order), so a warp owns
// one unit and walks those three rows -- three, not four: kGruRows is the walk's R -- first over x against W_ih, then
// over h against W_hh.  Lane i keeps row m0+i's gi = S_ih + b_ih and gh = S_hh + b_hh, each bit for bit
// qd_packed_linear's output, and applies torch's cell update in registers:
//   r = sig(gi_r + gh_r), z = sig(gi_z + gh_z), n = tanh(gi_n + r*gh_n), h' = n + z*(h - n).
// The n gate needs gh_n apart from gi_n (b_hn sits inside r*(...)), so unlike the LSTM cell the two sums are kept
// apart and added only in the activations, r and z included, as torch's fused CUDA cell and its composite both do.
constexpr int kGruRows = 3;

struct PackedGruArgs {
    CellOperand w[2];           // W_ih (over x), W_hh (over h)
    const float* x;             // x rows, stride ldx
    const float* h;             // h rows 0 .. m_prev-1, stride ldh
    const float* h0;            // h rows m_prev .. m-1, stride H
    const float* b_ih;          // may be NULL
    const float* b_hh;
    float* h_out;               // stride ldo
    float* h_n;                 // rows m_next .. m-1 also written here (stride H); may be NULL
    int64_t ldx, ldh, ldo;
    int64_t m, m_prev, m_next, H;
    float S;                    // uniform: levels - 1; 0: non-uniform
    bool x_vec, h_vec;          // every row of x (of h and h0) 16-byte aligned and I (H) a multiple of 4
};

// out[r] on lane i: row m0+i's sum of weight row orow[r], folded as qd_packed_linear folds it, plus bias[orow[r]]
// unless bias is NULL -- qd_packed_linear's y[m0+i, orow[r]] bit for bit
template <int MT, int R>
__device__ __forceinline__ void fold_rows(const float (&acc)[R][MT], const float* bias, const int64_t (&orow)[R], int lane, float (&out)[R]) {
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const float b = bias != nullptr ? __ldg(bias + orow[r]) : 0.f;
        out[r] = 0.f;
#pragma unroll
        for (int i = 0; i < MT; ++i) {
            float s = warp_sum(acc[r][i]);
            if (bias != nullptr) s = __fadd_rn(s, b);
            if (lane == i) out[r] = s;
        }
    }
}

template <int BI, int BH, int MT>
__global__ void __launch_bounds__(kPlThreads, 1) packed_gru_cell_kernel(PackedGruArgs a) {
    extern __shared__ float4 s_x[];
    __shared__ float s_unit[2][256];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t m0 = (int64_t)blockIdx.y * MT;
    const int64_t j = (int64_t)blockIdx.x * kPlWarps + warp;
    const int64_t ju = j < a.H ? j : a.H - 1;             // units past H repeat unit H-1: computed, never written
    load_cell_tables(a, s_unit);
    int64_t orow[kGruRows];
#pragma unroll
    for (int r = 0; r < kGruRows; ++r) orow[r] = r * a.H + ju;
    float acc[kGruRows][MT];
    float gi[kGruRows], gh[kGruRows];                      // lane i: row m0+i's two linear outputs
    auto x_row = [&](int64_t i) { return a.x + i * a.ldx; };
    gate_sums<BI, MT>(a.w[0], s_unit[0], s_x, x_row, m0, a.m, a.x_vec, lane, orow, acc);
    fold_rows(acc, a.b_ih, orow, lane, gi);
    auto h_row = [&](int64_t i) { return i < a.m_prev ? a.h + i * a.ldh : a.h0 + i * a.H; };
    gate_sums<BH, MT>(a.w[1], s_unit[1], s_x, h_row, m0, a.m, a.h_vec, lane, orow, acc);
    fold_rows(acc, a.b_hh, orow, lane, gh);
    const int64_t row = m0 + lane;
    if (j >= a.H || lane >= MT || row >= a.m) return;
    const float rg = lstm_sigmoid(__fadd_rn(gi[0], gh[0])), zg = lstm_sigmoid(__fadd_rn(gi[1], gh[1]));
    const float ng = tanhf(__fadd_rn(gi[2], __fmul_rn(rg, gh[2])));
    const float hp = h_row(row)[j];
    const float h = __fadd_rn(ng, __fmul_rn(zg, __fsub_rn(hp, ng)));
    a.h_out[row * a.ldo + j] = h;
    if (a.h_n != nullptr && row >= a.m_next) a.h_n[row * a.H + j] = h;
}

// ------------------------------------------------------------------ host side, shared by both cells
// Checks one packed operand of a cell ([G*H, K] at the model's levels) and fills its walk fields; `what` names it.
static int cell_operand(const qd_packed_tensor* t, int G, int64_t H, int64_t K, int levels, int64_t bucket, const char* what, CellOperand* w) {
    if (t == nullptr || t->packed == nullptr || t->alpha == nullptr || t->beta == nullptr) return fail(QD_ERR_INVALID_ARG, "%s: NULL argument", what);
    if (!bits_ok(t->bits)) return fail(QD_ERR_INVALID_ARG, "%s: bits must be 1, 2, 4 or 8", what);
    if (K > INT64_MAX / 32 / H) return fail(QD_ERR_INVALID_ARG, "%s: %d * hidden_size * %lld elements is too large", what, G, (long long)K);
    if (t->n != G * H * K)
        return fail(QD_ERR_INVALID_ARG, "%s: n = %lld, expected %d * %lld * %lld", what, (long long)t->n, G, (long long)H, (long long)K);
    if (levels != 0) {
        if (t->points != nullptr || t->num_points != 0) return fail(QD_ERR_INVALID_ARG, "%s: uniform weights have no points (points NULL, num_points 0)", what);
        if (levels < 2 || levels > (1 << t->bits)) return fail(QD_ERR_INVALID_ARG, "%s: levels must be in [2, 2^bits]", what);
    } else if (t->points == nullptr || t->num_points < 1 || t->num_points > (1 << t->bits)) {
        return fail(QD_ERR_INVALID_ARG, "%s: num_points must be in [1, 2^bits]", what);
    }
    Geometry geo;
    if (geometry_of(t->n, bucket, &geo)) return fail(QD_ERR_INVALID_ARG, "bucket must be >= 0");
    *w = CellOperand{};
    w->packed = t->packed, w->alpha = t->alpha, w->beta = t->beta, w->points = t->points;
    w->K = K;
    w->in_bytes = (t->n * t->bits + 7) / 8;
    w->L = geo.row_len, w->rows = geo.rows;
    const int64_t step_cols = 32 * 4 * (32 / t->bits);
    w->step_q = step_cols / w->L, w->step_r = step_cols % w->L;
    w->num_points = t->num_points;
    w->quad_aligned = aligned16(t->packed) && (K * t->bits) % 128 == 0;
    return QD_OK;
}

// [p, p + bytes) and [q, q + bytes_q) share a byte
static bool overlap(const void* p, int64_t bytes, const void* q, int64_t bytes_q) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(p), b = reinterpret_cast<uintptr_t>(q);
    return a < b + (uintptr_t)bytes_q && b < a + (uintptr_t)bytes;
}
// bytes spanned by `rows` float rows of `cols` at stride `ld`
static int64_t span(int64_t rows, int64_t cols, int64_t ld) { return ((rows - 1) * ld + cols) * (int64_t)sizeof(float); }

template <int BI, int BH, int MT>
static auto cell_kernel(const PackedLstmArgs&) { return packed_lstm_cell_kernel<BI, BH, MT>; }
template <int BI, int BH, int MT>
static auto cell_kernel(const PackedGruArgs&) { return packed_gru_cell_kernel<BI, BH, MT>; }

template <int MT, int BI, int BH, class Args>
static int launch_cell(Args a, cudaStream_t st) {
    a.w[0].kc = pl_chunk_cols<MT, BI>(a.w[0].K);
    a.w[1].kc = pl_chunk_cols<MT, BH>(a.w[1].K);
    const size_t smem = (size_t)MT * std::max(a.w[0].kc, a.w[1].kc) * sizeof(float);
    auto kern = cell_kernel<BI, BH, MT>(a);
    static size_t opted[64] = {};
    if (const int rc = opt_in_smem((const void*)kern, smem, opted)) return rc;
    const dim3 grid((unsigned)((a.H + kPlWarps - 1) / kPlWarps), (unsigned)((a.m + MT - 1) / MT));
    kern<<<grid, kPlThreads, smem, st>>>(a);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

// one cell launch for a.m rows, at the code widths of the two operands
template <class Args>
static int cell_step(const Args& a, int bits_ih, int bits_hh, cudaStream_t st) {
    auto go = [&](auto mt) {
        return with_bits(bits_ih, [&](auto bi) { return with_bits(bits_hh, [&](auto bh) { return launch_cell<mt, bi, bh>(a, st); }); });
    };
    if (a.m == 1) return go(std::integral_constant<int, 1>{});
    if (a.m == 2) return go(std::integral_constant<int, 2>{});
    if (a.m <= 4) return go(std::integral_constant<int, 4>{});
    return go(std::integral_constant<int, 8>{});
}

// Checks what a cell and its layer share -- sizes, both operands, levels -- and fills their part of `a`.
template <class Args>
static int cell_common(int G, int64_t I, int64_t H, const qd_packed_tensor* w_ih, const qd_packed_tensor* w_hh, int levels, int64_t bucket,
                       Args* a) {
    if (I < 1 || H < 1) return fail(QD_ERR_INVALID_ARG, "input_size and hidden_size must be >= 1");
    if (H > INT32_MAX) return fail(QD_ERR_INVALID_ARG, "hidden_size must be below 2^31");
    if (levels != 0 && (levels < 2 || levels > 256)) return fail(QD_ERR_INVALID_ARG, "levels must be in [2, 256] (uniform) or 0 (non-uniform)");
    if (const int rc = cell_operand(w_ih, G, H, I, levels, bucket, "w_ih", &a->w[0])) return rc;
    if (const int rc = cell_operand(w_hh, G, H, H, levels, bucket, "w_hh", &a->w[1])) return rc;
    a->H = H;
    a->S = levels != 0 ? (float)(levels - 1) : 0.f;
    return QD_OK;
}

// Checks a layer's host batch sizes (non-increasing, >= 1, the first at most max_rows rows of `cell`) and sums them.
static int layer_batch_sizes(const int64_t* batch_sizes, int64_t steps, int max_rows, const char* cell, int64_t* total) {
    const int64_t B = batch_sizes[0];
    *total = 0;
    for (int64_t t = 0; t < steps; ++t) {
        if (batch_sizes[t] < 1) return fail(QD_ERR_INVALID_ARG, "batch_sizes[%lld] = %lld: every step needs a row", (long long)t, (long long)batch_sizes[t]);
        if (batch_sizes[t] > B)
            return fail(QD_ERR_INVALID_ARG, "batch_sizes[%lld] = %lld exceeds batch_sizes[0] = %lld: batch sizes must not increase",
                        (long long)t, (long long)batch_sizes[t], (long long)B);
        if (t > 0 && batch_sizes[t] > batch_sizes[t - 1]) return fail(QD_ERR_INVALID_ARG, "batch sizes must not increase (step %lld)", (long long)t);
        *total += batch_sizes[t];
    }
    if (B > max_rows) return fail(QD_ERR_UNSUPPORTED, "a batch of %lld rows: the packed %s cell serves at most %d", (long long)B, cell, max_rows);
    return QD_OK;
}

// The step loop of a layer in one direction: step t reads x rows and writes out rows at its offset in the packed data
// (strides a.ldx, a.ldo), a row's previous h is the previous step's out row below m_prev, its h0 row above (a.h0), and
// a row's last step (rows at or past m_next) also writes it to a.h_n.  One cell_step per step, nothing synchronised.
template <class Args>
static int layer_steps(Args& a, const float* x, float* out, const int64_t* batch_sizes, int64_t steps, int reverse, int bits_ih, int bits_hh,
                       cudaStream_t st) {
    // row offset of every step in the packed data (kept per thread: no allocation once grown)
    thread_local std::vector<int64_t> off;
    off.resize((size_t)steps);
    for (int64_t t = 0, o = 0; t < steps; o += batch_sizes[t++]) off[(size_t)t] = o;
    int64_t m_prev = 0, prev = 0;
    for (int64_t s = 0; s < steps; ++s) {
        const int64_t t = reverse ? steps - 1 - s : s;
        const int64_t next = reverse ? t - 1 : t + 1;
        a.x = x + off[(size_t)t] * a.ldx;
        a.h = out + off[(size_t)prev] * a.ldo;            // read for rows below m_prev only
        a.h_out = out + off[(size_t)t] * a.ldo;
        a.m = batch_sizes[t];
        a.m_prev = m_prev;
        a.m_next = s + 1 < steps ? batch_sizes[next] : 0;
        if (const int rc = cell_step(a, bits_ih, bits_hh, st)) return rc;
        m_prev = a.m;
        prev = t;
    }
    return QD_OK;
}

// ------------------------------------------------------------------ the LSTM entry points
extern "C" int qd_packed_lstm_cell(const float* x, int64_t ldx, const float* h, int64_t ldh, const float* c, int64_t m, int64_t input_size,
                                   int64_t hidden_size, const qd_packed_tensor* w_ih, const qd_packed_tensor* w_hh, int levels,
                                   int64_t bucket, const float* b_ih, const float* b_hh, float* h_out, int64_t ldo, float* c_out,
                                   qd_stream_t stream) {
    if (x == nullptr || h == nullptr || c == nullptr || h_out == nullptr || c_out == nullptr) return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if (m < 1) return fail(QD_ERR_INVALID_ARG, "m must be >= 1 (got %lld)", (long long)m);
    PackedLstmArgs a{};
    if (const int rc = cell_common(4, input_size, hidden_size, w_ih, w_hh, levels, bucket, &a)) return rc;
    const int64_t I = input_size, H = hidden_size;
    if (ldx < I || ldh < H || ldo < H) return fail(QD_ERR_INVALID_ARG, "row strides must be at least the rows (ldx >= input_size, ldh and ldo >= hidden_size)");
    if (m > QD_PACKED_LSTM_MAX_ROWS)
        return fail(QD_ERR_UNSUPPORTED, "m = %lld rows: the packed LSTM cell serves at most %d", (long long)m, QD_PACKED_LSTM_MAX_ROWS);
    if (m > INT64_MAX / 4 / std::max(std::max(ldx, ldh), ldo)) return fail(QD_ERR_INVALID_ARG, "the rows overflow 64-bit indexing");
    const int64_t xs = span(m, I, ldx), hs = span(m, H, ldh), os = span(m, H, ldo), cs = span(m, H, H);
    if (overlap(h_out, os, x, xs) || overlap(h_out, os, h, hs)) return fail(QD_ERR_INVALID_ARG, "h_out must not overlap x or h");
    if (overlap(h_out, os, c, cs) || overlap(h_out, os, c_out, cs)) return fail(QD_ERR_INVALID_ARG, "h_out must not overlap c or c_out");
    if (c_out != c && overlap(c_out, cs, c, cs)) return fail(QD_ERR_INVALID_ARG, "c_out must be c or not overlap it");
    if (overlap(c_out, cs, x, xs) || overlap(c_out, cs, h, hs)) return fail(QD_ERR_INVALID_ARG, "c_out must not overlap x or h");
    a.x = x, a.h = h, a.h0 = h, a.c_in = c, a.b_ih = b_ih, a.b_hh = b_hh, a.h_out = h_out, a.c_out = c_out, a.h_n = nullptr;
    a.ldx = ldx, a.ldh = ldh, a.ldo = ldo;
    a.m = m, a.m_prev = m, a.m_next = m;
    a.x_vec = aligned16(x) && ldx % 4 == 0 && I % 4 == 0;
    a.h_vec = aligned16(h) && ldh % 4 == 0 && H % 4 == 0;
    return cell_step(a, w_ih->bits, w_hh->bits, as_stream(stream));
}

extern "C" int qd_packed_lstm_layer(const float* x, int64_t ldx, const int64_t* batch_sizes, int64_t steps, int reverse, int64_t input_size,
                                    int64_t hidden_size, const qd_packed_tensor* w_ih, const qd_packed_tensor* w_hh, int levels,
                                    int64_t bucket, const float* b_ih, const float* b_hh, const float* h0, const float* c0, float* out,
                                    int64_t ldo, float* h_n, float* c_n, qd_stream_t stream) {
    if (x == nullptr || batch_sizes == nullptr || h0 == nullptr || c0 == nullptr || out == nullptr || h_n == nullptr || c_n == nullptr)
        return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if (steps < 1) return fail(QD_ERR_INVALID_ARG, "steps must be >= 1 (got %lld)", (long long)steps);
    PackedLstmArgs a{};
    if (const int rc = cell_common(4, input_size, hidden_size, w_ih, w_hh, levels, bucket, &a)) return rc;
    const int64_t I = input_size, H = hidden_size;
    if (ldx < I || ldo < H) return fail(QD_ERR_INVALID_ARG, "row strides must be at least the rows (ldx >= input_size, ldo >= hidden_size)");
    const int64_t B = batch_sizes[0];
    int64_t total = 0;
    if (const int rc = layer_batch_sizes(batch_sizes, steps, QD_PACKED_LSTM_MAX_ROWS, "LSTM", &total)) return rc;
    if (total > INT64_MAX / 4 / std::max(ldx, ldo)) return fail(QD_ERR_INVALID_ARG, "the rows overflow 64-bit indexing");
    const int64_t xs = span(total, I, ldx), os = span(total, H, ldo), ss = span(B, H, H);
    if (overlap(out, os, x, xs) || overlap(out, os, h0, ss) || overlap(out, os, c0, ss)) return fail(QD_ERR_INVALID_ARG, "out must not overlap x, h0 or c0");
    for (const float* s : {(const float*)h_n, (const float*)c_n})
        if (overlap(s, ss, out, os) || overlap(s, ss, x, xs) || overlap(s, ss, h0, ss))
            return fail(QD_ERR_INVALID_ARG, "h_n and c_n must not overlap out, x or h0");
    if (overlap(h_n, ss, c_n, ss)) return fail(QD_ERR_INVALID_ARG, "h_n must not overlap c_n");
    if (c_n != c0 && overlap(c_n, ss, c0, ss)) return fail(QD_ERR_INVALID_ARG, "c_n must be c0 or not overlap it");
    cudaStream_t st = as_stream(stream);
    if (c_n != c0) QD_CUDA(cudaMemcpyAsync(c_n, c0, (size_t)ss, cudaMemcpyDeviceToDevice, st));
    a.h0 = h0, a.c_in = c_n, a.c_out = c_n, a.b_ih = b_ih, a.b_hh = b_hh, a.h_n = h_n;
    a.ldx = ldx, a.ldh = ldo, a.ldo = ldo;
    a.x_vec = aligned16(x) && ldx % 4 == 0 && I % 4 == 0;
    a.h_vec = aligned16(out) && ldo % 4 == 0 && aligned16(h0) && H % 4 == 0;
    return layer_steps(a, x, out, batch_sizes, steps, reverse, w_ih->bits, w_hh->bits, st);
}

// ------------------------------------------------------------------ the GRU entry points
extern "C" int qd_packed_gru_cell(const float* x, int64_t ldx, const float* h, int64_t ldh, int64_t m, int64_t input_size, int64_t hidden_size,
                                  const qd_packed_tensor* w_ih, const qd_packed_tensor* w_hh, int levels, int64_t bucket, const float* b_ih,
                                  const float* b_hh, float* h_out, int64_t ldo, qd_stream_t stream) {
    if (x == nullptr || h == nullptr || h_out == nullptr) return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if (m < 1) return fail(QD_ERR_INVALID_ARG, "m must be >= 1 (got %lld)", (long long)m);
    PackedGruArgs a{};
    if (const int rc = cell_common(3, input_size, hidden_size, w_ih, w_hh, levels, bucket, &a)) return rc;
    const int64_t I = input_size, H = hidden_size;
    if (ldx < I || ldh < H || ldo < H) return fail(QD_ERR_INVALID_ARG, "row strides must be at least the rows (ldx >= input_size, ldh and ldo >= hidden_size)");
    if (m > QD_PACKED_GRU_MAX_ROWS)
        return fail(QD_ERR_UNSUPPORTED, "m = %lld rows: the packed GRU cell serves at most %d", (long long)m, QD_PACKED_GRU_MAX_ROWS);
    if (m > INT64_MAX / 4 / std::max(std::max(ldx, ldh), ldo)) return fail(QD_ERR_INVALID_ARG, "the rows overflow 64-bit indexing");
    const int64_t xs = span(m, I, ldx), hs = span(m, H, ldh), os = span(m, H, ldo);
    if (overlap(h_out, os, x, xs) || overlap(h_out, os, h, hs)) return fail(QD_ERR_INVALID_ARG, "h_out must not overlap x or h");
    a.x = x, a.h = h, a.h0 = h, a.b_ih = b_ih, a.b_hh = b_hh, a.h_out = h_out, a.h_n = nullptr;
    a.ldx = ldx, a.ldh = ldh, a.ldo = ldo;
    a.m = m, a.m_prev = m, a.m_next = m;
    a.x_vec = aligned16(x) && ldx % 4 == 0 && I % 4 == 0;
    a.h_vec = aligned16(h) && ldh % 4 == 0 && H % 4 == 0;
    return cell_step(a, w_ih->bits, w_hh->bits, as_stream(stream));
}

extern "C" int qd_packed_gru_layer(const float* x, int64_t ldx, const int64_t* batch_sizes, int64_t steps, int reverse, int64_t input_size,
                                   int64_t hidden_size, const qd_packed_tensor* w_ih, const qd_packed_tensor* w_hh, int levels,
                                   int64_t bucket, const float* b_ih, const float* b_hh, const float* h0, float* out, int64_t ldo,
                                   float* h_n, qd_stream_t stream) {
    if (x == nullptr || batch_sizes == nullptr || h0 == nullptr || out == nullptr || h_n == nullptr) return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if (steps < 1) return fail(QD_ERR_INVALID_ARG, "steps must be >= 1 (got %lld)", (long long)steps);
    PackedGruArgs a{};
    if (const int rc = cell_common(3, input_size, hidden_size, w_ih, w_hh, levels, bucket, &a)) return rc;
    const int64_t I = input_size, H = hidden_size;
    if (ldx < I || ldo < H) return fail(QD_ERR_INVALID_ARG, "row strides must be at least the rows (ldx >= input_size, ldo >= hidden_size)");
    const int64_t B = batch_sizes[0];
    int64_t total = 0;
    if (const int rc = layer_batch_sizes(batch_sizes, steps, QD_PACKED_GRU_MAX_ROWS, "GRU", &total)) return rc;
    if (total > INT64_MAX / 4 / std::max(ldx, ldo)) return fail(QD_ERR_INVALID_ARG, "the rows overflow 64-bit indexing");
    const int64_t xs = span(total, I, ldx), os = span(total, H, ldo), ss = span(B, H, H);
    if (overlap(out, os, x, xs) || overlap(out, os, h0, ss)) return fail(QD_ERR_INVALID_ARG, "out must not overlap x or h0");
    if (overlap(h_n, ss, out, os) || overlap(h_n, ss, x, xs) || overlap(h_n, ss, h0, ss))
        return fail(QD_ERR_INVALID_ARG, "h_n must not overlap out, x or h0");
    a.h0 = h0, a.b_ih = b_ih, a.b_hh = b_hh, a.h_n = h_n;
    a.ldx = ldx, a.ldh = ldo, a.ldo = ldo;
    a.x_vec = aligned16(x) && ldx % 4 == 0 && I % 4 == 0;
    a.h_vec = aligned16(out) && ldo % 4 == 0 && aligned16(h0) && H % 4 == 0;
    return layer_steps(a, x, out, batch_sizes, steps, reverse, w_ih->bits, w_hh->bits, as_stream(stream));
}
