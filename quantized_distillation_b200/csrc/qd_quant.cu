// qd_quant.cu -- the fake-quantization ops: argument checking, path selection and the extern "C" entry points of
// scaling, uniform and non-uniform quantization (forward and backward), the abs scalings and the centroid index.
//
// Path selection by row length L (= bucket, or n when bucket is None / n < bucket):
//     L <= 1024                  warp path    (registers, 1 HBM pass)
//     L <= QD_MAX_STAGED_BUCKET  staged path  (TMA chunk ring in shared memory, 1 HBM pass; CTA size by L)
//     otherwise                  grid path    (two streaming passes)
// Thresholds inside these ranges were measured with tools/block_bench.py, every variant forced through a tuning hook
// that has since been removed.
#include <cstring>

#include "qd_abs_path.cuh"
#include "qd_block_path.cuh"
#include "qd_grid_path.cuh"
#include "qd_launch.h"
#include "qd_points_grad.cuh"
#include "qd_staged_path.cuh"
#include "qd_warp_path.cuh"

using namespace qd;

// ------------------------------------------------------------------ geometry / workspace
extern "C" int qd_bucket_geometry(int64_t n, int64_t bucket, int64_t* rows, int64_t* row_len, int64_t* padded_len) {
    Geometry g;
    if (geometry_of(n, bucket, &g)) return fail(QD_ERR_INVALID_ARG, "n must be > 0 and bucket >= 0 (n=%lld bucket=%lld)", (long long)n, (long long)bucket);
    if (rows) *rows = g.rows;
    if (row_len) *row_len = g.row_len;
    if (padded_len) *padded_len = g.rows * g.row_len;
    return QD_OK;
}

static constexpr size_t kPointsGradMaxCtas = 132 * 8;  // 8 CTAs per SM of a 132-SM H100 SXM; bigger parts are capped here
static size_t points_grad_ws_bytes() { return kPointsGradMaxCtas * 256 * sizeof(double); }

// the workspace a geometry needs: what qd_workspace_bytes states, and what the grid path checks it has
static size_t workspace_bytes_of(const Geometry& g) {
    size_t bytes = points_grad_ws_bytes();
    if (g.row_len > QD_MAX_STAGED_BUCKET) {
        size_t grid = (size_t)(g.rows * grid_chunks_per_row(g)) * sizeof(ChunkPartial) + (size_t)g.rows * sizeof(RowStat) + 256;
        if (grid > bytes) bytes = grid;
    }
    return bytes + 256;
}

extern "C" size_t qd_workspace_bytes(int64_t n, int64_t bucket) {
    Geometry g;
    if (geometry_of(n, bucket, &g)) return 0;
    return workspace_bytes_of(g);
}

// ------------------------------------------------------------------ launchers
template <int OP, int BWD, int R, bool VEC, int PACK = 0>
static int launch_warp_inst(const Params& P, cudaStream_t s) {
    auto kern = warp_rows_kernel<OP, BWD, R, VEC, false, PACK>;
    int grid = (int)warp_rows_grid(P.geo.rows);
    if constexpr (!kRowPerWarp<OP>) {
        int rc = resident_grid((const void*)kern, kWarpCtaThreads, 0, (P.geo.rows + kWarpsPerCta - 1) / kWarpsPerCta, &grid);
        if (rc) return rc;
    }
    if constexpr (OP == OP_UNIFORM && BWD == (int)BWD_MINMAX) {
        // r_b accumulation, chosen by A/B (64 Mi floats, both variants forced through a since-removed tuning hook):
        // the fused forward+backward is faster with one float64 add per element, the backward alone with the grouped
        // lane sum.  So the variant follows the presence of the q output.
        if (P.q != nullptr) {
            auto kern_a = warp_rows_kernel<OP, BWD, R, VEC, true>;
            kern_a<<<grid, kWarpCtaThreads, 0, s>>>(P);
            QD_CUDA(cudaGetLastError());
            return QD_OK;
        }
    }
    kern<<<grid, kWarpCtaThreads, 0, s>>>(P);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

template <int OP, int BWD>
static int launch_warp(const Params& P, bool vec, cudaStream_t s) {
    return with_row_regs(P.geo.row_len, [&](auto r) {
        return vec ? launch_warp_inst<OP, BWD, r, true>(P, s) : launch_warp_inst<OP, BWD, r, false>(P, s);
    });
}


template <int OP, int BWD, bool STAGED, int GROUP>
static int launch_block_inst(const Params& P, cudaStream_t s) {
    DevInfo* di;
    int rc = dev_info(&di);
    if (rc) return rc;
    auto kern = block_rows_kernel<OP, BWD, STAGED, GROUP>;
    const size_t smem = STAGED ? (size_t)P.geo.row_len * sizeof(float) : 0;
    if (smem + 8192 > di->smem_optin) return fail(QD_ERR_UNSUPPORTED, "row of %lld floats does not fit in shared memory", (long long)P.geo.row_len);
    if (STAGED) {
        static size_t opted[64] = {};  // largest dynamic size this instantiation was opted into, per device
        rc = opt_in_smem((const void*)kern, smem, opted);
        if (rc) return rc;
    }
    constexpr int64_t rows_per_cta = kBlockCtaThreads / GROUP;
    const int grid = di->grid((P.geo.rows + rows_per_cta - 1) / rows_per_cta,
                              resident_ctas((const void*)kern, di->device, kBlockCtaThreads, smem));
    kern<<<grid, kBlockCtaThreads, smem, s>>>(P);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

// CTA per row, TMA chunk ring (qd_staged_path.cuh)
template <int OP, int BWD, int STAGES, int T>
static int launch_staged_inst(const Params& P, cudaStream_t s) {
    DevInfo* di;
    int rc = dev_info(&di);
    if (rc) return rc;
    auto kern = staged_rows_kernel<OP, BWD, STAGES, T>;
    const int stage_floats = (int)((P.geo.row_len + 31) & ~(int64_t)31);
    const size_t smem = (size_t)STAGES * stage_floats * sizeof(float);
    if (smem + 8192 > di->smem_optin) return fail(QD_ERR_UNSUPPORTED, "row of %lld floats does not fit in shared memory", (long long)P.geo.row_len);
    static size_t opted[64] = {};  // largest dynamic size this instantiation was opted into, per device
    rc = opt_in_smem((const void*)kern, smem, opted);
    if (rc) return rc;
    const int grid = di->grid(P.geo.rows, resident_ctas((const void*)kern, di->device, T, smem));
    kern<<<grid, T, smem, s>>>(P, stage_floats);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

// CTA size and ring depth by row length (tools/block_bench.py, every variant forced through a since-removed tuning
// hook): 64 threads below 2048 floats (a 1280-float row is five full steps of a 64-thread CTA, three ragged ones of a
// 128-thread CTA), 128 up to 3072, 256 up to 12288, 512 up to 24576, 1024 beyond; two rows in flight per CTA up to
// 3072 floats, the chunk ring alone above (on H100 one row in flight is as fast or faster for every op at 4096 floats,
// and the min/max backward gains most: fused 459 vs 526 us, alone 371 vs 429 us at 64 Mi floats).
template <int OP, int BWD>
static int launch_staged(const Params& P, cudaStream_t s) {
    const int64_t L = P.geo.row_len;
    if (L <= kTwoStageMaxRow) return L < 2048 ? launch_staged_inst<OP, BWD, 2, 64>(P, s) : launch_staged_inst<OP, BWD, 2, 128>(P, s);
    if (L <= 12288) return launch_staged_inst<OP, BWD, 1, 256>(P, s);
    if (L <= 24576) return launch_staged_inst<OP, BWD, 1, 512>(P, s);
    return launch_staged_inst<OP, BWD, 1, 1024>(P, s);
}

// Rows of 1025 .. QD_MAX_STAGED_BUCKET floats, and the ragged 513 .. 1023-float rows of the min/max backward.
template <int OP, int BWD>
static int launch_block(const Params& P, cudaStream_t s) {
    if constexpr (OP == OP_UNIFORM || OP == OP_NONUNIFORM) {
        // the staged ring wins or ties at every row length for the ops it implements (tools/block_bench.py), except
        // the min/max backward on rows of 1025 .. 2048 floats, where the warp two-pass variant is faster on H100
        // (64 Mi floats: fused 460 vs 527 us at 1280 floats, 464 vs 531 us at 2048; backward alone 373 vs 409, 380 vs 407)
        if constexpr (OP == OP_UNIFORM && BWD == (int)BWD_MINMAX)
            if (P.geo.row_len > 1024 && P.geo.row_len <= kWarp2MinmaxMaxRow) return launch_block_inst<OP, BWD, false, 32>(P, s);
        return launch_staged<OP, BWD>(P, s);
    } else {
        // the ops the ring does not implement (stats / scale / stochastic) keep the round-1 kernels: warp per row, two
        // passes, then CTA per row, whole-row staging (stochastic rounding is a run-time branch of OP_UNIFORM there)
        constexpr int OP2 = (OP == OP_UNIFORM_STOCH) ? OP_UNIFORM : OP;
        if (P.geo.row_len <= 2 * kWarpTwoPassMaxRow) return launch_block_inst<OP2, BWD, false, 32>(P, s);
        return launch_block_inst<OP2, BWD, true, kBlockCtaThreads>(P, s);
    }
}

template <int OP, int BWD>
static int launch_grid(const Params& P, void* ws, size_t ws_bytes, cudaStream_t s) {
    const int64_t cpr = grid_chunks_per_row(P.geo);
    const int64_t items = P.geo.rows * cpr;
    // the stated size, not just the bytes used below: a caller that passes less is refused on every geometry alike
    const size_t need = workspace_bytes_of(P.geo);
    if (ws == nullptr || ws_bytes < need) return fail(QD_ERR_WORKSPACE, "workspace of %zu bytes needed, %zu given", need, ws_bytes);
    ChunkPartial* partial = reinterpret_cast<ChunkPartial*>(ws);
    RowStat* rowstat = reinterpret_cast<RowStat*>(partial + items);
    int grid;
    int rc = capped_grid(items, 4, &grid);
    if (rc) return rc;
    grid_stats_partial<<<grid, kGridCtaThreads, 0, s>>>(P, partial, cpr, P.argmin != nullptr ? 1 : 0);
    QD_CUDA(cudaGetLastError());
    grid_stats_final<<<(int)P.geo.rows, 256, 0, s>>>(P, partial, rowstat, cpr);
    QD_CUDA(cudaGetLastError());
    if (OP != OP_STATS) {
        grid_apply<(OP == OP_STATS ? OP_SCALE : OP), BWD><<<grid, kGridCtaThreads, 0, s>>>(P, rowstat, cpr);
        QD_CUDA(cudaGetLastError());
    }
    return QD_OK;
}

// true when every row of every non-null float tensor starts 16-byte aligned
static bool rows_vectorizable(const Params& P) {
    const bool ptrs = aligned16(P.x) && aligned16(P.g) && aligned16(P.q) && aligned16(P.gout) && aligned16(P.xhat) &&
                      ((reinterpret_cast<uintptr_t>(P.idx8) & 3) == 0);
    return ptrs && (P.geo.rows == 1 || (P.geo.row_len % 4) == 0);
}

template <int OP, int BWD>
static int run_rows(const Params& P, void* ws, size_t ws_bytes, cudaStream_t s) {
    if (P.geo.row_len >= (int64_t)1 << 31) return fail(QD_ERR_UNSUPPORTED, "rows of 2^31 elements or more are not supported");
    // ragged rows of 513..1023 floats with the min/max backward: the R = 8 register kernel runs its predicated
    // (non-FULL) variant at 128 registers there and loses to the staged ring (measured with tools/block_bench.py
    // --small, the ring forced down to these rows through a since-removed tuning hook); everything else up to 1024
    // floats is faster in registers
    const bool ragged_minmax = OP == OP_UNIFORM && BWD == (int)BWD_MINMAX && P.geo.row_len > 512 && P.geo.row_len < 1024;
    if (P.geo.row_len <= 1024 && !ragged_minmax)
        return launch_warp<OP, (OP == OP_NONUNIFORM ? 256 : BWD)>(P, rows_vectorizable(P), s);
    if (P.geo.row_len <= QD_MAX_STAGED_BUCKET) return launch_block<OP, BWD>(P, s);
    // the grid path keeps stochastic rounding as a run-time branch of OP_UNIFORM
    constexpr int OP2 = (OP == OP_UNIFORM_STOCH) ? OP_UNIFORM : OP;
    if (BWD == BWD_MINMAX)
        return fail(QD_ERR_UNSUPPORTED, "minmax backward needs bucket <= %d (reference: bucket_size None not supported, quant_functions.py:332-334)", QD_MAX_STAGED_BUCKET);
    return launch_grid<OP2, (BWD == BWD_MINMAX ? BWD_OFF : BWD)>(P, ws, ws_bytes, s);
}

static Params blank_params() {
    Params P;
    memset(&P, 0, sizeof(P));
    return P;
}

// ------------------------------------------------------------------ a2 / a3
extern "C" int qd_scale_down(const float* x, float* xhat, float* alpha, float* beta, int64_t* argmin, int64_t* argmax,
                             int64_t n, int64_t bucket, const float* mean, float max_element, void* workspace,
                             size_t workspace_bytes, qd_stream_t stream) {
    Params P = blank_params();
    if (x == nullptr) return fail(QD_ERR_INVALID_ARG, "x is NULL");
    if ((alpha == nullptr) != (beta == nullptr) || (argmin == nullptr) != (argmax == nullptr))
        return fail(QD_ERR_INVALID_ARG, "alpha/beta and argmin/argmax must be given in pairs");
    if (geometry_of(n, bucket, &P.geo)) return fail(QD_ERR_INVALID_ARG, "bad geometry n=%lld bucket=%lld", (long long)n, (long long)bucket);
    P.x = x; P.xhat = xhat; P.alpha = alpha; P.beta = beta; P.argmin = argmin; P.argmax = argmax;
    P.mean = mean; P.max_element = max_element;
    cudaStream_t s = as_stream(stream);
    if (xhat == nullptr) return run_rows<OP_STATS, BWD_OFF>(P, workspace, workspace_bytes, s);
    return run_rows<OP_SCALE, BWD_OFF>(P, workspace, workspace_bytes, s);
}
// (row, offset in row) of an element position that advances by fixed steps: one 64-bit division per THREAD, none per group
struct RowCursor {
    int64_t row, rem;
    __device__ __forceinline__ void advance(int64_t d_rows, int64_t d_rem, int64_t L) {
        row += d_rows;
        rem += d_rem;
        if (rem >= L) { rem -= L; ++row; }
    }
};

// y*alpha + beta (+ mean): groups of four consecutive elements, 128-bit accesses when the rows are multiples of four
// (every bucketed layout of the reference) and the pointers allow
__global__ void __launch_bounds__(256) inv_scale_kernel(const float* __restrict__ y, float* __restrict__ out, const float* __restrict__ alpha,
                                                        const float* __restrict__ beta, const float* __restrict__ mean, Geometry geo) {
    const float m = mean ? *mean : 0.f;
    const int64_t L = geo.row_len;
    const bool vec = (geo.rows == 1 || L % 4 == 0) && ((reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(out)) & 15) == 0;
    const int64_t groups = vec ? (geo.n >> 2) : 0;
    const int64_t tiles = (groups + kTileGroups - 1) / kTileGroups;
    const int64_t e_first = ((int64_t)blockIdx.x * kTileGroups + threadIdx.x) * 4;
    RowCursor cur{e_first / L, e_first % L};
    const int64_t du_rows = (256 * 4) / L, du_rem = (256 * 4) % L;
    const int64_t dt = (int64_t)gridDim.x * kTileGroups * 4;
    const int64_t dt_rows = dt / L, dt_rem = dt % L;
    for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int64_t g0 = tile * kTileGroups + threadIdx.x;
        float4 t[kTileU];
#pragma unroll
        for (int u = 0; u < kTileU; ++u)
            if (g0 + u * 256 < groups) t[u] = ld_stream4(y + (g0 + u * 256) * 4);
        RowCursor c = cur;
#pragma unroll
        for (int u = 0; u < kTileU; ++u) {
            if (g0 + u * 256 < groups) {
                const float a = alpha[c.row], b = beta[c.row];
                float4 o = make_float4(from_unit(t[u].x, a, b), from_unit(t[u].y, a, b), from_unit(t[u].z, a, b), from_unit(t[u].w, a, b));  // mul_, add_ (:142-143)
                if (mean) { o.x = __fadd_rn(o.x, m); o.y = __fadd_rn(o.y, m); o.z = __fadd_rn(o.z, m); o.w = __fadd_rn(o.w, m); }  // add_(mean) (:148)
                st_stream4(out + (g0 + u * 256) * 4, o);
            }
            c.advance(du_rows, du_rem, L);
        }
        cur.advance(dt_rows, dt_rem, L);
    }
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = groups * 4 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < geo.n; i += stride) {
        const int64_t row = (geo.rows == 1) ? 0 : i / L;
        float v = from_unit(y[i], alpha[row], beta[row]);
        if (mean) v = __fadd_rn(v, m);
        out[i] = v;
    }
}

extern "C" int qd_inv_scale_down(const float* y, float* out, const float* alpha, const float* beta, const float* mean,
                                 int64_t n, int64_t bucket, qd_stream_t stream) {
    Geometry g;
    if (y == nullptr || out == nullptr || alpha == nullptr || beta == nullptr) return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if (geometry_of(n, bucket, &g)) return fail(QD_ERR_INVALID_ARG, "bad geometry");
    int grid;
    int rc = capped_grid((n / 4 + kTileGroups - 1) / kTileGroups + 1, 8, &grid);
    if (rc) return rc;
    inv_scale_kernel<<<grid, 256, 0, as_stream(stream)>>>(y, out, alpha, beta, mean, g);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

// ------------------------------------------------------------------ a10 (extension, parity unpinned)
template <int MODE>
static int launch_abs(const AbsParams& P, cudaStream_t s) {
    DevInfo* di;
    int rc = dev_info(&di);
    if (rc) return rc;
    if (P.geo.row_len <= 1024) abs_rows_kernel<MODE, 32><<<di->grid((P.geo.rows + 7) / 8, 8), 256, 0, s>>>(P);
    else abs_rows_kernel<MODE, 256><<<di->grid(P.geo.rows, 8), 256, 0, s>>>(P);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

static int abs_common(AbsParams& P, const float* x, int64_t n, int64_t bucket, int kind, const float* mean, float max_element) {
    memset(&P, 0, sizeof(P));
    if (x == nullptr) return fail(QD_ERR_INVALID_ARG, "x is NULL");
    if (kind != QD_SCALE_ABSMAX && kind != QD_SCALE_ABSNORM) return fail(QD_ERR_INVALID_ARG, "unknown abs scaling kind %d", kind);
    if (geometry_of(n, bucket, &P.geo)) return fail(QD_ERR_INVALID_ARG, "bad geometry n=%lld bucket=%lld", (long long)n, (long long)bucket);
    P.x = x; P.kind = kind; P.mean = mean; P.max_element = max_element;
    return QD_OK;
}

extern "C" int qd_scale_down_abs(const float* x, float* xhat, float* sign, float* norm, int64_t n, int64_t bucket, int kind,
                                 const float* mean, float max_element, qd_stream_t stream) {
    AbsParams P;
    int rc = abs_common(P, x, n, bucket, kind, mean, max_element);
    if (rc) return rc;
    if (xhat == nullptr || norm == nullptr) return fail(QD_ERR_INVALID_ARG, "xhat and norm are required");
    P.out = xhat; P.sign = sign; P.norm = norm;
    return launch_abs<ABS_SCALE>(P, as_stream(stream));
}

extern "C" int qd_uniform_fwd_abs(const float* x, float* q, uint8_t* idx_u8, float* norm, int64_t n, int64_t bucket, int levels,
                                  int kind, const float* mean, float max_element, qd_stream_t stream) {
    AbsParams P;
    int rc = abs_common(P, x, n, bucket, kind, mean, max_element);
    if (rc) return rc;
    if (q == nullptr) return fail(QD_ERR_INVALID_ARG, "q is NULL");
    if (levels < 2) return fail(QD_ERR_INVALID_ARG, "levels (s) must be >= 2, got %d", levels);
    if (idx_u8 != nullptr && levels > 256) return fail(QD_ERR_INVALID_ARG, "idx_u8 needs levels <= 256");
    P.out = q; P.idx8 = idx_u8; P.norm = norm; P.S = (float)(levels - 1);
    return launch_abs<ABS_UNIFORM>(P, as_stream(stream));
}

extern "C" int qd_inv_scale_down_abs(const float* y, const float* sign, const float* norm, const float* mean, float* out,
                                     int64_t n, int64_t bucket, qd_stream_t stream) {
    Geometry g;
    if (y == nullptr || sign == nullptr || norm == nullptr || out == nullptr) return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if (geometry_of(n, bucket, &g)) return fail(QD_ERR_INVALID_ARG, "bad geometry");
    int grid;
    int rc = capped_grid((n + 255) / 256, 8, &grid);
    if (rc) return rc;
    abs_inv_scale_kernel<<<grid, 256, 0, as_stream(stream)>>>(y, sign, norm, mean, out, g);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

// ------------------------------------------------------------------ a4 / a5
static int uniform_common(Params& P, int64_t n, int64_t bucket, int levels) {
    if (levels < 2) return fail(QD_ERR_INVALID_ARG, "levels (s) must be >= 2, got %d", levels);
    if (geometry_of(n, bucket, &P.geo)) return fail(QD_ERR_INVALID_ARG, "bad geometry n=%lld bucket=%lld", (long long)n, (long long)bucket);
    P.S = (float)(levels - 1);
    P.rS = 1.0f / P.S;                                    // IEEE division on the host: RN(1/S)
    P.half_minus_band = 0.5f - P.S * 0x1p-20f;            // see qd_rowops.cuh "fast, still exact, level"
    return QD_OK;
}

extern "C" int qd_uniform_fwd(const float* x, float* q, uint8_t* idx_u8, float* alpha, float* beta, int64_t* argmin,
                              int64_t* argmax, int64_t n, int64_t bucket, int levels, const float* mean,
                              float max_element, int stochastic, uint64_t seed, uint64_t offset, void* workspace,
                              size_t workspace_bytes, qd_stream_t stream) {
    Params P = blank_params();
    if (x == nullptr || (q == nullptr && idx_u8 == nullptr)) return fail(QD_ERR_INVALID_ARG, "x and one of q / idx_u8 are required");
    if ((alpha == nullptr) != (beta == nullptr) || (argmin == nullptr) != (argmax == nullptr))
        return fail(QD_ERR_INVALID_ARG, "alpha/beta and argmin/argmax must be given in pairs");
    if (idx_u8 != nullptr && levels > 256) return fail(QD_ERR_INVALID_ARG, "idx_u8 needs levels <= 256");
    int rc = uniform_common(P, n, bucket, levels);
    if (rc) return rc;
    P.x = x; P.q = q; P.idx8 = idx_u8; P.alpha = alpha; P.beta = beta; P.argmin = argmin; P.argmax = argmax;
    P.mean = mean; P.max_element = max_element; P.stochastic = stochastic; P.seed = seed; P.offset = offset;
    if (stochastic) return run_rows<OP_UNIFORM_STOCH, BWD_OFF>(P, workspace, workspace_bytes, as_stream(stream));
    return run_rows<OP_UNIFORM, BWD_OFF>(P, workspace, workspace_bytes, as_stream(stream));
}

static int uniform_bwd_dispatch(Params& P, int mode, void* ws, size_t wsb, cudaStream_t s) {
    switch (mode) {
        case QD_BWD_STE: return run_rows<OP_UNIFORM, BWD_STE>(P, ws, wsb, s);
        case QD_BWD_TRUNCATED: return run_rows<OP_UNIFORM, BWD_TRUNC>(P, ws, wsb, s);
        case QD_BWD_MINMAX:
            if (P.geo.rows == 1 && P.geo.row_len == P.geo.n && P.geo.n > QD_MAX_STAGED_BUCKET)
                return fail(QD_ERR_UNSUPPORTED, "minmax backward needs a bucket size (quant_functions.py:332-334)");
            return run_rows<OP_UNIFORM, BWD_MINMAX>(P, ws, wsb, s);
        default: return fail(QD_ERR_INVALID_ARG, "unknown backward mode %d", mode);
    }
}

extern "C" int qd_uniform_bwd(const float* x, const float* g, float* gout, int64_t n, int64_t bucket, int levels,
                              int mode, void* workspace, size_t workspace_bytes, qd_stream_t stream) {
    Params P = blank_params();
    if (x == nullptr || g == nullptr || gout == nullptr) return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if (mode == QD_BWD_MINMAX && bucket == 0)
        return fail(QD_ERR_UNSUPPORTED, "minmax backward needs a bucket size (quant_functions.py:332-334)");
    int rc = uniform_common(P, n, bucket, levels);
    if (rc) return rc;
    cudaStream_t s = as_stream(stream);
    if (mode == QD_BWD_STE) {  // grad_input = grad_output
        if (gout != g) QD_CUDA(cudaMemcpyAsync(gout, g, (size_t)n * sizeof(float), cudaMemcpyDeviceToDevice, s));
        return QD_OK;
    }
    P.x = x; P.g = g; P.gout = gout;
    return uniform_bwd_dispatch(P, mode, workspace, workspace_bytes, s);
}

extern "C" int qd_uniform_fwd_bwd(const float* x, const float* g, float* q, float* gout, int64_t n, int64_t bucket,
                                  int levels, int mode, void* workspace, size_t workspace_bytes, qd_stream_t stream) {
    Params P = blank_params();
    if (x == nullptr || g == nullptr || q == nullptr || gout == nullptr) return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if (mode == QD_BWD_MINMAX && bucket == 0)
        return fail(QD_ERR_UNSUPPORTED, "minmax backward needs a bucket size (quant_functions.py:332-334)");
    int rc = uniform_common(P, n, bucket, levels);
    if (rc) return rc;
    P.x = x; P.g = g; P.q = q; P.gout = gout;
    return uniform_bwd_dispatch(P, mode, workspace, workspace_bytes, as_stream(stream));
}

// ------------------------------------------------------------------ a6 / a7 / a8
extern "C" int qd_nonuniform_fwd(const float* x, const float* points, int num_points, int rule, float* q,
                                 uint8_t* idx_u8, int64_t* idx_i64, float* alpha, float* beta, int64_t n,
                                 int64_t bucket, const float* mean, float max_element, void* workspace,
                                 size_t workspace_bytes, qd_stream_t stream) {
    Params P = blank_params();
    if (x == nullptr || points == nullptr) return fail(QD_ERR_INVALID_ARG, "x and points are required");
    if (q == nullptr && idx_u8 == nullptr && idx_i64 == nullptr) return fail(QD_ERR_INVALID_ARG, "no output requested");
    if (num_points < 1 || num_points > 256) return fail(QD_ERR_INVALID_ARG, "num_points must be in [1, 256], got %d", num_points);
    if (rule != QD_RULE_NEAREST && rule != QD_RULE_MIDPOINT) return fail(QD_ERR_INVALID_ARG, "unknown rule %d", rule);
    if ((alpha == nullptr) != (beta == nullptr)) return fail(QD_ERR_INVALID_ARG, "alpha/beta must be given in pairs");
    if (geometry_of(n, bucket, &P.geo)) return fail(QD_ERR_INVALID_ARG, "bad geometry n=%lld bucket=%lld", (long long)n, (long long)bucket);
    P.x = x; P.q = q; P.idx8 = idx_u8; P.idx64 = idx_i64; P.alpha = alpha; P.beta = beta;
    P.points = points; P.num_points = num_points; P.rule = rule; P.mean = mean; P.max_element = max_element;
    cudaStream_t s = as_stream(stream);
    if (P.geo.row_len <= 1024) {  // warp path: centroid tables of up to 32 points live in the lanes (AUX = table size class)
        const bool vec = rows_vectorizable(P);
        if (num_points <= 4) return launch_warp<OP_NONUNIFORM, 4>(P, vec, s);     // <= 32: table in the lanes (LaneSearch)
        if (num_points <= 8) return launch_warp<OP_NONUNIFORM, 8>(P, vec, s);
        if (num_points <= 16) return launch_warp<OP_NONUNIFORM, 16>(P, vec, s);
        if (num_points <= 32) return launch_warp<OP_NONUNIFORM, 32>(P, vec, s);
        if (num_points <= 64) return launch_warp<OP_NONUNIFORM, 64>(P, vec, s);   // unrolled search in shared memory
        return launch_warp<OP_NONUNIFORM, 256>(P, vec, s);
    }
    return run_rows<OP_NONUNIFORM, BWD_OFF>(P, workspace, workspace_bytes, s);
}

// per-tensor centroid gradient: the column scheme of qd_points_grad.cuh over one tensor
namespace qd {

template <typename IdxT>
__global__ void __launch_bounds__(kPgThreads) points_grad_partial(const float* __restrict__ g,
                                                                 const IdxT* __restrict__ idx,
                                                                 const float* __restrict__ alpha, int K, Geometry geo,
                                                                 double* __restrict__ partial /*[gridDim.x][K]*/) {
    __shared__ float s_col[kPgWarps][kPgSweep][32];
    extern __shared__ double s_acc[];  // [kPgWarps][K]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < kPgWarps * K; i += kPgThreads) s_acc[i] = 0.0;
    __syncthreads();
    float(*col)[32] = s_col[warp];

    // tile mode: 1024 consecutive elements of the flat tensor, alpha uniform per 128-element chunk
    const bool tile_mode = (geo.rows == 1) || (geo.row_len % 128 == 0);
    const int64_t tiles_per_row = (geo.row_len + kPgTile - 1) / kPgTile;
    const int64_t items = tile_mode ? (geo.n + kPgTile - 1) / kPgTile : geo.rows * tiles_per_row;
    const int64_t stride = (int64_t)gridDim.x * kPgWarps;
    // index minus sweep base, unsigned: negative indices and indices >= K fall outside [0, kcount) (int64: all 64 bits)
    using IdU = typename std::conditional<sizeof(IdxT) == 8, uint64_t, unsigned>::type;
    const bool vec_ok = sizeof(IdxT) == 1 && ((reinterpret_cast<uintptr_t>(g) & 15) == 0) &&
                        ((reinterpret_cast<uintptr_t>(idx) & 3) == 0);

    for (int kg = 0; kg < K; kg += kPgSweep) {
        const int kcount = min(kPgSweep, K - kg);
        for (int k = 0; k < kcount; ++k) col[k][lane] = 0.f;
        __syncwarp();
        int since_flush = 0;
        for (int64_t item = (int64_t)blockIdx.x * kPgWarps + warp; item < items; item += stride) {
            if (tile_mode) {
                const int64_t start = item * kPgTile;
                const int len = (int)min((int64_t)kPgTile, geo.n - start);
                if (vec_ok && len == kPgTile) {
                    float4 gv[8];
                    uint32_t iw[8];
#pragma unroll
                    for (int j = 0; j < 8; ++j) {  // all 16 loads in flight before the first use
                        gv[j] = ld_stream4(g + start + j * 128 + lane * 4);
                        iw[j] = *reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint8_t*>(idx) + start + j * 128 + lane * 4);
                    }
                    // row of each 128-element chunk: one division per tile, then increments
                    int64_t row = (geo.rows == 1) ? 0 : start / geo.row_len;
                    int64_t rem = (geo.rows == 1) ? 0 : start - row * geo.row_len;
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const float a = alpha[row];
                        if (geo.rows != 1) {
                            rem += 128;
                            if (rem >= geo.row_len) { rem -= geo.row_len; ++row; }
                        }
                        const float pv[4] = {__fmul_rn(gv[j].x, a), __fmul_rn(gv[j].y, a), __fmul_rn(gv[j].z, a),
                                             __fmul_rn(gv[j].w, a)};  // in-place multiply of the reference (:495)
#pragma unroll
                        for (int c = 0; c < 4; ++c) {
                            const unsigned id = ((iw[j] >> (8 * c)) & 0xffu) - (unsigned)kg;
                            if (id < (unsigned)kcount) col[id][lane] += pv[c];
                        }
                    }
                } else {
                    for (int e = lane; e < len; e += 32) {
                        const int64_t ge = start + e;
                        const float a = (geo.rows == 1) ? alpha[0] : alpha[ge / geo.row_len];
                        const IdU id = (IdU)idx[ge] - (IdU)kg;
                        if (id < (IdU)kcount) col[id][lane] += __fmul_rn(g[ge], a);
                    }
                }
            } else {
                const int64_t row = item / tiles_per_row, sub = item % tiles_per_row;
                const int64_t start = row * geo.row_len + sub * kPgTile;
                const int64_t row_end = min((row + 1) * geo.row_len, geo.n);
                const int len = (int)min((int64_t)kPgTile, row_end - start);
                const float a = alpha[row];
                for (int e = lane; e < len; e += 32) {
                    const IdU id = (IdU)idx[start + e] - (IdU)kg;
                    if (id < (IdU)kcount) col[id][lane] += __fmul_rn(g[start + e], a);
                }
            }
            if (++since_flush == kPgFlushEvery) {
                since_flush = 0;
                const double s = flush_column(col, lane, kcount);
                if (lane < kcount) s_acc[warp * K + kg + lane] += s;
            }
        }
        {
            const double s = flush_column(col, lane, kcount);
            if (lane < kcount) s_acc[warp * K + kg + lane] += s;
        }
        __syncwarp();
    }
    __syncthreads();
    for (int k = threadIdx.x; k < K; k += kPgThreads) {
        double s = 0.0;
        for (int w = 0; w < kPgWarps; ++w) s += s_acc[w * K + k];
        partial[(int64_t)blockIdx.x * K + k] = s;
    }
}

// one CTA per centroid: 256 threads stride over the CTA partials (a few loads each, all in flight), then a fixed
// tree (lanes by shuffle, warps in order).  One warp per centroid on ONE CTA serialised the fold into L2 round trips
// that took a visible share of the whole op at 64 Mi elements.
__global__ void __launch_bounds__(256) points_grad_final(const double* __restrict__ partial, int nblocks, int K,
                                                         float* __restrict__ out) {
    __shared__ double s_w[8];
    const int k = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double s = 0.0;
    for (int b = threadIdx.x; b < nblocks; b += 256) s += partial[(int64_t)b * K + k];
    s = warp_sum(s);
    if (lane == 0) s_w[warp] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < 8; ++w) t += s_w[w];
        out[k] = (float)t;
    }
}

}  // namespace qd

extern "C" int qd_nonuniform_bwd(const float* g, const uint8_t* idx_u8, const int64_t* idx_i64, const float* alpha,
                                 int num_points, float* grad_points, int64_t n, int64_t bucket, void* workspace,
                                 size_t workspace_bytes, qd_stream_t stream) {
    Geometry geo;
    if (g == nullptr || alpha == nullptr || grad_points == nullptr) return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if ((idx_u8 == nullptr) == (idx_i64 == nullptr)) return fail(QD_ERR_INVALID_ARG, "exactly one of idx_u8 / idx_i64 must be given");
    if (num_points < 1 || num_points > 256) return fail(QD_ERR_INVALID_ARG, "num_points must be in [1, 256], got %d", num_points);
    if (geometry_of(n, bucket, &geo)) return fail(QD_ERR_INVALID_ARG, "bad geometry");
    const int64_t items = (geo.n + kPgTile - 1) / kPgTile + geo.rows;  // upper bound of warp work items
    int grid;
    int rc = capped_grid((items + kPgWarps - 1) / kPgWarps, 8, &grid);
    if (rc) return rc;
    if (grid > (int)kPointsGradMaxCtas) grid = (int)kPointsGradMaxCtas;
    // the stated size, qd_workspace_bytes(n, bucket), not just the grid * K partials this launch uses: a caller
    // that sizes its buffer by some other rule is told so on every geometry, not only on the large ones
    const size_t need = workspace_bytes_of(geo);
    if (workspace == nullptr || workspace_bytes < need) return fail(QD_ERR_WORKSPACE, "workspace of %zu bytes needed, %zu given", need, workspace_bytes);
    double* partial = reinterpret_cast<double*>(workspace);
    cudaStream_t s = as_stream(stream);
    const size_t smem = (size_t)kPgWarps * num_points * sizeof(double);
    if (idx_u8)
        points_grad_partial<uint8_t><<<grid, kPgThreads, smem, s>>>(g, idx_u8, alpha, num_points, geo, partial);
    else
        points_grad_partial<int64_t><<<grid, kPgThreads, smem, s>>>(g, idx_i64, alpha, num_points, geo, partial);
    QD_CUDA(cudaGetLastError());
    points_grad_final<<<num_points, 256, 0, s>>>(partial, grid, num_points, grad_points);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

// index search on pre-scaled values (pre-processed path of the reference): 128-bit loads, lane-table search for
// K <= 32 (the loop runs the same number of times in every thread of a warp, so the shuffles are warp-uniform)
template <int KP>
__device__ __forceinline__ void centroid_index_body(const Centroids& cen, const float* s_k, const float* __restrict__ xhat, uint8_t* idx8,
                                                    int64_t* idx64, float* unit_out, int64_t n) {
    constexpr bool LANES = KP <= 32;
    LaneSearch<LANES ? KP : 1> ls;
    if constexpr (LANES) ls.load(cen, threadIdx.x & 31);
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const bool vec = ((reinterpret_cast<uintptr_t>(xhat) | reinterpret_cast<uintptr_t>(unit_out)) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(idx8) & 3) == 0;
    const int64_t groups = vec ? (n >> 2) : 0;
    for (int64_t base = (int64_t)blockIdx.x * blockDim.x; base < groups; base += stride) {
        const int64_t gi = base + threadIdx.x;
        const bool act = gi < groups;
        const float4 t = act ? ld_stream4(xhat + gi * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
        const float xv[4] = {t.x, t.y, t.z, t.w};
        int id[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if constexpr (LANES) id[j] = ls.index(xv[j]);
            else id[j] = padded_count<KP>(cen.t, xv[j]);
        }
        if (act) {
            if (idx8) *reinterpret_cast<uint32_t*>(idx8 + gi * 4) = (uint32_t)id[0] | ((uint32_t)id[1] << 8) | ((uint32_t)id[2] << 16) | ((uint32_t)id[3] << 24);
            if (idx64) { idx64[gi * 4] = id[0]; idx64[gi * 4 + 1] = id[1]; idx64[gi * 4 + 2] = id[2]; idx64[gi * 4 + 3] = id[3]; }
            if (unit_out) st_stream4(unit_out + gi * 4, make_float4(s_k[id[0]], s_k[id[1]], s_k[id[2]], s_k[id[3]]));
        }
    }
    for (int64_t i = groups * 4 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const int id = centroid_index(cen, xhat[i]);
        if (idx8) idx8[i] = (uint8_t)id;
        if (idx64) idx64[i] = id;
        if (unit_out) unit_out[i] = s_k[id];
    }
}

__global__ void __launch_bounds__(256) centroid_index_kernel(const float* __restrict__ xhat, const float* __restrict__ points,
                                                            int K, int rule, uint8_t* idx8, int64_t* idx64,
                                                            float* unit_out, int64_t n) {
    __shared__ float s_k[256];
    __shared__ float s_t[256];
    centroid_setup(s_k, s_t, points, K, rule);
    __syncthreads();
    Centroids cen{s_k, s_t, K};
    if (K <= 4) centroid_index_body<4>(cen, s_k, xhat, idx8, idx64, unit_out, n);
    else if (K <= 8) centroid_index_body<8>(cen, s_k, xhat, idx8, idx64, unit_out, n);
    else if (K <= 16) centroid_index_body<16>(cen, s_k, xhat, idx8, idx64, unit_out, n);
    else if (K <= 32) centroid_index_body<32>(cen, s_k, xhat, idx8, idx64, unit_out, n);
    else centroid_index_body<256>(cen, s_k, xhat, idx8, idx64, unit_out, n);
}

extern "C" int qd_centroid_index(const float* xhat, const float* points, int num_points, int rule, uint8_t* idx_u8,
                                 int64_t* idx_i64, float* unit_out, int64_t n, qd_stream_t stream) {
    if (xhat == nullptr || points == nullptr || n <= 0) return fail(QD_ERR_INVALID_ARG, "NULL argument or n <= 0");
    if (num_points < 1 || num_points > 256) return fail(QD_ERR_INVALID_ARG, "num_points must be in [1, 256], got %d", num_points);
    if (rule != QD_RULE_NEAREST && rule != QD_RULE_MIDPOINT) return fail(QD_ERR_INVALID_ARG, "unknown rule %d", rule);
    int grid;
    int rc = capped_grid((n / 4 + 255) / 256 + 1, 8, &grid);
    if (rc) return rc;
    centroid_index_kernel<<<grid, 256, 0, as_stream(stream)>>>(xhat, points, num_points, rule, idx_u8, idx_i64, unit_out, n);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

// ------------------------------------------------------------------ f2: quantize straight to packed codes
// The register warp path writes the packed stream itself (store_levels, qd_warp_path.cuh): 16-byte aligned rows of at
// most 1024 floats whose packed start is a whole byte, and a 4-byte aligned stream.  Every other layout runs the level
// kernel into the caller's workspace, then qd_pack_indices; the bytes are the same either way.
extern "C" size_t qd_packed_workspace_bytes(int64_t n, int64_t bucket) {
    const size_t ws = qd_workspace_bytes(n, bucket);
    return ws == 0 ? 0 : ((size_t)n + 255) / 256 * 256 + ws;
}

static bool packed_in_registers(const Params& P, int bits) {
    return P.geo.row_len <= 1024 && rows_vectorizable(P) && (reinterpret_cast<uintptr_t>(P.idx8) & 3) == 0 &&
           (P.geo.rows == 1 || (P.geo.row_len * bits) % 8 == 0);
}

// checks shared by both packed encoders; on success the fallback's uint8 levels and level-kernel scratch are split
// out of the workspace
static int packed_common(const float* x, uint8_t* packed, int bits, int symbols, const char* what, const float* alpha,
                         const float* beta, int64_t n, int64_t bucket, void* workspace, size_t workspace_bytes,
                         uint8_t** idx, void** ws_rest, size_t* ws_rest_bytes) {
    if (x == nullptr || packed == nullptr || alpha == nullptr || beta == nullptr) return fail(QD_ERR_INVALID_ARG, "x, packed, alpha and beta are required");
    if (!bits_ok(bits)) return fail(QD_ERR_INVALID_ARG, "bits must be 1, 2, 4 or 8");
    if (symbols < 1 || symbols > 256 || bits < bits_for(symbols))
        return fail(QD_ERR_INVALID_ARG, "%s = %d does not fit in %d-bit codes", what, symbols, bits);
    const size_t need = qd_packed_workspace_bytes(n, bucket);
    if (need == 0) return fail(QD_ERR_INVALID_ARG, "bad geometry n=%lld bucket=%lld", (long long)n, (long long)bucket);
    if (workspace == nullptr || workspace_bytes < need) return fail(QD_ERR_WORKSPACE, "workspace of %zu bytes needed, %zu given", need, workspace_bytes);
    const size_t idx_bytes = ((size_t)n + 255) / 256 * 256;
    *idx = static_cast<uint8_t*>(workspace);
    *ws_rest = static_cast<unsigned char*>(workspace) + idx_bytes;
    *ws_rest_bytes = workspace_bytes - idx_bytes;
    return QD_OK;
}

extern "C" int qd_uniform_fwd_packed(const float* x, uint8_t* packed, int bits, float* alpha, float* beta, int64_t n,
                                     int64_t bucket, int levels, void* workspace, size_t workspace_bytes, qd_stream_t stream) {
    uint8_t* idx;
    void* rest;
    size_t rest_bytes;
    if (levels < 2) return fail(QD_ERR_INVALID_ARG, "levels (s) must be >= 2, got %d", levels);
    int rc = packed_common(x, packed, bits, levels, "levels", alpha, beta, n, bucket, workspace, workspace_bytes, &idx, &rest, &rest_bytes);
    if (rc) return rc;
    Params P = blank_params();
    rc = uniform_common(P, n, bucket, levels);
    if (rc) return rc;
    P.x = x; P.idx8 = packed; P.alpha = alpha; P.beta = beta;
    cudaStream_t s = as_stream(stream);
    if (packed_in_registers(P, bits))
        return with_row_regs(P.geo.row_len, [&](auto r) {
            return with_bits(bits, [&](auto b) { return launch_warp_inst<OP_UNIFORM, BWD_OFF, decltype(r)::value, true, decltype(b)::value>(P, s); });
        });
    rc = qd_uniform_fwd(x, nullptr, idx, alpha, beta, nullptr, nullptr, n, bucket, levels, nullptr, 0.f, 0, 0, 0, rest, rest_bytes, stream);
    if (rc) return rc;
    return qd_pack_indices(idx, packed, n, bits, stream);
}

// smallest code width a centroid-table size class KP can need: KP = 4 holds K = 1 .. 4, every larger class K > KP / 2
template <int KP>
constexpr int kMinPackBits = KP <= 4 ? 1 : KP <= 16 ? 4 : 8;

extern "C" int qd_nonuniform_fwd_packed(const float* x, const float* points, int num_points, int rule, uint8_t* packed,
                                        int bits, float* alpha, float* beta, int64_t n, int64_t bucket, void* workspace,
                                        size_t workspace_bytes, qd_stream_t stream) {
    uint8_t* idx;
    void* rest;
    size_t rest_bytes;
    if (points == nullptr) return fail(QD_ERR_INVALID_ARG, "points is required");
    if (rule != QD_RULE_NEAREST && rule != QD_RULE_MIDPOINT) return fail(QD_ERR_INVALID_ARG, "unknown rule %d", rule);
    int rc = packed_common(x, packed, bits, num_points, "num_points", alpha, beta, n, bucket, workspace, workspace_bytes, &idx, &rest,
                           &rest_bytes);
    if (rc) return rc;
    Params P = blank_params();
    if (geometry_of(n, bucket, &P.geo)) return fail(QD_ERR_INVALID_ARG, "bad geometry n=%lld bucket=%lld", (long long)n, (long long)bucket);
    P.x = x; P.idx8 = packed; P.alpha = alpha; P.beta = beta;
    P.points = points; P.num_points = num_points; P.rule = rule;
    cudaStream_t s = as_stream(stream);
    if (packed_in_registers(P, bits)) {
        // same centroid-table classes as qd_nonuniform_fwd; widths below a class's smallest need are refused above
        auto go = [&](auto kp) {
            constexpr int KP = decltype(kp)::value;
            return with_row_regs(P.geo.row_len, [&](auto r) {
                return with_bits(bits, [&](auto b) {
                    constexpr int B = decltype(b)::value;
                    if constexpr (B >= kMinPackBits<KP>) return launch_warp_inst<OP_NONUNIFORM, KP, decltype(r)::value, true, B>(P, s);
                    else return fail(QD_ERR_INVALID_ARG, "%d points do not fit in %d-bit codes", num_points, B);
                });
            });
        };
        if (num_points <= 4) return go(std::integral_constant<int, 4>{});
        if (num_points <= 8) return go(std::integral_constant<int, 8>{});
        if (num_points <= 16) return go(std::integral_constant<int, 16>{});
        if (num_points <= 32) return go(std::integral_constant<int, 32>{});
        if (num_points <= 64) return go(std::integral_constant<int, 64>{});
        return go(std::integral_constant<int, 256>{});
    }
    rc = qd_nonuniform_fwd(x, points, num_points, rule, nullptr, idx, nullptr, alpha, beta, n, bucket, nullptr, 0.f, rest, rest_bytes, stream);
    if (rc) return rc;
    return qd_pack_indices(idx, packed, n, bits, stream);
}
