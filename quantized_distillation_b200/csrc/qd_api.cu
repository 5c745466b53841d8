// qd_api.cu -- host side of libqd_b200.so: argument checking, path selection
// and the extern "C" entry points declared in include/qd_b200.h.
//
// Path selection by row length L (= bucket, or n when bucket is None / n < bucket):
//     L <= 1024                  warp path    (registers, 1 HBM pass)
//     L <= QD_MAX_STAGED_BUCKET  staged path  (TMA chunk ring in shared memory, 1 HBM pass; CTA size by L)
//     otherwise                  grid path    (two streaming passes)
// Thresholds inside these ranges come from tools/block_bench.py (every variant forced through the tuning hook).
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdlib>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <unordered_map>
#include <vector>

#include "qd_abs_path.cuh"
#include "qd_block_path.cuh"
#include "qd_grid_path.cuh"
#include "qd_huffman.cuh"
#include "qd_plan.cuh"
#include "qd_points_grad.cuh"
#include "qd_select.cuh"
#include "qd_staged_path.cuh"
#include "qd_warp_path.cuh"

using namespace qd;

// ------------------------------------------------------------------ errors
static thread_local char g_err[512] = "";

static int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}
// same, for the other translation units of the library (qd_host.cu)
extern "C" int qd_internal_fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}
#define QD_CUDA(call)                                                                         \
    do {                                                                                      \
        cudaError_t e_ = (call);                                                              \
        if (e_ != cudaSuccess) return fail(QD_ERR_CUDA, "%s: %s", #call, cudaGetErrorString(e_)); \
    } while (0)

extern "C" int qd_version(void) { return 100; }
extern "C" const char* qd_last_error(void) { return g_err; }

// ------------------------------------------------------------------ device info
struct DevInfo {
    int sms = 0, major = 0, minor = 0;
    size_t smem_optin = 0;
};
static DevInfo g_dev[64];
static std::mutex g_mu;

static int dev_info(DevInfo** out) {
    int d = 0;
    QD_CUDA(cudaGetDevice(&d));
    if (d < 0 || d >= 64) return fail(QD_ERR_CUDA, "device ordinal %d out of range", d);
    std::lock_guard<std::mutex> lk(g_mu);
    if (g_dev[d].sms == 0) {
        int v = 0;
        QD_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, d)); g_dev[d].sms = v;
        QD_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMajor, d)); g_dev[d].major = v;
        QD_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMinor, d)); g_dev[d].minor = v;
        QD_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, d)); g_dev[d].smem_optin = (size_t)v;
    }
    *out = &g_dev[d];
    return QD_OK;
}

extern "C" int qd_device_info(int* sm_count, int* cc_major, int* cc_minor) {
    DevInfo* di;
    int rc = dev_info(&di);
    if (rc) return rc;
    if (sm_count) *sm_count = di->sms;
    if (cc_major) *cc_major = di->major;
    if (cc_minor) *cc_minor = di->minor;
    return QD_OK;
}

// resident CTAs per SM of a kernel, cached per (device, function)
static std::unordered_map<const void*, int> g_occ;
template <typename K>
static int resident_ctas(K kernel, int threads, size_t smem) {
    int d = 0;
    cudaGetDevice(&d);
    const void* key = reinterpret_cast<const void*>(reinterpret_cast<uintptr_t>(kernel) ^ ((uintptr_t)d << 56) ^ (smem << 20));
    {
        std::lock_guard<std::mutex> lk(g_mu);
        auto it = g_occ.find(key);
        if (it != g_occ.end()) return it->second;
    }
    int n = 1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, threads, smem) != cudaSuccess || n < 1) n = 1;
    std::lock_guard<std::mutex> lk(g_mu);
    g_occ[key] = n;
    return n;
}

// Opts a kernel instantiation into `smem` bytes of dynamic shared memory.  The attribute only ever grows (per
// instantiation and device: `opted` is that instantiation's own table) and changes under the library mutex, so two
// host threads launching the same instantiation with different row lengths can never lower it between the other
// thread's opt-in and its launch.
template <typename K>
static int opt_in_smem(K kernel, size_t smem, size_t* opted) {
    int d = 0;
    QD_CUDA(cudaGetDevice(&d));
    std::lock_guard<std::mutex> lk(g_mu);
    if (smem > opted[d & 63]) {
        QD_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        opted[d & 63] = smem;
    }
    return QD_OK;
}

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

extern "C" size_t qd_workspace_bytes(int64_t n, int64_t bucket) {
    Geometry g;
    if (geometry_of(n, bucket, &g)) return 0;
    size_t bytes = points_grad_ws_bytes();
    if (g.row_len > QD_MAX_STAGED_BUCKET) {
        size_t grid = (size_t)(g.rows * grid_chunks_per_row(g)) * sizeof(ChunkPartial) + (size_t)g.rows * sizeof(RowStat) + 256;
        if (grid > bytes) bytes = grid;
    }
    return bytes + 256;
}

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// ---- tuning hook (benchmarks only): -1 = built-in choice; keys are listed where they are used ----
static int64_t g_tune[8] = {-1, -1, -1, -1, -1, -1, -1, -1};
extern "C" int qd_debug_set_tuning(int key, int64_t value) {
    if (key < 0 || key >= 8) return fail(QD_ERR_INVALID_ARG, "unknown tuning key %d", key);
    g_tune[key] = value;
    return QD_OK;
}
extern "C" int64_t qd_internal_tuning(int key) { return (key >= 0 && key < 8) ? g_tune[key] : -1; }   // read by qd_host.cu

// ------------------------------------------------------------------ launchers
template <int OP, int BWD, int R, bool VEC>
static int launch_warp_inst(const Params& P, cudaStream_t s) {
    DevInfo* di;
    int rc = dev_info(&di);
    if (rc) return rc;
    auto kern = warp_rows_kernel<OP, BWD, R, VEC>;
    const int occ = resident_ctas(kern, kWarpCtaThreads, 0);
    int64_t need = (P.geo.rows + kWarpsPerCta - 1) / kWarpsPerCta;
    int64_t cap = (int64_t)di->sms * occ;
    int grid = (int)(need < cap ? need : cap);
    if constexpr (OP == OP_UNIFORM && BWD == (int)BWD_MINMAX) {
        // r_b accumulation, chosen by A/B (tools/headline_ab.py, 64 Mi floats): the fused forward+backward is faster
        // with one float64 add per element, the backward alone with the grouped lane sum.  So the variant follows the
        // presence of the q output (key 3: 1 forces the per-element sum, 0 the grouped one).
        const bool per_element = g_tune[3] >= 0 ? (g_tune[3] == 1) : (P.q != nullptr);
        if (per_element) {
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
    const int64_t L = P.geo.row_len;
    if (L <= 256) return vec ? launch_warp_inst<OP, BWD, 2, true>(P, s) : launch_warp_inst<OP, BWD, 2, false>(P, s);
    if (L <= 512) return vec ? launch_warp_inst<OP, BWD, 4, true>(P, s) : launch_warp_inst<OP, BWD, 4, false>(P, s);
    return vec ? launch_warp_inst<OP, BWD, 8, true>(P, s) : launch_warp_inst<OP, BWD, 8, false>(P, s);
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
        rc = opt_in_smem(kern, smem, opted);
        if (rc) return rc;
    }
    const int occ = resident_ctas(kern, kBlockCtaThreads, smem);
    constexpr int64_t rows_per_cta = kBlockCtaThreads / GROUP;
    int64_t need = (P.geo.rows + rows_per_cta - 1) / rows_per_cta;
    int64_t cap = (int64_t)di->sms * occ;
    int grid = (int)(need < cap ? need : cap);
    kern<<<grid, kBlockCtaThreads, smem, s>>>(P);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

// tuning keys of the block path:
//   key 0: longest row (floats) handled by the warp-per-row two-pass variant of the block path
//   key 1: longest row (floats) that keeps two rows in flight per CTA in the staged path
//   key 2: CTA size of the staged path (64 / 128 / 256 / 512 / 1024), 0 or -1 = by row length
//   key 3: 1 = headline kernel accumulates r_b with one float64 add per element (A/B measurement)

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
    rc = opt_in_smem(kern, smem, opted);
    if (rc) return rc;
    const int occ = resident_ctas(kern, T, smem);
    const int64_t cap = (int64_t)di->sms * occ;
    const int grid = (int)(P.geo.rows < cap ? P.geo.rows : cap);
    kern<<<grid, T, smem, s>>>(P, stage_floats);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

// CTA size and ring depth by row length (tools/block_bench.py, every variant forced through the tuning hook): 64
// threads below 2048 floats (a 1280-float row is five full steps of a 64-thread CTA, three ragged ones of a 128-thread
// CTA), 128 up to 3072, 256 up to 12288, 512 up to 24576, 1024 beyond; two rows in flight per CTA up to 3072 floats,
// the chunk ring alone above (on H100 one row in flight is as fast or faster for every op at 4096 floats, and the
// min/max backward gains most: fused 459 vs 526 us, alone 371 vs 429 us at 64 Mi floats).
// g_tune[1] = longest row with two rows in flight per CTA, g_tune[2] = forced CTA size.
template <int OP, int BWD>
static int launch_staged(const Params& P, cudaStream_t s) {
    const int64_t L = P.geo.row_len;
    const int64_t two_max = g_tune[1] >= 0 ? g_tune[1] : kTwoStageMaxRow;
    const bool two = L <= two_max && L <= 24576;
    int T = L < 2048 ? 64 : L <= 3072 ? 128 : L <= 12288 ? 256 : L <= 24576 ? 512 : 1024;
    if (g_tune[2] > 0) T = (int)g_tune[2];
    if (two) {
        if (T <= 64) return launch_staged_inst<OP, BWD, 2, 64>(P, s);
        if (T <= 128) return launch_staged_inst<OP, BWD, 2, 128>(P, s);
        if (T <= 256) return launch_staged_inst<OP, BWD, 2, 256>(P, s);
        return launch_staged_inst<OP, BWD, 2, 512>(P, s);
    }
    if (T <= 256) return launch_staged_inst<OP, BWD, 1, 256>(P, s);
    if (T <= 512) return launch_staged_inst<OP, BWD, 1, 512>(P, s);
    return launch_staged_inst<OP, BWD, 1, 1024>(P, s);
}

template <int OP, int BWD>
static int launch_block(const Params& P, cudaStream_t s) {
    // the staged ring wins or ties at every row length for the ops it implements (tools/block_bench.py);
    // the ops it does not implement (stats / scale / stochastic) keep the round-1 warp two-pass / whole-row staging
    constexpr bool kStagedOp = (OP == OP_UNIFORM || OP == OP_NONUNIFORM);
    const bool staged_ok = kStagedOp && !P.stochastic;
    // except the min/max backward on rows of 1025 .. 2048 floats, where the warp two-pass variant is faster on H100
    // (64 Mi floats: fused 460 vs 527 us at 1280 floats, 464 vs 531 us at 2048; backward alone 373 vs 409, 380 vs 407)
    constexpr bool kMinmax = OP == OP_UNIFORM && BWD == (int)BWD_MINMAX;
    const bool minmax_warp2 = kMinmax && staged_ok && P.geo.row_len > 1024 && P.geo.row_len <= kWarp2MinmaxMaxRow;
    const int64_t warp2_default = !staged_ok ? 2 * kWarpTwoPassMaxRow : minmax_warp2 ? kWarp2MinmaxMaxRow : 0;
    const int64_t warp2_max = g_tune[0] >= 0 ? g_tune[0] : warp2_default;
    if (P.geo.row_len <= warp2_max) return launch_block_inst<OP, BWD, false, 32>(P, s);               // warp per row, two passes
    if constexpr (kStagedOp) {
        if (staged_ok) return launch_staged<OP, BWD>(P, s);
    }
    return launch_block_inst<OP, BWD, true, kBlockCtaThreads>(P, s);  // scale / stats / stochastic: CTA per row, whole-row staging
}

template <int OP, int BWD>
static int launch_grid(const Params& P, void* ws, size_t ws_bytes, cudaStream_t s) {
    DevInfo* di;
    int rc = dev_info(&di);
    if (rc) return rc;
    const int64_t cpr = grid_chunks_per_row(P.geo);
    const int64_t items = P.geo.rows * cpr;
    const size_t need = (size_t)items * sizeof(ChunkPartial) + (size_t)P.geo.rows * sizeof(RowStat);
    if (ws == nullptr || ws_bytes < need) return fail(QD_ERR_WORKSPACE, "workspace of %zu bytes needed, %zu given", need, ws_bytes);
    ChunkPartial* partial = reinterpret_cast<ChunkPartial*>(ws);
    RowStat* rowstat = reinterpret_cast<RowStat*>(partial + items);
    const int64_t cap = (int64_t)di->sms * 4;
    const int grid = (int)(items < cap ? items : cap);
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

// longest row the register-resident warp path takes for (OP, BWD); set from tools/block_bench.py --small
template <int OP, int BWD>
static constexpr int64_t warp_path_max_row() { return 1024; }

template <int OP, int BWD>
static int run_rows(const Params& P, void* ws, size_t ws_bytes, cudaStream_t s) {
    if (P.geo.row_len >= (int64_t)1 << 31) return fail(QD_ERR_UNSUPPORTED, "rows of 2^31 elements or more are not supported");
    // longest row of the register-resident warp path (key 4 of the tuning hook moves the border for measurements)
    const int64_t warp_max = (g_tune[4] >= 0 && g_tune[4] <= 1024) ? g_tune[4] : warp_path_max_row<OP, BWD>();
    // ragged rows of 513..1023 floats with the min/max backward: the R = 8 register kernel runs its predicated
    // (non-FULL) variant at 128 registers there and loses to the staged ring (tools/block_bench.py --small);
    // everything else up to 1024 floats is faster in registers
    const bool ragged_minmax = OP == OP_UNIFORM && BWD == (int)BWD_MINMAX && P.geo.row_len > 512 && P.geo.row_len < 1024 && g_tune[4] < 0;
    if (P.geo.row_len <= warp_max && !ragged_minmax)
        return launch_warp<OP, (OP == OP_NONUNIFORM ? 256 : BWD)>(P, rows_vectorizable(P), s);
    // the CTA / grid paths keep stochastic rounding as a run-time branch of OP_UNIFORM
    constexpr int OP2 = (OP == OP_UNIFORM_STOCH) ? OP_UNIFORM : OP;
    if (P.geo.row_len <= QD_MAX_STAGED_BUCKET) return launch_block<OP2, BWD>(P, s);
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
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    if (xhat == nullptr) return run_rows<OP_STATS, BWD_OFF>(P, workspace, workspace_bytes, s);
    return run_rows<OP_SCALE, BWD_OFF>(P, workspace, workspace_bytes, s);
}

// Tiled helper kernels (inv_scale, pack, unpack): one CTA iteration = one contiguous tile of kTileGroups thread-groups,
// every thread owns kTileU groups of it, 256 groups apart, and issues all kTileU loads before the first use -- 64 B per
// thread in flight instead of 16 (Little: 132 SMs x 2048 threads x 16 B = 4.3 MB does not cover 3.35 TB/s x ~1.5 us).
constexpr int kTileU = 4;
constexpr int kTileGroups = 256 * kTileU;

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
    DevInfo* di;
    int rc = dev_info(&di);
    if (rc) return rc;
    int64_t need = (n / 4 + kTileGroups - 1) / kTileGroups + 1;
    int grid = (int)(need < (int64_t)di->sms * 8 ? need : (int64_t)di->sms * 8);
    inv_scale_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(y, out, alpha, beta, mean, g);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

// ------------------------------------------------------------------ a10 (extension, parity unpinned)
template <int MODE>
static int launch_abs(const AbsParams& P, cudaStream_t s) {
    DevInfo* di;
    int rc = dev_info(&di);
    if (rc) return rc;
    const int64_t cap = (int64_t)di->sms * 8;
    if (P.geo.row_len <= 1024) {
        const int64_t need = (P.geo.rows + 7) / 8;
        abs_rows_kernel<MODE, 32><<<(int)(need < cap ? need : cap), 256, 0, s>>>(P);
    } else {
        abs_rows_kernel<MODE, 256><<<(int)(P.geo.rows < cap ? P.geo.rows : cap), 256, 0, s>>>(P);
    }
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
    return launch_abs<ABS_SCALE>(P, reinterpret_cast<cudaStream_t>(stream));
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
    return launch_abs<ABS_UNIFORM>(P, reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int qd_inv_scale_down_abs(const float* y, const float* sign, const float* norm, const float* mean, float* out,
                                     int64_t n, int64_t bucket, qd_stream_t stream) {
    Geometry g;
    if (y == nullptr || sign == nullptr || norm == nullptr || out == nullptr) return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if (geometry_of(n, bucket, &g)) return fail(QD_ERR_INVALID_ARG, "bad geometry");
    DevInfo* di;
    int rc = dev_info(&di);
    if (rc) return rc;
    int64_t need = (n + 255) / 256;
    int grid = (int)(need < (int64_t)di->sms * 8 ? need : (int64_t)di->sms * 8);
    abs_inv_scale_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(y, sign, norm, mean, out, g);
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
    if (stochastic) return run_rows<OP_UNIFORM_STOCH, BWD_OFF>(P, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream));
    return run_rows<OP_UNIFORM, BWD_OFF>(P, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream));
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
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
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
    return uniform_bwd_dispatch(P, mode, workspace, workspace_bytes, reinterpret_cast<cudaStream_t>(stream));
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
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const int64_t warp_max = (g_tune[4] >= 0 && g_tune[4] <= 1024) ? g_tune[4] : warp_path_max_row<OP_NONUNIFORM, BWD_OFF>();
    if (P.geo.row_len <= warp_max) {  // warp path: centroid tables of up to 32 points live in the lanes (AUX = table size class)
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

extern "C" int qd_nonuniform_bwd(const float* g, const uint8_t* idx_u8, const int64_t* idx_i64, const float* alpha,
                                 int num_points, float* grad_points, int64_t n, int64_t bucket, void* workspace,
                                 size_t workspace_bytes, qd_stream_t stream) {
    Geometry geo;
    if (g == nullptr || alpha == nullptr || grad_points == nullptr) return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if ((idx_u8 == nullptr) == (idx_i64 == nullptr)) return fail(QD_ERR_INVALID_ARG, "exactly one of idx_u8 / idx_i64 must be given");
    if (num_points < 1 || num_points > 256) return fail(QD_ERR_INVALID_ARG, "num_points must be in [1, 256], got %d", num_points);
    if (geometry_of(n, bucket, &geo)) return fail(QD_ERR_INVALID_ARG, "bad geometry");
    DevInfo* di;
    int rc = dev_info(&di);
    if (rc) return rc;
    const int64_t items = (geo.n + kPgTile - 1) / kPgTile + geo.rows;  // upper bound of warp work items
    int64_t need_ctas = (items + kPgWarps - 1) / kPgWarps;
    int64_t cap = (int64_t)di->sms * 8;
    if (cap > (int64_t)kPointsGradMaxCtas) cap = kPointsGradMaxCtas;
    const int grid = (int)(need_ctas < cap ? need_ctas : cap);
    const size_t need = (size_t)grid * num_points * sizeof(double);
    if (workspace == nullptr || workspace_bytes < need) return fail(QD_ERR_WORKSPACE, "workspace of %zu bytes needed, %zu given", need, workspace_bytes);
    double* partial = reinterpret_cast<double*>(workspace);
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
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
    DevInfo* di;
    int rc = dev_info(&di);
    if (rc) return rc;
    int64_t need = (n / 4 + 255) / 256 + 1;
    int grid = (int)(need < (int64_t)di->sms * 8 ? need : (int64_t)di->sms * 8);
    centroid_index_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(xhat, points, num_points, rule, idx_u8,
                                                                                  idx_i64, unit_out, n);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

// ------------------------------------------------------------------ f2: histogram of indices
__global__ void __launch_bounds__(256) index_histogram_kernel(const uint8_t* __restrict__ idx, int64_t n, int bins,
                                                             unsigned long long* __restrict__ counts) {
    __shared__ unsigned int s_h[8][256];
    for (int i = threadIdx.x; i < 8 * 256; i += 256) (&s_h[0][0])[i] = 0u;
    __syncthreads();
    unsigned int* h = s_h[threadIdx.x >> 5];
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const bool vec = (reinterpret_cast<uintptr_t>(idx) & 15) == 0;
    const int64_t nv = vec ? (n >> 4) : 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += stride) {
        uint4 w = reinterpret_cast<const uint4*>(idx)[i];
        unsigned int ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int b = 0; b < 4; ++b) atomicAdd(&h[(ws[a] >> (8 * b)) & 0xffu], 1u);
    }
    for (int64_t i = nv * 16 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) atomicAdd(&h[idx[i]], 1u);
    __syncthreads();
    for (int b = threadIdx.x; b < bins; b += 256) {
        unsigned long long s = 0;
        for (int w = 0; w < 8; ++w) s += s_h[w][b];
        if (s) atomicAdd(&counts[b], s);
    }
}

extern "C" int qd_index_histogram(const uint8_t* idx_u8, int64_t n, int num_bins, int64_t* counts, qd_stream_t stream) {
    if (idx_u8 == nullptr || counts == nullptr || n <= 0) return fail(QD_ERR_INVALID_ARG, "NULL argument or n <= 0");
    if (num_bins < 1 || num_bins > 256) return fail(QD_ERR_INVALID_ARG, "num_bins must be in [1, 256]");
    DevInfo* di;
    int rc = dev_info(&di);
    if (rc) return rc;
    int64_t need = (n / 16 + 255) / 256 + 1;
    int grid = (int)(need < (int64_t)di->sms * 4 ? need : (int64_t)di->sms * 4);
    index_histogram_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        idx_u8, n, num_bins, reinterpret_cast<unsigned long long*>(counts));
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

// ------------------------------------------------------------------ f2: packed codec
// one thread-group = 16 consecutive codes in (one 128-bit load), 2*BITS bytes out (one store of that width); BITS is a
// template parameter so that every shift, mask and access width is a compile-time constant
template <int BITS>
__device__ __forceinline__ uint32_t squeeze4(uint32_t w) {  // four codes in four bytes -> 4*BITS bits
    constexpr unsigned mask = (1u << BITS) - 1u;
    return (w & mask) | (((w >> 8) & mask) << BITS) | (((w >> 16) & mask) << (2 * BITS)) | (((w >> 24) & mask) << (3 * BITS));
}

template <int BITS>
__global__ void __launch_bounds__(256) pack_kernel(const uint8_t* __restrict__ idx, uint8_t* __restrict__ packed, int64_t n) {
    const int64_t groups = (n + 15) / 16;
    const int64_t full = n / 16;   // groups with all sixteen codes present
    const int64_t tiles = (groups + kTileGroups - 1) / kTileGroups;
    const int64_t out_bytes = (n * BITS + 7) / 8;
    const bool in_vec = (reinterpret_cast<uintptr_t>(idx) & 15) == 0;
    const bool out_vec = (reinterpret_cast<uintptr_t>(packed) & 15) == 0;
    for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int64_t g0 = tile * kTileGroups + threadIdx.x;
        uint4 c[kTileU];
#pragma unroll
        for (int u = 0; u < kTileU; ++u) {
            const int64_t g = g0 + u * 256;
            if (in_vec && g < full) {
                c[u] = __ldcs(reinterpret_cast<const uint4*>(idx) + g);
            } else {
                uint32_t w[4] = {0u, 0u, 0u, 0u};
                if (g < groups)
                    for (int j = 0; j < 16; ++j)
                        if (g * 16 + j < n) w[j >> 2] |= (uint32_t)idx[g * 16 + j] << (8 * (j & 3));
                c[u] = make_uint4(w[0], w[1], w[2], w[3]);
            }
        }
#pragma unroll
        for (int u = 0; u < kTileU; ++u) {
            const int64_t g = g0 + u * 256;
            if (g >= groups) continue;
            // 16*BITS output bits, low codes first, as two 64-bit halves (the second one is only used for BITS = 8)
            unsigned long long lo, hi = 0;
            if constexpr (BITS == 8) {
                lo = (unsigned long long)c[u].x | ((unsigned long long)c[u].y << 32);
                hi = (unsigned long long)c[u].z | ((unsigned long long)c[u].w << 32);
            } else {
                lo = (unsigned long long)squeeze4<BITS>(c[u].x) | ((unsigned long long)squeeze4<BITS>(c[u].y) << (4 * BITS)) |
                     ((unsigned long long)squeeze4<BITS>(c[u].z) << (8 * BITS)) | ((unsigned long long)squeeze4<BITS>(c[u].w) << (12 * BITS));
            }
            uint8_t* dst = packed + g * (2 * BITS);
            if (out_vec && g < full) {
                if constexpr (BITS == 8) __stcs(reinterpret_cast<uint4*>(dst), make_uint4((uint32_t)lo, (uint32_t)(lo >> 32), (uint32_t)hi, (uint32_t)(hi >> 32)));
                else if constexpr (BITS == 4) __stcs(reinterpret_cast<unsigned long long*>(dst), lo);
                else if constexpr (BITS == 2) __stcs(reinterpret_cast<uint32_t*>(dst), (uint32_t)lo);
                else __stcs(reinterpret_cast<uint16_t*>(dst), (uint16_t)lo);
            } else {
                for (int b = 0; b < 2 * BITS; ++b)
                    if (g * (2 * BITS) + b < out_bytes) dst[b] = (uint8_t)((b < 8 ? lo >> (8 * b) : hi >> (8 * (b - 8))));
            }
        }
    }
}

extern "C" int qd_pack_indices(const uint8_t* idx_u8, uint8_t* packed, int64_t n, int bits, qd_stream_t stream) {
    if (idx_u8 == nullptr || packed == nullptr || n <= 0) return fail(QD_ERR_INVALID_ARG, "NULL argument or n <= 0");
    if (bits != 1 && bits != 2 && bits != 4 && bits != 8) return fail(QD_ERR_INVALID_ARG, "bits must be 1, 2, 4 or 8");
    DevInfo* di;
    int rc = dev_info(&di);
    if (rc) return rc;
    int64_t need = ((n + 15) / 16 + kTileGroups - 1) / kTileGroups;
    int grid = (int)(need < (int64_t)di->sms * 8 ? need : (int64_t)di->sms * 8);
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    if (bits == 8) pack_kernel<8><<<grid, 256, 0, s>>>(idx_u8, packed, n);
    else if (bits == 4) pack_kernel<4><<<grid, 256, 0, s>>>(idx_u8, packed, n);
    else if (bits == 2) pack_kernel<2><<<grid, 256, 0, s>>>(idx_u8, packed, n);
    else pack_kernel<1><<<grid, 256, 0, s>>>(idx_u8, packed, n);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

// one thread-group = FOUR consecutive elements: their codes are one aligned load of 4*BITS bits (a nibble for BITS = 1),
// the four dequantized values leave as one 128-bit store (a warp writes 512 contiguous bytes).  The unit value of a
// code comes from a 256-entry table in shared memory: c/S for the uniform scheme (the reference's division, done once
// per code instead of once per element), the centroid for the non-uniform one.
template <int BITS>
__device__ __forceinline__ uint32_t load_codes4(const uint8_t* __restrict__ packed, int64_t e0, int64_t in_bytes, bool ivec) {
    if constexpr (BITS == 8) {
        if (ivec && e0 + 4 <= in_bytes) return __ldcs(reinterpret_cast<const uint32_t*>(packed + e0));
        uint32_t word = 0;
        for (int b = 0; b < 4; ++b)
            if (e0 + b < in_bytes) word |= (uint32_t)packed[e0 + b] << (8 * b);
        return word;
    } else if constexpr (BITS == 4) {
        const int64_t b0 = e0 >> 1;
        if (ivec && b0 + 2 <= in_bytes) return __ldcs(reinterpret_cast<const uint16_t*>(packed + b0));
        uint32_t word = packed[b0];
        if (b0 + 1 < in_bytes) word |= (uint32_t)packed[b0 + 1] << 8;
        return word;
    } else if constexpr (BITS == 2) {
        return packed[e0 >> 2];
    } else {
        return (uint32_t)packed[e0 >> 3] >> (unsigned)(e0 & 4);
    }
}

// codes of group g (four elements) when the packed pointer is 4-byte aligned and the group is complete
template <int BITS>
__device__ __forceinline__ uint32_t load_codes4_fast(const uint8_t* __restrict__ packed, int64_t g) {
    if constexpr (BITS == 8) return __ldcs(reinterpret_cast<const uint32_t*>(packed) + g);
    else if constexpr (BITS == 4) return __ldcs(reinterpret_cast<const uint16_t*>(packed) + g);
    else if constexpr (BITS == 2) return __ldcs(packed + g);
    else return (uint32_t)__ldcs(packed + (g >> 1)) >> (unsigned)((g & 1) * 4);
}

template <bool UNIFORM, int BITS>
__global__ void __launch_bounds__(256, 4) unpack_dequant_kernel(const uint8_t* __restrict__ packed,
                                                            const float* __restrict__ points, int K,
                                                            const float* __restrict__ alpha, const float* __restrict__ beta,
                                                            float* __restrict__ q, Geometry geo, float S) {
    __shared__ float s_unit[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) {
        if (UNIFORM) s_unit[i] = ((float)i <= S) ? level_to_unit((float)i, S) : 0.f;
        else s_unit[i] = (i < K) ? points[i] : 0.f;
    }
    __syncthreads();
    const int64_t L = geo.row_len;
    const int64_t groups = (geo.n + 3) / 4;
    constexpr unsigned mask = (1u << BITS) - 1u;
    const bool single = geo.rows == 1;
    // fast tiles: complete tiles of kTileGroups groups, aligned pointers, the four elements of a group in one row, and
    // a row cursor that fits 32 bits (rows x row length beyond that only exist for buckets of < 32 floats on > 8 G
    // elements; they take the general loop below)
    const bool fast_ok = ((reinterpret_cast<uintptr_t>(q) & 15) == 0) && ((reinterpret_cast<uintptr_t>(packed) & 3) == 0) &&
                         (single || (L % 4 == 0 && L < (1ll << 30) && geo.rows < (1ll << 31)));
    const int64_t full_tiles = fast_ok ? geo.n / (kTileGroups * 4) : 0;
    if (full_tiles > (int64_t)blockIdx.x) {
        const uint32_t L32 = single ? 1u : (uint32_t)L;
        const int64_t e_first = ((int64_t)blockIdx.x * kTileGroups + threadIdx.x) * 4;
        int row = single ? 0 : (int)(e_first / L);
        uint32_t rem = single ? 0u : (uint32_t)(e_first % L);
        const int du_rows = single ? 0 : (int)((256 * 4) / L);
        const uint32_t du_rem = single ? 0u : (uint32_t)((256 * 4) % L);
        const int64_t dt = (int64_t)gridDim.x * kTileGroups * 4;
        const int dt_rows = single ? 0 : (int)(dt / L);
        const uint32_t dt_rem = single ? 0u : (uint32_t)(dt % L);
        // Everything a tile READS (codes, alpha, beta of its kTileU groups) is fetched one tile ahead: the stores of a
        // tile are asm volatile (no load moves across them), and under a store-dominated stream a read round trip is
        // several microseconds -- without the prefetch every group of four stores waited for its own alpha/beta read.
        struct Fetched { uint32_t w[kTileU]; float a[kTileU], b[kTileU]; };
        auto fetch = [&](int64_t tile, int r, uint32_t m, Fetched& f) {
            const int64_t g0 = tile * kTileGroups + threadIdx.x;
#pragma unroll
            for (int u = 0; u < kTileU; ++u) f.w[u] = load_codes4_fast<BITS>(packed, g0 + u * 256);
#pragma unroll
            for (int u = 0; u < kTileU; ++u) {
                f.a[u] = __ldg(alpha + r);
                f.b[u] = __ldg(beta + r);
                r += du_rows;
                m += du_rem;
                if (m >= L32) { m -= L32; ++r; }
            }
        };
        Fetched cur;
        fetch(blockIdx.x, row, rem, cur);
        for (int64_t tile = blockIdx.x; tile < full_tiles; tile += gridDim.x) {
            Fetched nxt = cur;
            row += dt_rows;
            rem += dt_rem;
            if (rem >= L32) { rem -= L32; ++row; }
            if (tile + gridDim.x < full_tiles) fetch(tile + gridDim.x, row, rem, nxt);
            float* dst = q + (tile * kTileGroups + threadIdx.x) * 4;
#pragma unroll
            for (int u = 0; u < kTileU; ++u) {
                float o[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) o[j] = from_unit(s_unit[(cur.w[u] >> (j * BITS)) & mask], cur.a[u], cur.b[u]);
                st_stream4(dst + u * 1024, make_float4(o[0], o[1], o[2], o[3]));
            }
            cur = nxt;
        }
    }
    // general loop: the last partial tile, unaligned pointers, ragged buckets
    const int64_t in_bytes = (geo.n * BITS + 7) / 8;
    const bool ivec = (reinterpret_cast<uintptr_t>(packed) & 3) == 0;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t g = full_tiles * kTileGroups + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += stride) {
        const int64_t e0 = g * 4;
        const uint32_t w = load_codes4<BITS>(packed, e0, in_bytes, ivec);
        for (int j = 0; j < 4; ++j) {
            if (e0 + j >= geo.n) break;
            const int64_t r = single ? 0 : (e0 + j) / L;
            q[e0 + j] = from_unit(s_unit[(w >> (j * BITS)) & mask], alpha[r], beta[r]);
        }
    }
}

static int unpack_common(const uint8_t* packed, int bits, const float* alpha, const float* beta, float* q, int64_t n,
                         int64_t bucket, Geometry* geo, int* grid) {
    if (packed == nullptr || alpha == nullptr || beta == nullptr || q == nullptr) return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if (bits != 1 && bits != 2 && bits != 4 && bits != 8) return fail(QD_ERR_INVALID_ARG, "bits must be 1, 2, 4 or 8");
    if (geometry_of(n, bucket, geo)) return fail(QD_ERR_INVALID_ARG, "bad geometry");
    DevInfo* di;
    int rc = dev_info(&di);
    if (rc) return rc;
    int64_t need = ((n + 3) / 4 + kTileGroups - 1) / kTileGroups;
    *grid = (int)(need < (int64_t)di->sms * 4 ? need : (int64_t)di->sms * 4);   // one resident wave (__launch_bounds__(256, 4))
    return QD_OK;
}

extern "C" int qd_unpack_dequant_uniform(const uint8_t* packed, int bits, const float* alpha, const float* beta, float* q,
                                         int64_t n, int64_t bucket, int levels, qd_stream_t stream) {
    Geometry geo;
    int grid = 0;
    if (levels < 2 || levels > (1 << bits)) return fail(QD_ERR_INVALID_ARG, "levels must be in [2, 2^bits]");
    int rc = unpack_common(packed, bits, alpha, beta, q, n, bucket, &geo, &grid);
    if (rc) return rc;
    const float S = (float)(levels - 1);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (bits == 8) unpack_dequant_kernel<true, 8><<<grid, 256, 0, st>>>(packed, nullptr, 0, alpha, beta, q, geo, S);
    else if (bits == 4) unpack_dequant_kernel<true, 4><<<grid, 256, 0, st>>>(packed, nullptr, 0, alpha, beta, q, geo, S);
    else if (bits == 2) unpack_dequant_kernel<true, 2><<<grid, 256, 0, st>>>(packed, nullptr, 0, alpha, beta, q, geo, S);
    else unpack_dequant_kernel<true, 1><<<grid, 256, 0, st>>>(packed, nullptr, 0, alpha, beta, q, geo, S);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

extern "C" int qd_unpack_dequant_nonuniform(const uint8_t* packed, int bits, const float* points, int num_points,
                                            const float* alpha, const float* beta, float* q, int64_t n, int64_t bucket,
                                            qd_stream_t stream) {
    Geometry geo;
    int grid = 0;
    if (points == nullptr || num_points < 1 || num_points > (1 << bits)) return fail(QD_ERR_INVALID_ARG, "num_points must be in [1, 2^bits]");
    int rc = unpack_common(packed, bits, alpha, beta, q, n, bucket, &geo, &grid);
    if (rc) return rc;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (bits == 8) unpack_dequant_kernel<false, 8><<<grid, 256, 0, st>>>(packed, points, num_points, alpha, beta, q, geo, 0.f);
    else if (bits == 4) unpack_dequant_kernel<false, 4><<<grid, 256, 0, st>>>(packed, points, num_points, alpha, beta, q, geo, 0.f);
    else if (bits == 2) unpack_dequant_kernel<false, 2><<<grid, 256, 0, st>>>(packed, points, num_points, alpha, beta, q, geo, 0.f);
    else unpack_dequant_kernel<false, 1><<<grid, 256, 0, st>>>(packed, points, num_points, alpha, beta, q, geo, 0.f);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

// ------------------------------------------------------------------ f2: Huffman-coded storage (qd_huffman.cuh)
extern "C" int qd_huffman_encode(const uint8_t* idx_u8, int64_t n, const qd_huffman_table* table, uint32_t* words_out,
                                 int64_t words_capacity, uint32_t* chunk_offsets, uint64_t* total_words, qd_stream_t stream) {
    if (idx_u8 == nullptr || table == nullptr || chunk_offsets == nullptr || total_words == nullptr || n <= 0)
        return fail(QD_ERR_INVALID_ARG, "NULL argument or n <= 0");
    if (words_capacity < 0 || (words_capacity > 0 && words_out == nullptr)) return fail(QD_ERR_INVALID_ARG, "bad words_out / capacity");
    DevInfo* di;
    int rc = dev_info(&di);
    if (rc) return rc;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const int64_t chunks = (n + kHuffChunk - 1) / kHuffChunk;
    const int64_t cap = (int64_t)di->sms * 8;
    const int64_t need1 = (chunks + 7) / 8;
    huff_chunk_words_kernel<<<(int)(need1 < cap ? need1 : cap), 256, 0, s>>>(idx_u8, n, table, chunk_offsets, chunks);
    huff_scan_kernel<<<1, 1024, 0, s>>>(chunk_offsets, chunks, reinterpret_cast<unsigned long long*>(total_words));
    const int64_t need2 = (chunks + kHuffEncWarps - 1) / kHuffEncWarps;
    if (words_capacity > 0)
        huff_encode_kernel<<<(int)(need2 < cap ? need2 : cap), kHuffEncWarps * 32, 0, s>>>(
            idx_u8, n, table, chunk_offsets, reinterpret_cast<const unsigned long long*>(total_words), chunks, words_out, words_capacity);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

static int huff_decode_common(const uint32_t* words, int64_t num_words, const uint32_t* chunk_offsets, const qd_huffman_table* table,
                              const float* alpha, const float* beta, float* q, int64_t n, int64_t bucket, Geometry* geo, int* grid) {
    if (chunk_offsets == nullptr || table == nullptr || alpha == nullptr || beta == nullptr || q == nullptr)
        return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if (num_words < 0 || (num_words > 0 && words == nullptr)) return fail(QD_ERR_INVALID_ARG, "bad words / num_words");
    if (geometry_of(n, bucket, geo)) return fail(QD_ERR_INVALID_ARG, "bad geometry");
    DevInfo* di;
    int rc = dev_info(&di);
    if (rc) return rc;
    const int64_t need = ((n + kHuffChunk - 1) / kHuffChunk + kHuffDecThreads - 1) / kHuffDecThreads;
    const int64_t cap = (int64_t)di->sms * 16;
    *grid = (int)(need < cap ? need : cap);
    return QD_OK;
}

extern "C" int qd_huffman_decode_dequant_uniform(const uint32_t* words, int64_t num_words, const uint32_t* chunk_offsets,
                                                 const qd_huffman_table* table, const float* alpha, const float* beta, float* q,
                                                 int64_t n, int64_t bucket, int levels, qd_stream_t stream) {
    Geometry geo;
    int grid = 0;
    if (levels < 2 || levels > 256) return fail(QD_ERR_INVALID_ARG, "levels must be in [2, 256]");
    int rc = huff_decode_common(words, num_words, chunk_offsets, table, alpha, beta, q, n, bucket, &geo, &grid);
    if (rc) return rc;
    huff_decode_dequant_kernel<true><<<grid, kHuffDecThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        words, num_words, chunk_offsets, table, nullptr, 0, alpha, beta, q, geo, (float)(levels - 1), (n + kHuffChunk - 1) / kHuffChunk);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

extern "C" int qd_huffman_decode_dequant_nonuniform(const uint32_t* words, int64_t num_words, const uint32_t* chunk_offsets,
                                                    const qd_huffman_table* table, const float* points, int num_points,
                                                    const float* alpha, const float* beta, float* q, int64_t n, int64_t bucket,
                                                    qd_stream_t stream) {
    Geometry geo;
    int grid = 0;
    if (points == nullptr || num_points < 1 || num_points > 256) return fail(QD_ERR_INVALID_ARG, "num_points must be in [1, 256]");
    int rc = huff_decode_common(words, num_words, chunk_offsets, table, alpha, beta, q, n, bucket, &geo, &grid);
    if (rc) return rc;
    huff_decode_dequant_kernel<false><<<grid, kHuffDecThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        words, num_words, chunk_offsets, table, points, num_points, alpha, beta, q, geo, 0.f, (n + kHuffChunk - 1) / kHuffChunk);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

// workspace of the model decode: the tensor array, then cta_start[count + 1] (int32)
static_assert(sizeof(qd_huffman_tensor) == 72 && sizeof(qd_huffman_tensor) % alignof(int32_t) == 0,
              "qd_huffman_tensor layout is shared with codec.py");

extern "C" size_t qd_huffman_model_workspace_bytes(int count) {
    return count < 1 ? 0 : (size_t)count * sizeof(qd_huffman_tensor) + ((size_t)count + 1) * sizeof(int32_t);
}

extern "C" int qd_huffman_decode_dequant_model(const qd_huffman_tensor* tensors, int count, const qd_huffman_table* table,
                                               int64_t bucket, int levels, void* workspace, size_t workspace_bytes,
                                               qd_stream_t stream) {
    if (tensors == nullptr || count < 1 || table == nullptr) return fail(QD_ERR_INVALID_ARG, "NULL tensors / table or count < 1");
    if (bucket < 0) return fail(QD_ERR_INVALID_ARG, "bucket must be >= 0");
    if (levels != 0 && (levels < 2 || levels > 256)) return fail(QD_ERR_INVALID_ARG, "levels must be in [2, 256] (uniform) or 0 (non-uniform)");
    const size_t need = qd_huffman_model_workspace_bytes(count);
    if (workspace == nullptr || (reinterpret_cast<uintptr_t>(workspace) & 15) || workspace_bytes < need)
        return fail(QD_ERR_WORKSPACE, "workspace must be 16-byte aligned and hold %zu bytes (got %zu)", need, workspace_bytes);
    const bool uniform = levels != 0;
    // host image of the workspace, consumed by the pageable copy before it returns (kept per thread: no allocation once grown)
    thread_local std::vector<unsigned char> image;
    image.resize(need);
    int32_t* cta_start = reinterpret_cast<int32_t*>(image.data() + (size_t)count * sizeof(qd_huffman_tensor));
    int64_t ctas = 0;
    for (int i = 0; i < count; ++i) {
        const qd_huffman_tensor& t = tensors[i];
        if (t.chunk_offsets == nullptr || t.alpha == nullptr || t.beta == nullptr || t.q == nullptr)
            return fail(QD_ERR_INVALID_ARG, "tensor %d: NULL argument", i);
        if (t.num_words < 0 || (t.num_words > 0 && t.words == nullptr)) return fail(QD_ERR_INVALID_ARG, "tensor %d: bad words / num_words", i);
        if (t.n < 1) return fail(QD_ERR_INVALID_ARG, "tensor %d: n must be >= 1", i);
        if (t.reserved != 0) return fail(QD_ERR_INVALID_ARG, "tensor %d: reserved must be 0", i);
        if (uniform && (t.points != nullptr || t.num_points != 0))
            return fail(QD_ERR_INVALID_ARG, "tensor %d: a uniform model has no points (points NULL, num_points 0)", i);
        if (!uniform && (t.points == nullptr || t.num_points < 1 || t.num_points > 256))
            return fail(QD_ERR_INVALID_ARG, "tensor %d: num_points must be in [1, 256]", i);
        cta_start[i] = (int32_t)ctas;
        ctas += ((t.n + kHuffChunk - 1) / kHuffChunk + kHuffDecThreads - 1) / kHuffDecThreads;
        if (ctas > INT32_MAX) return fail(QD_ERR_INVALID_ARG, "the model has more than 2^31 - 1 blocks of %d chunks", kHuffDecThreads);
    }
    cta_start[count] = (int32_t)ctas;
    memcpy(image.data(), tensors, (size_t)count * sizeof(qd_huffman_tensor));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    QD_CUDA(cudaMemcpyAsync(workspace, image.data(), need, cudaMemcpyHostToDevice, st));
    const qd_huffman_tensor* dev_tensors = static_cast<const qd_huffman_tensor*>(workspace);
    const int32_t* dev_start = reinterpret_cast<const int32_t*>(static_cast<const unsigned char*>(workspace) + (size_t)count * sizeof(qd_huffman_tensor));
    if (uniform)
        huff_decode_dequant_model_kernel<true><<<(unsigned)ctas, kHuffDecThreads, 0, st>>>(dev_tensors, dev_start, count, table, bucket,
                                                                                           (float)(levels - 1));
    else
        huff_decode_dequant_model_kernel<false><<<(unsigned)ctas, kHuffDecThreads, 0, st>>>(dev_tensors, dev_start, count, table, bucket, 0.f);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

// ------------------------------------------------------------------ plans (f1)
struct qd_plan {
    int count = 0;
    int64_t bucket = 0;
    int64_t total_rows = 0;
    int64_t max_row_len = 0;
    bool warp_path = true;
    bool has_shadow = false;
    bool has_momentum = false;
    std::vector<PlanEntry> host;
    PlanEntry* dev = nullptr;
    float** dev_grads = nullptr;  // count pointers, refreshed per backward call
    // bucket_size None: every tensor is one row -> the long-row plan (three launches for the whole model)
    bool long_path = false;
    std::vector<LongEntry> long_host;
    LongEntry* long_dev = nullptr;
    int64_t* long_chunk_starts = nullptr;
    int64_t* long_row_starts = nullptr;
    ChunkMinMax* long_partial = nullptr;
    RowScale* long_rowscale = nullptr;
    int64_t long_chunks = 0;
    void* workspace = nullptr;    // for tensors that need the grid path
    size_t workspace_bytes = 0;
    int device = 0;
};

extern "C" int qd_plan_create(qd_plan** out, int count, const float* const* src, float* const* dst, const int64_t* n,
                              const int32_t* levels, int64_t bucket) {
    if (out == nullptr || count <= 0 || src == nullptr || dst == nullptr || n == nullptr || levels == nullptr)
        return fail(QD_ERR_INVALID_ARG, "bad plan arguments");
    qd_plan* p = new qd_plan();
    p->count = count;
    p->bucket = bucket;
    p->host.resize(count);
    cudaGetDevice(&p->device);
    int64_t row = 0;
    size_t ws = 0;
    for (int i = 0; i < count; ++i) {
        Geometry g;
        if (geometry_of(n[i], bucket, &g) || levels[i] < 2 || src[i] == nullptr || dst[i] == nullptr) {
            delete p;
            return fail(QD_ERR_INVALID_ARG, "bad tensor %d in plan (n=%lld levels=%d)", i, (long long)n[i], levels[i]);
        }
        PlanEntry& e = p->host[i];
        e.src = src[i]; e.dst = dst[i]; e.save = nullptr; e.mom = nullptr; e.n = n[i]; e.row_start = row; e.rows = g.rows; e.row_len = g.row_len;
        e.S = (float)(levels[i] - 1);
        e.rS = 1.0f / e.S;
        e.lim = 0.5f - e.S * 0x1p-20f;
        e.vec = (aligned16(src[i]) && aligned16(dst[i]) && (g.rows == 1 || g.row_len % 4 == 0)) ? 1 : 0;
        row += g.rows;
        if (g.row_len > p->max_row_len) p->max_row_len = g.row_len;
        size_t w = qd_workspace_bytes(n[i], bucket);
        if (w > ws) ws = w;
    }
    p->total_rows = row;
    p->warp_path = p->max_row_len <= 1024;
    p->long_path = !p->warp_path && bucket == 0;
    if (p->long_path) {
        p->long_host.resize(count);
        std::vector<int64_t> cs(count), rs(count);
        int64_t chunk = 0;
        for (int i = 0; i < count; ++i) {
            const PlanEntry& pe = p->host[i];
            LongEntry& le = p->long_host[i];
            le.src = pe.src; le.dst = pe.dst; le.save = nullptr; le.n = pe.n; le.row_len = pe.row_len; le.rows = pe.rows;
            le.chunks_per_row = (pe.row_len + kPlanChunk - 1) / kPlanChunk;
            le.chunk_start = chunk; le.row_start = pe.row_start; le.S = pe.S; le.rS = pe.rS; le.lim = pe.lim;
            cs[i] = chunk; rs[i] = pe.row_start;
            chunk += le.chunks_per_row * pe.rows;
        }
        p->long_chunks = chunk;
        cudaError_t le_ = cudaMalloc(&p->long_dev, sizeof(LongEntry) * count);
        if (le_ == cudaSuccess) le_ = cudaMalloc(&p->long_chunk_starts, sizeof(int64_t) * count);
        if (le_ == cudaSuccess) le_ = cudaMalloc(&p->long_row_starts, sizeof(int64_t) * count);
        if (le_ == cudaSuccess) le_ = cudaMalloc(&p->long_partial, sizeof(ChunkMinMax) * (size_t)chunk);
        if (le_ == cudaSuccess) le_ = cudaMalloc(&p->long_rowscale, sizeof(RowScale) * (size_t)row);
        if (le_ == cudaSuccess) le_ = cudaMemcpy(p->long_dev, p->long_host.data(), sizeof(LongEntry) * count, cudaMemcpyHostToDevice);
        if (le_ == cudaSuccess) le_ = cudaMemcpy(p->long_chunk_starts, cs.data(), sizeof(int64_t) * count, cudaMemcpyHostToDevice);
        if (le_ == cudaSuccess) le_ = cudaMemcpy(p->long_row_starts, rs.data(), sizeof(int64_t) * count, cudaMemcpyHostToDevice);
        if (le_ != cudaSuccess) {
            qd_plan_destroy(p);
            return fail(QD_ERR_CUDA, "plan allocation: %s", cudaGetErrorString(le_));
        }
    }
    cudaError_t e = cudaMalloc(&p->dev, sizeof(PlanEntry) * count);
    if (e == cudaSuccess) e = cudaMalloc(&p->dev_grads, sizeof(float*) * count);
    if (e == cudaSuccess && !p->warp_path) { e = cudaMalloc(&p->workspace, ws); p->workspace_bytes = ws; }
    if (e == cudaSuccess) e = cudaMemcpy(p->dev, p->host.data(), sizeof(PlanEntry) * count, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        qd_plan_destroy(p);
        return fail(QD_ERR_CUDA, "plan allocation: %s", cudaGetErrorString(e));
    }
    *out = p;
    return QD_OK;
}

extern "C" int qd_plan_destroy(qd_plan* p) {
    if (p == nullptr) return QD_OK;
    if (p->dev) cudaFree(p->dev);
    if (p->dev_grads) cudaFree(p->dev_grads);
    if (p->workspace) cudaFree(p->workspace);
    if (p->long_dev) cudaFree(p->long_dev);
    if (p->long_chunk_starts) cudaFree(p->long_chunk_starts);
    if (p->long_row_starts) cudaFree(p->long_row_starts);
    if (p->long_partial) cudaFree(p->long_partial);
    if (p->long_rowscale) cudaFree(p->long_rowscale);
    delete p;
    return QD_OK;
}

// three launches for the whole model (qd_plan.cuh, "Long-row plan")
static int plan_long_forward(const qd_plan* p, int with_save, cudaStream_t s) {
    DevInfo* di;
    int rc = dev_info(&di);
    if (rc) return rc;
    const int64_t cap = (int64_t)di->sms * 4;
    const int grid = (int)(p->long_chunks < cap ? p->long_chunks : cap);
    plan_long_stats_partial<<<grid, kPlanChunkThreads, 0, s>>>(p->long_dev, p->count, p->long_chunk_starts, p->long_chunks, p->long_partial);
    plan_long_stats_final<<<(int)((p->total_rows + 7) / 8), 256, 0, s>>>(p->long_dev, p->count, p->long_row_starts, p->total_rows,
                                                                        p->long_partial, p->long_rowscale);
    plan_long_apply<BWD_OFF><<<grid, kPlanChunkThreads, 0, s>>>(p->long_dev, p->count, p->long_chunk_starts, p->long_chunks,
                                                               p->long_rowscale, with_save, nullptr);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

extern "C" int qd_plan_set_shadow(qd_plan* p, float* const* shadow) {
    if (p == nullptr || shadow == nullptr) return fail(QD_ERR_INVALID_ARG, "plan or shadow is NULL");
    for (int i = 0; i < p->count; ++i) {
        if (shadow[i] == nullptr) return fail(QD_ERR_INVALID_ARG, "shadow[%d] is NULL", i);
        p->host[i].save = shadow[i];
        if (p->long_path) p->long_host[i].save = shadow[i];
    }
    QD_CUDA(cudaMemcpy(p->dev, p->host.data(), sizeof(PlanEntry) * p->count, cudaMemcpyHostToDevice));
    if (p->long_path) QD_CUDA(cudaMemcpy(p->long_dev, p->long_host.data(), sizeof(LongEntry) * p->count, cudaMemcpyHostToDevice));
    p->has_shadow = true;
    return QD_OK;
}

extern "C" int qd_plan_set_momentum(qd_plan* p, float* const* momentum) {
    if (p == nullptr || momentum == nullptr) return fail(QD_ERR_INVALID_ARG, "plan or momentum is NULL");
    for (int i = 0; i < p->count; ++i) {
        if (momentum[i] == nullptr) return fail(QD_ERR_INVALID_ARG, "momentum[%d] is NULL", i);
        p->host[i].mom = momentum[i];
    }
    QD_CUDA(cudaMemcpy(p->dev, p->host.data(), sizeof(PlanEntry) * p->count, cudaMemcpyHostToDevice));
    p->has_momentum = true;
    return QD_OK;
}

template <int BWD>
static int plan_sgd_launch(const qd_plan* p, float* const* dev_grads, const GradTable& gt, const SgdParams& sp, cudaStream_t s) {
    DevInfo* di;
    int rc = dev_info(&di);
    if (rc) return rc;
    const int64_t need = (p->total_rows + kWarpsPerCta - 1) / kWarpsPerCta;
#define QD_SGD_LAUNCH(RR)                                                                          \
    {                                                                                              \
        auto kern = plan_sgd_step_kernel<BWD, RR>;                                                 \
        const int64_t cap = (int64_t)di->sms * resident_ctas(kern, kWarpCtaThreads, 0);            \
        const int grid = (int)(need < cap ? need : cap);                                           \
        kern<<<grid, kWarpCtaThreads, 0, s>>>(p->dev, p->count, p->total_rows, dev_grads, gt, sp); \
    }
    if (p->max_row_len <= 256) QD_SGD_LAUNCH(2)
    else QD_SGD_LAUNCH(4)
#undef QD_SGD_LAUNCH
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

extern "C" int qd_plan_sgd_step(const qd_plan* p, float* const* grad, int mode, double lr, double momentum,
                                double weight_decay, int nesterov, qd_stream_t stream) {
    if (p == nullptr || grad == nullptr) return fail(QD_ERR_INVALID_ARG, "plan or grad is NULL");
    if (!p->has_shadow || !p->has_momentum) return fail(QD_ERR_INVALID_ARG, "qd_plan_set_shadow and qd_plan_set_momentum must be called first");
    if (p->max_row_len > 512) return fail(QD_ERR_UNSUPPORTED, "fused optimizer step needs rows of at most 512 elements (plan has %lld)", (long long)p->max_row_len);
    if (mode == QD_BWD_MINMAX && p->bucket == 0)
        return fail(QD_ERR_UNSUPPORTED, "minmax backward needs a bucket size (quant_functions.py:332-334)");
    if (nesterov && !(momentum > 0.0)) return fail(QD_ERR_INVALID_ARG, "Nesterov momentum requires a momentum");   // torch.optim.SGD's own check
    for (int i = 0; i < p->count; ++i)
        if (grad[i] == nullptr) return fail(QD_ERR_INVALID_ARG, "grad[%d] is NULL", i);
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    SgdParams sp;
    sp.lr = (float)lr; sp.momentum = (float)momentum; sp.weight_decay = (float)weight_decay; sp.nesterov = nesterov ? 1 : 0;
    static const GradTable kEmpty = {};
    GradTable gt = {};
    float* const* dev_grads = nullptr;
    if (p->count <= kPlanGradsByValue) {
        for (int i = 0; i < p->count; ++i) gt.g[i] = grad[i];
    } else {
        QD_CUDA(cudaMemcpyAsync(p->dev_grads, grad, sizeof(float*) * p->count, cudaMemcpyHostToDevice, s));
        dev_grads = p->dev_grads;
    }
    const GradTable& g = dev_grads ? kEmpty : gt;
    switch (mode) {
        case QD_BWD_STE: return plan_sgd_launch<BWD_STE>(p, dev_grads, g, sp, s);
        case QD_BWD_TRUNCATED: return plan_sgd_launch<BWD_TRUNC>(p, dev_grads, g, sp, s);
        case QD_BWD_MINMAX: return plan_sgd_launch<BWD_MINMAX>(p, dev_grads, g, sp, s);
        default: return fail(QD_ERR_INVALID_ARG, "unknown backward mode %d", mode);
    }
}

template <int BWD>
static int plan_launch(const qd_plan* p, float* const* dev_grads, cudaStream_t s, int with_save = 0,
                       const GradTable* gtab = nullptr) {
    static const GradTable kEmpty = {};
    const GradTable& gt = gtab ? *gtab : kEmpty;
    DevInfo* di;
    int rc = dev_info(&di);
    if (rc) return rc;
    int64_t need = (p->total_rows + kWarpsPerCta - 1) / kWarpsPerCta;
#define QD_PLAN_LAUNCH(RR)                                                                        \
    {                                                                                             \
        auto kern = plan_rows_kernel<BWD, RR>;                                                    \
        int64_t cap = (int64_t)di->sms * resident_ctas(kern, kWarpCtaThreads, 0);                 \
        int grid = (int)(need < cap ? need : cap);                                                \
        kern<<<grid, kWarpCtaThreads, 0, s>>>(p->dev, p->count, p->total_rows, dev_grads, with_save, gt); \
    }
    if (p->max_row_len <= 256) QD_PLAN_LAUNCH(2)
    else if (p->max_row_len <= 512) QD_PLAN_LAUNCH(4)
    else QD_PLAN_LAUNCH(8)
#undef QD_PLAN_LAUNCH
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

extern "C" int qd_plan_uniform_fwd(const qd_plan* p, qd_stream_t stream) {
    if (p == nullptr) return fail(QD_ERR_INVALID_ARG, "plan is NULL");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    if (p->warp_path) return plan_launch<BWD_OFF>(p, nullptr, s);
    if (p->long_path) return plan_long_forward(p, 0, s);
    for (int i = 0; i < p->count; ++i) {  // buckets of 1025..49152: per-tensor block path
        const PlanEntry& e = p->host[i];
        int rc = qd_uniform_fwd(e.src, e.dst, nullptr, nullptr, nullptr, nullptr, nullptr, e.n, p->bucket, (int)e.S + 1,
                                nullptr, 0.f, 0, 0, 0, p->workspace, p->workspace_bytes, stream);
        if (rc) return rc;
    }
    return QD_OK;
}

extern "C" int qd_plan_uniform_fwd_save(const qd_plan* p, qd_stream_t stream) {
    if (p == nullptr) return fail(QD_ERR_INVALID_ARG, "plan is NULL");
    if (!p->has_shadow) return fail(QD_ERR_INVALID_ARG, "qd_plan_set_shadow has not been called");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    if (p->warp_path) return plan_launch<BWD_OFF>(p, nullptr, s, 1);
    if (p->long_path) return plan_long_forward(p, 1, s);
    for (int i = 0; i < p->count; ++i) {  // buckets of 1025..49152: copy, then the per-tensor block path
        const PlanEntry& e = p->host[i];
        QD_CUDA(cudaMemcpyAsync(e.save, e.src, (size_t)e.n * sizeof(float), cudaMemcpyDeviceToDevice, s));
    }
    return qd_plan_uniform_fwd(p, stream);
}

extern "C" int qd_plan_uniform_bwd(const qd_plan* p, float* const* grad, int mode, qd_stream_t stream) {
    if (p == nullptr || grad == nullptr) return fail(QD_ERR_INVALID_ARG, "plan or grad is NULL");
    if (mode == QD_BWD_STE) return QD_OK;  // identity
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    if (p->long_path) {
        if (mode == QD_BWD_MINMAX)
            return fail(QD_ERR_UNSUPPORTED, "minmax backward needs a bucket size (quant_functions.py:332-334)");
        if (mode != QD_BWD_TRUNCATED) return fail(QD_ERR_INVALID_ARG, "unknown backward mode %d", mode);
        DevInfo* di;
        int rc = dev_info(&di);
        if (rc) return rc;
        QD_CUDA(cudaMemcpyAsync(p->dev_grads, grad, sizeof(float*) * p->count, cudaMemcpyHostToDevice, s));
        const int64_t cap = (int64_t)di->sms * 4;
        const int grid = (int)(p->long_chunks < cap ? p->long_chunks : cap);
        plan_long_apply<BWD_TRUNC><<<grid, kPlanChunkThreads, 0, s>>>(p->long_dev, p->count, p->long_chunk_starts, p->long_chunks,
                                                                     p->long_rowscale, 0, p->dev_grads);
        QD_CUDA(cudaGetLastError());
        return QD_OK;
    }
    if (!p->warp_path) {
        for (int i = 0; i < p->count; ++i) {
            const PlanEntry& e = p->host[i];
            int rc = qd_uniform_bwd(e.src, grad[i], grad[i], e.n, p->bucket, (int)e.S + 1, mode, p->workspace,
                                    p->workspace_bytes, stream);
            if (rc) return rc;
        }
        return QD_OK;
    }
    if (mode == QD_BWD_MINMAX && p->bucket == 0)
        return fail(QD_ERR_UNSUPPORTED, "minmax backward needs a bucket size (quant_functions.py:332-334)");
    if (mode != QD_BWD_TRUNCATED && mode != QD_BWD_MINMAX) return fail(QD_ERR_INVALID_ARG, "unknown backward mode %d", mode);
    for (int i = 0; i < p->count; ++i)
        if (grad[i] == nullptr) return fail(QD_ERR_INVALID_ARG, "grad[%d] is NULL", i);
    if (p->count <= kPlanGradsByValue) {  // pointers ride in the launch parameters (graph-capturable)
        GradTable gt = {};
        for (int i = 0; i < p->count; ++i) gt.g[i] = grad[i];
        return mode == QD_BWD_TRUNCATED ? plan_launch<BWD_TRUNC>(p, nullptr, s, 0, &gt)
                                        : plan_launch<BWD_MINMAX>(p, nullptr, s, 0, &gt);
    }
    QD_CUDA(cudaMemcpyAsync(p->dev_grads, grad, sizeof(float*) * p->count, cudaMemcpyHostToDevice, s));
    if (mode == QD_BWD_TRUNCATED) return plan_launch<BWD_TRUNC>(p, p->dev_grads, s);
    if (mode == QD_BWD_MINMAX) return plan_launch<BWD_MINMAX>(p, p->dev_grads, s);
    return fail(QD_ERR_INVALID_ARG, "unknown backward mode %d", mode);
}

// ------------------------------------------------------------------ plan of the differentiable-quantization loop
struct qd_nu_plan {
    int count = 0;
    int64_t bucket = 0;
    int64_t total_rows = 0, max_row_len = 0, total_blocks = 0;
    int block_tiles = 1;
    std::vector<NuEntry> host;
    NuEntry* dev = nullptr;
    double* partial = nullptr;
    float** dev_grads = nullptr;
};

extern "C" int qd_plan_nonuniform_destroy(qd_nu_plan* p) {
    if (p == nullptr) return QD_OK;
    if (p->dev) cudaFree(p->dev);
    if (p->partial) cudaFree(p->partial);
    if (p->dev_grads) cudaFree(p->dev_grads);
    delete p;
    return QD_OK;
}

extern "C" int qd_plan_nonuniform_create(qd_nu_plan** out, int count, const float* const* src, float* const* dst,
                                         uint8_t* const* idx, float* const* alpha, float* const* beta,
                                         const float* const* points, float* const* grad_points, const int64_t* n,
                                         const int32_t* num_points, int64_t bucket) {
    if (out == nullptr || count <= 0 || !src || !dst || !idx || !alpha || !beta || !points || !grad_points || !n || !num_points)
        return fail(QD_ERR_INVALID_ARG, "bad plan arguments");
    qd_nu_plan* p = new qd_nu_plan();
    p->count = count;
    p->bucket = bucket;
    p->host.resize(count);
    int64_t row = 0, tiles = 0;
    for (int i = 0; i < count; ++i) {
        Geometry g;
        if (geometry_of(n[i], bucket, &g) || !src[i] || !dst[i] || !idx[i] || !alpha[i] || !beta[i] || !points[i] || !grad_points[i]) {
            delete p;
            return fail(QD_ERR_INVALID_ARG, "bad tensor %d in plan (n=%lld)", i, (long long)n[i]);
        }
        if (num_points[i] < 1 || num_points[i] > kNuMaxK || g.row_len > 1024) {
            delete p;
            return fail(QD_ERR_UNSUPPORTED, "plan of the centroid op needs 1..%d points and rows of at most 1024 elements "
                                            "(tensor %d: %d points, rows of %lld)", kNuMaxK, i, num_points[i], (long long)g.row_len);
        }
        NuEntry& e = p->host[i];
        e.src = src[i]; e.dst = dst[i]; e.idx = idx[i]; e.alpha = alpha[i]; e.beta = beta[i]; e.points = points[i];
        e.grad_points = grad_points[i]; e.n = n[i]; e.row_start = row; e.rows = g.rows; e.row_len = g.row_len; e.K = num_points[i];
        e.vec = (aligned16(src[i]) && aligned16(dst[i]) && ((reinterpret_cast<uintptr_t>(idx[i]) & 3) == 0) &&
                 (g.rows == 1 || g.row_len % 4 == 0)) ? 1 : 0;
        row += g.rows;
        tiles += (n[i] + kPgTile - 1) / kPgTile;
        if (g.row_len > p->max_row_len) p->max_row_len = g.row_len;
    }
    p->total_rows = row;
    // gradient blocks: enough of them to fill the machine, fixed for the life of the plan (determinism)
    int64_t bt = (tiles + 4735) / 4736;
    p->block_tiles = (int)(bt < 1 ? 1 : (bt > 16 ? 16 : bt));
    int64_t blk = 0;
    for (int i = 0; i < count; ++i) {
        NuEntry& e = p->host[i];
        const int64_t t = (e.n + kPgTile - 1) / kPgTile;
        e.blk_start = blk;
        e.blocks = (t + p->block_tiles - 1) / p->block_tiles;
        blk += e.blocks;
    }
    p->total_blocks = blk;
    cudaError_t e = cudaMalloc(&p->dev, sizeof(NuEntry) * count);
    if (e == cudaSuccess) e = cudaMalloc(&p->partial, sizeof(double) * kNuMaxK * (size_t)blk);
    if (e == cudaSuccess) e = cudaMalloc(&p->dev_grads, sizeof(float*) * count);
    if (e == cudaSuccess) e = cudaMemcpy(p->dev, p->host.data(), sizeof(NuEntry) * count, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        qd_plan_nonuniform_destroy(p);
        return fail(QD_ERR_CUDA, "plan allocation: %s", cudaGetErrorString(e));
    }
    *out = p;
    return QD_OK;
}

extern "C" int qd_plan_nonuniform_fwd(const qd_nu_plan* p, qd_stream_t stream) {
    if (p == nullptr) return fail(QD_ERR_INVALID_ARG, "plan is NULL");
    DevInfo* di;
    int rc = dev_info(&di);
    if (rc) return rc;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const int64_t need = (p->total_rows + kWarpsPerCta - 1) / kWarpsPerCta;
#define QD_NU_LAUNCH(RR)                                                                  \
    {                                                                                     \
        auto kern = plan_nonuniform_fwd_kernel<RR>;                                       \
        const int64_t cap = (int64_t)di->sms * resident_ctas(kern, kWarpCtaThreads, 0);   \
        const int grid = (int)(need < cap ? need : cap);                                  \
        kern<<<grid, kWarpCtaThreads, 0, s>>>(p->dev, p->count, p->total_rows);           \
    }
    if (p->max_row_len <= 256) QD_NU_LAUNCH(2)
    else if (p->max_row_len <= 512) QD_NU_LAUNCH(4)
    else QD_NU_LAUNCH(8)
#undef QD_NU_LAUNCH
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

extern "C" int qd_plan_nonuniform_bwd(const qd_nu_plan* p, const float* const* grad, qd_stream_t stream) {
    if (p == nullptr || grad == nullptr) return fail(QD_ERR_INVALID_ARG, "plan or grad is NULL");
    for (int i = 0; i < p->count; ++i)
        if (grad[i] == nullptr) return fail(QD_ERR_INVALID_ARG, "grad[%d] is NULL", i);
    DevInfo* di;
    int rc = dev_info(&di);
    if (rc) return rc;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const int64_t need = (p->total_blocks + kPgWarps - 1) / kPgWarps;
    const int64_t cap = (int64_t)di->sms * 4;
    const int grid = (int)(need < cap ? need : cap);
    if (p->count <= kPlanGradsByValue) {  // pointers ride in the launch parameters (graph-capturable)
        GradTable gt = {};
        for (int i = 0; i < p->count; ++i) gt.g[i] = const_cast<float*>(grad[i]);
        plan_points_grad_partial<0><<<grid, kPgThreads, 0, s>>>(p->dev, p->count, p->total_blocks, p->block_tiles, gt, nullptr, p->partial);
    } else {
        static const GradTable kEmpty = {};
        QD_CUDA(cudaMemcpyAsync(p->dev_grads, grad, sizeof(float*) * p->count, cudaMemcpyHostToDevice, s));
        plan_points_grad_partial<0><<<grid, kPgThreads, 0, s>>>(p->dev, p->count, p->total_blocks, p->block_tiles, kEmpty, p->dev_grads, p->partial);
    }
    QD_CUDA(cudaGetLastError());
    plan_points_grad_final<<<(p->count + 7) / 8, 256, 0, s>>>(p->dev, p->count, p->partial);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

// ------------------------------------------------------------------ f3: order statistics / multi-tensor norms
static size_t select_header_bytes() {
    size_t h = sizeof(unsigned long long) * kSelBins + sizeof(SelectState);
    return (h + 255) & ~(size_t)255;
}
extern "C" size_t qd_order_statistics_workspace_bytes(int64_t n) {
    return n > 0 ? select_header_bytes() + (size_t)n * sizeof(uint32_t) : 0;
}

extern "C" int qd_order_statistics(const float* v, int64_t n, const int64_t* ranks, int num_ranks, float* out,
                                   void* workspace, size_t workspace_bytes, qd_stream_t stream) {
    if (v == nullptr || ranks == nullptr || out == nullptr || n <= 0) return fail(QD_ERR_INVALID_ARG, "NULL argument or n <= 0");
    if (num_ranks < 1 || num_ranks > kSelMaxRanks) return fail(QD_ERR_INVALID_ARG, "num_ranks must be in [1, %d]", kSelMaxRanks);
    if (workspace == nullptr || workspace_bytes < qd_order_statistics_workspace_bytes(n))
        return fail(QD_ERR_WORKSPACE, "workspace of %zu bytes needed, %zu given", qd_order_statistics_workspace_bytes(n), workspace_bytes);
    DevInfo* di;
    int rc = dev_info(&di);
    if (rc) return rc;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    unsigned long long* hist = reinterpret_cast<unsigned long long*>(workspace);
    SelectState* st = reinterpret_cast<SelectState*>(hist + kSelBins);
    uint32_t* buf = reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(workspace) + select_header_bytes());
    QD_CUDA(cudaMemsetAsync(hist, 0, sizeof(unsigned long long) * kSelBins, s));
    const int64_t need = (n / 4 + kSelThreads - 1) / kSelThreads + 1;
    const int grid = (int)(need < (int64_t)di->sms * 4 ? need : (int64_t)di->sms * 4);
    select_hist_kernel<<<grid, kSelThreads, 0, s>>>(v, n, hist);
    select_plan_kernel<<<1, kSelThreads, 0, s>>>(hist, ranks, num_ranks, st);
    select_compact_kernel<<<grid, kSelThreads, 0, s>>>(v, n, st, buf);
    select_final_kernel<<<num_ranks, kSelThreads, 0, s>>>(st, buf, out);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

extern "C" int qd_multi_l2norm(const float* const* tensors, const int64_t* n, int count, float* out, qd_stream_t stream) {
    if (tensors == nullptr || n == nullptr || out == nullptr || count <= 0) return fail(QD_ERR_INVALID_ARG, "bad arguments");
    DevInfo* di;
    int rc = dev_info(&di);
    if (rc) return rc;
    std::vector<NormEntry> host(count);
    int64_t chunks = 0;
    for (int i = 0; i < count; ++i) {
        if (tensors[i] == nullptr || n[i] <= 0) return fail(QD_ERR_INVALID_ARG, "bad tensor %d", i);
        host[i].ptr = tensors[i]; host[i].n = n[i]; host[i].chunk_start = chunks;
        host[i].chunks = (n[i] + kNormChunk - 1) / kNormChunk;
        chunks += host[i].chunks;
    }
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    NormEntry* dev = nullptr;
    double* partial = nullptr;
    // setup-time call (once per bit allocation): stream-ordered scratch, table copied before the launch
    QD_CUDA(cudaMallocAsync(&dev, sizeof(NormEntry) * count, s));
    QD_CUDA(cudaMallocAsync(&partial, sizeof(double) * (size_t)chunks, s));
    QD_CUDA(cudaMemcpyAsync(dev, host.data(), sizeof(NormEntry) * count, cudaMemcpyHostToDevice, s));
    QD_CUDA(cudaStreamSynchronize(s));   // `host` goes out of scope; this entry point is not on the per-step path
    const int64_t cap = (int64_t)di->sms * 8;
    multi_norm_partial<<<(int)(chunks < cap ? chunks : cap), 256, 0, s>>>(dev, count, chunks, partial);
    multi_norm_final<<<(count + 255) / 256, 256, 0, s>>>(dev, count, partial, out);
    QD_CUDA(cudaGetLastError());
    QD_CUDA(cudaFreeAsync(dev, s));
    QD_CUDA(cudaFreeAsync(partial, s));
    return QD_OK;
}

// ------------------------------------------------------------------ self test
// Checks the float32 pipeline pieces on device against double arithmetic where
// double rounding cannot occur: quotient in [0,1] of 24-bit operands.
__global__ void selftest_division_kernel(int64_t pairs, uint64_t seed, unsigned long long* mismatches) {
    Philox rng(seed);
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < pairs; i += stride) {
        uint4 r = rng((uint64_t)i);
        float d = __uint_as_float((r.x & 0x007fffffu) | (((r.y % 60u) + 97u) << 23));  // 2^-30 .. 2^29
        float frac = u01(r.z);
        float a = __fmul_rn(d, frac);
        float q = __fdiv_rn(a, d);
        double qd = (double)a / (double)d;  // exact to 53 bits; rounding to 24 is then correct
        float qr = (float)qd;               // unless qd sits within 2^-29 rel. of a tie (never for 24-bit a, d)
        if (q != qr) atomicAdd(mismatches, 1ull);
        // hoisted-reciprocal division used by the kernels, incl. its guard and slow path
        const RowDivider div(d);
        if (div.exact(a) != q) atomicAdd(mismatches, 1ull);
        float tiny = __fmul_rn(a, (r.w & 1u) ? 0x1p-28f : 0x1p-33f);  // around and below the guard threshold
        if (div.exact(tiny) != __fdiv_rn(tiny, d)) atomicAdd(mismatches, 1ull);
        // level / S for S <= 255
        const float S = (float)(1u + (r.w >> 8) % 255u), k = (float)((r.w >> 16) % ((unsigned)S + 1u));
        if (small_level_to_unit(k, S, __fdiv_rn(1.0f, S)) != __fdiv_rn(k, S)) atomicAdd(mismatches, 1ull);
    }
}

extern "C" int qd_selftest_division(int64_t pairs, uint64_t seed, int64_t* mismatches, qd_stream_t stream) {
    unsigned long long* d = nullptr;
    QD_CUDA(cudaMalloc(&d, sizeof(unsigned long long)));
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    QD_CUDA(cudaMemsetAsync(d, 0, sizeof(unsigned long long), s));
    selftest_division_kernel<<<1184, 256, 0, s>>>(pairs, seed, d);
    unsigned long long h = 0;
    QD_CUDA(cudaMemcpyAsync(&h, d, sizeof(h), cudaMemcpyDeviceToHost, s));
    QD_CUDA(cudaStreamSynchronize(s));
    QD_CUDA(cudaFree(d));
    if (mismatches) *mismatches = (int64_t)h;
    return QD_OK;
}
