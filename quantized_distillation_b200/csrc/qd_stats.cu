// qd_stats.cu -- entry points of the setup reductions (qd_select.cuh): exact order statistics and multi-tensor L2
// norms; and the device self-test of the division helpers.
#include <vector>

#include "qd_launch.h"
#include "qd_select.cuh"

using namespace qd;

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
    int grid;
    int rc = capped_grid((n / 4 + kSelThreads - 1) / kSelThreads + 1, 4, &grid);
    if (rc) return rc;
    cudaStream_t s = as_stream(stream);
    unsigned long long* hist = reinterpret_cast<unsigned long long*>(workspace);
    SelectState* st = reinterpret_cast<SelectState*>(hist + kSelBins);
    uint32_t* buf = reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(workspace) + select_header_bytes());
    QD_CUDA(cudaMemsetAsync(hist, 0, sizeof(unsigned long long) * kSelBins, s));
    select_hist_kernel<<<grid, kSelThreads, 0, s>>>(v, n, hist);
    select_plan_kernel<<<1, kSelThreads, 0, s>>>(hist, ranks, num_ranks, st);
    select_compact_kernel<<<grid, kSelThreads, 0, s>>>(v, n, st, buf);
    select_final_kernel<<<num_ranks, kSelThreads, 0, s>>>(st, buf, out);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

extern "C" int qd_multi_l2norm(const float* const* tensors, const int64_t* n, int count, float* out, qd_stream_t stream) {
    if (tensors == nullptr || n == nullptr || out == nullptr || count <= 0) return fail(QD_ERR_INVALID_ARG, "bad arguments");
    std::vector<NormEntry> host(count);
    int64_t chunks = 0;
    for (int i = 0; i < count; ++i) {
        if (tensors[i] == nullptr || n[i] <= 0) return fail(QD_ERR_INVALID_ARG, "bad tensor %d", i);
        host[i].ptr = tensors[i]; host[i].n = n[i]; host[i].chunk_start = chunks;
        host[i].chunks = (n[i] + kNormChunk - 1) / kNormChunk;
        chunks += host[i].chunks;
    }
    int grid;
    int rc = capped_grid(chunks, 8, &grid);
    if (rc) return rc;
    cudaStream_t s = as_stream(stream);
    NormEntry* dev = nullptr;
    double* partial = nullptr;
    // setup-time call (once per bit allocation): stream-ordered scratch, table copied before the launch
    QD_CUDA(cudaMallocAsync(&dev, sizeof(NormEntry) * count, s));
    QD_CUDA(cudaMallocAsync(&partial, sizeof(double) * (size_t)chunks, s));
    QD_CUDA(cudaMemcpyAsync(dev, host.data(), sizeof(NormEntry) * count, cudaMemcpyHostToDevice, s));
    QD_CUDA(cudaStreamSynchronize(s));   // `host` goes out of scope; this entry point is not on the per-step path
    multi_norm_partial<<<grid, 256, 0, s>>>(dev, count, chunks, partial);
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
    cudaStream_t s = as_stream(stream);
    QD_CUDA(cudaMemsetAsync(d, 0, sizeof(unsigned long long), s));
    selftest_division_kernel<<<1184, 256, 0, s>>>(pairs, seed, d);
    unsigned long long h = 0;
    QD_CUDA(cudaMemcpyAsync(&h, d, sizeof(h), cudaMemcpyDeviceToHost, s));
    QD_CUDA(cudaStreamSynchronize(s));
    QD_CUDA(cudaFree(d));
    if (mismatches) *mismatches = (int64_t)h;
    return QD_OK;
}
