// qd_host.cu -- host-buffer entry points: what a caller holding CPU tensors
// gets (the reference's functions accept CPU tensors; here the arithmetic still
// runs on the GPU).  The tensor is cut into row-aligned chunks and each chunk
// travels H2D -> fused kernel -> D2H on one of three streams, so the two PCIe
// directions and the kernel overlap; end-to-end time is bounded by the slower
// PCIe direction, not by their sum.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <mutex>

#include "qd_launch.h"

using qd::fail;

namespace {

// pipeline depth and chunk size: three slots of 8-16 MiB per buffer sit on the plateau of the sweeps (slots and chunk
// sizes forced through a since-removed tuning hook: slots beyond 2 and chunks beyond 16 MiB changed nothing)
constexpr int kSlots = 3;
constexpr int64_t kChunkElems = 4 << 20;
constexpr int64_t kDirectMaxElems = 8 << 20;   // largest tensor run as ONE launch on pinned host pointers

struct Slot {
    cudaStream_t stream = nullptr;
    float *x = nullptr, *g = nullptr, *q = nullptr, *gout = nullptr;
    void* ws = nullptr;
    size_t ws_bytes = 0;
};

struct HostCtx {
    int slots = 0;              // allocated slots
    int64_t chunk_cap = 0;      // their capacity in elements
    Slot slot[kSlots];
    float *big_x = nullptr, *big_g = nullptr, *big_q = nullptr, *big_gout = nullptr;  // bucket=None path
    int64_t big_cap = 0;
    void* big_ws = nullptr;
    size_t big_ws_bytes = 0;
};

HostCtx g_ctx[64];
std::mutex g_mu[64];  // one lock per device: callers on different GPUs never wait for each other

// the caller's current device is put back when the call returns, whatever the path
struct DeviceGuard {
    int prev = -1;
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

int ensure_ctx(int device, int64_t chunk_elems, HostCtx** out) {
    HostCtx& c = g_ctx[device];
    if (c.slots < kSlots || c.chunk_cap < chunk_elems) {
        for (int i = 0; i < c.slots; ++i) {
            Slot& s = c.slot[i];
            cudaFree(s.x); cudaFree(s.g); cudaFree(s.q); cudaFree(s.gout); cudaFree(s.ws);
            s.x = s.g = s.q = s.gout = nullptr;
            s.ws = nullptr;
        }
        c.slots = 0;
        c.chunk_cap = 0;
        for (int i = 0; i < kSlots; ++i) {
            Slot& s = c.slot[i];
            if (s.stream == nullptr) QD_CUDA(cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking));
            const size_t bytes = (size_t)chunk_elems * sizeof(float);
            QD_CUDA(cudaMalloc(&s.x, bytes));
            QD_CUDA(cudaMalloc(&s.g, bytes));
            QD_CUDA(cudaMalloc(&s.q, bytes));
            QD_CUDA(cudaMalloc(&s.gout, bytes));
            s.ws_bytes = qd_workspace_bytes(chunk_elems, 0);
            QD_CUDA(cudaMalloc(&s.ws, s.ws_bytes));
        }
        c.slots = kSlots;
        c.chunk_cap = chunk_elems;
    }
    *out = &c;
    return QD_OK;
}

int run_host(const float* hx, const float* hg, float* hq, float* hgout, int64_t n, int64_t bucket, int levels, int mode,
             int device) {
    if (hx == nullptr || hq == nullptr || n <= 0 || bucket < 0)
        return fail(QD_ERR_INVALID_ARG, "host entry point: NULL buffer, n <= 0 or bucket < 0 (n=%lld bucket=%lld)", (long long)n, (long long)bucket);
    const bool bwd = hg != nullptr;
    if (bwd && hgout == nullptr) return fail(QD_ERR_INVALID_ARG, "gout_host is NULL");
    if (device < 0 || device >= 64) return fail(QD_ERR_INVALID_ARG, "device ordinal %d out of range", device);
    DeviceGuard guard;
    QD_CUDA(cudaGetDevice(&guard.prev));
    QD_CUDA(cudaSetDevice(device));
    std::lock_guard<std::mutex> lk(g_mu[device]);
    // Pinned (cudaHostAlloc'd / registered) host buffers are device-addressable under UVA: the kernel can read its
    // inputs and write its outputs straight over PCIe.  Such a launch moves less per direction than the copy engines
    // but has no pipeline to fill and drain, so it wins on small tensors; the crossover is set at 8 Mi elements
    // (measured with both paths forced through a since-removed tuning hook; mixed forms -- DMA one way, the kernel the
    // other -- lost at every size).
    auto device_view = [](const void* p) -> void* {
        if (p == nullptr) return nullptr;
        cudaPointerAttributes at;
        if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return nullptr; }
        return at.type == cudaMemoryTypeHost ? at.devicePointer : nullptr;
    };
    bool direct = n <= kDirectMaxElems;
    const float *dev_x = nullptr, *dev_g = nullptr;
    float *dev_q = nullptr, *dev_gout = nullptr;
    if (direct) {
        dev_x = static_cast<const float*>(device_view(hx));
        dev_g = static_cast<const float*>(device_view(hg));
        dev_q = static_cast<float*>(device_view(hq));
        dev_gout = static_cast<float*>(device_view(hgout));
        direct = dev_x != nullptr && dev_q != nullptr && (!bwd || (dev_g != nullptr && dev_gout != nullptr));
    }
    // staged pipeline: ~8 chunks per tensor, 8 MiB (below that per-copy overhead wins) to 16 MiB per buffer
    const int64_t chunk_elems = n >= (32ll << 20) ? kChunkElems : kChunkElems / 2;
    HostCtx* c;
    int rc = ensure_ctx(device, chunk_elems, &c);
    if (rc) return rc;

    int64_t rows, row_len, padded;
    rc = qd_bucket_geometry(n, bucket, &rows, &row_len, &padded);
    if (rc) return rc;
    // what the fused op refuses, refused before any copy is enqueued: an error return leaves no transfer in flight on
    // the caller's buffers and nothing written to the outputs
    if (bwd && mode != QD_BWD_STE && mode != QD_BWD_TRUNCATED && mode != QD_BWD_MINMAX)
        return fail(QD_ERR_INVALID_ARG, "unknown backward mode %d", mode);
    if (bwd && mode == QD_BWD_MINMAX && (bucket == 0 || row_len > QD_MAX_STAGED_BUCKET))
        return fail(QD_ERR_UNSUPPORTED, "minmax backward needs a bucket of at most %d floats (quant_functions.py:332-334)",
                    QD_MAX_STAGED_BUCKET);

    if (row_len > chunk_elems) {
        // one row spans more than a chunk (bucket None on a large tensor): no row-aligned
        // cut exists, so stage the whole tensor; copies still run at PCIe rate.
        if (c->big_cap < n) {
            cudaFree(c->big_x); cudaFree(c->big_g); cudaFree(c->big_q); cudaFree(c->big_gout); cudaFree(c->big_ws);
            const size_t bytes = (size_t)n * sizeof(float);
            c->big_ws_bytes = qd_workspace_bytes(n, bucket);
            c->big_cap = 0;
            c->big_x = c->big_g = c->big_q = c->big_gout = nullptr;
            c->big_ws = nullptr;
            QD_CUDA(cudaMalloc(&c->big_x, bytes));
            QD_CUDA(cudaMalloc(&c->big_g, bytes));
            QD_CUDA(cudaMalloc(&c->big_q, bytes));
            QD_CUDA(cudaMalloc(&c->big_gout, bytes));
            QD_CUDA(cudaMalloc(&c->big_ws, c->big_ws_bytes));
            c->big_cap = n;
        }
        cudaStream_t s = c->slot[0].stream;
        const size_t bytes = (size_t)n * sizeof(float);
        QD_CUDA(cudaMemcpyAsync(c->big_x, hx, bytes, cudaMemcpyHostToDevice, s));
        if (bwd) QD_CUDA(cudaMemcpyAsync(c->big_g, hg, bytes, cudaMemcpyHostToDevice, s));
        rc = bwd ? qd_uniform_fwd_bwd(c->big_x, c->big_g, c->big_q, c->big_gout, n, bucket, levels, mode, c->big_ws,
                                      c->big_ws_bytes, s)
                 : qd_uniform_fwd(c->big_x, c->big_q, nullptr, nullptr, nullptr, nullptr, nullptr, n, bucket, levels,
                                  nullptr, 0.f, 0, 0, 0, c->big_ws, c->big_ws_bytes, s);
        if (rc) {
            cudaStreamSynchronize(s);  // the copies above still read the caller's buffers
            return rc;
        }
        QD_CUDA(cudaMemcpyAsync(hq, c->big_q, bytes, cudaMemcpyDeviceToHost, s));
        if (bwd) QD_CUDA(cudaMemcpyAsync(hgout, c->big_gout, bytes, cudaMemcpyDeviceToHost, s));
        QD_CUDA(cudaStreamSynchronize(s));
        return QD_OK;
    }

    // row-aligned chunks; the kernel sees each chunk as an independent tensor with the
    // same bucket size, which is exact because rows never straddle a chunk boundary and
    // only the last chunk holds the (short) tail row.
    // (A ramp of smaller chunks at the head and the tail to shorten the half-duplex fill / drain was measured and
    // dropped: copies below 16 MiB lose more to per-copy overhead than the ramp saves; chunk sizes were forced through a
    // since-removed tuning hook.)
    // the register / staged-row kernels read and write every element once; the grid path (rows beyond
    // QD_MAX_STAGED_BUCKET floats) makes several passes and keeps its staging
    if (direct && row_len <= QD_MAX_STAGED_BUCKET) {
        Slot& s = c->slot[0];
        rc = bwd ? qd_uniform_fwd_bwd(dev_x, dev_g, dev_q, dev_gout, n, bucket, levels, mode, s.ws, s.ws_bytes, s.stream)
                 : qd_uniform_fwd(dev_x, dev_q, nullptr, nullptr, nullptr, nullptr, nullptr, n, bucket, levels, nullptr, 0.f, 0,
                                  0, 0, s.ws, s.ws_bytes, s.stream);
        if (rc) return rc;
        QD_CUDA(cudaStreamSynchronize(s.stream));
        QD_CUDA(cudaGetLastError());
        return QD_OK;
    }
    const int64_t rows_per_chunk = chunk_elems / row_len;
    const int64_t chunk = rows_per_chunk * row_len;
    int k = 0;
    for (int64_t off = 0; off < n; off += chunk, ++k) {
        Slot& s = c->slot[k % kSlots];
        const int64_t len = (n - off < chunk) ? (n - off) : chunk;
        const size_t bytes = (size_t)len * sizeof(float);
        // a chunk shorter than the bucket must still be bucketed like the tail of the
        // full tensor: with rows >= 2 overall the tail row is "padded", never a short
        // single row -- both cases give the same min/max, so passing bucket is exact.
        QD_CUDA(cudaMemcpyAsync(s.x, hx + off, bytes, cudaMemcpyHostToDevice, s.stream));
        if (bwd) QD_CUDA(cudaMemcpyAsync(s.g, hg + off, bytes, cudaMemcpyHostToDevice, s.stream));
        rc = bwd ? qd_uniform_fwd_bwd(s.x, s.g, s.q, s.gout, len, bucket, levels, mode, s.ws, s.ws_bytes, s.stream)
                 : qd_uniform_fwd(s.x, s.q, nullptr, nullptr, nullptr, nullptr, nullptr, len, bucket, levels, nullptr,
                                  0.f, 0, 0, 0, s.ws, s.ws_bytes, s.stream);
        if (rc) {
            for (int i = 0; i < kSlots; ++i) cudaStreamSynchronize(c->slot[i].stream);  // copies of earlier chunks in flight
            return rc;
        }
        QD_CUDA(cudaMemcpyAsync(hq + off, s.q, bytes, cudaMemcpyDeviceToHost, s.stream));
        if (bwd) QD_CUDA(cudaMemcpyAsync(hgout + off, s.gout, bytes, cudaMemcpyDeviceToHost, s.stream));
    }
    for (int i = 0; i < kSlots; ++i) QD_CUDA(cudaStreamSynchronize(c->slot[i].stream));
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

}  // namespace

extern "C" int qd_uniform_fwd_host(const float* x_host, float* q_host, int64_t n, int64_t bucket, int levels, int device) {
    return run_host(x_host, nullptr, q_host, nullptr, n, bucket, levels, 0, device);
}

extern "C" int qd_uniform_fwd_bwd_host(const float* x_host, const float* g_host, float* q_host, float* gout_host,
                                       int64_t n, int64_t bucket, int levels, int mode, int device) {
    if (g_host == nullptr) return fail(QD_ERR_INVALID_ARG, "g_host is NULL");
    return run_host(x_host, g_host, q_host, gout_host, n, bucket, levels, mode, device);
}
