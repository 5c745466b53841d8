// qd_plans.cu -- plans: every tensor of a model in one launch (qd_plan.cuh).  qd_plan_* for the uniform op, the
// fused optimizer step and the long-row (bucket None) path; qd_plan_nonuniform_* for the centroid op and its gradient.
#include <vector>

#include "qd_launch.h"
#include "qd_plan.cuh"

using namespace qd;

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
    int grid;
    int rc = capped_grid(p->long_chunks, 4, &grid);
    if (rc) return rc;
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

// Gradient pointers of a backward launch: by value in `gt` up to kPlanGradsByValue tensors (graph-capturable), else
// copied to p->dev_grads on the stream and returned in `dev_grads` (gt stays zero).
template <class Plan>
static int plan_grads(const Plan* p, const float* const* grad, cudaStream_t s, GradTable* gt, float* const** dev_grads) {
    *gt = {};
    *dev_grads = nullptr;
    if (p->count <= kPlanGradsByValue) {
        for (int i = 0; i < p->count; ++i) gt->g[i] = const_cast<float*>(grad[i]);
    } else {
        QD_CUDA(cudaMemcpyAsync(p->dev_grads, grad, sizeof(float*) * p->count, cudaMemcpyHostToDevice, s));
        *dev_grads = p->dev_grads;
    }
    return QD_OK;
}

template <int BWD>
static int plan_sgd_launch(const qd_plan* p, float* const* dev_grads, const GradTable& gt, const SgdParams& sp, cudaStream_t s) {
    return with_row_regs<4>(p->max_row_len, [&](auto r) -> int {   // rows of more than 512 floats are refused before
        auto kern = plan_sgd_step_kernel<BWD, r>;
        int grid;
        int rc = resident_grid((const void*)kern, kWarpCtaThreads, 0, (p->total_rows + kWarpsPerCta - 1) / kWarpsPerCta, &grid);
        if (rc) return rc;
        kern<<<grid, kWarpCtaThreads, 0, s>>>(p->dev, p->count, p->total_rows, dev_grads, gt, sp);
        QD_CUDA(cudaGetLastError());
        return QD_OK;
    });
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
    cudaStream_t s = as_stream(stream);
    SgdParams sp;
    sp.lr = (float)lr; sp.momentum = (float)momentum; sp.weight_decay = (float)weight_decay; sp.nesterov = nesterov ? 1 : 0;
    GradTable gt;
    float* const* dev_grads;
    int rc = plan_grads(p, grad, s, &gt, &dev_grads);
    if (rc) return rc;
    switch (mode) {
        case QD_BWD_STE: return plan_sgd_launch<BWD_STE>(p, dev_grads, gt, sp, s);
        case QD_BWD_TRUNCATED: return plan_sgd_launch<BWD_TRUNC>(p, dev_grads, gt, sp, s);
        case QD_BWD_MINMAX: return plan_sgd_launch<BWD_MINMAX>(p, dev_grads, gt, sp, s);
        default: return fail(QD_ERR_INVALID_ARG, "unknown backward mode %d", mode);
    }
}

template <int BWD>
static int plan_launch(const qd_plan* p, float* const* dev_grads, cudaStream_t s, int with_save = 0,
                       const GradTable* gtab = nullptr) {
    static const GradTable kEmpty = {};
    const GradTable& gt = gtab ? *gtab : kEmpty;
    return with_row_regs(p->max_row_len, [&](auto r) -> int {
        auto kern = plan_rows_kernel<BWD, r>;
        int grid;
        int rc = resident_grid((const void*)kern, kWarpCtaThreads, 0, (p->total_rows + kWarpsPerCta - 1) / kWarpsPerCta, &grid);
        if (rc) return rc;
        kern<<<grid, kWarpCtaThreads, 0, s>>>(p->dev, p->count, p->total_rows, dev_grads, with_save, gt);
        QD_CUDA(cudaGetLastError());
        return QD_OK;
    });
}

extern "C" int qd_plan_uniform_fwd(const qd_plan* p, qd_stream_t stream) {
    if (p == nullptr) return fail(QD_ERR_INVALID_ARG, "plan is NULL");
    cudaStream_t s = as_stream(stream);
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
    cudaStream_t s = as_stream(stream);
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
    if (mode != QD_BWD_TRUNCATED && mode != QD_BWD_MINMAX) return fail(QD_ERR_INVALID_ARG, "unknown backward mode %d", mode);
    // Every refusal comes before the first launch, so a refused call leaves every gradient untouched: the per-tensor
    // fallback below fixes the tensors up in place one after the other, and the op refuses min/max rows beyond the
    // staged path (qd_quant.cu run_rows) only when it reaches them.
    if (mode == QD_BWD_MINMAX && p->bucket == 0)
        return fail(QD_ERR_UNSUPPORTED, "minmax backward needs a bucket size (quant_functions.py:332-334)");
    if (mode == QD_BWD_MINMAX && p->max_row_len > QD_MAX_STAGED_BUCKET)
        return fail(QD_ERR_UNSUPPORTED, "minmax backward needs rows of at most %d elements (plan has %lld)", QD_MAX_STAGED_BUCKET,
                    (long long)p->max_row_len);
    for (int i = 0; i < p->count; ++i)
        if (grad[i] == nullptr) return fail(QD_ERR_INVALID_ARG, "grad[%d] is NULL", i);
    cudaStream_t s = as_stream(stream);
    if (p->long_path) {
        int grid;
        int rc = capped_grid(p->long_chunks, 4, &grid);
        if (rc) return rc;
        QD_CUDA(cudaMemcpyAsync(p->dev_grads, grad, sizeof(float*) * p->count, cudaMemcpyHostToDevice, s));
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
    GradTable gt;
    float* const* dev_grads;
    int rc = plan_grads(p, grad, s, &gt, &dev_grads);
    if (rc) return rc;
    return mode == QD_BWD_TRUNCATED ? plan_launch<BWD_TRUNC>(p, dev_grads, s, 0, &gt) : plan_launch<BWD_MINMAX>(p, dev_grads, s, 0, &gt);
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
    return with_row_regs(p->max_row_len, [&](auto r) -> int {
        auto kern = plan_nonuniform_fwd_kernel<r>;
        int grid;
        int rc = resident_grid((const void*)kern, kWarpCtaThreads, 0, (p->total_rows + kWarpsPerCta - 1) / kWarpsPerCta, &grid);
        if (rc) return rc;
        kern<<<grid, kWarpCtaThreads, 0, as_stream(stream)>>>(p->dev, p->count, p->total_rows);
        QD_CUDA(cudaGetLastError());
        return QD_OK;
    });
}

// the gradient blocks of every tensor -> p->partial (first launch of every backward entry point)
static int nu_grad_partials(const qd_nu_plan* p, const float* const* grad, cudaStream_t s) {
    if (grad == nullptr) return fail(QD_ERR_INVALID_ARG, "grad is NULL");
    for (int i = 0; i < p->count; ++i)
        if (grad[i] == nullptr) return fail(QD_ERR_INVALID_ARG, "grad[%d] is NULL", i);
    int grid;
    int rc = capped_grid((p->total_blocks + kPgWarps - 1) / kPgWarps, 4, &grid);
    if (rc) return rc;
    GradTable gt;
    float* const* dev_grads;
    rc = plan_grads(p, grad, s, &gt, &dev_grads);
    if (rc) return rc;
    plan_points_grad_partial<0><<<grid, kPgThreads, 0, s>>>(p->dev, p->count, p->total_blocks, p->block_tiles, gt, dev_grads, p->partial);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

extern "C" int qd_plan_nonuniform_bwd(const qd_nu_plan* p, const float* const* grad, qd_stream_t stream) {
    if (p == nullptr) return fail(QD_ERR_INVALID_ARG, "plan is NULL");
    cudaStream_t s = as_stream(stream);
    int rc = nu_grad_partials(p, grad, s);
    if (rc) return rc;
    plan_points_grad_final<<<(p->count + 7) / 8, 256, 0, s>>>(p->dev, p->count, p->partial);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

extern "C" int qd_plan_nonuniform_bwd_partial(const qd_nu_plan* p, const float* const* grad, double* sums, qd_stream_t stream) {
    if (p == nullptr || sums == nullptr) return fail(QD_ERR_INVALID_ARG, "plan or sums is NULL");
    if ((reinterpret_cast<uintptr_t>(sums) & 7) != 0) return fail(QD_ERR_INVALID_ARG, "sums must be 8-byte aligned");
    cudaStream_t s = as_stream(stream);
    int rc = nu_grad_partials(p, grad, s);
    if (rc) return rc;
    plan_points_grad_sums<<<(p->count + 7) / 8, 256, 0, s>>>(p->dev, p->count, p->partial, sums);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

extern "C" int qd_plan_nonuniform_bwd_finish(const qd_nu_plan* p, const double* sums, double scale, qd_stream_t stream) {
    if (p == nullptr || sums == nullptr) return fail(QD_ERR_INVALID_ARG, "plan or sums is NULL");
    if ((reinterpret_cast<uintptr_t>(sums) & 7) != 0) return fail(QD_ERR_INVALID_ARG, "sums must be 8-byte aligned");
    plan_points_grad_finish<<<(p->count + 7) / 8, 256, 0, as_stream(stream)>>>(p->dev, p->count, sums, scale);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}
