// stream_ceiling.cu -- measurement only: the copy ceiling of the headline's traffic (64 Mi floats, rows of 256 floats,
// x and g read, q = x and gout = g written: 16 B per element) under several row -> warp -> CTA orders, and the library's
// headline call (qd_uniform_fwd_bwd, min/max backward) timed in the same process.  Built and run by
// tools/stream_ceiling.py, which adds the card's name, power limit and clock and writes profiles/stream_ceiling.json:
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -Iinclude -Iquantized_distillation_b200/csrc \
//        -o /tmp/stream_ceiling tools/stream_ceiling.cu -Lquantized_distillation_b200 -lqd_b200 \
//        -Xlinker -rpath=$PWD/quantized_distillation_b200 && /tmp/stream_ceiling [launches] [rounds]
// Prints one JSON object: per variant the microseconds per launch of every round.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "qd_b200.h"
#include "qd_common.cuh"

#define CK(x)                                                                                  \
    do {                                                                                       \
        cudaError_t e_ = (x);                                                                  \
        if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } \
    } while (0)

using namespace qd;

constexpr int kRowFloats = 256;  // the headline's bucket: 2 float4 per lane
constexpr int kWarps = 8;        // 256-thread CTAs

template <bool EF>
__device__ __forceinline__ float4 ld4(const float* p, uint64_t pol) {
    if constexpr (EF) return ld_hint4(p, pol);
    else return ld_stream4(p);
}
template <bool EF>
__device__ __forceinline__ void st4(float* p, float4 v, uint64_t pol) {
    if constexpr (EF) st_hint4(p, v, pol);
    else st_stream4(p, v);
}

// SPAN = false: warp w of CTA b starts at row b*8 + w and strides by gridDim*8 (the headline's order).
// SPAN = true:  CTA b owns rows [b*span, (b+1)*span); its 8 warps walk them 8 consecutive rows at a time.
// K rows are loaded per warp before the first store.  Lane L owns floats r*128 + 4L .. +3 of a row (r = 0, 1).
template <bool SPAN, int K, bool EF_LD, bool EF_ST>
__global__ void __launch_bounds__(256) copy_rows(const float* __restrict__ x, const float* __restrict__ g, float* __restrict__ q,
                                                 float* __restrict__ go, int64_t rows, int64_t span) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint64_t pol = (EF_LD || EF_ST) ? l2_policy_evict_first() : 0;
    int64_t row, end, step;
    if (SPAN) {
        row = (int64_t)blockIdx.x * span + warp;
        end = min(rows, ((int64_t)blockIdx.x + 1) * span);
        step = kWarps;
    } else {
        row = (int64_t)blockIdx.x * kWarps + warp;
        end = rows;
        step = (int64_t)gridDim.x * kWarps;
    }
    for (; row < end; row += K * step) {
        float4 vx[K][2], vg[K][2];
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const int64_t r = row + k * step;
            if (r < end) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    vx[k][h] = ld4<EF_LD>(x + r * kRowFloats + h * 128 + lane * 4, pol);
                    vg[k][h] = ld4<EF_LD>(g + r * kRowFloats + h * 128 + lane * 4, pol);
                }
            }
        }
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const int64_t r = row + k * step;
            if (r < end) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    st4<EF_ST>(q + r * kRowFloats + h * 128 + lane * 4, vx[k][h], pol);
                    st4<EF_ST>(go + r * kRowFloats + h * 128 + lane * 4, vg[k][h], pol);
                }
            }
        }
    }
}

// x -> q only: the V1 order over one input and one output stream (launched once for x -> q, once for g -> gout)
__global__ void __launch_bounds__(256) copy_rows_single(const float* __restrict__ x, float* __restrict__ q, int64_t rows) {
    const int lane = threadIdx.x & 31;
    const int64_t step = (int64_t)gridDim.x * kWarps;
    for (int64_t r = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5); r < rows; r += step) {
        float4 v[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) v[h] = ld_stream4(x + r * kRowFloats + h * 128 + lane * 4);
#pragma unroll
        for (int h = 0; h < 2; ++h) st_stream4(q + r * kRowFloats + h * 128 + lane * 4, v[h]);
    }
}

struct Variant {
    std::string id;
    void (*kern)(const float*, const float*, float*, float*, int64_t, int64_t);  // null: not a copy kernel
    int ctas_per_sm;  // 0: one CTA per 8 rows (no grid stride)
    int kind;  // 0 = copy kernel, 1 = cudaMemcpyAsync, 2 = library headline, 3 = one stream pair at a time
};

int main(int argc, char** argv) {
    const int launches = argc > 1 ? atoi(argv[1]) : 200;
    const int rounds = argc > 2 ? atoi(argv[2]) : 5;
    const int64_t n = (int64_t)1 << 26, rows = n / kRowFloats;
    int sms = 0, dev = 0;
    CK(cudaGetDevice(&dev));
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));

    float *x, *g, *q, *go;
    CK(cudaMalloc(&x, n * 4)); CK(cudaMalloc(&g, n * 4)); CK(cudaMalloc(&q, n * 4)); CK(cudaMalloc(&go, n * 4));
    {
        // x ~ 0.05 * N(0, 1) (Irwin-Hall of 4 uniforms), g ~ U(-1, 1): the headline's rows take its usual fast path
        std::vector<float> hx(n), hg(n);
        uint64_t s = 0x9E3779B97F4A7C15ull;
        auto u = [&]() { s = s * 6364136223846793005ull + 1442695040888963407ull; return (float)((s >> 40) * (1.0 / 16777216.0)); };
        for (int64_t i = 0; i < n; ++i) {
            hx[i] = 0.05f * (u() + u() + u() + u() - 2.0f) * 1.7320508f;
            hg[i] = 2.0f * u() - 1.0f;
        }
        CK(cudaMemcpy(x, hx.data(), n * 4, cudaMemcpyHostToDevice));
        CK(cudaMemcpy(g, hg.data(), n * 4, cudaMemcpyHostToDevice));
    }
    const size_t ws_bytes = qd_workspace_bytes(n, kRowFloats);
    void* ws;
    CK(cudaMalloc(&ws, ws_bytes));
    cudaStream_t st;
    CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));

    const std::vector<Variant> vs = {
        {"V0_memcpy", nullptr, 0, 1},
        {"V1_interleaved_3cta", copy_rows<false, 1, false, false>, 3, 0},
        {"V2_interleaved_2cta", copy_rows<false, 1, false, false>, 2, 0},
        {"V2_interleaved_4cta", copy_rows<false, 1, false, false>, 4, 0},
        {"V3_span_3cta", copy_rows<true, 1, false, false>, 3, 0},
        {"V3_span_2cta", copy_rows<true, 1, false, false>, 2, 0},
        {"V3_span_4cta", copy_rows<true, 1, false, false>, 4, 0},
        {"V4_interleaved_k2_3cta", copy_rows<false, 2, false, false>, 3, 0},
        {"V4_span_k2_3cta", copy_rows<true, 2, false, false>, 3, 0},
        {"V5_interleaved_st_evict_first", copy_rows<false, 1, false, true>, 3, 0},
        {"V5_interleaved_ldst_evict_first", copy_rows<false, 1, true, true>, 3, 0},
        {"V5_span_st_evict_first", copy_rows<true, 1, false, true>, 3, 0},
        {"V5_span_ldst_evict_first", copy_rows<true, 1, true, true>, 3, 0},
        {"V6_one_pair_at_a_time_3cta", nullptr, 3, 3},
        {"V7_one_row_per_warp_grid", copy_rows<false, 1, false, false>, 0, 0},
        {"headline_qd_uniform_fwd_bwd_minmax", nullptr, 0, 2},
    };

    auto launch = [&](const Variant& v) {
        if (v.kind == 1) {
            CK(cudaMemcpyAsync(q, x, n * 4, cudaMemcpyDeviceToDevice, st));
            CK(cudaMemcpyAsync(go, g, n * 4, cudaMemcpyDeviceToDevice, st));
        } else if (v.kind == 2) {
            int rc = qd_uniform_fwd_bwd(x, g, q, go, n, kRowFloats, 16, QD_BWD_MINMAX, ws, ws_bytes, st);
            if (rc) { fprintf(stderr, "qd_uniform_fwd_bwd: %s\n", qd_last_error()); exit(1); }
        } else if (v.kind == 3) {
            copy_rows_single<<<sms * v.ctas_per_sm, 256, 0, st>>>(x, q, rows);
            copy_rows_single<<<sms * v.ctas_per_sm, 256, 0, st>>>(g, go, rows);
            CK(cudaGetLastError());
        } else {
            const int grid = v.ctas_per_sm ? sms * v.ctas_per_sm : (int)((rows + kWarps - 1) / kWarps);
            const int64_t span = (rows + grid - 1) / grid;
            v.kern<<<grid, 256, 0, st>>>(x, g, q, go, rows, span);
            CK(cudaGetLastError());
        }
    };

    // every copy variant must reproduce its inputs exactly
    {
        std::vector<float> hx(n), hq(n), hg(n), hgo(n);
        CK(cudaMemcpy(hx.data(), x, n * 4, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(hg.data(), g, n * 4, cudaMemcpyDeviceToHost));
        for (const auto& v : vs) {
            if (v.kind != 0 && v.kind != 3) continue;
            CK(cudaMemsetAsync(q, 0xff, n * 4, st));
            CK(cudaMemsetAsync(go, 0xff, n * 4, st));
            launch(v);
            CK(cudaStreamSynchronize(st));
            CK(cudaMemcpy(hq.data(), q, n * 4, cudaMemcpyDeviceToHost));
            CK(cudaMemcpy(hgo.data(), go, n * 4, cudaMemcpyDeviceToHost));
            for (int64_t i = 0; i < n; ++i)
                if (hq[i] != hx[i] || hgo[i] != hg[i]) { fprintf(stderr, "%s: wrong copy at %lld\n", v.id.c_str(), (long long)i); return 1; }
        }
    }

    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    std::vector<std::vector<double>> us(vs.size());
    for (int rd = 0; rd < rounds; ++rd) {
        for (size_t i = 0; i < vs.size(); ++i) {
            for (int w = 0; w < 10; ++w) launch(vs[i]);
            CK(cudaEventRecord(e0, st));
            for (int l = 0; l < launches; ++l) launch(vs[i]);
            CK(cudaEventRecord(e1, st));
            CK(cudaEventSynchronize(e1));
            float ms = 0;
            CK(cudaEventElapsedTime(&ms, e0, e1));
            us[i].push_back(ms * 1e3 / launches);
        }
    }
    printf("{\"n\": %lld, \"row_floats\": %d, \"bytes_per_elem\": 16, \"sms\": %d, \"launches\": %d, \"rounds\": %d, \"us\": {",
           (long long)n, kRowFloats, sms, launches, rounds);
    for (size_t i = 0; i < vs.size(); ++i) {
        printf("%s\"%s\": [", i ? ", " : "", vs[i].id.c_str());
        for (int rd = 0; rd < rounds; ++rd) printf("%s%.3f", rd ? ", " : "", us[i][rd]);
        printf("]");
    }
    printf("}}\n");
    CK(cudaFree(x)); CK(cudaFree(g)); CK(cudaFree(q)); CK(cudaFree(go)); CK(cudaFree(ws));
    return 0;
}
