// qd_codec.cu -- stored-model codecs: histogram of level indices, fixed-width 1/2/4/8-bit packing and its fused
// unpack + dequantization, and the Huffman-coded stream (qd_huffman.cuh) per tensor and per model.
#include <algorithm>
#include <cstring>
#include <vector>

#include "qd_huffman.cuh"
#include "qd_launch.h"
#include "qd_packed_walk.cuh"

using namespace qd;

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
    int grid;
    int rc = capped_grid((n / 16 + 255) / 256 + 1, 4, &grid);
    if (rc) return rc;
    index_histogram_kernel<<<grid, 256, 0, as_stream(stream)>>>(idx_u8, n, num_bins, reinterpret_cast<unsigned long long*>(counts));
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

// ------------------------------------------------------------------ f2: packed codec
// one thread-group = 16 consecutive codes in (one 128-bit load), 2*BITS bytes out (one store of that width); BITS is a
// template parameter so that every shift, mask and access width is a compile-time constant
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
    if (!bits_ok(bits)) return fail(QD_ERR_INVALID_ARG, "bits must be 1, 2, 4 or 8");
    int grid;
    int rc = capped_grid(((n + 15) / 16 + kTileGroups - 1) / kTileGroups, 8, &grid);
    if (rc) return rc;
    with_bits(bits, [&](auto b) { pack_kernel<b><<<grid, 256, 0, as_stream(stream)>>>(idx_u8, packed, n); });
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

// inverse of pack_kernel: one thread-group = 16 consecutive codes, read as four load_codes4 groups, written as one
// 128-bit store when the output is 16-byte aligned and the group complete, else byte by byte
template <int BITS>
__global__ void __launch_bounds__(256) unpack_indices_kernel(const uint8_t* __restrict__ packed, uint8_t* __restrict__ idx, int64_t n) {
    constexpr uint32_t mask = (1u << BITS) - 1u;
    const int64_t groups = (n + 15) / 16;
    const int64_t in_bytes = (n * BITS + 7) / 8;
    const bool ivec = (reinterpret_cast<uintptr_t>(packed) & 3) == 0;
    const bool ovec = (reinterpret_cast<uintptr_t>(idx) & 15) == 0;
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += (int64_t)gridDim.x * blockDim.x) {
        uint32_t w[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int64_t e0 = g * 16 + u * 4;
            const uint32_t c = e0 < n ? load_codes4<BITS>(packed, e0, in_bytes, ivec) : 0u;
            w[u] = (c & mask) | (((c >> BITS) & mask) << 8) | (((c >> (2 * BITS)) & mask) << 16) | (((c >> (3 * BITS)) & mask) << 24);
        }
        if (ovec && g * 16 + 16 <= n) {
            __stcs(reinterpret_cast<uint4*>(idx + g * 16), make_uint4(w[0], w[1], w[2], w[3]));
        } else {
            for (int j = 0; j < 16 && g * 16 + j < n; ++j) idx[g * 16 + j] = (uint8_t)(w[j >> 2] >> (8 * (j & 3)));
        }
    }
}

extern "C" int qd_unpack_indices(const uint8_t* packed, int bits, uint8_t* idx_u8, int64_t n, qd_stream_t stream) {
    if (packed == nullptr || idx_u8 == nullptr || n <= 0) return fail(QD_ERR_INVALID_ARG, "NULL argument or n <= 0");
    if (!bits_ok(bits)) return fail(QD_ERR_INVALID_ARG, "bits must be 1, 2, 4 or 8");
    int grid;
    int rc = capped_grid(((n + 15) / 16 + 255) / 256, 8, &grid);
    if (rc) return rc;
    with_bits(bits, [&](auto b) { unpack_indices_kernel<b><<<grid, 256, 0, as_stream(stream)>>>(packed, idx_u8, n); });
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

// The element loop of one tensor's unpack, as CTA `block` of the `nblocks` CTAs that serve the tensor: the per-tensor
// kernel calls it with its own grid, the whole-model kernel with the tensor's share of its grid, so both write the
// same bits by construction.
template <int BITS>
__device__ __forceinline__ void unpack_dequant_body(const float* s_unit, const uint8_t* __restrict__ packed,
                                                    const float* __restrict__ alpha, const float* __restrict__ beta,
                                                    float* __restrict__ q, const Geometry& geo, unsigned block, unsigned nblocks) {
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
    if (full_tiles > (int64_t)block) {
        const uint32_t L32 = single ? 1u : (uint32_t)L;
        const int64_t e_first = ((int64_t)block * kTileGroups + threadIdx.x) * 4;
        int row = single ? 0 : (int)(e_first / L);
        uint32_t rem = single ? 0u : (uint32_t)(e_first % L);
        const int du_rows = single ? 0 : (int)((256 * 4) / L);
        const uint32_t du_rem = single ? 0u : (uint32_t)((256 * 4) % L);
        const int64_t dt = (int64_t)nblocks * kTileGroups * 4;
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
        fetch(block, row, rem, cur);
        for (int64_t tile = block; tile < full_tiles; tile += nblocks) {
            Fetched nxt = cur;
            row += dt_rows;
            rem += dt_rem;
            if (rem >= L32) { rem -= L32; ++row; }
            if (tile + nblocks < full_tiles) fetch(tile + nblocks, row, rem, nxt);
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
    const int64_t stride = (int64_t)nblocks * blockDim.x;
    for (int64_t g = full_tiles * kTileGroups + (int64_t)block * blockDim.x + threadIdx.x; g < groups; g += stride) {
        const int64_t e0 = g * 4;
        const uint32_t w = load_codes4<BITS>(packed, e0, in_bytes, ivec);
        for (int j = 0; j < 4; ++j) {
            if (e0 + j >= geo.n) break;
            const int64_t r = single ? 0 : (e0 + j) / L;
            q[e0 + j] = from_unit(s_unit[(w >> (j * BITS)) & mask], alpha[r], beta[r]);
        }
    }
}

template <bool UNIFORM, int BITS>
__global__ void __launch_bounds__(256, 4) unpack_dequant_kernel(const uint8_t* __restrict__ packed,
                                                            const float* __restrict__ points, int K,
                                                            const float* __restrict__ alpha, const float* __restrict__ beta,
                                                            float* __restrict__ q, Geometry geo, float S) {
    __shared__ float s_unit[256];
    load_unit_table<UNIFORM>(s_unit, points, K, S);
    __syncthreads();
    unpack_dequant_body<BITS>(s_unit, packed, alpha, beta, q, geo, blockIdx.x, gridDim.x);
}

// Checks the arguments both unpacks share and launches unpack_dequant_kernel<UNIFORM, bits>.
template <bool UNIFORM>
static int unpack_dequant(const uint8_t* packed, int bits, const float* points, int K, const float* alpha, const float* beta,
                          float* q, int64_t n, int64_t bucket, float S, qd_stream_t stream) {
    Geometry geo;
    if (packed == nullptr || alpha == nullptr || beta == nullptr || q == nullptr) return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if (!bits_ok(bits)) return fail(QD_ERR_INVALID_ARG, "bits must be 1, 2, 4 or 8");
    if (geometry_of(n, bucket, &geo)) return fail(QD_ERR_INVALID_ARG, "bad geometry");
    int grid;   // one resident wave (__launch_bounds__(256, 4))
    int rc = capped_grid(((n + 3) / 4 + kTileGroups - 1) / kTileGroups, 4, &grid);
    if (rc) return rc;
    with_bits(bits, [&](auto b) {
        unpack_dequant_kernel<UNIFORM, b><<<grid, 256, 0, as_stream(stream)>>>(packed, points, K, alpha, beta, q, geo, S);
    });
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

extern "C" int qd_unpack_dequant_uniform(const uint8_t* packed, int bits, const float* alpha, const float* beta, float* q,
                                         int64_t n, int64_t bucket, int levels, qd_stream_t stream) {
    if (levels < 2 || levels > (1 << bits)) return fail(QD_ERR_INVALID_ARG, "levels must be in [2, 2^bits]");
    return unpack_dequant<true>(packed, bits, nullptr, 0, alpha, beta, q, n, bucket, (float)(levels - 1), stream);
}

extern "C" int qd_unpack_dequant_nonuniform(const uint8_t* packed, int bits, const float* points, int num_points,
                                            const float* alpha, const float* beta, float* q, int64_t n, int64_t bucket,
                                            qd_stream_t stream) {
    if (points == nullptr || num_points < 1 || num_points > (1 << bits)) return fail(QD_ERR_INVALID_ARG, "num_points must be in [1, 2^bits]");
    return unpack_dequant<false>(packed, bits, points, num_points, alpha, beta, q, n, bucket, 0.f, stream);
}

// A whole model in one launch.  Tensor t owns CTAs [cta_start[t], cta_start[t + 1]), one per tile of kTileGroups groups
// of four elements, found by binary search; every CTA loads its tensor's unit table once and runs the per-tensor body
// as CTA (blockIdx.x - cta_start[t]) of the tensor's share of the grid, at the tensor's own code width.
template <bool UNIFORM>
__global__ void __launch_bounds__(256, 4) unpack_dequant_model_kernel(const qd_packed_tensor* __restrict__ tensors,
                                                                  const int32_t* __restrict__ cta_start, int count,
                                                                  int64_t bucket, float S) {
    __shared__ float s_unit[256];
    const int b = (int)blockIdx.x;
    const int lo = model_tensor_of(cta_start, count, b);
    const qd_packed_tensor& t = tensors[lo];
    load_unit_table<UNIFORM>(s_unit, t.points, t.num_points, S);
    __syncthreads();
    Geometry geo;                                 // geometry_of
    geo.n = t.n;
    geo.row_len = (bucket == 0 || t.n < bucket) ? t.n : bucket;
    geo.rows = (t.n + geo.row_len - 1) / geo.row_len;
    const int first = __ldg(cta_start + lo);
    const unsigned block = (unsigned)(b - first), nblocks = (unsigned)(__ldg(cta_start + lo + 1) - first);
    switch (t.bits) {
        case 8: unpack_dequant_body<8>(s_unit, t.packed, t.alpha, t.beta, t.q, geo, block, nblocks); break;
        case 4: unpack_dequant_body<4>(s_unit, t.packed, t.alpha, t.beta, t.q, geo, block, nblocks); break;
        case 2: unpack_dequant_body<2>(s_unit, t.packed, t.alpha, t.beta, t.q, geo, block, nblocks); break;
        default: unpack_dequant_body<1>(s_unit, t.packed, t.alpha, t.beta, t.q, geo, block, nblocks); break;
    }
}

// ------------------------------------------------------------------ whole-model launches
// qd_unpack_dequant_model, qd_huffman_decode_dequant_model and qd_huffman_decode_packed_model read one workspace: the caller's descriptor array, then
// cta_start[count + 1] (int32); the kernel finds a CTA's tensor with model_tensor_of.
template <typename Desc>
static size_t model_workspace_bytes(int count) {
    static_assert(sizeof(Desc) % alignof(int32_t) == 0, "cta_start follows the descriptors");
    return count < 1 ? 0 : (size_t)count * sizeof(Desc) + ((size_t)count + 1) * sizeof(int32_t);
}

// Checks the workspace and every tensor -- ctas_of(i, tensors[i], &ctas) returns QD_OK with the tensor's CTA count, or
// the status of fail() -- refuses grids of more than 2^31 - 1 CTAs (each `unit` of `size` `what`), then uploads the
// image with one copy on `st`.  On QD_OK, *grid is the launch's CTA count and *dev_start the device cta_start; the
// descriptors are at the start of the workspace.
template <typename Desc, typename CtasOf>
static int upload_model(const Desc* tensors, int count, void* workspace, size_t workspace_bytes, cudaStream_t st, CtasOf ctas_of,
                        const char* unit, int size, const char* what, unsigned* grid, const int32_t** dev_start) {
    const size_t need = model_workspace_bytes<Desc>(count);
    if (workspace == nullptr || (reinterpret_cast<uintptr_t>(workspace) & 15) || workspace_bytes < need)
        return fail(QD_ERR_WORKSPACE, "workspace must be 16-byte aligned and hold %zu bytes (got %zu)", need, workspace_bytes);
    // host image of the workspace, consumed by the pageable copy before it returns (kept per thread: no allocation once grown)
    thread_local std::vector<unsigned char> image;
    image.resize(need);
    int32_t* cta_start = reinterpret_cast<int32_t*>(image.data() + (size_t)count * sizeof(Desc));
    int64_t ctas = 0;
    for (int i = 0; i < count; ++i) {
        int64_t c = 0;
        if (const int rc = ctas_of(i, tensors[i], &c)) return rc;
        cta_start[i] = (int32_t)ctas;
        ctas += c;
        if (ctas > INT32_MAX) return fail(QD_ERR_INVALID_ARG, "the model has more than 2^31 - 1 %s of %d %s", unit, size, what);
    }
    cta_start[count] = (int32_t)ctas;
    memcpy(image.data(), tensors, (size_t)count * sizeof(Desc));
    QD_CUDA(cudaMemcpyAsync(workspace, image.data(), need, cudaMemcpyHostToDevice, st));
    *grid = (unsigned)ctas;
    *dev_start = reinterpret_cast<const int32_t*>(static_cast<const unsigned char*>(workspace) + (size_t)count * sizeof(Desc));
    return QD_OK;
}

static_assert(sizeof(qd_packed_tensor) == 56, "qd_packed_tensor layout is shared with codec.py");

extern "C" size_t qd_unpack_model_workspace_bytes(int count) { return model_workspace_bytes<qd_packed_tensor>(count); }

extern "C" int qd_unpack_dequant_model(const qd_packed_tensor* tensors, int count, int64_t bucket, int levels, void* workspace,
                                       size_t workspace_bytes, qd_stream_t stream) {
    if (tensors == nullptr || count < 1) return fail(QD_ERR_INVALID_ARG, "NULL tensors or count < 1");
    if (bucket < 0) return fail(QD_ERR_INVALID_ARG, "bucket must be >= 0");
    if (levels != 0 && (levels < 2 || levels > 256)) return fail(QD_ERR_INVALID_ARG, "levels must be in [2, 256] (uniform) or 0 (non-uniform)");
    const bool uniform = levels != 0;
    auto ctas_of = [&](int i, const qd_packed_tensor& t, int64_t* ctas) {
        if (t.packed == nullptr || t.alpha == nullptr || t.beta == nullptr || t.q == nullptr)
            return fail(QD_ERR_INVALID_ARG, "tensor %d: NULL argument", i);
        if (t.n < 1) return fail(QD_ERR_INVALID_ARG, "tensor %d: n must be >= 1", i);
        if (!bits_ok(t.bits)) return fail(QD_ERR_INVALID_ARG, "tensor %d: bits must be 1, 2, 4 or 8", i);
        if (uniform && (t.points != nullptr || t.num_points != 0))
            return fail(QD_ERR_INVALID_ARG, "tensor %d: a uniform model has no points (points NULL, num_points 0)", i);
        if (uniform && levels > (1 << t.bits)) return fail(QD_ERR_INVALID_ARG, "tensor %d: %d levels do not fit in %d-bit codes", i, levels, t.bits);
        if (!uniform && (t.points == nullptr || t.num_points < 1 || t.num_points > (1 << t.bits)))
            return fail(QD_ERR_INVALID_ARG, "tensor %d: num_points must be in [1, 2^bits]", i);
        *ctas = ((t.n + 3) / 4 + kTileGroups - 1) / kTileGroups;
        return (int)QD_OK;
    };
    cudaStream_t st = as_stream(stream);
    unsigned ctas;
    const int32_t* dev_start;
    if (const int rc = upload_model(tensors, count, workspace, workspace_bytes, st, ctas_of, "tiles", kTileGroups * 4, "elements",
                                    &ctas, &dev_start))
        return rc;
    const qd_packed_tensor* dev_tensors = static_cast<const qd_packed_tensor*>(workspace);
    if (uniform)
        unpack_dequant_model_kernel<true><<<ctas, 256, 0, st>>>(dev_tensors, dev_start, count, bucket, (float)(levels - 1));
    else
        unpack_dequant_model_kernel<false><<<ctas, 256, 0, st>>>(dev_tensors, dev_start, count, bucket, 0.f);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

// ------------------------------------------------------------------ f2: fully-connected layer on packed weights
// y[i, o] = sum_k x[i, k] * q[o*K + k] (+ bias[o]) where q is the tensor qd_unpack_dequant_* writes: every weight is
// from_unit(unit[code], alpha[bucket], beta[bucket]) with the unit table of load_unit_table.
//
// A warp owns four consecutive output features and walks their rows with the quad walk of qd_packed_walk.cuh, then
// folds its 32 partial sums with warp_sum's fixed xor butterfly: the order is fixed by K and BITS alone, so neither the
// grid, the chunking of x nor the batch size m changes a single bit of y[i, o].
//
// x rows m0 .. m0+MT-1 (MT = 1, 2, 4, 8 accumulators per lane and row, blockIdx.y = row tile) are staged in shared
// memory, in chunks of kc columns when MT*K floats exceed kPlSmemBytes.  With one chunk the tile is staged once and
// the CTA walks its slabs of output features; with several, each slab restages them.
constexpr int kPlSlab = kPlWarps * kPlRowsPerWarp;   // output features per CTA iteration

struct PackedLinearArgs {
    const float* x;
    const uint8_t* packed;
    const float* alpha;
    const float* beta;
    const float* points;
    const float* bias;
    float* y;
    int64_t m, K, O;
    int64_t in_bytes;           // ceil(O*K*bits/8)
    int64_t L, rows;            // bucket row length and bucket count (geometry_of)
    int64_t step_q, step_r;     // (128*E) / L and (128*E) % L: a lane's bucket cursor from one of its quads to the next
    int64_t kc;                 // columns per chunk of the x tile, a multiple of 128*E
    int num_points;
    float S;
    bool quad_aligned;          // packed 16-byte aligned and K*bits a multiple of 128: every quad is one aligned load
    bool x_vec;                 // x 16-byte aligned and K a multiple of 4
};

template <bool UNIFORM, int BITS, int MT>
__global__ void __launch_bounds__(kPlThreads, 1) packed_linear_kernel(PackedLinearArgs a) {
    constexpr int E = 32 / BITS;
    extern __shared__ float4 s_x[];
    __shared__ float s_unit[256];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t m0 = (int64_t)blockIdx.y * MT;
    const int kc4 = (int)(a.kc / 4);
    const int64_t kq = a.kc / (4 * E);                    // quads per chunk (a multiple of 32)
    const int64_t qpr = (a.K + 4 * E - 1) / (4 * E);      // quads per weight row
    const int64_t chunks = (a.K + a.kc - 1) / a.kc;
    const int64_t slabs = (a.O + kPlSlab - 1) / kPlSlab;
    auto x_row = [&](int64_t i) { return a.x + i * a.K; };
    load_unit_table<UNIFORM>(s_unit, a.points, a.num_points, a.S);
    if (chunks == 1) pl_stage<BITS, MT>(s_x, x_row, m0, a.m, a.K, a.kc, kc4, a.x_vec, 0);
    __syncthreads();
    for (int64_t slab = blockIdx.x; slab < slabs; slab += gridDim.x) {
        // rows past O repeat row O-1: computed, never written
        int64_t orow[kPlRowsPerWarp];
#pragma unroll
        for (int r = 0; r < kPlRowsPerWarp; ++r) {
            const int64_t o = slab * kPlSlab + warp * kPlRowsPerWarp + r;
            orow[r] = o < a.O ? o : a.O - 1;
        }
        float acc[kPlRowsPerWarp][MT];
#pragma unroll
        for (int r = 0; r < kPlRowsPerWarp; ++r)
#pragma unroll
            for (int i = 0; i < MT; ++i) acc[r][i] = 0.f;
        for (int64_t c = 0; c < chunks; ++c) {
            if (chunks > 1) {
                __syncthreads();
                pl_stage<BITS, MT>(s_x, x_row, m0, a.m, a.K, a.kc, kc4, a.x_vec, c);
                __syncthreads();
            }
            pl_walk<BITS, MT>(a, s_unit, s_x, kc4, kq, qpr, c, lane, orow, acc);
        }
#pragma unroll
        for (int r = 0; r < kPlRowsPerWarp; ++r) {
            const int64_t o = slab * kPlSlab + warp * kPlRowsPerWarp + r;
            const float b = (a.bias != nullptr && o < a.O) ? __ldg(a.bias + o) : 0.f;
#pragma unroll
            for (int i = 0; i < MT; ++i) {
                float s = warp_sum(acc[r][i]);
                if (a.bias != nullptr) s = __fadd_rn(s, b);
                if (lane == 0 && o < a.O && m0 + i < a.m) a.y[(m0 + i) * a.O + o] = s;
            }
        }
    }
}

template <int MT, bool UNIFORM, int BITS>
static int launch_packed_linear(PackedLinearArgs a, cudaStream_t st) {
    constexpr int64_t step_cols = 32 * 4 * (32 / BITS);   // columns of one warp-wide step
    a.kc = pl_chunk_cols<MT, BITS>(a.K);
    a.step_q = step_cols / a.L;
    a.step_r = step_cols % a.L;
    const size_t smem = (size_t)MT * a.kc * sizeof(float);
    auto kern = packed_linear_kernel<UNIFORM, BITS, MT>;
    static size_t opted[64] = {};
    int rc = opt_in_smem((const void*)kern, smem, opted);
    if (rc) return rc;
    const int64_t row_tiles = (a.m + MT - 1) / MT;
    int grid;
    const int64_t slabs = (a.O + kPlSlab - 1) / kPlSlab;
    rc = resident_grid((const void*)kern, kPlThreads, smem, slabs * row_tiles, &grid);
    if (rc) return rc;
    grid = std::max(1, grid / (int)row_tiles);           // at most one resident wave over all row tiles
    kern<<<dim3((unsigned)grid, (unsigned)row_tiles), kPlThreads, smem, st>>>(a);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

extern "C" int qd_packed_linear(const float* x, int64_t m, int64_t in_features, int64_t out_features, const uint8_t* packed,
                                int bits, const float* alpha, const float* beta, const float* points, int num_points, int levels,
                                int64_t bucket, const float* bias, float* y, qd_stream_t stream) {
    if (x == nullptr || packed == nullptr || alpha == nullptr || beta == nullptr || y == nullptr)
        return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if (m < 1) return fail(QD_ERR_INVALID_ARG, "m must be >= 1 (got %lld)", (long long)m);
    if (m > QD_PACKED_LINEAR_MAX_ROWS)
        return fail(QD_ERR_UNSUPPORTED, "m = %lld rows: the packed linear kernel serves at most %d", (long long)m, QD_PACKED_LINEAR_MAX_ROWS);
    if (in_features < 1 || out_features < 1) return fail(QD_ERR_INVALID_ARG, "in_features and out_features must be >= 1");
    if (in_features > INT64_MAX / 8 / out_features) return fail(QD_ERR_INVALID_ARG, "in_features * out_features is too large");
    if (!bits_ok(bits)) return fail(QD_ERR_INVALID_ARG, "bits must be 1, 2, 4 or 8");
    const bool uniform = levels != 0;
    if (uniform) {
        if (points != nullptr || num_points != 0) return fail(QD_ERR_INVALID_ARG, "uniform weights have no points (points NULL, num_points 0)");
        if (levels < 2 || levels > (1 << bits)) return fail(QD_ERR_INVALID_ARG, "levels must be in [2, 2^bits]");
    } else if (points == nullptr || num_points < 1 || num_points > (1 << bits)) {
        return fail(QD_ERR_INVALID_ARG, "num_points must be in [1, 2^bits]");
    }
    Geometry geo;
    const int64_t n = in_features * out_features;
    if (geometry_of(n, bucket, &geo)) return fail(QD_ERR_INVALID_ARG, "bucket must be >= 0");
    const uintptr_t xb = reinterpret_cast<uintptr_t>(x), xe = xb + (uintptr_t)(m * in_features) * sizeof(float);
    const uintptr_t yb = reinterpret_cast<uintptr_t>(y), ye = yb + (uintptr_t)(m * out_features) * sizeof(float);
    if (xb < ye && yb < xe) return fail(QD_ERR_INVALID_ARG, "y must not overlap x");
    PackedLinearArgs a{};
    a.x = x, a.packed = packed, a.alpha = alpha, a.beta = beta, a.points = points, a.bias = bias, a.y = y;
    a.m = m, a.K = in_features, a.O = out_features;
    a.in_bytes = (n * bits + 7) / 8;
    a.L = geo.row_len;
    a.rows = geo.rows;
    a.num_points = num_points;
    a.S = uniform ? (float)(levels - 1) : 0.f;
    a.quad_aligned = aligned16(packed) && (in_features * bits) % 128 == 0;
    a.x_vec = aligned16(x) && in_features % 4 == 0;
    cudaStream_t st = as_stream(stream);
    auto go = [&](auto mt) {
        return with_bits(bits, [&](auto b) {
            return uniform ? launch_packed_linear<mt, true, b>(a, st) : launch_packed_linear<mt, false, b>(a, st);
        });
    };
    if (m == 1) return go(std::integral_constant<int, 1>{});
    if (m == 2) return go(std::integral_constant<int, 2>{});
    if (m <= 4) return go(std::integral_constant<int, 4>{});
    return go(std::integral_constant<int, 8>{});
}

// ------------------------------------------------------------------ f2: convolution on packed weights
// y[n, o, ho, wo] = sum_k x[n, c, ho*sh - ph + r, wo*sw - pw + s] * q[o*K + k] (+ bias[o]), k = (c*kh + r)*kw + s,
// K = C*kh*kw, taps outside the input read 0.  q is the tensor qd_unpack_dequant_* writes: every weight is
// from_unit(unit[code], alpha[bucket], beta[bucket]) with the unit table of load_unit_table.
//
// Implicit GEMM over M = N*Ho*Wo output positions x O channels x K taps.  A CTA owns a tile of kPcBM positions and
// kPcBO channels and walks K in slabs of kPcBK taps: it decodes the slab's weights from the codes into shared memory
// (each thread four consecutive taps of one channel, a bucket cursor instead of a division), gathers the matching
// input patch (each thread four consecutive taps of one position, a (c, r, s) cursor, padding zero-filled), then every
// thread runs a 4 x 4 register micro-tile.  Each output is one fmaf chain over k = 0 .. K-1 in order, the bias added
// last: the order depends on the layer alone, not on N, H, W, the grid or timing.
constexpr int kPcBM = 64, kPcBO = 64, kPcBK = 16;
constexpr int kPcThreads = 256;

struct PackedConvArgs {
    const float* x;
    const uint8_t* packed;
    const float* alpha;
    const float* beta;
    const float* points;
    const float* bias;
    float* y;
    int64_t M, O, C, HW, HoWo;  // positions, channels, input channels, input and output plane sizes
    int64_t L, rows;            // bucket row length and bucket count (geometry_of)
    int64_t step_q, step_r;     // kPcBK / L and kPcBK % L: a bucket cursor from one slab to the next
    int K, H, W, Wo, kh, kw, sh, sw, ph, pw;
    int step_c, step_rr, step_s;  // kPcBK taps as (channels, rows, columns) of the window
    int num_points;
    float S;
};

template <bool UNIFORM, int BITS>
__global__ void __launch_bounds__(kPcThreads, 2) packed_conv2d_kernel(PackedConvArgs a) {
    constexpr unsigned mask = (1u << BITS) - 1u;
    __shared__ float s_unit[256];
    __shared__ __align__(16) float s_x[kPcBK][kPcBM];
    __shared__ __align__(16) float s_w[kPcBK][kPcBO];
    const int t = threadIdx.x;
    const int64_t m0 = (int64_t)blockIdx.x * kPcBM, o0 = (int64_t)blockIdx.y * kPcBO;
    const int lane4 = (t >> 6) * 4;     // first of the four taps this thread gathers and decodes per slab

    // gather role: position m0 + (t & 63); tap cursor (gc, gr, gs) of tap lane4 of the slab
    const int64_t gpos = m0 + (t & 63);
    const bool gvalid = gpos < a.M;
    const float* xb = a.x;
    int hi0 = 0, wi0 = 0;
    if (gvalid) {
        const int64_t n = gpos / a.HoWo;
        const int p = (int)(gpos - n * a.HoWo);
        const int ho = p / a.Wo, wo = p - ho * a.Wo;
        xb = a.x + n * a.C * a.HW;
        hi0 = ho * a.sh - a.ph;
        wi0 = wo * a.sw - a.pw;
    }
    int gc = lane4 / (a.kh * a.kw), gr = lane4 - gc * a.kh * a.kw, gs = gr % a.kw;
    gr /= a.kw;

    // decode role: channel o0 + (t & 63), elements o*K + k0 + lane4 .. +3; bucket cursor (bc, rc) of the first
    const int64_t o = o0 + (t & 63);
    const bool ovalid = o < a.O;
    const int64_t e_first = (ovalid ? o : 0) * a.K + lane4;
    int64_t bc = e_first / a.L, rc = e_first - bc * a.L;

    load_unit_table<UNIFORM>(s_unit, a.points, a.num_points, a.S);
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    const int tx = t & 15, ty = t >> 4;   // micro-tile: positions m0 + 4*tx .. +3, channels o0 + 4*ty .. +3

    for (int k0 = 0; k0 < a.K; k0 += kPcBK) {
        __syncthreads();                  // the previous slab is consumed (and, at the first, the unit table written)
        {   // input patch: taps k0 + lane4 + j of position gpos
            int c = gc, r = gr, s = gs;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int hi = hi0 + r, wi = wi0 + s;
                float v = 0.f;
                if (gvalid && c < a.C && (unsigned)hi < (unsigned)a.H && (unsigned)wi < (unsigned)a.W)
                    v = __ldg(xb + (int64_t)c * a.HW + (int64_t)hi * a.W + wi);
                s_x[lane4 + j][t & 63] = v;
                if (++s == a.kw) {
                    s = 0;
                    if (++r == a.kh) { r = 0; ++c; }
                }
            }
        }
        {   // weights: elements o*K + k0 + lane4 + j, walked with the bucket cursor
            int64_t b = bc, rr = rc;
            float al = __ldg(a.alpha + min(b, a.rows - 1)), be = __ldg(a.beta + min(b, a.rows - 1));
            const int64_t e0 = o * a.K + k0 + lane4;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                float w = 0.f;
                if (ovalid && k0 + lane4 + j < a.K) {
                    const int64_t bit = (e0 + j) * BITS;
                    const unsigned code = ((unsigned)__ldg(a.packed + (bit >> 3)) >> (unsigned)(bit & 7)) & mask;
                    w = from_unit(s_unit[code], al, be);
                }
                s_w[lane4 + j][t & 63] = w;
                if (++rr == a.L) {        // next element starts bucket b + 1
                    rr = 0;
                    ++b;
                    al = __ldg(a.alpha + min(b, a.rows - 1));
                    be = __ldg(a.beta + min(b, a.rows - 1));
                }
            }
        }
        // advance both cursors by one slab
        bc += a.step_q;
        rc += a.step_r;
        if (rc >= a.L) { rc -= a.L; ++bc; }
        gs += a.step_s;
        if (gs >= a.kw) { gs -= a.kw; ++gr; }
        gr += a.step_rr;
        if (gr >= a.kh) { gr -= a.kh; ++gc; }
        gc += a.step_c;
        __syncthreads();
        const int kn = min(kPcBK, a.K - k0);
#pragma unroll
        for (int kk = 0; kk < kPcBK; ++kk) {
            if (kk < kn) {
                const float4 xv = *reinterpret_cast<const float4*>(&s_x[kk][4 * tx]);
                const float4 wv = *reinterpret_cast<const float4*>(&s_w[kk][4 * ty]);
                const float xs[4] = {xv.x, xv.y, xv.z, xv.w}, ws[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) acc[i][j] = __fmaf_rn(xs[i], ws[j], acc[i][j]);
            }
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int64_t m = m0 + 4 * tx + i;
        if (m >= a.M) break;
        const int64_t n = m / a.HoWo;
        float* yb = a.y + n * a.O * a.HoWo + (m - n * a.HoWo);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int64_t oc = o0 + 4 * ty + j;
            if (oc < a.O) yb[oc * a.HoWo] = a.bias != nullptr ? __fadd_rn(acc[i][j], __ldg(a.bias + oc)) : acc[i][j];
        }
    }
}

static bool mul_ok(int64_t p, int64_t q, int64_t* out) { return !__builtin_mul_overflow(p, q, out); }

extern "C" int qd_packed_conv2d(const float* x, int64_t batch, int64_t in_channels, int64_t height, int64_t width,
                                int64_t out_channels, int kernel_h, int kernel_w, int stride_h, int stride_w, int pad_h, int pad_w,
                                const uint8_t* packed, int bits, const float* alpha, const float* beta, const float* points,
                                int num_points, int levels, int64_t bucket, const float* bias, float* y, qd_stream_t stream) {
    if (x == nullptr || packed == nullptr || alpha == nullptr || beta == nullptr || y == nullptr)
        return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if (batch < 1 || in_channels < 1 || height < 1 || width < 1 || out_channels < 1 || kernel_h < 1 || kernel_w < 1)
        return fail(QD_ERR_INVALID_ARG, "batch, channels, input and kernel sizes must be >= 1");
    if (stride_h < 1 || stride_w < 1 || pad_h < 0 || pad_w < 0) return fail(QD_ERR_INVALID_ARG, "strides must be >= 1 and padding >= 0");
    if (height > INT32_MAX / 4 || width > INT32_MAX / 4 || pad_h > INT32_MAX / 4 || pad_w > INT32_MAX / 4)
        return fail(QD_ERR_UNSUPPORTED, "input sides and padding must be below 2^29");
    const int64_t hp = height + 2 * (int64_t)pad_h, wp = width + 2 * (int64_t)pad_w;
    if (hp < kernel_h || wp < kernel_w)
        return fail(QD_ERR_INVALID_ARG, "the %dx%d kernel is larger than the padded %lldx%lld input: the output is empty", kernel_h,
                    kernel_w, (long long)hp, (long long)wp);
    const int64_t ho = (hp - kernel_h) / stride_h + 1, wo = (wp - kernel_w) / stride_w + 1;
    int64_t K, n, hw, howo, x_n, y_n, m;
    if (!mul_ok(in_channels, (int64_t)kernel_h * kernel_w, &K) || !mul_ok(K, out_channels, &n) || n > INT64_MAX / 8 ||
        !mul_ok(height, width, &hw) || !mul_ok(ho, wo, &howo) || !mul_ok(hw, in_channels, &x_n) || !mul_ok(x_n, batch, &x_n) ||
        !mul_ok(howo, out_channels, &y_n) || !mul_ok(y_n, batch, &y_n) || !mul_ok(howo, batch, &m) || x_n > INT64_MAX / 4 ||
        y_n > INT64_MAX / 4)
        return fail(QD_ERR_INVALID_ARG, "the layer's sizes overflow 64-bit indexing");
    if (K > INT32_MAX) return fail(QD_ERR_UNSUPPORTED, "K = in_channels * kernel_h * kernel_w = %lld: at most 2^31 - 1", (long long)K);
    const int64_t m_tiles = (m + kPcBM - 1) / kPcBM, o_tiles = (out_channels + kPcBO - 1) / kPcBO;
    if (m_tiles > INT32_MAX || o_tiles > 65535)
        return fail(QD_ERR_UNSUPPORTED, "%lld output positions x %lld channels: more tiles than one launch holds", (long long)m,
                    (long long)out_channels);
    if (!bits_ok(bits)) return fail(QD_ERR_INVALID_ARG, "bits must be 1, 2, 4 or 8");
    const bool uniform = levels != 0;
    if (uniform) {
        if (points != nullptr || num_points != 0) return fail(QD_ERR_INVALID_ARG, "uniform weights have no points (points NULL, num_points 0)");
        if (levels < 2 || levels > (1 << bits)) return fail(QD_ERR_INVALID_ARG, "levels must be in [2, 2^bits]");
    } else if (points == nullptr || num_points < 1 || num_points > (1 << bits)) {
        return fail(QD_ERR_INVALID_ARG, "num_points must be in [1, 2^bits]");
    }
    Geometry geo;
    if (geometry_of(n, bucket, &geo)) return fail(QD_ERR_INVALID_ARG, "bucket must be >= 0");
    const uintptr_t xb = reinterpret_cast<uintptr_t>(x), xe = xb + (uintptr_t)x_n * sizeof(float);
    const uintptr_t yb = reinterpret_cast<uintptr_t>(y), ye = yb + (uintptr_t)y_n * sizeof(float);
    if (xb < ye && yb < xe) return fail(QD_ERR_INVALID_ARG, "y must not overlap x");
    PackedConvArgs a{};
    a.x = x, a.packed = packed, a.alpha = alpha, a.beta = beta, a.points = points, a.bias = bias, a.y = y;
    a.M = m, a.O = out_channels, a.C = in_channels, a.HW = hw, a.HoWo = howo;
    a.L = geo.row_len, a.rows = geo.rows;
    a.step_q = kPcBK / a.L, a.step_r = kPcBK % a.L;
    a.K = (int)K, a.H = (int)height, a.W = (int)width, a.Wo = (int)wo;
    a.kh = kernel_h, a.kw = kernel_w, a.sh = stride_h, a.sw = stride_w, a.ph = pad_h, a.pw = pad_w;
    const int taps = kernel_h * kernel_w;
    a.step_c = kPcBK / taps, a.step_rr = (kPcBK % taps) / kernel_w, a.step_s = (kPcBK % taps) % kernel_w;
    a.num_points = num_points;
    a.S = uniform ? (float)(levels - 1) : 0.f;
    const dim3 grid((unsigned)m_tiles, (unsigned)o_tiles);
    cudaStream_t st = as_stream(stream);
    with_bits(bits, [&](auto b) {
        if (uniform) packed_conv2d_kernel<true, b><<<grid, kPcThreads, 0, st>>>(a);
        else packed_conv2d_kernel<false, b><<<grid, kPcThreads, 0, st>>>(a);
    });
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

// ------------------------------------------------------------------ f2: embedding lookup on packed weights
// out[i, d] = q[idx_i*D + d] where q is the tensor qd_unpack_dequant_* writes: every value is
// from_unit(unit[code], alpha[bucket], beta[bucket]) with the unit table of load_unit_table, and nothing else.
//
// A row of D outputs is served by lpr lanes, the power of two >= ceil(D/4) up to 32, so a warp serves 32/lpr rows at
// once and the grid covers the count rows once, without a grid stride.  Lane l of a row takes the groups of four
// columns 4*l, 4*(l + lpr), ...: so the lanes of a row read one contiguous span of codes per step.  A group's 4*bits
// code bits are one or two aligned 32-bit words funnel-shifted (a row starts inside a byte whenever D*bits is not a
// multiple of 8); a word that reaches past the last code byte is read byte by byte up to it.  A bucket cursor per
// group (one division per row, then one compare per element) gives each element its (alpha, beta).  An index outside
// [0, V) is never dereferenced: its row is written NaN and counted once in *invalid.
constexpr int kPeThreads = 256;

struct PackedEmbeddingArgs {
    const void* indices;
    const uint8_t* packed;
    const float* alpha;
    const float* beta;
    const float* points;
    float* out;
    int32_t* invalid;           // may be NULL
    int64_t count, V, D;
    int64_t in_bytes;           // ceil(V*D*bits/8)
    int64_t L, rows;            // bucket row length and bucket count (geometry_of)
    int64_t step_q, step_r;     // (4*lpr) / L and (4*lpr) % L: a lane's bucket cursor from one of its groups to the next
    int lpr_log2;               // log2 of the lanes per row
    int index_bytes;            // 4 or 8
    int num_points;
    float S;
    bool words_aligned;         // packed 4-byte aligned: a code word inside the tensor is one load
};

// 32-bit code word w (bytes 4w .. 4w+3 of packed); bytes at or past in_bytes read as 0 and are never loaded
__device__ __forceinline__ uint32_t pe_word(const PackedEmbeddingArgs& a, int64_t w) {
    const int64_t b0 = 4 * w;
    if (a.words_aligned && b0 + 4 <= a.in_bytes) return __ldg(reinterpret_cast<const unsigned int*>(a.packed) + w);
    uint32_t v = 0;
    for (int i = 0; i < 4; ++i)
        if (b0 + i < a.in_bytes) v |= (uint32_t)__ldg(a.packed + b0 + i) << (8 * i);
    return v;
}

template <bool UNIFORM, int BITS>
__global__ void __launch_bounds__(kPeThreads) packed_embedding_kernel(PackedEmbeddingArgs a) {
    constexpr unsigned mask = (1u << BITS) - 1u;
    __shared__ float s_unit[256];
    const int lpr = 1 << a.lpr_log2, step = 4 << a.lpr_log2;
    const int sub = (int)threadIdx.x & (lpr - 1);
    const int64_t i = ((int64_t)blockIdx.x * kPeThreads + threadIdx.x) >> a.lpr_log2;
    int64_t r = 0;
    if (i < a.count)                                        // in flight while the unit table is built
        r = a.index_bytes == 8 ? (int64_t)__ldg(static_cast<const long long*>(a.indices) + i)
                               : (int64_t)__ldg(static_cast<const int*>(a.indices) + i);
    load_unit_table<UNIFORM>(s_unit, a.points, a.num_points, a.S);
    __syncthreads();
    // lpr is a power of two, so D of 9-12, 17-28, ... leaves lanes with no group in the row: their first element would
    // lie past the row, its bucket past the scale arrays at the tensor's end
    if (i >= a.count || 4 * sub >= a.D) return;
    float* dst = a.out + i * a.D;
    const bool vec = (reinterpret_cast<uintptr_t>(dst) & 15) == 0;
    auto store = [&](int64_t c, const float (&o)[4]) {
        if (vec && c + 4 <= a.D) {
            *reinterpret_cast<float4*>(dst + c) = make_float4(o[0], o[1], o[2], o[3]);
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (c + j < a.D) dst[c + j] = o[j];
        }
    };
    if (r < 0 || r >= a.V) {
        const float nan = __int_as_float(0x7fc00000);
        const float o[4] = {nan, nan, nan, nan};
        for (int64_t c = 4 * sub; c < a.D; c += step) store(c, o);
        if (sub == 0 && a.invalid != nullptr) atomicAdd(a.invalid, 1);
        return;
    }
    // what a group reads -- its one or two code words and the (alpha, beta) of its first bucket -- is fetched one group
    // ahead, so that the loads of the next group are in flight while this one is decoded and stored
    struct Fetched { uint32_t lo, hi; float al, be; };
    auto fetch = [&](int64_t e, int64_t b, Fetched& f) {
        const int64_t bit = e * BITS;
        f.lo = pe_word(a, bit >> 5);
        f.hi = (int)(bit & 31) + 4 * BITS > 32 ? pe_word(a, (bit >> 5) + 1) : 0u;
        f.al = __ldg(a.alpha + b);
        f.be = __ldg(a.beta + b);
    };
    int64_t e = r * a.D + 4 * sub;                          // first element of the lane's group
    int64_t bg = e / a.L, rg = e - bg * a.L;                // its bucket and offset in it
    Fetched cur;
    fetch(e, bg, cur);
    for (int64_t c = 4 * sub; c < a.D; c += step, e += step) {
        int64_t nb = bg + a.step_q, nr = rg + a.step_r;     // the cursor of the lane's next group
        if (nr >= a.L) { nr -= a.L; ++nb; }
        Fetched nxt = cur;
        if (c + step < a.D) fetch(e + step, nb, nxt);
        const uint32_t codes = __funnelshift_r(cur.lo, cur.hi, (unsigned)(e * BITS) & 31u);
        int64_t b = bg, rr = rg;
        float al = cur.al, be = cur.be;
        float o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            o[j] = from_unit(s_unit[(codes >> (j * BITS)) & mask], al, be);
            if (j < 3 && ++rr == a.L) {                     // the next element starts bucket b + 1
                rr = 0;
                b = min(b + 1, a.rows - 1);                 // past the last bucket only beyond the tensor's end
                al = __ldg(a.alpha + b);
                be = __ldg(a.beta + b);
            }
        }
        store(c, o);
        bg = nb;
        rg = nr;
        cur = nxt;
    }
}

extern "C" int qd_packed_embedding(const void* indices, int index_bytes, int64_t count, int64_t num_embeddings, int64_t dim,
                                   const uint8_t* packed, int bits, const float* alpha, const float* beta, const float* points,
                                   int num_points, int levels, int64_t bucket, float* out, int32_t* invalid, qd_stream_t stream) {
    if (indices == nullptr || packed == nullptr || alpha == nullptr || beta == nullptr || out == nullptr)
        return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if (index_bytes != 4 && index_bytes != 8) return fail(QD_ERR_INVALID_ARG, "index_bytes must be 4 (int32) or 8 (int64), got %d", index_bytes);
    if (count < 1 || num_embeddings < 1 || dim < 1) return fail(QD_ERR_INVALID_ARG, "count, num_embeddings and dim must be >= 1");
    if (num_embeddings > INT64_MAX / 8 / dim) return fail(QD_ERR_INVALID_ARG, "num_embeddings * dim is too large");
    if (count > INT64_MAX / 4 / dim) return fail(QD_ERR_INVALID_ARG, "count * dim overflows 64-bit indexing");
    if (!bits_ok(bits)) return fail(QD_ERR_INVALID_ARG, "bits must be 1, 2, 4 or 8");
    const bool uniform = levels != 0;
    if (uniform) {
        if (points != nullptr || num_points != 0) return fail(QD_ERR_INVALID_ARG, "uniform weights have no points (points NULL, num_points 0)");
        if (levels < 2 || levels > (1 << bits)) return fail(QD_ERR_INVALID_ARG, "levels must be in [2, 2^bits]");
    } else if (points == nullptr || num_points < 1 || num_points > (1 << bits)) {
        return fail(QD_ERR_INVALID_ARG, "num_points must be in [1, 2^bits]");
    }
    Geometry geo;
    const int64_t n = num_embeddings * dim;
    if (geometry_of(n, bucket, &geo)) return fail(QD_ERR_INVALID_ARG, "bucket must be >= 0");
    int lpr_log2 = 0;
    while (lpr_log2 < 5 && (int64_t)4 << lpr_log2 < dim) ++lpr_log2;
    const int64_t rows_per_cta = kPeThreads >> lpr_log2;
    const int64_t ctas = (count + rows_per_cta - 1) / rows_per_cta;
    if (ctas > INT32_MAX) return fail(QD_ERR_UNSUPPORTED, "%lld indices: more rows than one launch holds", (long long)count);
    const uintptr_t ib = reinterpret_cast<uintptr_t>(indices), ie = ib + (uintptr_t)count * index_bytes;
    const uintptr_t ob = reinterpret_cast<uintptr_t>(out), oe = ob + (uintptr_t)(count * dim) * sizeof(float);
    if (ib < oe && ob < ie) return fail(QD_ERR_INVALID_ARG, "out must not overlap the indices");
    PackedEmbeddingArgs a{};
    a.indices = indices, a.packed = packed, a.alpha = alpha, a.beta = beta, a.points = points, a.out = out, a.invalid = invalid;
    a.count = count, a.V = num_embeddings, a.D = dim;
    a.in_bytes = (n * bits + 7) / 8;
    a.L = geo.row_len, a.rows = geo.rows;
    a.step_q = ((int64_t)4 << lpr_log2) / a.L, a.step_r = ((int64_t)4 << lpr_log2) % a.L;
    a.lpr_log2 = lpr_log2;
    a.index_bytes = index_bytes;
    a.num_points = num_points;
    a.S = uniform ? (float)(levels - 1) : 0.f;
    a.words_aligned = (reinterpret_cast<uintptr_t>(packed) & 3) == 0;
    cudaStream_t st = as_stream(stream);
    with_bits(bits, [&](auto b) {
        if (uniform) packed_embedding_kernel<true, b><<<(unsigned)ctas, kPeThreads, 0, st>>>(a);
        else packed_embedding_kernel<false, b><<<(unsigned)ctas, kPeThreads, 0, st>>>(a);
    });
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
    cudaStream_t s = as_stream(stream);
    const int64_t chunks = (n + kHuffChunk - 1) / kHuffChunk;
    huff_chunk_words_kernel<<<di->grid((chunks + 7) / 8, 8), 256, 0, s>>>(idx_u8, n, table, chunk_offsets, chunks);
    huff_scan_kernel<<<1, 1024, 0, s>>>(chunk_offsets, chunks, reinterpret_cast<unsigned long long*>(total_words));
    if (words_capacity > 0)
        huff_encode_kernel<<<di->grid((chunks + kHuffEncWarps - 1) / kHuffEncWarps, 8), kHuffEncWarps * 32, 0, s>>>(
            idx_u8, n, table, chunk_offsets, reinterpret_cast<const unsigned long long*>(total_words), chunks, words_out, words_capacity);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

// Checks the arguments both per-tensor decodes share and launches huff_decode_dequant_kernel<UNIFORM>.
template <bool UNIFORM>
static int huff_decode_dequant(const uint32_t* words, int64_t num_words, const uint32_t* chunk_offsets, const qd_huffman_table* table,
                               const float* points, int K, const float* alpha, const float* beta, float* q, int64_t n,
                               int64_t bucket, float S, qd_stream_t stream) {
    Geometry geo;
    if (chunk_offsets == nullptr || table == nullptr || alpha == nullptr || beta == nullptr || q == nullptr)
        return fail(QD_ERR_INVALID_ARG, "NULL argument");
    if (num_words < 0 || (num_words > 0 && words == nullptr)) return fail(QD_ERR_INVALID_ARG, "bad words / num_words");
    if (geometry_of(n, bucket, &geo)) return fail(QD_ERR_INVALID_ARG, "bad geometry");
    const int64_t chunks = (n + kHuffChunk - 1) / kHuffChunk;
    int grid;
    int rc = capped_grid((chunks + kHuffDecThreads - 1) / kHuffDecThreads, 16, &grid);
    if (rc) return rc;
    huff_decode_dequant_kernel<UNIFORM><<<grid, kHuffDecThreads, 0, as_stream(stream)>>>(
        words, num_words, chunk_offsets, table, points, K, alpha, beta, q, geo, S, chunks);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

extern "C" int qd_huffman_decode_dequant_uniform(const uint32_t* words, int64_t num_words, const uint32_t* chunk_offsets,
                                                 const qd_huffman_table* table, const float* alpha, const float* beta, float* q,
                                                 int64_t n, int64_t bucket, int levels, qd_stream_t stream) {
    if (levels < 2 || levels > 256) return fail(QD_ERR_INVALID_ARG, "levels must be in [2, 256]");
    return huff_decode_dequant<true>(words, num_words, chunk_offsets, table, nullptr, 0, alpha, beta, q, n, bucket,
                                     (float)(levels - 1), stream);
}

extern "C" int qd_huffman_decode_dequant_nonuniform(const uint32_t* words, int64_t num_words, const uint32_t* chunk_offsets,
                                                    const qd_huffman_table* table, const float* points, int num_points,
                                                    const float* alpha, const float* beta, float* q, int64_t n, int64_t bucket,
                                                    qd_stream_t stream) {
    if (points == nullptr || num_points < 1 || num_points > 256) return fail(QD_ERR_INVALID_ARG, "num_points must be in [1, 256]");
    return huff_decode_dequant<false>(words, num_words, chunk_offsets, table, points, num_points, alpha, beta, q, n, bucket, 0.f,
                                      stream);
}

static_assert(sizeof(qd_huffman_tensor) == 72, "qd_huffman_tensor layout is shared with codec.py");

extern "C" size_t qd_huffman_model_workspace_bytes(int count) { return model_workspace_bytes<qd_huffman_tensor>(count); }

extern "C" int qd_huffman_decode_dequant_model(const qd_huffman_tensor* tensors, int count, const qd_huffman_table* table,
                                               int64_t bucket, int levels, void* workspace, size_t workspace_bytes,
                                               qd_stream_t stream) {
    if (tensors == nullptr || count < 1 || table == nullptr) return fail(QD_ERR_INVALID_ARG, "NULL tensors / table or count < 1");
    if (bucket < 0) return fail(QD_ERR_INVALID_ARG, "bucket must be >= 0");
    if (levels != 0 && (levels < 2 || levels > 256)) return fail(QD_ERR_INVALID_ARG, "levels must be in [2, 256] (uniform) or 0 (non-uniform)");
    const bool uniform = levels != 0;
    auto ctas_of = [&](int i, const qd_huffman_tensor& t, int64_t* ctas) {
        if (t.chunk_offsets == nullptr || t.alpha == nullptr || t.beta == nullptr || t.q == nullptr)
            return fail(QD_ERR_INVALID_ARG, "tensor %d: NULL argument", i);
        if (t.num_words < 0 || (t.num_words > 0 && t.words == nullptr)) return fail(QD_ERR_INVALID_ARG, "tensor %d: bad words / num_words", i);
        if (t.n < 1) return fail(QD_ERR_INVALID_ARG, "tensor %d: n must be >= 1", i);
        if (t.reserved != 0) return fail(QD_ERR_INVALID_ARG, "tensor %d: reserved must be 0", i);
        if (uniform && (t.points != nullptr || t.num_points != 0))
            return fail(QD_ERR_INVALID_ARG, "tensor %d: a uniform model has no points (points NULL, num_points 0)", i);
        if (!uniform && (t.points == nullptr || t.num_points < 1 || t.num_points > 256))
            return fail(QD_ERR_INVALID_ARG, "tensor %d: num_points must be in [1, 256]", i);
        *ctas = ((t.n + kHuffChunk - 1) / kHuffChunk + kHuffDecThreads - 1) / kHuffDecThreads;
        return (int)QD_OK;
    };
    cudaStream_t st = as_stream(stream);
    unsigned ctas;
    const int32_t* dev_start;
    if (const int rc = upload_model(tensors, count, workspace, workspace_bytes, st, ctas_of, "blocks", kHuffDecThreads, "chunks",
                                    &ctas, &dev_start))
        return rc;
    const qd_huffman_tensor* dev_tensors = static_cast<const qd_huffman_tensor*>(workspace);
    if (uniform)
        huff_decode_dequant_model_kernel<true><<<ctas, kHuffDecThreads, 0, st>>>(dev_tensors, dev_start, count, table, bucket,
                                                                                 (float)(levels - 1));
    else
        huff_decode_dequant_model_kernel<false><<<ctas, kHuffDecThreads, 0, st>>>(dev_tensors, dev_start, count, table, bucket, 0.f);
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}

static_assert(sizeof(qd_huffman_repack_tensor) == 48, "qd_huffman_repack_tensor layout is shared with codec.py");

extern "C" size_t qd_huffman_repack_model_workspace_bytes(int count) { return model_workspace_bytes<qd_huffman_repack_tensor>(count); }

extern "C" int qd_huffman_decode_packed_model(const qd_huffman_repack_tensor* tensors, int count, const qd_huffman_table* table,
                                              int64_t* out_of_range, void* workspace, size_t workspace_bytes, qd_stream_t stream) {
    if (tensors == nullptr || count < 1 || table == nullptr || out_of_range == nullptr)
        return fail(QD_ERR_INVALID_ARG, "NULL tensors / table / out_of_range or count < 1");
    auto ctas_of = [&](int i, const qd_huffman_repack_tensor& t, int64_t* ctas) {
        if (t.chunk_offsets == nullptr || t.packed == nullptr) return fail(QD_ERR_INVALID_ARG, "tensor %d: NULL argument", i);
        if (t.num_words < 0 || (t.num_words > 0 && t.words == nullptr)) return fail(QD_ERR_INVALID_ARG, "tensor %d: bad words / num_words", i);
        if (t.n < 1) return fail(QD_ERR_INVALID_ARG, "tensor %d: n must be >= 1", i);
        if (!bits_ok(t.bits)) return fail(QD_ERR_INVALID_ARG, "tensor %d: bits must be 1, 2, 4 or 8", i);
        if (t.limit < 1 || t.limit > (1 << t.bits)) return fail(QD_ERR_INVALID_ARG, "tensor %d: limit must be in [1, 2^bits]", i);
        *ctas = ((t.n + kHuffChunk - 1) / kHuffChunk + kHuffDecThreads - 1) / kHuffDecThreads;
        return (int)QD_OK;
    };
    cudaStream_t st = as_stream(stream);
    unsigned ctas;
    const int32_t* dev_start;
    if (const int rc = upload_model(tensors, count, workspace, workspace_bytes, st, ctas_of, "blocks", kHuffDecThreads, "chunks",
                                    &ctas, &dev_start))
        return rc;
    huff_decode_packed_model_kernel<<<ctas, kHuffDecThreads, 0, st>>>(static_cast<const qd_huffman_repack_tensor*>(workspace), dev_start,
                                                                      count, table, reinterpret_cast<unsigned long long*>(out_of_range));
    QD_CUDA(cudaGetLastError());
    return QD_OK;
}
