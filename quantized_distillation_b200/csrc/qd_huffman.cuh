// qd_huffman.cuh -- Huffman-coded model storage: encoder (uint8 levels -> canonical-code bit stream) and
// decoder fused with the dequantization (bit stream -> float32 q) or with the fixed-width packing (bit stream ->
// 1/2/4/8-bit codes).
//
// Stream format (include/qd_b200.h, codec.py): every tensor's symbols are cut into chunks of QD_HUFFMAN_CHUNK;
// each chunk's codes are written MSB-first into 32-bit words starting on a fresh word, chunk_offsets[c] is the
// word where chunk c starts.  Chunks are the unit of parallelism on both sides: the encoder never has to merge
// two chunks' bits into one word, the decoder starts every chunk at a known word.
#pragma once
#include "qd_common.cuh"

namespace qd {

static_assert(sizeof(qd_huffman_table) == 13328, "qd_huffman_table layout is shared with codec.py");

constexpr int kHuffChunk = QD_HUFFMAN_CHUNK;
constexpr int kHuffLutBits = QD_HUFFMAN_LUT_BITS;
constexpr int kHuffImgWords = kHuffChunk * QD_HUFFMAN_MAX_LENGTH / 32;  // longest possible chunk, in words
constexpr int kHuffEncWarps = 4;
constexpr int kHuffDecThreads = 128;   // one chunk per thread
constexpr int kHuffDecRound = 32;      // symbols per thread between two coalesced store phases
constexpr int kHuffStageStride = kHuffDecRound / 4 + 1;  // words per thread row of the stage (+1: no bank conflicts)

// ---- encoder pass 1: one warp per chunk, words the chunk's codes occupy (written into chunk_offsets) ----------
__global__ void __launch_bounds__(256) huff_chunk_words_kernel(const uint8_t* __restrict__ idx, int64_t n,
                                                               const qd_huffman_table* __restrict__ tab,
                                                               uint32_t* __restrict__ chunk_words, int64_t chunks) {
    __shared__ uint32_t s_len[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) s_len[i] = tab->length[i];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    const bool vec = (reinterpret_cast<uintptr_t>(idx) & 3) == 0;
    for (int64_t c = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); c < chunks; c += warps) {
        const int64_t e0 = c * kHuffChunk;
        const int m = (int)(n - e0 < kHuffChunk ? n - e0 : kHuffChunk);
        uint32_t bits = 0;
        if (vec && m == kHuffChunk) {
            const uint32_t* w = reinterpret_cast<const uint32_t*>(idx + e0);
#pragma unroll
            for (int k = 0; k < kHuffChunk / 128; ++k) {
                const uint32_t v = __ldcs(w + k * 32 + lane);
                bits += s_len[v & 0xffu] + s_len[(v >> 8) & 0xffu] + s_len[(v >> 16) & 0xffu] + s_len[v >> 24];
            }
        } else {
            for (int j = lane; j < m; j += 32) bits += s_len[idx[e0 + j]];
        }
        bits = __reduce_add_sync(kFullMask, bits);
        if (lane == 0) chunk_words[c] = (bits + 31u) >> 5;
    }
}

// ---- encoder scan: exclusive prefix sum of the chunk word counts, in place, and the total ---------------------
// One CTA: the array has n/1024 entries (0.1 % of the bytes pass 1 reads), so a single CTA costs a few
// microseconds and needs no inter-CTA protocol; the sums are 64-bit so that an oversized stream is detected.
__global__ void __launch_bounds__(1024) huff_scan_kernel(uint32_t* __restrict__ offs, int64_t chunks,
                                                         unsigned long long* __restrict__ total) {
    __shared__ unsigned long long s_warp[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t per = (chunks + blockDim.x - 1) / blockDim.x;
    const int64_t b = (int64_t)threadIdx.x * per;
    const int64_t e = b + per < chunks ? b + per : chunks;
    unsigned long long sum = 0;
    for (int64_t i = b; i < e; ++i) sum += offs[i];
    unsigned long long incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long v = __shfl_up_sync(kFullMask, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        unsigned long long w = lane < (int)(blockDim.x >> 5) ? s_warp[lane] : 0ull;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long v = __shfl_up_sync(kFullMask, w, o);
            if (lane >= o) w += v;
        }
        s_warp[lane] = w;
    }
    __syncthreads();
    unsigned long long run = incl - sum + (warp ? s_warp[warp - 1] : 0ull);
    for (int64_t i = b; i < e; ++i) {
        const uint32_t w = offs[i];
        offs[i] = (uint32_t)run;
        run += w;
    }
    if (threadIdx.x == blockDim.x - 1) *total = run;
}

// code (len bits, right-aligned) at bit p of a chunk image, MSB-first; len + (p & 31) <= 88 spans <= 3 words
__device__ __forceinline__ void huff_place(uint32_t* img, unsigned long long code, uint32_t len, uint32_t p) {
    const uint32_t w = p >> 5, t = (p & 31u) + len;
    if (t <= 64) {
        const unsigned long long v = code << (64 - t);
        atomicOr(&img[w], (uint32_t)(v >> 32));
        if (t > 32) atomicOr(&img[w + 1], (uint32_t)v);
    } else {
        const unsigned long long v = code >> (t - 64);
        atomicOr(&img[w], (uint32_t)(v >> 32));
        atomicOr(&img[w + 1], (uint32_t)v);
        atomicOr(&img[w + 2], (uint32_t)(code << (96 - t)));
    }
}

// ---- encoder pass 2: one warp per chunk.  32 symbols per step: warp scan of the code lengths gives each code's
// bit position, the code is ORed into the chunk's image in shared memory, then the image leaves as coalesced word
// stores.  No global atomics: the output bytes do not depend on scheduling.  A chunk that would end beyond
// `capacity` words is not written (the caller compares *total with its capacity).
__global__ void __launch_bounds__(kHuffEncWarps * 32) huff_encode_kernel(const uint8_t* __restrict__ idx, int64_t n,
                                                                         const qd_huffman_table* __restrict__ tab,
                                                                         const uint32_t* __restrict__ offs,
                                                                         const unsigned long long* __restrict__ total,
                                                                         int64_t chunks, uint32_t* __restrict__ out,
                                                                         int64_t capacity) {
    __shared__ uint32_t s_img[kHuffEncWarps][kHuffImgWords];
    __shared__ unsigned long long s_code[256];
    __shared__ uint32_t s_len[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) {
        s_code[i] = tab->code[i];
        s_len[i] = tab->length[i];
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t* img = s_img[warp];
    const unsigned long long tot = *total;
    for (int64_t c = (int64_t)blockIdx.x * kHuffEncWarps + warp; c < chunks; c += (int64_t)gridDim.x * kHuffEncWarps) {
        const unsigned long long start = offs[c];
        const unsigned long long end = c + 1 < chunks ? (unsigned long long)offs[c + 1] : tot;
        if (end < start || end > (unsigned long long)capacity || end - start > (unsigned long long)kHuffImgWords) continue;
        const int words = (int)(end - start);
        for (int i = lane; i < words; i += 32) img[i] = 0u;
        __syncwarp();
        const int64_t e0 = c * kHuffChunk;
        const int m = (int)(n - e0 < kHuffChunk ? n - e0 : kHuffChunk);
        uint32_t base = 0;
        for (int j0 = 0; j0 < m; j0 += 32) {
            const int j = j0 + lane;
            const uint32_t sym = j < m ? idx[e0 + j] : 0u;
            const uint32_t len = j < m ? s_len[sym] : 0u;
            uint32_t incl = len;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t v = __shfl_up_sync(kFullMask, incl, o);
                if (lane >= o) incl += v;
            }
            if (len) huff_place(img, s_code[sym], len, base + incl - len);
            base += __shfl_sync(kFullMask, incl, 31);
        }
        __syncwarp();
        for (int i = lane; i < words; i += 32) out[start + i] = img[i];
        __syncwarp();
    }
}

// ---- decoder fused with dequantization, or with packing ---------------------------------------------------------
// One thread decodes one chunk sequentially from a 64-bit bit buffer (refilled a word at a time, >= 33 valid bits
// after a refill): the next 11 bits index a lookup table in shared memory; a miss (code longer than 11 bits) walks
// the canonical per-length ranges.  After every 32 symbols the CTA's decoded codes (staged in shared memory as
// bytes) are either dequantized with the same unit table and (unit*alpha)+beta arithmetic as unpack_dequant_kernel and
// leave as 128-bit stores (8 threads write one chunk's 128 contiguous bytes), or packed into the fixed-width layout
// of qd_pack_indices.
struct HuffDecodeShared {
    uint32_t lut[1 << kHuffLutBits];
    unsigned long long first[64];
    uint32_t count[64], index[64], symbols[256];
    float unit[256];
    uint32_t stage[kHuffDecThreads * kHuffStageStride];
};

__device__ __forceinline__ uint32_t huff_next_word(const uint32_t* __restrict__ words, int64_t num_words, int64_t& wi) {
    const uint32_t w = wi < num_words ? __ldg(words + wi) : 0u;
    ++wi;
    return w;
}

__device__ __forceinline__ uint32_t huff_decode_one(const HuffDecodeShared& s, int max_len, const uint32_t* __restrict__ words,
                                                    int64_t num_words, int64_t& wi, unsigned long long& buf, int& nb) {
    if (nb <= 32) {
        buf |= (unsigned long long)huff_next_word(words, num_words, wi) << (32 - nb);
        nb += 32;
    }
    const uint32_t e = s.lut[buf >> (64 - kHuffLutBits)];
    int len = (int)(e >> 16);
    uint32_t sym = e & 0xffffu;
    if (len == 0) {
        // the window extends the buffer with the next (unconsumed) word: 64 valid bits >= the longest code
        const uint32_t w2 = wi < num_words ? __ldg(words + wi) : 0u;
        const unsigned long long window = buf | ((unsigned long long)w2 >> (nb - 32));
        for (int l = kHuffLutBits + 1; l <= max_len; ++l) {
            const unsigned long long d = (window >> (64 - l)) - s.first[l];
            if (d < s.count[l]) {
                sym = s.symbols[s.index[l] + (uint32_t)d];
                len = l;
                break;
            }
        }
        if (len == 0) len = 1;   // not a codeword (corrupt stream): consume a bit, never loop
        if (len > nb) {          // the code runs into w2: absorb it
            const int k = len - nb;
            ++wi;
            buf = (unsigned long long)w2 << (32 + k);
            nb = 32 - k;
            return sym;
        }
    }
    buf <<= len;
    nb -= len;
    return sym;
}

// the code (model-wide) and, with UNIT, the unit table (per tensor: level / S, or the tensor's points) into shared
// memory; the caller synchronises the CTA before decoding
template <bool UNIFORM, bool UNIT = true>
__device__ __forceinline__ void huff_load_tables(HuffDecodeShared& s, const qd_huffman_table* __restrict__ tab, float S,
                                                 const float* __restrict__ points, int K) {
    for (int i = threadIdx.x; i < (1 << kHuffLutBits); i += blockDim.x) s.lut[i] = tab->lut[i];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) {
        s.symbols[i] = tab->symbols[i];
        if (UNIT && UNIFORM) s.unit[i] = ((float)i <= S) ? level_to_unit((float)i, S) : 0.f;
        else if (UNIT) s.unit[i] = (i < K) ? points[i] : 0.f;
    }
    for (int i = threadIdx.x; i < 64; i += blockDim.x) {
        s.first[i] = tab->first[i];
        s.count[i] = tab->count[i];
        s.index[i] = tab->index[i];
    }
}

// Output of the packing decode: one tensor's codes in the qd_pack_indices layout at `bits` per code.
struct HuffPackOut {
    uint8_t* packed;
    int64_t bytes;       // ceil(n * bits / 8)
    uint32_t limit;      // symbols >= limit are counted into `bad`
    int bits;
    uint32_t bad;
};

// Store stage of the packing decode, after one round: chunk c0 + cl's kHuffDecRound codes are 4*BITS bytes at byte
// (c0 + cl) * 128*BITS + r*BITS/8 (a chunk fills 128*BITS bytes, so chunks never share a byte).  Thread i writes
// 32-bit word i % BITS of chunk i / BITS: consecutive threads write consecutive words of a chunk's piece.  Codes past n
// are staged as 0, so the last byte's high bits are 0, and no byte past the tensor is written.  Every staged symbol
// >= limit is added to o.bad.
template <int BITS>
__device__ __forceinline__ void huff_store_packed(const HuffDecodeShared& s, HuffPackOut& o, int64_t c0, int r) {
    constexpr int per = 8 / BITS;                 // staged words (four codes each) per output word (32 / BITS codes)
    const bool vec = (reinterpret_cast<uintptr_t>(o.packed) & 3) == 0;
    for (int i = threadIdx.x; i < kHuffDecThreads * BITS; i += kHuffDecThreads) {
        const int cl = i / BITS, part = i % BITS;
        const int64_t b = (c0 + cl) * (kHuffChunk / 8 * BITS) + (r / kHuffDecRound) * (kHuffDecRound / 8 * BITS) + part * 4;
        if (b >= o.bytes) continue;
        uint32_t w = 0u;
#pragma unroll
        for (int j = 0; j < per; ++j) {
            const uint32_t codes = s.stage[cl * kHuffStageStride + part * per + j];
#pragma unroll
            for (int k = 0; k < 4; ++k) o.bad += ((codes >> (8 * k)) & 0xffu) >= o.limit;
            w |= (BITS == 8 ? codes : squeeze4<BITS>(codes)) << (4 * BITS * j);
        }
        if (vec && b + 4 <= o.bytes) {
            __stcs(reinterpret_cast<uint32_t*>(o.packed + b), w);
        } else {
            for (int k = 0; k < 4 && b + k < o.bytes; ++k) o.packed[b + k] = (uint8_t)(w >> (8 * k));
        }
    }
}

// Decodes chunks [c0, c0 + kHuffDecThreads) of one tensor (c0 < chunks), one chunk per thread.  Every thread of the
// CTA calls it with the same arguments (the staging rounds synchronise the CTA).  The decode loop is shared; the store
// stage that follows every round is chosen at compile time: PACK = false dequantizes into q (alpha, beta, L,
// single_row; pk is NULL), PACK = true writes the codes to *pk and counts out-of-range symbols into pk->bad.
template <bool PACK>
__device__ __forceinline__ void huff_decode_chunks(HuffDecodeShared& s, int max_len, const uint32_t* __restrict__ words,
                                                   int64_t num_words, const uint32_t* __restrict__ offs,
                                                   const float* __restrict__ alpha, const float* __restrict__ beta,
                                                   float* __restrict__ q, int64_t n, int64_t L, bool single_row, int64_t chunks,
                                                   int64_t c0, HuffPackOut* pk) {
    const bool qvec = (reinterpret_cast<uintptr_t>(q) & 15) == 0;
    const int64_t c = c0 + threadIdx.x;
    const int64_t e0 = c * kHuffChunk;
    const int m = c < chunks ? (int)(n - e0 < kHuffChunk ? n - e0 : kHuffChunk) : 0;
    const int m_cta = (int)(n - c0 * kHuffChunk < kHuffChunk ? n - c0 * kHuffChunk : kHuffChunk);  // first chunk is the longest
    int64_t wi = c < chunks ? (int64_t)offs[c] : 0;
    unsigned long long buf = 0ull;
    int nb = 0;
    for (int r = 0; r < m_cta; r += kHuffDecRound) {
        const int cnt = m - r;
#pragma unroll 1
        for (int g = 0; g < kHuffDecRound / 4; ++g) {
            uint32_t acc = 0u;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                if (g * 4 + k < cnt) {
                    const uint32_t sym = max_len == 0 ? s.symbols[0] : huff_decode_one(s, max_len, words, num_words, wi, buf, nb);
                    acc |= (sym & 0xffu) << (8 * k);
                }
            }
            s.stage[threadIdx.x * kHuffStageStride + g] = acc;
        }
        __syncthreads();
        if constexpr (PACK) {
            switch (pk->bits) {
                case 8: huff_store_packed<8>(s, *pk, c0, r); break;
                case 4: huff_store_packed<4>(s, *pk, c0, r); break;
                case 2: huff_store_packed<2>(s, *pk, c0, r); break;
                default: huff_store_packed<1>(s, *pk, c0, r); break;
            }
        } else {
#pragma unroll 2
            for (int i = threadIdx.x; i < kHuffDecThreads * (kHuffDecRound / 4); i += kHuffDecThreads) {
                const int cl = i / (kHuffDecRound / 4), part = i % (kHuffDecRound / 4);
                const int64_t e = (c0 + cl) * kHuffChunk + r + part * 4;
                if (c0 + cl >= chunks || e >= n || r + part * 4 >= kHuffChunk) continue;
                const uint32_t codes = s.stage[cl * kHuffStageStride + part];
                if (qvec && e + 4 <= n && (single_row || L % 4 == 0)) {
                    const int64_t row = single_row ? 0 : e / L;
                    const float a = __ldg(alpha + row), b = __ldg(beta + row);
                    st_stream4(q + e, make_float4(from_unit(s.unit[codes & 0xffu], a, b), from_unit(s.unit[(codes >> 8) & 0xffu], a, b),
                                                  from_unit(s.unit[(codes >> 16) & 0xffu], a, b), from_unit(s.unit[codes >> 24], a, b)));
                } else {
                    for (int j = 0; j < 4 && e + j < n; ++j) {
                        const int64_t row = single_row ? 0 : (e + j) / L;
                        q[e + j] = from_unit(s.unit[(codes >> (8 * j)) & 0xffu], __ldg(alpha + row), __ldg(beta + row));
                    }
                }
            }
        }
        __syncthreads();
    }
}

// one tensor: a grid-stride loop over its chunks, kHuffDecThreads chunks per CTA step
template <bool UNIFORM>
__global__ void __launch_bounds__(kHuffDecThreads) huff_decode_dequant_kernel(
    const uint32_t* __restrict__ words, int64_t num_words, const uint32_t* __restrict__ offs,
    const qd_huffman_table* __restrict__ tab, const float* __restrict__ points, int K, const float* __restrict__ alpha,
    const float* __restrict__ beta, float* __restrict__ q, Geometry geo, float S, int64_t chunks) {
    __shared__ HuffDecodeShared s;
    huff_load_tables<UNIFORM>(s, tab, S, points, K);
    const int max_len = (int)tab->max_length;
    __syncthreads();
    for (int64_t c0 = (int64_t)blockIdx.x * kHuffDecThreads; c0 < chunks; c0 += (int64_t)gridDim.x * kHuffDecThreads)
        huff_decode_chunks<false>(s, max_len, words, num_words, offs, alpha, beta, q, geo.n, geo.row_len, geo.rows == 1, chunks, c0,
                                  nullptr);
}

// A whole model in one launch.  Tensor t owns CTAs [cta_start[t], cta_start[t + 1]), ceil(chunks_t / kHuffDecThreads)
// of them, so every CTA serves one tensor (found by binary search) and loads that tensor's unit table once.  The
// tensor's fields live in registers rather than kernel parameters: 10 CTAs per SM (<= 51 registers) keep them without
// spills, where ptxas's default budget for 128 threads (40) spills.
template <bool UNIFORM>
__global__ void __launch_bounds__(kHuffDecThreads, 10) huff_decode_dequant_model_kernel(
    const qd_huffman_tensor* __restrict__ tensors, const int32_t* __restrict__ cta_start, int count,
    const qd_huffman_table* __restrict__ tab, int64_t bucket, float S) {
    __shared__ HuffDecodeShared s;
    const int b = (int)blockIdx.x;
    const int lo = model_tensor_of(cta_start, count, b);
    const qd_huffman_tensor& t = tensors[lo];
    huff_load_tables<UNIFORM>(s, tab, S, t.points, t.num_points);
    const int max_len = (int)tab->max_length;
    __syncthreads();
    const int64_t n = t.n;
    const int64_t L = (bucket == 0 || n < bucket) ? n : bucket;   // geometry_of; one row exactly when L == n
    const int64_t chunks = (n + kHuffChunk - 1) / kHuffChunk;
    huff_decode_chunks<false>(s, max_len, t.words, t.num_words, t.chunk_offsets, t.alpha, t.beta, t.q, n, L, L == n, chunks,
                              (int64_t)(b - __ldg(cta_start + lo)) * kHuffDecThreads, nullptr);
}

// A whole model's streams to fixed-width codes in one launch: the CTA map of huff_decode_dequant_model_kernel, no
// unit table, and the packing store stage at the tensor's own width.  A CTA that staged symbols >= the tensor's limit
// adds their count to out_of_range[t].
__global__ void __launch_bounds__(kHuffDecThreads, 10) huff_decode_packed_model_kernel(
    const qd_huffman_repack_tensor* __restrict__ tensors, const int32_t* __restrict__ cta_start, int count,
    const qd_huffman_table* __restrict__ tab, unsigned long long* __restrict__ out_of_range) {
    __shared__ HuffDecodeShared s;
    const int b = (int)blockIdx.x;
    const int lo = model_tensor_of(cta_start, count, b);
    const qd_huffman_repack_tensor& t = tensors[lo];
    huff_load_tables<true, false>(s, tab, 0.f, nullptr, 0);
    const int max_len = (int)tab->max_length;
    __syncthreads();
    const int64_t n = t.n;
    const int64_t chunks = (n + kHuffChunk - 1) / kHuffChunk;
    HuffPackOut pk{t.packed, (n * t.bits + 7) / 8, (uint32_t)t.limit, t.bits, 0u};
    huff_decode_chunks<true>(s, max_len, t.words, t.num_words, t.chunk_offsets, nullptr, nullptr, nullptr, n, n, true, chunks,
                             (int64_t)(b - __ldg(cta_start + lo)) * kHuffDecThreads, &pk);
    if (pk.bad) atomicAdd(out_of_range + lo, (unsigned long long)pk.bad);
}

}  // namespace qd
