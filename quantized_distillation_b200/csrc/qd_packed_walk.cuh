// qd_packed_walk.cuh -- the device half of the layers that run from fixed-width packed codes: the unit table, and
// the quad walk of qd_packed_linear (staging of the activation tile, one warp's weight rows summed against it) that
// the packed LSTM and GRU cells (qd_recurrent.cu) run twice, once per weight.  Everything here is __forceinline__, so
// each kernel compiles it as if written in place.
#pragma once
#include <algorithm>

#include "qd_common.cuh"

namespace qd {

// unit value of every code: c/S for the uniform scheme (the reference's division, done once per code instead of once
// per element), the centroid for the non-uniform one
template <bool UNIFORM>
__device__ __forceinline__ void load_unit_table(float* s_unit, const float* __restrict__ points, int K, float S) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) {
        if (UNIFORM) s_unit[i] = ((float)i <= S) ? level_to_unit((float)i, S) : 0.f;
        else s_unit[i] = (i < K) ? points[i] : 0.f;
    }
}

// ------------------------------------------------------------------ the quad walk
// A warp owns R weight rows (four; three in the GRU cell) and walks them together, so that one shared-memory read of x
// feeds R rows.  A row is cut into quads of 4*E codes (E = 32/BITS per 32-bit word; quad d holds columns
// 4*E*d .. 4*E*d+4*E-1, one 128-bit load when rows start on 16-byte boundaries); lane L takes quads L, L+32, ... in
// increasing order and sums its
// elements in column order, one fmaf per element and x row; the caller then folds the 32 partial sums with warp_sum's
// fixed xor butterfly.  The order is therefore fixed by K and BITS alone: neither the grid, the chunking of x nor the
// row count m changes a single bit of a sum.
//
// x rows m0 .. m0+MT-1 are staged in shared memory, in chunks of kc columns (a multiple of 128*E).  The float4 groups
// of the tile are XOR-swizzled within blocks of eight so that the 32 lanes' reads (stride 4*E floats) hit distinct
// banks.
//
// The walk reads a weight through an argument struct A with the fields packed, alpha, beta, in_bytes (ceil(n*bits/8)),
// K (columns), L and rows (bucket geometry), step_q and step_r ((128*E) / L and (128*E) % L: a lane's bucket cursor
// from one of its quads to the next) and quad_aligned (packed 16-byte aligned and K*bits a multiple of 128).
constexpr int kPlWarps = 8;
constexpr int kPlThreads = kPlWarps * 32;
constexpr int kPlRowsPerWarp = 4;                    // rows per warp of qd_packed_linear and the LSTM cell
constexpr size_t kPlSmemBytes = 96 * 1024;           // x tile, unless one warp-wide step of MT rows needs more

// position of float4 group g of a tile row: bits 0-2 XOR-ed with the quad index (E float4 groups per quad)
template <int BITS>
__device__ __forceinline__ int pl_slot(int g) {
    constexpr int shift = BITS == 8 ? 2 : BITS == 4 ? 3 : BITS == 2 ? 4 : 5;   // log2(E)
    return g ^ ((g >> shift) & 7);
}

// the 32 code bits of elements e0 .. e0+E-1 (e0*BITS need not be a multiple of 32); bytes past the tensor read as 0
template <int BITS, class A>
__device__ __forceinline__ uint32_t pl_word(const A& a, int64_t e0) {
    const int64_t bit = e0 * BITS;
    const int64_t b0 = bit >> 3;
    unsigned long long v = 0;
    for (int i = 0; i < 5; ++i)
        if (b0 + i < a.in_bytes) v |= (unsigned long long)a.packed[b0 + i] << (8 * i);
    return (uint32_t)(v >> (unsigned)(bit & 7));
}

template <int BITS, class A>
__device__ __forceinline__ uint4 pl_quad(const A& a, int64_t e0) {
    if (a.quad_aligned) return __ldcs(reinterpret_cast<const uint4*>(a.packed + ((e0 * BITS) >> 3)));
    constexpr int E = 32 / BITS;
    return make_uint4(pl_word<BITS>(a, e0), pl_word<BITS>(a, e0 + E), pl_word<BITS>(a, e0 + 2 * E), pl_word<BITS>(a, e0 + 3 * E));
}

// Stages chunk c (columns c*kc .. c*kc+kc-1, kc4 = kc/4) of rows m0 .. m0+MT-1 of x into s_x; row(i) is the first
// float of x row i, rows at or past m and columns at or past K read 0.  vec: every row 16-byte aligned and K a
// multiple of 4.
template <int BITS, int MT, class Row>
__device__ __forceinline__ void pl_stage(float4* s_x, Row row, int64_t m0, int64_t m, int64_t K, int64_t kc, int kc4, bool vec,
                                         int64_t c) {
    const int64_t c0 = c * kc;
    for (int t = threadIdx.x; t < MT * kc4; t += kPlThreads) {
        const int i = t / kc4, g = t - i * kc4;
        const int64_t k = c0 + 4 * (int64_t)g;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (m0 + i < m && k < K) {
            const float* xr = row(m0 + i);
            if (vec) {
                v = __ldg(reinterpret_cast<const float4*>(xr + k));
            } else {
                v.x = xr[k];
                if (k + 1 < K) v.y = xr[k + 1];
                if (k + 2 < K) v.z = xr[k + 2];
                if (k + 3 < K) v.w = xr[k + 3];
            }
        }
        s_x[i * kc4 + pl_slot<BITS>(g)] = v;
    }
}

// Adds this lane's share of chunk c of the R weight rows orow[] times the staged x rows to acc[row][x row]: quads
// d = c*kq + lane, +32, ... below min(qpr, (c+1)*kq), where kq = kc / (4*E) is the quads per chunk and qpr the quads
// per weight row.  Each row's sum is walked on its own (its codes, its bucket cursor, its accumulators), so a row's
// bits do not depend on R: qd_packed_linear and the LSTM cell walk four rows per warp, the GRU cell three.
template <int BITS, int MT, int R, class A>
__device__ __forceinline__ void pl_walk(const A& a, const float* s_unit, const float4* s_x, int kc4, int64_t kq, int64_t qpr, int64_t c,
                                        int lane, const int64_t (&orow)[R], float (&acc)[R][MT]) {
    constexpr int E = 32 / BITS, E4 = E / 4;
    constexpr unsigned mask = (1u << BITS) - 1u;
    const int64_t d_first = c * kq + lane, d_end = min(qpr, (c + 1) * kq);
    if (d_first >= d_end) return;
    int64_t bk[R], rk[R];                           // bucket of the quad's first element, offset in it
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const int64_t e0 = orow[r] * a.K + d_first * 4 * E;
        bk[r] = e0 / a.L;
        rk[r] = e0 - bk[r] * a.L;
    }
    for (int64_t d = d_first; d < d_end; d += 32) {
        uint4 cq[R];
#pragma unroll
        for (int r = 0; r < R; ++r) cq[r] = pl_quad<BITS>(a, orow[r] * a.K + d * 4 * E);
        // per row, a cursor (bucket bc, offset rc) that walks the quad's elements in order: alpha / beta are
        // fetched once per bucket, and a bucket ending inside the quad costs one compare per element
        float al[R], be[R];
        int64_t bc[R], rc[R];
#pragma unroll
        for (int r = 0; r < R; ++r) {
            bc[r] = bk[r];
            rc[r] = rk[r];
            al[r] = __ldg(a.alpha + bc[r]);
            be[r] = __ldg(a.beta + bc[r]);
        }
        // columns of the quad inside the row: < 4*E only in its last quad
        const int valid = (int)min((int64_t)(4 * E), a.K - d * 4 * E);
        const int gbase = (int)(d - c * kq) * E;
        // loops over the quad's words and float4 groups stay rolled: the kernel body must fit the instruction
        // cache, since a lane runs it only a few times per launch
#pragma unroll 1
        for (int u = 0; u < 4; ++u) {
#pragma unroll 1
            for (int t = 0; t < E4; ++t) {
                float q[R][4];
#pragma unroll
                for (int r = 0; r < R; ++r) {
                    const uint32_t cw = u == 0 ? cq[r].x : u == 1 ? cq[r].y : u == 2 ? cq[r].z : cq[r].w;
#pragma unroll
                    for (int jj = 0; jj < 4; ++jj) {
                        const int jw = 4 * t + jj, j = u * E + jw;
                        q[r][jj] = j < valid ? from_unit(s_unit[(cw >> (jw * BITS)) & mask], al[r], be[r]) : 0.f;
                        if (++rc[r] == a.L) {                  // next element starts bucket bc + 1
                            rc[r] = 0;
                            const int64_t b = min(++bc[r], a.rows - 1);
                            al[r] = __ldg(a.alpha + b);
                            be[r] = __ldg(a.beta + b);
                        }
                    }
                }
#pragma unroll
                for (int i = 0; i < MT; ++i) {
                    const float4 xv = s_x[i * kc4 + pl_slot<BITS>(gbase + u * E4 + t)];
#pragma unroll
                    for (int r = 0; r < R; ++r) {
                        acc[r][i] = __fmaf_rn(xv.x, q[r][0], acc[r][i]);
                        acc[r][i] = __fmaf_rn(xv.y, q[r][1], acc[r][i]);
                        acc[r][i] = __fmaf_rn(xv.z, q[r][2], acc[r][i]);
                        acc[r][i] = __fmaf_rn(xv.w, q[r][3], acc[r][i]);
                    }
                }
            }
        }
#pragma unroll
        for (int r = 0; r < R; ++r) {
            bk[r] += a.step_q;
            rk[r] += a.step_r;
            if (rk[r] >= a.L) { rk[r] -= a.L; ++bk[r]; }
        }
    }
}

// Columns per chunk of the x tile for MT rows of a K-column weight at BITS: all of K when MT*K floats fit
// kPlSmemBytes, else the most whole warp-wide steps (128*E columns) that do, at least one.
template <int MT, int BITS>
inline int64_t pl_chunk_cols(int64_t K) {
    constexpr int64_t step_cols = 32 * 4 * (32 / BITS);   // columns of one warp-wide step
    const int64_t room = (kPlSmemBytes / (MT * sizeof(float))) / step_cols;
    return std::min((room > 1 ? room : 1) * step_cols, (K + step_cols - 1) / step_cols * step_cols);
}

}  // namespace qd
