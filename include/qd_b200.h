/*
 * qd_b200.h -- C ABI of libqd_b200.so: the H100 (sm_90a) implementation of the
 * fake-quantization hot path of antspy/quantized_distillation.
 *
 * The reference has no FFI layer: its boundary for this path is the Python
 * package `quantization` (quantization/__init__.py:3-8).  This header is the
 * boundary *behind* that package in the new implementation: every entry point
 * below replaces the body of one reference function (cited as
 * path:line in the reference checkout) and is what a ctypes / cffi / pybind
 * stub on the reference side would bind (see INTEGRATION.md).
 *
 * Conventions
 *   - all tensor pointers are DEVICE pointers to contiguous float32 storage in
 *     C order unless the name ends in `_host`; no torch types cross the ABI.
 *   - `n` is the number of elements, `bucket` the bucket size, 0 meaning the
 *     reference's `bucket_size=None` (one bucket spanning the tensor).
 *   - bucket geometry follows create_bucket_tensor
 *     (quantization/help_functions.py:67-94): rows = ceil(n/bucket) unless
 *     n < bucket (one short row); the tail row behaves as if padded with copies
 *     of the last element, but the padding is never materialised except in the
 *     `xhat` output of qd_scale_down, whose length is padded_len.
 *   - per-row outputs (alpha, beta: float32[rows]; argmin, argmax: int64[rows],
 *     index inside the row, first occurrence) may be NULL when not wanted.
 *   - device: kernels launch on the calling thread's CURRENT CUDA device (one
 *     process per GPU is the deployment model); the device pointers and
 *     `stream` of a call must belong to it.  Only the *_host entry points take
 *     a device ordinal and switch (and restore) the device themselves.
 *   - `stream` is a cudaStream_t; every call only enqueues work on it (no host
 *     synchronisation) except the *_host entry points, which return after the
 *     result is in host memory.
 *   - `workspace` is device scratch of at least qd_workspace_bytes(n, bucket)
 *     bytes, owned by the caller, private to the stream for the call.
 *   - return value: 0 (QD_OK) or a qd_status; qd_last_error() gives the
 *     message for the calling thread.  Nothing throws, nothing aborts.
 *   - arithmetic: float32, one IEEE round-to-nearest-even per reference torch
 *     op, no FMA contraction, true division, rintf -- results are bit-identical
 *     to the reference's CPU path for q / idx / alpha / beta / argmin / argmax.
 */
#ifndef QD_B200_H
#define QD_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* qd_stream_t; /* cudaStream_t */

typedef enum {
    QD_OK = 0,
    QD_ERR_INVALID_ARG = 1,  /* reference raises ValueError (quant_functions.py:22-33,138-139,230-236) */
    QD_ERR_UNSUPPORTED = 2,  /* reference raises NotImplementedError (quant_functions.py:329-334) */
    QD_ERR_CUDA = 3,         /* a CUDA runtime call failed; message holds cudaGetErrorString */
    QD_ERR_WORKSPACE = 4     /* workspace missing or too small */
} qd_status;

/* gradient fix-up styles of the training loop (cnn_models/conv_forward_model.py:249-266) */
typedef enum {
    QD_BWD_STE = 0,       /* 'none': straight-through, gout = g */
    QD_BWD_TRUNCATED = 1, /* 'truncated': gout = |x| > 1 ? 0 : g          (:263-264) */
    QD_BWD_MINMAX = 2     /* 'complicated': uniformQuantization_variable.backward (quant_functions.py:319-406) */
} qd_bwd_mode;

/* index rule of the non-uniform op */
typedef enum {
    QD_RULE_NEAREST = 0,  /* nonUniformQuantization direct path (quant_functions.py:267-273) */
    QD_RULE_MIDPOINT = 1  /* SearchSorted.query, pre-processed path  (quant_functions.py:531-573) */
} qd_rule;

/* ---- library ----------------------------------------------------------- */
int qd_version(void);
const char* qd_last_error(void);
/* SM count and compute capability of the current device. */
int qd_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ---- a1: create_bucket_tensor geometry (help_functions.py:67-94) -------- */
int qd_bucket_geometry(int64_t n, int64_t bucket, int64_t* rows, int64_t* row_len, int64_t* padded_len);
size_t qd_workspace_bytes(int64_t n, int64_t bucket);

/* ---- a2: ScalingFunction.scale_down, linear (quant_functions.py:56-107) --
 * xhat[padded_len] = (x' - beta)/alpha with x' = clamp(x - *mean, +-max_element);
 * mean NULL = no mean subtraction, max_element <= 0 = no clamp.  xhat may be
 * NULL to compute only the per-row state. */
int qd_scale_down(const float* x, float* xhat, float* alpha, float* beta, int64_t* argmin, int64_t* argmax,
                  int64_t n, int64_t bucket, const float* mean, float max_element,
                  void* workspace, size_t workspace_bytes, qd_stream_t stream);

/* ---- a3: ScalingFunction.inv_scale_down (quant_functions.py:131-152) -----
 * out[n] = (y*alpha + beta) + *mean over the first n of y[padded_len]. */
int qd_inv_scale_down(const float* y, float* out, const float* alpha, const float* beta, const float* mean,
                      int64_t n, int64_t bucket, qd_stream_t stream);

/* ---- a10: absmax / absnorm scaling -- EXTENSION, parity unpinned ---------
 * quant_functions.py:109-127, 144-146 cannot execute in the reference (`tensor.max(p=2)`, a bound method stored
 * as the scale), so no output of the reference exists to compare with.  These entry points implement what the
 * lines intend once the two slips are repaired: sign = sign(x), v = |x|, norm_b = max v (ABSMAX) or
 * sqrt(sum v^2) over the padded bucket (ABSNORM), norm_b < 1e-10 -> 1, x_hat = v / norm_b; inverse
 * y * norm_b * sign (+ mean).  xhat / sign use the padded layout of qd_scale_down; norm: float32[rows]. */
typedef enum { QD_SCALE_ABSMAX = 1, QD_SCALE_ABSNORM = 2 } qd_abs_scaling;
int qd_scale_down_abs(const float* x, float* xhat, float* sign, float* norm, int64_t n, int64_t bucket, int kind,
                      const float* mean, float max_element, qd_stream_t stream);
int qd_inv_scale_down_abs(const float* y, const float* sign, const float* norm, const float* mean, float* out,
                          int64_t n, int64_t bucket, qd_stream_t stream);
/* uniformQuantization(type_of_scaling='absmax'|'absnorm'): q = ((rint(x_hat*S)/S) * norm_b) * sign (+ mean) */
int qd_uniform_fwd_abs(const float* x, float* q, uint8_t* idx_u8, float* norm, int64_t n, int64_t bucket, int levels,
                       int kind, const float* mean, float max_element, qd_stream_t stream);

/* ---- a4: uniformQuantization (quant_functions.py:155-194) ----------------
 * q[n] (may alias x: modify_in_place); idx_u8[n] optional integer levels
 * (levels <= 256); levels = s >= 2.  stochastic != 0 selects stochastic
 * rounding (:174-187) with a Philox stream (seed, offset) -- distributional
 * parity only, the reference draws from torch.rand on the host. */
int qd_uniform_fwd(const float* x, float* q, uint8_t* idx_u8, float* alpha, float* beta, int64_t* argmin,
                   int64_t* argmax, int64_t n, int64_t bucket, int levels, const float* mean, float max_element,
                   int stochastic, uint64_t seed, uint64_t offset,
                   void* workspace, size_t workspace_bytes, qd_stream_t stream);

/* ---- a5: backward of the uniform op --------------------------------------
 * gout[n] (may alias g).  QD_BWD_MINMAX requires bucket != 0 like the
 * reference (quant_functions.py:332-334) and bucket <= QD_MAX_STAGED_BUCKET. */
int qd_uniform_bwd(const float* x, const float* g, float* gout, int64_t n, int64_t bucket, int levels, int mode,
                   void* workspace, size_t workspace_bytes, qd_stream_t stream);

/* forward + backward in one pass over (x, g): 16 bytes per element.  q may alias x and gout may alias g, one or both
 * (the same pointer, as an in-place training step passes them); the results are the bits of the call without aliasing.
 * No other overlap of the four arrays is allowed.  q is qd_uniform_fwd's q; gout is qd_uniform_bwd's in the same mode,
 * refused where that one is (for QD_BWD_MINMAX the two may add the terms of r_b in another order). */
int qd_uniform_fwd_bwd(const float* x, const float* g, float* q, float* gout, int64_t n, int64_t bucket,
                       int levels, int mode, void* workspace, size_t workspace_bytes, qd_stream_t stream);

/* ---- a6/a7: nonUniformQuantization (quant_functions.py:196-290, 509-573) -
 * points[K] device, sorted ascending; idx_u8 (K <= 256) and/or idx_i64 optional. */
int qd_nonuniform_fwd(const float* x, const float* points, int num_points, int rule, float* q, uint8_t* idx_u8,
                      int64_t* idx_i64, float* alpha, float* beta, int64_t n, int64_t bucket, const float* mean,
                      float max_element, void* workspace, size_t workspace_bytes, qd_stream_t stream);

/* ---- a8: nonUniformQuantization_variable.backward (quant_functions.py:471-506)
 * grad_points[K] = sum_{i: idx_i = k} fl32(g_i * alpha_row(i)); exactly one of
 * idx_u8 / idx_i64 non-NULL.  Deterministic (fixed reduction tree, float64
 * accumulation), so data-parallel replicas stay bit-identical. */
int qd_nonuniform_bwd(const float* g, const uint8_t* idx_u8, const int64_t* idx_i64, const float* alpha,
                      int num_points, float* grad_points, int64_t n, int64_t bucket,
                      void* workspace, size_t workspace_bytes, qd_stream_t stream);

/* index search alone, on values that are already scaled to [0,1] (the
 * reference's pre-processed path hands SearchSorted an already scaled tensor,
 * quant_functions.py:432-447, 275): idx = rule(xhat_i), unit_out_i = points[idx].
 * Any of idx_u8 / idx_i64 / unit_out may be NULL. */
int qd_centroid_index(const float* xhat, const float* points, int num_points, int rule, uint8_t* idx_u8,
                      int64_t* idx_i64, float* unit_out, int64_t n, qd_stream_t stream);

/* ---- next row f2: index histogram for the Huffman statistics
 * (help_functions.py:223-225): counts[b] += #{ i : idx_i = b }, b < num_bins <= 256;
 * counts is a device int64[num_bins] the caller zeroes (it accumulates across tensors). */
int qd_index_histogram(const uint8_t* idx_u8, int64_t n, int num_bins, int64_t* counts, qd_stream_t stream);

/* ---- next row f2: packed integer codec (the compressed-model deliverable the reference only
 * accounts for: helpers/functions.py:216-262).  bits in {1, 2, 4, 8}; code i of element e sits in
 * byte e*bits/8 at bit offset (e*bits)%8 (little endian).  packed has ceil(n*bits/8) bytes. */
int qd_pack_indices(const uint8_t* idx_u8, uint8_t* packed, int64_t n, int bits, qd_stream_t stream);
/* the inverse: idx_u8[e] = code of element e (any alignment of either pointer) */
int qd_unpack_indices(const uint8_t* packed, int bits, uint8_t* idx_u8, int64_t n, qd_stream_t stream);
/* q[n] rebuilt from packed uniform levels and the per-row (alpha, beta): bit-identical to the
 * output of qd_uniform_fwd that produced the levels. */
int qd_unpack_dequant_uniform(const uint8_t* packed, int bits, const float* alpha, const float* beta, float* q,
                              int64_t n, int64_t bucket, int levels, qd_stream_t stream);
/* same for centroid codes: q = points[code]*alpha + beta */
int qd_unpack_dequant_nonuniform(const uint8_t* packed, int bits, const float* points, int num_points,
                                 const float* alpha, const float* beta, float* q, int64_t n, int64_t bucket,
                                 qd_stream_t stream);
/* Quantize straight to packed codes: packed (ceil(n*bits/8) bytes), alpha and beta are byte-identical to
 * qd_uniform_fwd / qd_nonuniform_fwd (uint8 levels) followed by qd_pack_indices, and no level array is written.
 * bits in {1, 2, 4, 8} and 2^bits >= levels (num_points).  Rows of at most 1024 floats with a 16-byte aligned x, a
 * 4-byte aligned packed and a packed row start on a whole byte (one row, or bucket*bits a multiple of 8) are packed in
 * registers by the fake-quantization kernel itself; other layouts write uint8 levels into the workspace and pack them.
 * workspace: qd_packed_workspace_bytes(n, bucket) bytes (required in either case). */
size_t qd_packed_workspace_bytes(int64_t n, int64_t bucket);
int qd_uniform_fwd_packed(const float* x, uint8_t* packed, int bits, float* alpha, float* beta, int64_t n,
                          int64_t bucket, int levels, void* workspace, size_t workspace_bytes, qd_stream_t stream);
int qd_nonuniform_fwd_packed(const float* x, const float* points, int num_points, int rule, uint8_t* packed, int bits,
                             float* alpha, float* beta, int64_t n, int64_t bucket,
                             void* workspace, size_t workspace_bytes, qd_stream_t stream);
/* Whole model in one launch: every quantized tensor of a model at its own code width, with the model-wide levels and
 * bucket; q of each tensor is bit-identical to qd_unpack_dequant_* on it.  The host array is validated, then copied
 * into `workspace` (device, 16-byte aligned, >= qd_unpack_model_workspace_bytes(count) bytes, private to the stream
 * until the launch has run) with a stream-ordered copy; the call neither allocates nor synchronises, and the host
 * array may be reused as soon as it returns. */
typedef struct {                 /* one quantized tensor of a model; every pointer is DEVICE memory */
    const uint8_t* packed;       /* ceil(n*bits/8) bytes */
    const float* alpha;          /* float32[rows] */
    const float* beta;
    const float* points;         /* non-uniform: this tensor's points; NULL for uniform */
    float* q;                    /* n floats, contiguous; 4-byte alignment is enough */
    int64_t n;                   /* >= 1 */
    int32_t bits;                /* 1, 2, 4 or 8 */
    int32_t num_points;          /* non-uniform: 1..2^bits; uniform: 0 */
} qd_packed_tensor;
size_t qd_unpack_model_workspace_bytes(int count);
int qd_unpack_dequant_model(const qd_packed_tensor* tensors /* HOST array */, int count, int64_t bucket,
                            int levels /* uniform: s in [2, 2^bits]; 0: non-uniform */,
                            void* workspace, size_t workspace_bytes, qd_stream_t stream);
/* Fully-connected layer straight from packed weights: y[i, o] = sum_k x[i, k] * q[o*K + k] (+ bias[o]) for
 * x float32[m, K] and y float32[m, O] (K = in_features, O = out_features, both C order), where q is the tensor of
 * O*K elements that qd_unpack_dequant_* writes from (packed, alpha, beta) at this bucket: the weights are the stored
 * ones, bit for bit.  levels: uniform s in [2, 2^bits] (points NULL, num_points 0); 0: non-uniform, points[num_points]
 * with num_points in [1, 2^bits].  bias may be NULL.  Accumulation is float32 fmaf in an order fixed by K and bits
 * alone (no atomics, no dependence on m, the grid or timing): repeated calls and replicas give identical bits.
 * 1 <= m <= QD_PACKED_LINEAR_MAX_ROWS, larger m is QD_ERR_UNSUPPORTED (decode, then a dense GEMM).  y must not
 * overlap x.  Needs no workspace; only enqueues work on `stream`. */
#define QD_PACKED_LINEAR_MAX_ROWS 64
int qd_packed_linear(const float* x, int64_t m, int64_t in_features, int64_t out_features, const uint8_t* packed, int bits,
                     const float* alpha, const float* beta, const float* points, int num_points, int levels, int64_t bucket,
                     const float* bias, float* y, qd_stream_t stream);

/* Convolution on packed weights: y = conv2d(x, W) (+ bias) for x float32[batch, in_channels, height, width] and
 * y float32[batch, out_channels, Ho, Wo] (NCHW, C order), groups 1, dilation 1, zero padding pad_h / pad_w on both
 * sides, Ho = (height + 2*pad_h - kernel_h) / stride_h + 1 (Wo likewise).  W is the tensor of
 * out_channels*in_channels*kernel_h*kernel_w elements (flattened [O, C, kh, kw]) that qd_unpack_dequant_* writes from
 * (packed, alpha, beta) at this bucket: the weights are the stored ones, bit for bit.  levels, points, num_points and
 * bias as for qd_packed_linear.  Each output is one float32 fmaf chain over k = (c*kh + r)*kw + s in increasing order,
 * the bias added last: the order depends on (in_channels, kernel_h, kernel_w) alone, so an image gives the same bits
 * alone or in any batch, and repeated calls and replicas agree.  QD_ERR_INVALID_ARG: NULL pointers, sizes < 1,
 * strides < 1, padding < 0, an empty output, bits too narrow, y overlapping x.  QD_ERR_UNSUPPORTED: sides or padding
 * of 2^29 or more, K = in_channels*kernel_h*kernel_w of 2^31 or more, more output tiles than one launch holds.  Needs
 * no workspace; only enqueues work on `stream`. */
int qd_packed_conv2d(const float* x, int64_t batch, int64_t in_channels, int64_t height, int64_t width, int64_t out_channels,
                     int kernel_h, int kernel_w, int stride_h, int stride_w, int pad_h, int pad_w, const uint8_t* packed,
                     int bits, const float* alpha, const float* beta, const float* points, int num_points, int levels,
                     int64_t bucket, const float* bias, float* y, qd_stream_t stream);

/* Embedding lookup on packed weights: out[i, :] = row indices[i] of W, for W the tensor of num_embeddings*dim elements
 * (flattened [num_embeddings, dim]) that qd_unpack_dequant_* writes from (packed, alpha, beta) at this bucket: every
 * value is from_unit(unit[code], alpha, beta), bit for bit what the unpack writes for that row.  indices: `count`
 * contiguous int32 (index_bytes 4) or int64 (index_bytes 8), repeats allowed; out: float32[count, dim], C order, any
 * 4-byte alignment, not overlapping the indices.  levels, points and num_points as for qd_packed_linear.  An index
 * outside [0, num_embeddings) is never dereferenced: its row of out is written NaN and *invalid (a device int32, may be
 * NULL) is incremented once per such index; the kernel does not trap.  QD_ERR_INVALID_ARG: NULL pointers, index_bytes
 * not 4 or 8, sizes < 1, sizes past 64-bit indexing, bits too narrow, out overlapping the indices.  QD_ERR_UNSUPPORTED:
 * more rows than one launch holds.  Needs no workspace; only enqueues work on `stream` (graph-capturable). */
int qd_packed_embedding(const void* indices, int index_bytes, int64_t count, int64_t num_embeddings, int64_t dim,
                        const uint8_t* packed, int bits, const float* alpha, const float* beta, const float* points,
                        int num_points, int levels, int64_t bucket, float* out, int32_t* invalid, qd_stream_t stream);

/* One LSTM step on packed weights for m rows (1 <= m <= QD_PACKED_LSTM_MAX_ROWS; larger m is QD_ERR_UNSUPPORTED):
 * x float32[m, I] (row stride ldx >= I), h float32[m, H] (stride ldh >= H), c float32[m, H] (C order); w_ih and w_hh
 * describe the packed [4H, I] and [4H, H] weights (HOST structs holding device pointers; n must be 4*H*I and 4*H*H,
 * each its own bits and, non-uniform, its own points; q is not read), decoded as qd_unpack_dequant_* decodes them at
 * the model's levels and bucket; b_ih and b_hh float32[4H] may be NULL.  Gate order is torch's: i, f, g, o (rows j,
 * H+j, 2H+j, 3H+j of each weight for hidden unit j).  Writes h_out[m, H] (stride ldo >= H) and c_out[m, H].
 * Numerical contract: with S_ih and S_hh the sums qd_packed_linear forms (so S_ih + b_ih is bit for bit
 * qd_packed_linear(x, W_ih, b_ih) and S_hh is qd_packed_linear(h, W_hh, NULL)), each gate's preactivation is
 * ((S_ih + b_ih) + S_hh) + b_hh in float32 (a NULL bias is not added); then c' = (sig(f)*c) + (sig(i)*tanh(g)) and
 * h' = sig(o)*tanh(c'), sig(z) = 1/(1 + expf(-z)), every op rounded to float32 in that order (IEEE expf / tanhf, no
 * contraction).  The order depends on (I, H, bits) alone: a row gives the same bits alone or in any batch, on any
 * stream, in any replay.  c_out may be exactly c (each element is read and written by one thread) but must not overlap
 * it otherwise; h_out must not overlap x, h, c or c_out, nor c_out x or h.  QD_ERR_INVALID_ARG: NULL pointers, sizes
 * below 1, strides below the rows, bits too narrow for levels or points, the overlaps above.  No workspace; only
 * enqueues work on `stream` (graph-capturable). */
#define QD_PACKED_LSTM_MAX_ROWS 64
int qd_packed_lstm_cell(const float* x, int64_t ldx, const float* h, int64_t ldh, const float* c, int64_t m, int64_t input_size,
                        int64_t hidden_size, const qd_packed_tensor* w_ih, const qd_packed_tensor* w_hh, int levels, int64_t bucket,
                        const float* b_ih, const float* b_hh, float* h_out, int64_t ldo, float* c_out, qd_stream_t stream);
/* One LSTM layer in one direction over `steps` steps, one qd_packed_lstm_cell launch per step enqueued from a C loop
 * (no host synchronisation: graph-capturable).  batch_sizes: HOST int64[steps], non-increasing, >= 1, the first at
 * most QD_PACKED_LSTM_MAX_ROWS (PackedSequence layout; a padded batch passes `steps` equal entries).  Step t reads x
 * rows and writes out rows at its offset sum(batch_sizes[0..t-1]) in the packed data (strides ldx >= I, ldo >= H: a
 * bidirectional layer writes its half of a [., 2H] output).  reverse != 0 runs the steps T-1 .. 0.  h0, c0, h_n, c_n:
 * float32[batch_sizes[0], H], C order.  A row's previous h is the previous step's out row when the row was active
 * there, else its h0 row; c_n is first set from c0 (a stream-ordered copy, none when c_n == c0), then updated in place
 * (rows inactive at a step are left untouched); a row's h_n is written by its last step.  Arithmetic as
 * qd_packed_lstm_cell.  QD_ERR_INVALID_ARG as there, plus batch sizes that increase or are below 1, and out, h_n or
 * c_n overlapping x, h0 or each other (c_n may be c0). */
int qd_packed_lstm_layer(const float* x, int64_t ldx, const int64_t* batch_sizes, int64_t steps, int reverse, int64_t input_size,
                         int64_t hidden_size, const qd_packed_tensor* w_ih, const qd_packed_tensor* w_hh, int levels, int64_t bucket,
                         const float* b_ih, const float* b_hh, const float* h0, const float* c0, float* out, int64_t ldo,
                         float* h_n, float* c_n, qd_stream_t stream);

/* One GRU step on packed weights for m rows (1 <= m <= QD_PACKED_GRU_MAX_ROWS; larger m is QD_ERR_UNSUPPORTED):
 * x float32[m, I] (row stride ldx >= I), h float32[m, H] (stride ldh >= H); w_ih and w_hh describe the packed [3H, I]
 * and [3H, H] weights (HOST structs holding device pointers; n must be 3*H*I and 3*H*H, each its own bits and,
 * non-uniform, its own points; q is not read), decoded as qd_unpack_dequant_* decodes them at the model's levels and
 * bucket; b_ih and b_hh float32[3H] may be NULL.  Gate order is torch's: r, z, n (rows j, H+j, 2H+j of each weight for
 * hidden unit j).  Writes h_out[m, H] (stride ldo >= H).
 * Numerical contract: with gi = qd_packed_linear(x, W_ih, b_ih) and gh = qd_packed_linear(h, W_hh, b_hh), bit for bit
 * (a NULL bias is not added), r = sig(gi_r + gh_r), z = sig(gi_z + gh_z), n = tanh(gi_n + r*gh_n) and
 * h' = n + z*(h - n): torch's GRU cell, b_hn inside r*(...).  sig(v) = 1/(1 + expf(-v)); every op is rounded to float32
 * in that order (IEEE expf / tanhf, no contraction).  Unlike the LSTM cell's ((S_ih + b_ih) + S_hh) + b_hh, gi and gh
 * are each complete before they meet, for r and z too, since n needs gh_n on its own.  The order depends on (I, H,
 * bits) alone: a row gives the same bits alone or in any batch, on any stream, in any replay.  h_out must not overlap x
 * or h (every warp reads all of h).  QD_ERR_INVALID_ARG: NULL pointers, sizes below 1, strides below the rows, bits too
 * narrow for levels or points, the overlaps above.  No workspace; only enqueues work on `stream` (graph-capturable). */
#define QD_PACKED_GRU_MAX_ROWS 64
int qd_packed_gru_cell(const float* x, int64_t ldx, const float* h, int64_t ldh, int64_t m, int64_t input_size, int64_t hidden_size,
                       const qd_packed_tensor* w_ih, const qd_packed_tensor* w_hh, int levels, int64_t bucket, const float* b_ih,
                       const float* b_hh, float* h_out, int64_t ldo, qd_stream_t stream);
/* One GRU layer in one direction over `steps` steps, one qd_packed_gru_cell launch per step enqueued from a C loop (no
 * host synchronisation: graph-capturable), with qd_packed_lstm_layer's protocol: batch_sizes is HOST int64[steps],
 * non-increasing, >= 1, the first at most QD_PACKED_GRU_MAX_ROWS; step t reads x rows and writes out rows at its
 * offset sum(batch_sizes[0..t-1]) (strides ldx >= I, ldo >= H); reverse != 0 runs the steps T-1 .. 0; a row's
 * previous h is the previous step's out row when the row was active there, else its h0 row; a row's h_n is written by
 * its last step.  h0, h_n: float32[batch_sizes[0], H], C order.  Arithmetic as qd_packed_gru_cell.  QD_ERR_INVALID_ARG
 * as there, plus batch sizes that increase or are below 1, and out or h_n overlapping x, h0 or each other. */
int qd_packed_gru_layer(const float* x, int64_t ldx, const int64_t* batch_sizes, int64_t steps, int reverse, int64_t input_size,
                        int64_t hidden_size, const qd_packed_tensor* w_ih, const qd_packed_tensor* w_hh, int levels, int64_t bucket,
                        const float* b_ih, const float* b_hh, const float* h0, float* out, int64_t ldo, float* h_n, qd_stream_t stream);

/* ---- the NMT loss over the target vocabulary (onmt/Loss.py:97-120, NMTLossCompute.compute_loss) ----------
 * logits, teacher_logits: float32[rows, V], C order, any 4-byte alignment (16-byte aligned rows load 128 bits at a
 * time; the results do not depend on alignment).  teacher_logits may be NULL (no distillation term).  target: int64[rows].
 * padding_idx: -1 (none) or in [0, V).  w (weight_teacher_loss) in [0, 1]; ignored without a teacher.  Per row with
 * target y, lse_s = log sum_c exp(z_s), lse_t likewise over z_t, S_t = sum_c exp(z_t - m_t) for the row maximum m_t,
 * A = sum_c exp(z_t - m_t) (z_t - z_s), where a column with z_t = -inf adds 0 and a column with z_t finite and
 * z_s = -inf makes A (and the loss) +inf, however small its teacher probability:
 *   y == padding_idx: loss_i = 0, counted nowhere, gradient row 0;
 *   y outside [0, V) otherwise: never dereferenced; loss_i and the gradient row are NaN, counted in n_invalid;
 *   else without a teacher: loss_i = lse_s - z_s[y]; with one: (1-w)(lse_s - z_s[y]) + w (A/S_t - lse_t + lse_s);
 *        counted in n_words, and in n_correct when y is the first-occurrence argmax of z_s.
 * The sums run in float64 over IEEE expf terms, in an order fixed by V alone: a row gives the same bits alone or at any
 * position of any batch, and two calls give the same bits.  A row whose student logits are all -inf has lse_s = -inf
 * and a NaN loss and gradient, as the log-softmax has; the argmax of a row holding NaN is unspecified.
 * Neither call synchronises or allocates (graph-capturable). */
size_t qd_nmt_loss_workspace_bytes(int64_t rows);
/* row_lse: float32[rows][2] = (lse_s, lse_t; 0 without a teacher), read by the backward.  loss: one device float32,
 * sum_i loss_i rounded once.  counts: device int64[3] = n_words, n_correct, n_invalid.  workspace: device, 16-byte
 * aligned, >= qd_nmt_loss_workspace_bytes(rows) bytes (may be NULL when that is 0), else QD_ERR_WORKSPACE.  rows may be
 * 0 (loss 0, counts 0).  QD_ERR_INVALID_ARG: NULL or misaligned pointers, rows < 0, V < 1, rows*V past 64-bit
 * indexing, padding_idx or w out of range, outputs overlapping the inputs or each other. */
int qd_nmt_loss_fwd(const float* logits, const float* teacher_logits, const int64_t* target, int64_t rows, int64_t V,
                    int64_t padding_idx, float w, float* row_lse, float* loss, int64_t* counts, void* workspace,
                    size_t workspace_bytes, qd_stream_t stream);
/* grad_logits[i, c] = g (exp(z_s - lse_s) - w exp(z_t - lse_t) - (1-w)[c = y]), g = *grad_loss (a device float32
 * read by the kernel), float32 ops in that order; row_lse from qd_nmt_loss_fwd on the same inputs.  Padding rows get 0,
 * invalid targets NaN.  grad_logits: float32[rows, V], must not overlap the inputs.  Same checks as the forward. */
int qd_nmt_loss_bwd(const float* logits, const float* teacher_logits, const int64_t* target, const float* row_lse,
                    const float* grad_loss, int64_t rows, int64_t V, int64_t padding_idx, float w, float* grad_logits,
                    qd_stream_t stream);

/* ---- one beam search step of B sentences (onmt/Beam.py:55-106, Beam.advance; Translator.translateBatch) ----------
 * Rows follow onmt's beam-major decoder batch: row r = k*B + b is beam k of sentence b (K = beam).  out: float32
 * [K*B, V], C order, any 4-byte alignment.  With normalize = 0 it holds log-probabilities lp; with normalize = 1 the
 * generator Linear's logits x, and lp = fl(x - lse) with lse bit-identical to qd_nmt_loss_fwd's lse_s of the same row.
 * scores, last_tokens, origin, flat_origin, tokens: [K*B]; n_finished, eos_top: [B].  Per sentence b, the key of row k,
 * column j is lp[0, j] on the first step (rows k > 0 take no part and last_tokens is not read); otherwise -1e20f in
 * every column when last_tokens[r] == eos (such a row is never read), else fl(lp[k, j] + scores[k]).  The K selected
 * entries are the top K of the K*V keys, keys descending, a tie to the lower flat index k*V + j, NaN above every number
 * (as torch.topk) and -0 equal to +0.  Selected entry i of sentence b goes to row i*B + b: scores = its key,
 * origin = flat / V, tokens = flat mod V, flat_origin = origin*B + b (the index that reorders the decoder state);
 * n_finished[b] += the selected tokens equal to eos; eos_top[b] = 1 when beam 0's token is eos (else unchanged).
 * scores, n_finished and eos_top are updated in place; nothing else may overlap.  workspace: device, 16-byte aligned,
 * >= qd_beam_workspace_bytes(batch, beam).  No atomics, no synchronisation, no allocation: deterministic and
 * graph-capturable.  QD_ERR_INVALID_ARG: NULL or misaligned pointers (float arrays 4 bytes, int64 arrays 8,
 * n_finished 4), beam outside [1, QD_BEAM_MAX], batch < 0, normalize not 0 or 1, V < beam or V >= 2^32, eos outside
 * [0, V), batch*beam*V past 64-bit indexing, overlapping arrays; QD_ERR_WORKSPACE: a short workspace.  batch 0 does
 * nothing. */
#define QD_BEAM_MAX 16
size_t qd_beam_workspace_bytes(int64_t batch, int beam);
int qd_beam_step(const float* out, int normalize, int64_t batch, int beam, int64_t V, int64_t eos, int first_step,
                 float* scores, const int64_t* last_tokens, int64_t* origin, int64_t* flat_origin, int64_t* tokens,
                 int32_t* n_finished, uint8_t* eos_top, void* workspace, size_t workspace_bytes, qd_stream_t stream);

/* ---- next row f2: Huffman-coded storage (the model helpers/functions.py:226-262 only sizes) ----------
 * Canonical code over uint8 symbols, codes of 1..QD_HUFFMAN_MAX_LENGTH bits (built on the host: codec.py).
 * Stream: a tensor's symbols are cut into chunks of QD_HUFFMAN_CHUNK; each chunk's codes are written MSB-first
 * into 32-bit words (stored little-endian), starting on a fresh word; chunk_offsets[c] (uint32, one per chunk)
 * is the word at which chunk c starts.  A single-symbol code has length 0: no stream, every element is that
 * symbol.  The table is DEVICE memory in this layout (13328 bytes): */
#define QD_HUFFMAN_CHUNK 1024
#define QD_HUFFMAN_MAX_LENGTH 57 /* a 64-bit window at any bit of a word, minus the in-word offset slack */
#define QD_HUFFMAN_LUT_BITS 11
typedef struct {
    uint64_t code[256];    /* codeword of each symbol, right-aligned */
    uint64_t first[64];    /* first codeword of length l, right-aligned (canonical order) */
    uint32_t length[256];  /* code length of each symbol, 0 when absent */
    uint32_t count[64];    /* codewords of length l */
    uint32_t index[64];    /* position in symbols[] of the first codeword of length l */
    uint32_t symbols[256]; /* symbols in canonical order (length, then symbol) */
    uint32_t lut[1 << QD_HUFFMAN_LUT_BITS]; /* next 11 stream bits -> (length << 16) | symbol; length 0: longer code */
    uint32_t max_length;   /* longest code; 0: single-symbol code, every element is symbols[0] */
    uint32_t reserved[3];
} qd_huffman_table;
/* Encoder: pass 1 (per-chunk word counts), a one-CTA exclusive scan into chunk_offsets[ceil(n/C)] and
 * *total_words (device uint64), pass 2 (one warp per chunk) writes words_out.  The caller allocates
 * words_capacity words from its own bound (code bits of the tensor's histogram / 32 + one word per chunk) and
 * trims to *total_words after a synchronise; chunks that would end beyond the capacity are not written. */
int qd_huffman_encode(const uint8_t* idx_u8, int64_t n, const qd_huffman_table* table, uint32_t* words_out,
                      int64_t words_capacity, uint32_t* chunk_offsets, uint64_t* total_words, qd_stream_t stream);
/* Decoder fused with the dequantization of qd_unpack_dequant_*: q is bit-identical to the output of the op that
 * produced the levels.  words may be NULL when num_words is 0 (single-symbol code). */
int qd_huffman_decode_dequant_uniform(const uint32_t* words, int64_t num_words, const uint32_t* chunk_offsets,
                                      const qd_huffman_table* table, const float* alpha, const float* beta, float* q,
                                      int64_t n, int64_t bucket, int levels, qd_stream_t stream);
int qd_huffman_decode_dequant_nonuniform(const uint32_t* words, int64_t num_words, const uint32_t* chunk_offsets,
                                         const qd_huffman_table* table, const float* points, int num_points,
                                         const float* alpha, const float* beta, float* q, int64_t n, int64_t bucket,
                                         qd_stream_t stream);
/* Whole model in one launch: every chunk of every tensor, with the model-wide table, levels and bucket; q of each
 * tensor is bit-identical to the per-tensor entry points above.  The host array is validated, then copied into
 * `workspace` (device, 16-byte aligned, >= qd_huffman_model_workspace_bytes(count) bytes, private to the stream
 * until the launch has run) with a stream-ordered copy; the call neither allocates nor synchronises, and the host
 * array may be reused as soon as it returns. */
typedef struct {                 /* one quantized tensor of a model; every pointer is DEVICE memory */
    const uint32_t* words;       /* may be NULL when num_words == 0 (single-symbol code) */
    const uint32_t* chunk_offsets;
    const float* alpha;
    const float* beta;
    const float* points;         /* non-uniform: this tensor's points; NULL for uniform */
    float* q;                    /* n floats, contiguous; 4-byte alignment is enough */
    int64_t num_words;
    int64_t n;                   /* >= 1 */
    int32_t num_points;          /* non-uniform: 1..256; uniform: 0 */
    int32_t reserved;            /* 0 */
} qd_huffman_tensor;
size_t qd_huffman_model_workspace_bytes(int count);
int qd_huffman_decode_dequant_model(const qd_huffman_tensor* tensors /* HOST array */, int count,
                                    const qd_huffman_table* table, int64_t bucket,
                                    int levels /* uniform: s in [2,256]; 0: non-uniform */,
                                    void* workspace, size_t workspace_bytes, qd_stream_t stream);

/* Transcoding, Huffman stream -> fixed-width codes, a whole model in one launch: every tensor's symbols are decoded
 * with the model-wide table and written to `packed` at the tensor's own width, byte-identical to qd_pack_indices of
 * the decoded levels (the high bits of the last byte included).  A symbol >= the tensor's limit is counted into
 * out_of_range[t] (device int64[count], zeroed by the caller); that tensor's bytes are then unspecified.  Same
 * protocol as qd_huffman_decode_dequant_model: the host array is validated, then copied into `workspace` (device,
 * 16-byte aligned, >= qd_huffman_repack_model_workspace_bytes(count) bytes, else QD_ERR_WORKSPACE) with a
 * stream-ordered copy; the call neither allocates nor synchronises. */
typedef struct {                 /* one quantized tensor; every pointer is DEVICE memory */
    const uint32_t* words;       /* may be NULL when num_words == 0 (single-symbol code) */
    const uint32_t* chunk_offsets;
    uint8_t* packed;             /* out: ceil(n*bits/8) bytes, the qd_pack_indices layout */
    int64_t num_words;
    int64_t n;                   /* >= 1 */
    int32_t bits;                /* 1, 2, 4 or 8 */
    int32_t limit;               /* every symbol must be < limit: uniform s, non-uniform K_t; 1 <= limit <= 2^bits */
} qd_huffman_repack_tensor;
size_t qd_huffman_repack_model_workspace_bytes(int count);
int qd_huffman_decode_packed_model(const qd_huffman_repack_tensor* tensors /* HOST array */, int count,
                                   const qd_huffman_table* table, int64_t* out_of_range, void* workspace,
                                   size_t workspace_bytes, qd_stream_t stream);

/* ---- next row f1: one launch over every parameter tensor of a model ------
 * (replaces the per-tensor loop of cnn_models/conv_forward_model.py:236-247).
 * A plan owns a device-side table of (src, dst, n, levels); pointers must stay
 * valid while the plan lives.  src[i] == dst[i] quantizes in place. */
typedef struct qd_plan qd_plan;
int qd_plan_create(qd_plan** plan, int count, const float* const* src, float* const* dst, const int64_t* n,
                   const int32_t* levels, int64_t bucket);
int qd_plan_destroy(qd_plan* plan);
/* Optional shadow buffers (one per tensor, n[i] floats): when set, qd_plan_uniform_fwd with
 * save != 0 also writes the untouched full-precision row there -- the reference's
 * `model_state_dict = model.state_dict()` (conv_forward_model.py:286) for free in the same pass. */
int qd_plan_set_shadow(qd_plan* plan, float* const* shadow);
int qd_plan_uniform_fwd(const qd_plan* plan, qd_stream_t stream);
int qd_plan_uniform_fwd_save(const qd_plan* plan, qd_stream_t stream);
/* gout_i = bwd(src_i, grad_i) for every tensor, in place in grad. */
int qd_plan_uniform_bwd(const qd_plan* plan, float* const* grad, int mode, qd_stream_t stream);

/* Fused end-of-step: for every tensor, in ONE pass (24 bytes per element):
 *   grad    <- fix-up of `mode` evaluated at the full-precision shadow copy   (conv_forward_model.py:249-266, :315)
 *   shadow, momentum <- torch.optim.SGD update (momentum, Nesterov, weight decay, dampening 0)   (:317)
 *   dst     <- uniformQuantization(shadow)   -- the next step's quantized weights            (:286-287)
 * QD_BWD_TRUNCATED also clamps the updated weights to [-1, 1] (the next step's clamp, :240-241).
 * momentum[i]: n[i] floats, zero before the first step.  Rows of at most 512 elements, else QD_ERR_UNSUPPORTED.
 * Arithmetic = torch's CUDA SGD kernels (a + alpha*b contracted to one FMA): see qd_plan.cuh. */
int qd_plan_set_momentum(qd_plan* plan, float* const* momentum);
int qd_plan_sgd_step(const qd_plan* plan, float* const* grad, int mode, double lr, double momentum,
                     double weight_decay, int nesterov, qd_stream_t stream);

/* ---- the same for the differentiable-quantization loop (cnn_models/conv_forward_model.py:501-551):
 * one launch re-quantizes every tensor with its own current list of points (midpoint rule of the
 * pre-processed path, quant_functions.py:531-573), two small launches produce every tensor's centroid
 * gradient (:471-506), deterministically.  Per tensor i: src[i] the fixed full-precision tensor,
 * dst[i] the live parameter (receives q), idx[i] uint8[n], alpha[i] / beta[i] float[rows] (written by
 * the forward, read by the backward), points[i] float[num_points[i]] ascending, device memory, re-read
 * at every launch, grad_points[i] float[num_points[i]].  1 <= num_points <= 32 and rows of at most
 * 1024 elements, otherwise QD_ERR_UNSUPPORTED (use the per-tensor entry points). */
typedef struct qd_nu_plan qd_nu_plan;
int qd_plan_nonuniform_create(qd_nu_plan** plan, int count, const float* const* src, float* const* dst,
                              uint8_t* const* idx, float* const* alpha, float* const* beta,
                              const float* const* points, float* const* grad_points, const int64_t* n,
                              const int32_t* num_points, int64_t bucket);
int qd_plan_nonuniform_destroy(qd_nu_plan* plan);
int qd_plan_nonuniform_fwd(const qd_nu_plan* plan, qd_stream_t stream);
/* grad[i]: dLoss/d(quantized tensor i), float[n[i]] */
int qd_plan_nonuniform_bwd(const qd_nu_plan* plan, const float* const* grad, qd_stream_t stream);
/* The same backward split in two for data-parallel training, where the centroid gradient of the global
 * batch is the rank average of the per-rank ones.  _partial runs the same launches and writes each tensor's
 * float64 sum into sums, a caller-owned device table double[count][32] (zeros past num_points[i]) instead
 * of casting it; the caller may reduce that table across ranks.  _finish writes
 * grad_points[i][k] = (float)(sums[i][k] * scale).  _partial then _finish(scale = 1) equals
 * qd_plan_nonuniform_bwd bit for bit.  Both are stream-ordered only (no allocation, no synchronisation),
 * so they can be captured in a CUDA graph. */
int qd_plan_nonuniform_bwd_partial(const qd_nu_plan* plan, const float* const* grad, double* sums, qd_stream_t stream);
int qd_plan_nonuniform_bwd_finish(const qd_nu_plan* plan, const double* sums, double scale, qd_stream_t stream);

/* ---- next row f3: the reductions of the differentiable-quantization setup -----------------
 * Exact order statistics without a sort: out[r] = the ranks[r]-th smallest element of v (0-based; ranks
 * is a DEVICE array of num_ranks <= 512 entries, clamped to [0, n-1]).  This is what
 * np.percentile(x_hat, linspace(0, 100, K)) reads (help_functions.py:140-154).  Two reads of v
 * (value histogram, then compaction of the selected bins) plus a radix select on the compacted keys.
 * workspace: qd_order_statistics_workspace_bytes(n) bytes. */
size_t qd_order_statistics_workspace_bytes(int64_t n);
int qd_order_statistics(const float* v, int64_t n, const int64_t* ranks, int num_ranks, float* out,
                        void* workspace, size_t workspace_bytes, qd_stream_t stream);
/* out[i] = ||tensors[i]||_2 for count tensors (host array of device pointers) in two launches, float64
 * partial sums in a fixed order: the gradient norms of assign_bits_automatically
 * (cnn_models/conv_forward_model.py:424-448).  Setup-time call: synchronises the stream once. */
int qd_multi_l2norm(const float* const* tensors, const int64_t* n, int count, float* out, qd_stream_t stream);

/* ---- host-buffer entry points (what a CPU-tensor caller gets) ------------
 * Inputs and outputs in HOST memory (pinned for full PCIe rate); the call
 * pipelines H2D, the fused kernel and D2H in row-aligned chunks on internal
 * streams of `device` -- or, for pinned tensors of at most 8 Mi elements, runs
 * one launch straight on the (device-addressable) host pointers -- and returns
 * when the outputs are complete.  Pageable memory is accepted (slower copies). */
int qd_uniform_fwd_host(const float* x_host, float* q_host, int64_t n, int64_t bucket, int levels, int device);
int qd_uniform_fwd_bwd_host(const float* x_host, const float* g_host, float* q_host, float* gout_host,
                            int64_t n, int64_t bucket, int levels, int mode, int device);

/* ---- self tests used by tests/ (device side arithmetic checks) ---------- */
int qd_selftest_division(int64_t pairs, uint64_t seed, int64_t* mismatches, qd_stream_t stream);

#define QD_MAX_STAGED_BUCKET 49152 /* floats; largest bucket staged in shared memory */

#ifdef __cplusplus
}
#endif
#endif /* QD_B200_H */
