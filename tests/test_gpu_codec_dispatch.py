"""Every branch of the stored-model codecs, against the oracles.

The Huffman encoder and decoder (csrc/qd_huffman.cuh) and the fixed-width unpack (csrc/qd_codec.cu) pick their branches
from the code lengths, the bit position of every code inside its word, the symbol count of the tensor, the bucket and
the alignment of every pointer.  This file walks each of them through both sides of every edge:

  * synthetic canonical codes built from explicit lengths (CODES): the longest the format carries (1, 2, ..., 56, 57, 57),
    codes whose longest length is exactly QD_HUFFMAN_LUT_BITS and one past it, many 11- and 12-bit codes, lengths 30-36
    on both sides of the encoder's three-word placement, the two-symbol and the single-symbol code; a 58-bit code is
    refused by codec.huffman_table;
  * symbol layouts: uniform draws, chunks made only of the longest code (a 57-bit chunk fills the encoder's shared-memory
    image exactly), chunks of the longest code alternating with chunks of the shortest, random runs;
  * sizes (N_SIZES) on both sides of QD_HUFFMAN_CHUNK, of the kHuffDecRound-symbol rounds inside a chunk, of
    kHuffEncWarps chunks per encoder CTA and of kHuffDecThreads chunks per decoder CTA;
  * per-tensor decode at every bucket of BUCKETS (ragged ones included) into q at float offsets 0-3, from symbols read
    at byte offsets 0-3; the encoder's capacity contract; the three whole-model launches; the fixed-width unpack at row
    lengths (UNPACK_L) around its fast tiles, with more tiles than the resident grid.

Stream words and chunk offsets are compared bit for bit with oracle/huffman_oracle.py, decoded floats with
quant_oracle.dequantize_levels, decoded symbols through identity points, fixed-width bytes with the qd_pack_indices
layout.  Output buffers start as a sentinel, and the guard elements around every view must keep it.
test_boundary_lists_track_the_codec_constants runs without a GPU and fails when a constant in the sources moves without
these lists."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from oracle import huffman_oracle as HO
from oracle import quant_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
gpu = pytest.mark.gpu

CHUNK = 1024                    # QD_HUFFMAN_CHUNK (checked against the header below)
CTA_CHUNKS = 128                # kHuffDecThreads: chunks one decoder CTA serves


def _lengths(*pairs):
    out = {}
    for syms, l in pairs:
        for s in syms:
            out[int(s)] = int(l)
    return out


# Synthetic canonical codes, {symbol: length}; every one is Kraft-complete.
CODES = {
    # 1, 2, ..., 56, 57, 57 with the two 57-bit codes on symbols 0 and 1 (so 1-bit-wide transcodes carry only them) ...
    "long_lo": _lengths(([0, 1], 57), *[([s], 58 - s) for s in range(2, 58)]),
    # ... and on symbols 56 and 57 (so a limit of 56 leaves only 57-bit codes out of range)
    "long_hi": _lengths(*[([s], min(s + 1, 57)) for s in range(58)]),
    "lut11": _lengths(*[([s], min(s + 1, 11)) for s in range(12)]),         # longest = QD_HUFFMAN_LUT_BITS
    "lut12": _lengths(*[([s], min(s + 1, 12)) for s in range(13)]),         # longest = one past it
    "many_11_12": _lengths(([0], 1), ([1], 2), ([2], 3), ([3], 4), (range(4, 68), 11), (range(68, 196), 12)),
    # 1 .. 28, then 16 codes of 30 .. 36 bits: placed at any in-word offset they end on both sides of t = 64
    "mid_30_36": _lengths(*[([s], s + 1) for s in range(28)], ([28, 29], 30), ([30, 31], 31), ([32, 33], 32), ([34, 35], 33),
                          ([36, 37], 34), ([38, 39], 35), ([40, 41, 42, 43], 36)),
    "two": {0: 1, 1: 1},
    "single": {1: 0},
}
REFUSED = {"58_bits": _lengths(*[([s], s + 1) for s in range(58)], ([58], 58))}   # 1 .. 57, 58, 58
# symbols the uniform draws and runs take (default: every symbol of the code)
POOLS = {"mid_30_36": list(range(28, 44))}
LAYOUTS = ["uniform", "longest", "long_short", "runs"]

N_SIZES = [
    1, 31, 32, 33,                          # inside one round; kHuffDecRound +- 1
    1023, 1024, 1025,                       # QD_HUFFMAN_CHUNK +- 1
    2 * CHUNK + 31, 3 * CHUNK + 32, 4 * CHUNK + 33,   # rounds inside the last chunk; 3, 4 and 5 chunks (kHuffEncWarps)
    4 * CHUNK,                              # kHuffEncWarps chunks, every one full
    CTA_CHUNKS * CHUNK - 1, CTA_CHUNKS * CHUNK, CTA_CHUNKS * CHUNK + 1,   # one decoder CTA; one symbol into the next
    (CTA_CHUNKS + 1) * CHUNK,               # kHuffDecThreads + 1 chunks, the last one full
    3 * CTA_CHUNKS * CHUNK + 517,           # several decoder CTAs
]
# per-tensor buckets: None, multiples of 4 (vector stores with several rows) and ragged ones (per-element rows)
BUCKETS = [None, 4, 12, 100, 256, 3, 6, 10, 1001]
# whole-model tensor sizes: 1, a partial round, one past a chunk, one past a decoder CTA, several CTAs, one fast unpack
# tile (kTileGroups groups of four) and one past it
MODEL_NS = [1, 31, 1025, CTA_CHUNKS * CHUNK + 1, 3 * CTA_CHUNKS * CHUNK + 7, 4096, 4097, 5000]
# fixed-width unpack row lengths: kTileU = 4 and kTileGroups = 1024 (one thread's groups are 1024 floats apart) and one
# past each, lengths that do not divide 1024, longer than 1024 and not a multiple of it, and ragged ones (general loop)
UNPACK_L = [None, 3, 4, 5, 6, 10, 12, 100, 1001, 1024, 1025, 1028, 5000]

PAD = 8                         # guard elements after every view (and up to 3 before it)
SENT = 0x7FBADBAD               # NaN payload no kernel writes
SENT8 = 0xAB
LEVELS = 256                    # uniform decodes: every symbol of every code is a level


# ----------------------------------------------------------------------------------------------- no GPU needed
def _constant(text, name):
    m = re.search(rf"constexpr\s+int\s+{name}\s*=\s*(\d+)\s*;", text)
    assert m, f"{name} not found"
    return int(m.group(1))


def test_boundary_lists_track_the_codec_constants():
    """Each constant the codec kernels branch on, and one past it, is in this file's lists: a pull request that moves
    one without moving these tests fails here, on any machine."""
    csrc = os.path.join(ROOT, "quantized_distillation_b200", "csrc")
    read = lambda *p: open(os.path.join(*p)).read()  # noqa: E731
    header, huff, common = read(ROOT, "include", "qd_b200.h"), read(csrc, "qd_huffman.cuh"), read(csrc, "qd_common.cuh")

    def define(name):
        m = re.search(rf"#define\s+{name}\s+(\d+)", header)
        assert m, f"{name} not found"
        return int(m.group(1))

    chunk = define("QD_HUFFMAN_CHUNK")
    assert chunk == CHUNK and _constant(huff, "kHuffDecThreads") == CTA_CHUNKS
    tile_u = _constant(common, "kTileU")
    m = re.search(r"constexpr\s+int\s+kTileGroups\s*=\s*(\d+)\s*\*\s*kTileU\s*;", common)
    assert m, "kTileGroups not found"
    tile_groups = int(m.group(1)) * tile_u
    longest = {max(c.values()) for c in CODES.values()} | {max(c.values()) for c in REFUSED.values()}
    rounds = {n % chunk for n in N_SIZES}
    chunk_counts = {-(-n // chunk) for n in N_SIZES}
    checks = [("QD_HUFFMAN_CHUNK", chunk, N_SIZES), ("QD_HUFFMAN_MAX_LENGTH", define("QD_HUFFMAN_MAX_LENGTH"), longest),
              ("QD_HUFFMAN_LUT_BITS", define("QD_HUFFMAN_LUT_BITS"), longest),
              ("kHuffDecThreads", CTA_CHUNKS, chunk_counts), ("kHuffDecRound", _constant(huff, "kHuffDecRound"), rounds),
              ("kHuffEncWarps", _constant(huff, "kHuffEncWarps"), chunk_counts),
              ("QD_HUFFMAN_CHUNK * kHuffDecThreads", chunk * CTA_CHUNKS, N_SIZES),
              ("kTileU", tile_u, UNPACK_L), ("kTileGroups", tile_groups, UNPACK_L), ("4 * kTileGroups", 4 * tile_groups, MODEL_NS)]
    for what, v, where in checks:
        assert v in where and v + 1 in where, f"{what} = {v}: add {v} and {v + 1} to the boundary lists"
    # the longest code fills the encoder's chunk image (kHuffImgWords = chunk * max / 32 words) exactly
    assert chunk * define("QD_HUFFMAN_MAX_LENGTH") % 32 == 0


def test_codes_are_canonical_and_the_58_bit_code_is_refused():
    from quantized_distillation_b200 import codec
    for name, lengths in CODES.items():
        codec.check_code_lengths(lengths)
        assert codec.huffman_table(lengths).nbytes == codec.HUFFMAN_TABLE_BYTES, name
    assert max(CODES["long_lo"].values()) == codec.HUFFMAN_MAX_LENGTH
    assert max(CODES["lut11"].values()) == codec.HUFFMAN_LUT_BITS
    for lengths in REFUSED.values():
        with pytest.raises(ValueError, match="at most 57"):
            codec.huffman_table(lengths)


def test_dequantize_levels_restates_the_forward_ops():
    """The oracle the decoded floats are checked against gives the q of O.uniform_fwd / O.nonuniform_fwd from their
    levels, at regular and ragged buckets."""
    rng = np.random.default_rng(5)
    for n, bucket in [(1, None), (1000, None), (1000, 3), (1000, 6), (1001, 256), (5000, 1001), (4096, 4)]:
        x = (rng.standard_normal(n) * 0.3 + 0.1).astype(np.float32)
        q, idx, st = O.uniform_fwd(x, 16, bucket)
        got = O.dequantize_levels(idx, st["alpha"], st["beta"], bucket, s=16)
        assert np.array_equal(got.view(np.int32), q.reshape(-1).view(np.int32)), (n, bucket)
        pts = np.sort(rng.random(7)).astype(np.float32)
        q, idx, st = O.nonuniform_fwd(x, pts, bucket)
        got = O.dequantize_levels(idx, st["alpha"], st["beta"], bucket, points=pts)
        assert np.array_equal(got.view(np.int32), q.reshape(-1).view(np.int32)), (n, bucket)


# ----------------------------------------------------------------------------------------------- helpers
@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from quantized_distillation_b200 import _native as N
    from quantized_distillation_b200 import codec
    tables = {k: torch.from_numpy(codec.huffman_table(v)).cuda() for k, v in CODES.items()}
    return N, codec, tables


def sm_count(N):
    sms = ctypes.c_int(0)
    N.check(N.lib().qd_device_info(ctypes.byref(sms), None, None))
    return sms.value


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def np_pack(codes, bits):
    """The qd_pack_indices layout: the code of element e in byte e*bits/8 at bit (e*bits)%8, low bits first."""
    per = 8 // bits
    c = np.zeros(-(-codes.size // per) * per, np.uint32)
    c[:codes.size] = codes
    return (c.reshape(-1, per) << (np.arange(per, dtype=np.uint32) * bits)).sum(1).astype(np.uint8)


def symbols(code, layout, n, rng):
    lengths = CODES[code]
    pool = np.array(POOLS.get(code, sorted(lengths)))
    top, bottom = max(lengths.values()), min(lengths.values())
    longest = np.array([s for s, l in lengths.items() if l == top])
    shortest = np.array([s for s, l in lengths.items() if l == bottom])
    if layout == "uniform":
        out = rng.choice(pool, n)
    elif layout == "longest":
        out = rng.choice(longest, n)
    elif layout == "long_short":
        out = np.where((np.arange(n) // CHUNK) % 2 == 0, rng.choice(longest, n), rng.choice(shortest, n))
    else:
        runs = rng.geometric(1 / 40, n // 8 + 8)
        while runs.sum() < n:
            runs = np.concatenate([runs, rng.geometric(1 / 40, n // 8 + 8)])
        out = np.repeat(rng.choice(pool, runs.size), runs)[:n]
    return out.astype(np.uint8)


def scales(n, bucket, rng):
    rows = O.bucket_geometry(n, bucket)[0]
    return rng.uniform(0.5, 2.0, rows).astype(np.float32), rng.standard_normal(rows).astype(np.float32)


def guarded_floats(n, off):
    """(int32 buffer full of SENT, float32 view of n elements at element offset off)."""
    buf = torch.full((off + n + PAD,), SENT, dtype=torch.int32, device="cuda")
    return buf, buf.view(torch.float32)[off:off + n]


def check_guarded(buf, off, n, want, what):
    got = buf.cpu().numpy()
    assert np.all(got[:off] == SENT) and np.all(got[off + n:] == SENT), f"{what}: guard overwritten"
    w = np.ascontiguousarray(want).view(np.int32)
    bad = np.nonzero(got[off:off + n] != w)[0]
    assert bad.size == 0, f"{what}: {bad.size} mismatches, first at {bad[:5].tolist()}"


def gpu_encode(N, sym, table, off=0, capacity=None):
    """qd_huffman_encode of `sym` read at byte offset `off`: (words buffer, chunk offsets + 1 guard, total).  The words
    buffer holds `capacity` words (default: enough) and PAD guard words, all starting as SENT; capacity 0 passes NULL."""
    n = sym.size
    chunks = -(-n // CHUNK)
    base = torch.zeros(n + off, dtype=torch.uint8, device="cuda")
    base[off:] = cuda(sym)
    if capacity is None:
        capacity = (n * 57 + 31) // 32 + chunks
    words = torch.full((capacity + PAD,), SENT, dtype=torch.int32, device="cuda") if capacity else None
    offs = torch.full((chunks + 1,), SENT, dtype=torch.int32, device="cuda")
    total = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    N.check(N.lib().qd_huffman_encode(N.ptr(base[off:]), n, N.ptr(table), N.ptr(words) if capacity else None, capacity, N.ptr(offs),
                                      N.ptr(total), N.stream_ptr()))
    w = words.cpu().numpy().view(np.uint32) if capacity else None
    return w, offs.cpu().numpy().view(np.uint32), int(total.item())


def gpu_decode(N, words, offs, table, alpha, beta, n, bucket, qoff, levels=None, points=None):
    """The per-tensor decode into q at float offset qoff of a guarded buffer; returns the buffer."""
    buf, q = guarded_floats(n, qoff)
    w = cuda(words.view(np.int32))
    o = cuda(offs.view(np.int32))
    wp = N.ptr(w) if w.numel() else None
    a, b = cuda(alpha), cuda(beta)
    if points is None:
        N.check(N.lib().qd_huffman_decode_dequant_uniform(wp, w.numel(), N.ptr(o), N.ptr(table), N.ptr(a), N.ptr(b), N.ptr(q), n,
                                                           bucket or 0, levels, N.stream_ptr()))
    else:
        p = cuda(points)
        N.check(N.lib().qd_huffman_decode_dequant_nonuniform(wp, w.numel(), N.ptr(o), N.ptr(table), N.ptr(p), p.numel(), N.ptr(a),
                                                              N.ptr(b), N.ptr(q), n, bucket or 0, N.stream_ptr()))
    return buf


IDENTITY = (np.arange(256) / 256).astype(np.float32)    # q * 256 is the decoded symbol (alpha 1, beta 0)


def decoded_symbols(N, words, offs, table, n):
    buf = gpu_decode(N, words, offs, table, np.ones(1, np.float32), np.zeros(1, np.float32), n, None, 0, points=IDENTITY)
    return (buf.view(torch.float32)[:n] * 256).to(torch.uint8).cpu().numpy()


# ----------------------------------------------------------------------------------------------- per-tensor streams
@gpu
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("code", sorted(CODES))
def test_stream_every_code_layout_and_size(env, code, layout):
    """At every size of N_SIZES: the encoder's words and chunk offsets from symbols at byte offsets 0-3 equal the
    oracle's; the decoded symbols equal the input; the decoded floats equal the oracle's at a bucket, q offset and
    scheme that cycle through BUCKETS, 0-3 and uniform / non-uniform."""
    N, codec, tables = env
    lengths, table = CODES[code], tables[code]
    rng = np.random.default_rng(sorted(CODES).index(code) * 10 + LAYOUTS.index(layout))
    start = sorted(CODES).index(code) + LAYOUTS.index(layout)
    for i, n in enumerate(N_SIZES):
        what = f"{code}/{layout} n={n}"
        sym = symbols(code, layout, n, rng)
        ow, oo = HO.encode(sym, lengths)
        w, offs, total = gpu_encode(N, sym, table, off=i % 4)
        assert total == ow.size and np.array_equal(offs[:-1], oo) and offs[-1] == np.uint32(SENT), what
        assert np.array_equal(w[:total], ow), f"{what}: words differ at {np.nonzero(w[:total] != ow)[0][:5].tolist()}"
        assert np.all(w[total:] == np.uint32(SENT)), what
        got = decoded_symbols(N, ow, oo, table, n)
        assert np.array_equal(got, sym), f"{what}: symbols differ at {np.nonzero(got != sym)[0][:5].tolist()}"
        k = start + i
        bucket, qoff = BUCKETS[k % len(BUCKETS)], k % 4
        alpha, beta = scales(n, bucket, rng)
        if k % 2:
            buf = gpu_decode(N, ow, oo, table, alpha, beta, n, bucket, qoff, levels=LEVELS)
            want = O.dequantize_levels(sym, alpha, beta, bucket, s=LEVELS)
        else:
            pts = np.sort(rng.standard_normal(256)).astype(np.float32)
            buf = gpu_decode(N, ow, oo, table, alpha, beta, n, bucket, qoff, points=pts)
            want = O.dequantize_levels(sym, alpha, beta, bucket, points=pts)
        check_guarded(buf, qoff, n, want, f"{what} bucket={bucket} qoff={qoff}")


@gpu
@pytest.mark.parametrize("code", ["long_lo", "long_hi", "mid_30_36", "many_11_12", "lut12", "two", "single"])
def test_decode_every_bucket_and_q_offset(env, code):
    """Several decoder CTAs and rows: every bucket of BUCKETS at q offsets 0-3, both schemes.  At offset 0 the buckets
    that are multiples of 4 take the vector stores with a row per group of four, the ragged ones the per-element rows."""
    N, codec, tables = env
    rng = np.random.default_rng(sorted(CODES).index(code))
    n = 3 * CTA_CHUNKS * CHUNK + 517
    sym = symbols(code, "uniform", n, rng)
    ow, oo = HO.encode(sym, CODES[code])
    for bucket in BUCKETS:
        alpha, beta = scales(n, bucket, rng)
        pts = np.sort(rng.standard_normal(256)).astype(np.float32)
        want_u = O.dequantize_levels(sym, alpha, beta, bucket, s=LEVELS)
        want_n = O.dequantize_levels(sym, alpha, beta, bucket, points=pts)
        for qoff in range(4):
            buf = gpu_decode(N, ow, oo, tables[code], alpha, beta, n, bucket, qoff, levels=LEVELS)
            check_guarded(buf, qoff, n, want_u, f"{code} uniform bucket={bucket} qoff={qoff}")
            buf = gpu_decode(N, ow, oo, tables[code], alpha, beta, n, bucket, qoff, points=pts)
            check_guarded(buf, qoff, n, want_n, f"{code} non-uniform bucket={bucket} qoff={qoff}")


@gpu
def test_encoder_grid_stride(env):
    """More chunks than both encoder passes' grids hold (8 CTAs per SM of 8 and 4 warps, one chunk per warp): every
    warp encodes several chunks, and the scan gives each of its threads several."""
    N, codec, tables = env
    n = (64 * sm_count(N) + 5) * CHUNK + 77
    rng = np.random.default_rng(9)
    for code in ("many_11_12", "long_lo"):
        sym = symbols(code, "runs" if code == "long_lo" else "uniform", n, rng)
        ow, oo = HO.encode(sym, CODES[code])
        w, offs, total = gpu_encode(N, sym, tables[code], off=1)
        assert total == ow.size and np.array_equal(offs[:-1], oo) and np.array_equal(w[:total], ow), code
        assert np.array_equal(decoded_symbols(N, ow, oo, tables[code], n), sym), code


@gpu
@pytest.mark.parametrize("code", ["long_lo", "mid_30_36", "lut12"])
def test_encoder_capacity_contract(env, code):
    """Exactly *total_words: the whole stream.  One word less, and a capacity that ends inside chunk 3: every chunk that
    ends within the capacity is the oracle's, every word of the other chunks and past the capacity keeps its sentinel.
    Capacity 0 with words_out NULL: only the sizing runs."""
    N, codec, tables = env
    rng = np.random.default_rng(21)
    n = 9 * CHUNK + 100                     # 10 chunks: more than one encoder CTA's kHuffEncWarps
    sym = symbols(code, "uniform", n, rng)
    ow, oo = HO.encode(sym, CODES[code])
    total = ow.size
    ends = np.append(oo[1:].astype(np.int64), total)
    for cap in (total, total - 1, int(oo[3]) + 1):
        w, offs, t = gpu_encode(N, sym, tables[code], capacity=cap)
        assert t == total and np.array_equal(offs[:-1], oo), (code, cap)
        written = np.zeros(cap + PAD, bool)
        for c in range(len(oo)):
            lo, hi = int(oo[c]), int(ends[c])
            if hi <= cap:
                assert np.array_equal(w[lo:hi], ow[lo:hi]), (code, cap, c)
                written[lo:hi] = True
        assert np.all(w[~written] == np.uint32(SENT)), (code, cap)
        assert written.sum() == int(ends[ends <= cap].max()), (code, cap)
    w, offs, t = gpu_encode(N, sym, tables[code], capacity=0)
    assert w is None and t == total and np.array_equal(offs[:-1], oo), code


# ----------------------------------------------------------------------------------------------- whole-model launches
def _model_streams(code, ns, rng, layouts=None):
    syms = [symbols(code, (layouts or LAYOUTS)[i % len(layouts or LAYOUTS)], n, rng) for i, n in enumerate(ns)]
    streams = [HO.encode(s, CODES[code]) for s in syms]
    return syms, [(cuda(w.view(np.int32)), cuda(o.view(np.int32))) for w, o in streams]


def _float_arena(ns):
    """Int32 buffer full of SENT holding every output with at least one guard element around each; output t starts at
    a float offset of t % 4 from a 16-byte boundary."""
    starts, pos = [], 4
    for i, n in enumerate(ns):
        pos = -(-pos // 4) * 4 + i % 4
        starts.append(pos)
        pos += n + 1
    return torch.full((pos + PAD,), SENT, dtype=torch.int32, device="cuda"), starts


def _check_float_arena(arena, starts, ns, wants, what):
    got = arena.cpu().numpy()
    covered = np.zeros(got.size, bool)
    for t, (st, n, want) in enumerate(zip(starts, ns, wants)):
        bad = np.nonzero(got[st:st + n] != want.view(np.int32))[0]
        assert bad.size == 0, f"{what} tensor {t} (n={n}): {bad.size} mismatches, first at {bad[:5].tolist()}"
        covered[st:st + n] = True
    assert np.all(got[~covered] == SENT), f"{what}: guard overwritten"


@gpu
@pytest.mark.parametrize("bucket", BUCKETS)
@pytest.mark.parametrize("code", ["long_lo", "mid_30_36", "many_11_12", "single"])
def test_model_decode(env, code, bucket):
    """qd_huffman_decode_dequant_model over tensors of MODEL_NS (one with several CTAs), each in its own layout, q at
    float offsets 0-3: uniform, and non-uniform with each tensor's own points."""
    N, codec, tables = env
    rng = np.random.default_rng(BUCKETS.index(bucket) * 10 + sorted(CODES).index(code))
    syms, streams = _model_streams(code, MODEL_NS, rng)
    sc = [scales(n, bucket, rng) for n in MODEL_NS]
    for uniform in (True, False):
        arena, starts = _float_arena(MODEL_NS)
        desc = np.zeros(len(MODEL_NS), codec._MODEL_TENSOR)
        keep, wants = [], []
        for i, (n, (w, o), (al, be), s) in enumerate(zip(MODEL_NS, streams, sc, syms)):
            a, b = cuda(al), cuda(be)
            pts = None if uniform else cuda(np.sort(rng.standard_normal(256 - i)).astype(np.float32))   # K_t > every symbol
            keep += [a, b, pts]
            desc[i] = (N.ptr(w) if w.numel() else 0, N.ptr(o), N.ptr(a), N.ptr(b), 0 if uniform else N.ptr(pts),
                       arena.data_ptr() + 4 * starts[i], w.numel(), n, 0 if uniform else pts.numel(), 0)
            wants.append(O.dequantize_levels(s, al, be, bucket, s=LEVELS) if uniform else
                         O.dequantize_levels(s, al, be, bucket, points=pts.cpu().numpy()))
        ws = torch.empty(int(N.lib().qd_huffman_model_workspace_bytes(len(MODEL_NS))), dtype=torch.uint8, device="cuda")
        N.check(N.lib().qd_huffman_decode_dequant_model(desc.ctypes.data, len(MODEL_NS), N.ptr(tables[code]), bucket or 0,
                                                        LEVELS if uniform else 0, N.ptr(ws), ws.numel(), N.stream_ptr()))
        _check_float_arena(arena, starts, MODEL_NS, wants, f"{code} bucket={bucket} uniform={uniform}")


# (n, bits, limit, symbols in range): widths 1/2/4/8 with byte tails (n*bits not a multiple of 32), tensors of one and of
# several decoder CTAs, limits below 2^bits.  Out-of-range tensors draw from every symbol of the code.
TRANSCODE = [(1, 1, 2, True), (31, 2, 4, True), (1025, 4, 16, True), (CTA_CHUNKS * CHUNK + 1, 1, 2, True),
             (3 * CTA_CHUNKS * CHUNK + 7, 2, 3, True), (4099, 8, 256, True), (33, 8, 200, True), (1000, 4, 5, True),
             (5 * CHUNK + 3, 1, 1, True), (2 * CTA_CHUNKS * CHUNK + 5, 8, 256, True),
             (5000, 8, 56, False), (3 * CTA_CHUNKS * CHUNK + 7, 8, 57, False), (777, 4, 3, False), (CHUNK + 1, 2, 2, False),
             (1, 1, 1, False)]


@gpu
@pytest.mark.parametrize("code", sorted(CODES))
def test_model_transcode(env, code):
    """qd_huffman_decode_packed_model: every in-range tensor's bytes equal qd_pack_indices' layout of its symbols, the
    guard bytes around packed views at byte offsets 0-3 keep their sentinel, and every tensor's out_of_range count is the
    number of its symbols >= its limit -- with long_hi at limits 56 and 57, only 57-bit codes are out of range."""
    N, codec, tables = env
    rng = np.random.default_rng(100 + sorted(CODES).index(code))
    lengths = CODES[code]
    allsym = np.array(sorted(lengths))
    syms = []
    for i, (n, bits, limit, ok) in enumerate(TRANSCODE):
        pool = allsym[allsym < min(limit, 1 << bits)] if ok else allsym
        if pool.size == 0:
            pool = allsym[:1]
        layout = LAYOUTS[i % len(LAYOUTS)]
        if layout == "longest" or layout == "long_short":
            top = max(lengths[int(s)] for s in pool)
            pool = pool[[lengths[int(s)] == top for s in pool]] if layout == "longest" else pool
        syms.append(rng.choice(pool, n).astype(np.uint8) if layout != "runs" else
                    np.repeat(rng.choice(pool, n), rng.geometric(1 / 40, n))[:n].astype(np.uint8))
    streams = [HO.encode(s, lengths) for s in syms]
    sizes = [(n * bits + 7) // 8 for n, bits, _, _ in TRANSCODE]
    starts, pos = [], 4
    for i, nb in enumerate(sizes):
        pos = -(-pos // 4) * 4 + i % 4
        starts.append(pos)
        pos += nb + 1
    arena = torch.full((pos + PAD,), SENT8, dtype=torch.uint8, device="cuda")
    desc = np.zeros(len(TRANSCODE), codec._REPACK_TENSOR)
    keep = []
    for i, ((n, bits, limit, _), (w, o)) in enumerate(zip(TRANSCODE, streams)):
        wd, od = cuda(w.view(np.int32)), cuda(o.view(np.int32))
        keep += [wd, od]
        desc[i] = (N.ptr(wd) if wd.numel() else 0, N.ptr(od), arena.data_ptr() + starts[i], wd.numel(), n, bits, limit)
    oor = torch.zeros(len(TRANSCODE), dtype=torch.int64, device="cuda")
    ws = torch.empty(int(N.lib().qd_huffman_repack_model_workspace_bytes(len(TRANSCODE))), dtype=torch.uint8, device="cuda")
    N.check(N.lib().qd_huffman_decode_packed_model(desc.ctypes.data, len(TRANSCODE), N.ptr(tables[code]), N.ptr(oor), N.ptr(ws),
                                                   ws.numel(), N.stream_ptr()))
    got, counts = arena.cpu().numpy(), oor.cpu().numpy()
    want_counts = [int((s >= limit).sum()) for s, (_, _, limit, _) in zip(syms, TRANSCODE)]
    assert counts.tolist() == want_counts, code
    covered = np.zeros(got.size, bool)
    for i, ((n, bits, limit, ok), s) in enumerate(zip(TRANSCODE, syms)):
        covered[starts[i]:starts[i] + sizes[i]] = True
        if want_counts[i] == 0:
            assert np.array_equal(got[starts[i]:starts[i] + sizes[i]], np_pack(s, bits)), (code, i, n, bits)
    assert np.all(got[~covered] == SENT8), f"{code}: guard byte overwritten"
    if code == "long_hi":                    # the out-of-range symbols of limits 56 and 57 are 57-bit codes only
        assert want_counts[10] > 0 and want_counts[11] > 0 and all(lengths[v] == 57 for v in range(56, 58))


# ----------------------------------------------------------------------------------------------- fixed-width unpack
def _unpack_inputs(n, bits, uniform, rng):
    k = (1 << bits) if uniform else max(1, (1 << bits) - int(rng.integers(0, 2)))
    sym = rng.integers(0, k, n).astype(np.uint8)
    pts = None if uniform else np.sort(rng.standard_normal(k)).astype(np.float32)
    return sym, k, pts


@gpu
@pytest.mark.parametrize("L", UNPACK_L)
def test_unpack_per_tensor(env, L):
    """qd_unpack_dequant_uniform / _nonuniform at row length L: with q 16-byte and packed 4-byte aligned, the fast tiles
    carry a row cursor across groups 1024 floats apart and, with more tiles than the resident grid (4 CTAs per SM),
    prefetch one tile ahead; unaligned q or packed, and every ragged L, take the general loop with several rows."""
    N, codec, tables = env
    rng = np.random.default_rng(1000 + UNPACK_L.index(L))
    tile = 4096                              # floats per fast tile: kTileGroups groups of four
    big = (2 * 4 * sm_count(N) + 3) * tile + 4093
    small = 3 * (L or 1000) + 1 if L is None or L < 4000 else 2 * L + 3
    runs = [(big, 0, 0, True), (big, 1, 0, False), (big, 0, 2, False), (small, 0, 0, False), (small, 3, 1, True),
            (tile, 0, 0, True), (tile + 1, 2, 3, False)]
    for j, (n, qoff, poff, uniform) in enumerate(runs):
        bits = (1, 2, 4, 8)[(j + UNPACK_L.index(L)) % 4]
        sym, k, pts = _unpack_inputs(n, bits, uniform, rng)
        alpha, beta = scales(n, L, rng)
        packed = np_pack(sym, bits)
        pbuf = torch.zeros(packed.size + poff, dtype=torch.uint8, device="cuda")
        pbuf[poff:] = cuda(packed)
        buf, q = guarded_floats(n, qoff)
        a, b = cuda(alpha), cuda(beta)
        if uniform:
            N.check(N.lib().qd_unpack_dequant_uniform(N.ptr(pbuf[poff:]), bits, N.ptr(a), N.ptr(b), N.ptr(q), n, L or 0, k,
                                                      N.stream_ptr()))
            want = O.dequantize_levels(sym, alpha, beta, L, s=k)
        else:
            p = cuda(pts)
            N.check(N.lib().qd_unpack_dequant_nonuniform(N.ptr(pbuf[poff:]), bits, N.ptr(p), k, N.ptr(a), N.ptr(b), N.ptr(q), n,
                                                         L or 0, N.stream_ptr()))
            want = O.dequantize_levels(sym, alpha, beta, L, points=pts)
        check_guarded(buf, qoff, n, want, f"L={L} n={n} bits={bits} qoff={qoff} poff={poff} uniform={uniform}")


@gpu
@pytest.mark.parametrize("uniform", [True, False])
@pytest.mark.parametrize("bucket", BUCKETS)
def test_model_unpack(env, bucket, uniform):
    """qd_unpack_dequant_model over tensors of MODEL_NS at widths 1/2/4/8 (uniform: 2/4/8 at 3 levels), q at float
    offsets 0-3 and packed codes at byte offsets 0-3, each tensor against the oracle."""
    N, codec, tables = env
    rng = np.random.default_rng(200 + BUCKETS.index(bucket) * 2 + uniform)
    ns = MODEL_NS + MODEL_NS[::-1]
    arena, starts = _float_arena(ns)
    widths = (2, 4, 8) if uniform else (1, 2, 4, 8)
    desc = np.zeros(len(ns), codec._PACKED_TENSOR)
    keep, wants = [], []
    for i, n in enumerate(ns):
        bits = widths[i % len(widths)]
        if uniform:
            sym, k, pts = rng.integers(0, 3, n).astype(np.uint8), 0, None
        else:
            sym, k, pts = _unpack_inputs(n, bits, False, rng)
        alpha, beta = scales(n, bucket, rng)
        poff = (i + 1) % 4
        pk = torch.zeros(n + 8, dtype=torch.uint8, device="cuda")
        packed = np_pack(sym, bits)
        pk[poff:poff + packed.size] = cuda(packed)
        a, b = cuda(alpha), cuda(beta)
        p = None if uniform else cuda(pts)
        keep += [pk, a, b, p]
        desc[i] = (pk.data_ptr() + poff, N.ptr(a), N.ptr(b), 0 if uniform else N.ptr(p), arena.data_ptr() + 4 * starts[i], n, bits, k)
        wants.append(O.dequantize_levels(sym, alpha, beta, bucket, s=3) if uniform else
                     O.dequantize_levels(sym, alpha, beta, bucket, points=pts))
    ws = torch.empty(int(N.lib().qd_unpack_model_workspace_bytes(len(ns))), dtype=torch.uint8, device="cuda")
    N.check(N.lib().qd_unpack_dequant_model(desc.ctypes.data, len(ns), bucket or 0, 3 if uniform else 0, N.ptr(ws), ws.numel(),
                                            N.stream_ptr()))
    _check_float_arena(arena, starts, ns, wants, f"bucket={bucket} uniform={uniform}")
