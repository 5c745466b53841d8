"""Packed integer codec and size accounting (SURVEY.md section 8 f2).

The reference's deliverable is a *small* model, but it only ever computes the size it would
have (helpers/functions.py:216-262: Huffman mean bit length x parameter count + 8 bytes per
bucket); the weights themselves stay float32.  Here a quantized tensor can actually be stored:
bit-packed codes (1/2/4/8 bits) + (alpha, beta) per bucket, produced and decoded on the GPU,
and decoding reproduces the fake-quantized float tensor bit for bit."""
from __future__ import annotations

import json
import math
import struct
from dataclasses import dataclass, field

import numpy as np
import torch

from . import _native as N
from .quantization import help_functions as qhf


def bits_for(levels: int) -> int:
    b = max(1, math.ceil(math.log2(levels)))
    return 1 if b <= 1 else 2 if b <= 2 else 4 if b <= 4 else 8


@dataclass
class PackedTensor:
    packed: torch.Tensor        # uint8, ceil(n*bits/8) bytes
    alpha: torch.Tensor         # float32 [rows]
    beta: torch.Tensor          # float32 [rows]
    shape: torch.Size
    bits: int
    levels: int                 # uniform: s; non-uniform: number of points
    bucket_size: object
    points: object = None       # centroid table for the non-uniform codec

    @property
    def nbytes(self) -> int:
        extra = 0 if self.points is None else self.points.numel() * 4
        return self.packed.numel() + (self.alpha.numel() + self.beta.numel()) * 4 + extra


def _rows(n, bucket_size):
    return N.geometry(n, 0 if bucket_size is None else int(bucket_size))[0]


def _bucket(bucket_size) -> int:
    """The C ABI's bucket argument: 0 for one bucket per tensor."""
    return 0 if bucket_size is None else int(bucket_size)


def _levels(x, s, pts, bucket_size, rule, sp):
    """(uint8 level indices, alpha, beta) of x (contiguous float32 on the current device) from the fused forward op:
    uniformQuantization's s levels when ``pts`` is None, else nonUniformQuantization's over ``pts`` with ``rule``."""
    n, b = x.numel(), _bucket(bucket_size)
    rows = _rows(n, bucket_size)
    alpha = torch.empty(rows, device=x.device)
    beta = torch.empty(rows, device=x.device)
    idx = torch.empty(n, dtype=torch.uint8, device=x.device)
    ws = N.workspace(n, b, x.device)
    if pts is None:
        N.check(N.lib().qd_uniform_fwd(N.ptr(x), None, N.ptr(idx), N.ptr(alpha), N.ptr(beta), None, None, n, b, int(s), None, 0.0,
                                       0, 0, 0, N.ptr(ws), ws.numel(), sp))
    else:
        N.check(N.lib().qd_nonuniform_fwd(N.ptr(x), N.ptr(pts), pts.numel(), N.RULE_MIDPOINT if rule == "midpoint" else N.RULE_NEAREST,
                                          None, N.ptr(idx), None, N.ptr(alpha), N.ptr(beta), n, b, None, 0.0, N.ptr(ws), ws.numel(), sp))
    return idx, alpha, beta


def _encode(tensor, s, bucket_size, points=None, rule="nearest") -> PackedTensor:
    """Level indices of ``tensor`` (uniform with s levels, or non-uniform on ``points``) packed at the width they need."""
    x = tensor.detach().cuda().contiguous().float()
    pts = None if points is None else torch.as_tensor(points, dtype=torch.float32).detach().to(x.device).contiguous()
    sp = N.stream_ptr(x.device)
    idx, alpha, beta = _levels(x, s, pts, bucket_size, rule, sp)
    levels = int(s) if pts is None else pts.numel()
    bits = bits_for(levels)
    packed = torch.empty((x.numel() * bits + 7) // 8, dtype=torch.uint8, device=x.device)
    N.check(N.lib().qd_pack_indices(N.ptr(idx), N.ptr(packed), x.numel(), bits, sp))
    return PackedTensor(packed, alpha, beta, tensor.shape, bits, levels, bucket_size, points=pts)


def encode_uniform(tensor: torch.Tensor, s: int, bucket_size=None) -> PackedTensor:
    """uniformQuantization (quant_functions.py:155-194) straight to packed codes: the float
    fake-quantized tensor is never written."""
    N.require_cuda()
    if s > 256:
        raise ValueError("the packed codec stores at most 8 bits per weight")
    return _encode(tensor, s, bucket_size)


def encode_nonuniform(tensor: torch.Tensor, points, bucket_size=None, rule="nearest") -> PackedTensor:
    N.require_cuda()
    return _encode(tensor, None, bucket_size, points, rule)


def _unpack(packed, bits, alpha, beta, points, levels, bucket_size, out: torch.Tensor) -> torch.Tensor:
    """Decodes one tensor's packed codes into ``out`` (contiguous float32, on their device): qd_unpack_dequant_uniform
    with ``levels``, or qd_unpack_dequant_nonuniform on ``points`` when they are given."""
    n, b, sp = out.numel(), _bucket(bucket_size), N.stream_ptr(out.device)
    if points is None:
        N.check(N.lib().qd_unpack_dequant_uniform(N.ptr(packed), bits, N.ptr(alpha), N.ptr(beta), N.ptr(out), n, b, levels, sp))
    else:
        N.check(N.lib().qd_unpack_dequant_nonuniform(N.ptr(packed), bits, N.ptr(points), points.numel(), N.ptr(alpha), N.ptr(beta),
                                                     N.ptr(out), n, b, sp))
    return out


def decode(pt: PackedTensor) -> torch.Tensor:
    """Packed codes -> the fake-quantized float32 tensor (bit-identical to the fused op)."""
    N.require_cuda()
    out = torch.empty(int(math.prod(pt.shape)), dtype=torch.float32, device=pt.packed.device)
    return _unpack(pt.packed, pt.bits, pt.alpha, pt.beta, pt.points, pt.levels, pt.bucket_size, out).view(pt.shape)


# ---------------------------------------------------------------------------------------------------------------
# Stored models.  Two containers share one file layout -- magic, version, reserved 0, JSON header length, the JSON
# header, then 16-byte-aligned little-endian sections -- one reader with one set of checks, and one whole-model decode
# protocol (a descriptor per quantized tensor, every tensor's points in one upload, one launch per device).
#
# Huffman-coded: the code is the one the size accounting uses (huffman_code_of_histogram over the level histogram of
# every quantized tensor), made canonical; the stream and table layout are declared in include/qd_b200.h and produced /
# consumed by csrc/qd_huffman.cuh.
HUFFMAN_CHUNK = 1024            # symbols per independently decodable chunk (QD_HUFFMAN_CHUNK)
HUFFMAN_MAX_LENGTH = 57         # QD_HUFFMAN_MAX_LENGTH
HUFFMAN_LUT_BITS = 11           # QD_HUFFMAN_LUT_BITS
HUFFMAN_TABLE_BYTES = 13328     # sizeof(qd_huffman_table)
FILE_MAGIC = b"QDHUFF\x00\x00"
FILE_VERSION = 1                # parameters only
FILE_VERSION_BUFFERS = 2        # parameters + persistent buffers: a version-1 reader refuses it rather than drop them
# Fixed-width: every quantized tensor is stored as its packed codes (qd_pack_indices layout, its own width
# bits_for(levels or points)) + (alpha, beta) per bucket: the size get_size_reduction accounts for.  It decodes at HBM
# rate in one launch (qd_unpack_dequant_model) and can be read at any bucket without a chunk index.  Buffers are stored
# as in Huffman version 2.
PACKED_MAGIC = b"QDPACK\x00\x00"
PACKED_VERSION = 1
_PREFIX = struct.Struct("<8sIIQ")   # magic, version, reserved (0), JSON header length
_ALIGN = 16
# dtypes a stored buffer may have, by their name in the header
_BUFFER_DTYPES = {"float32": torch.float32, "int64": torch.int64}
# qd_huffman_tensor (include/qd_b200.h): one entry of the whole-model decode
_MODEL_TENSOR = np.dtype([("words", "<u8"), ("chunk_offsets", "<u8"), ("alpha", "<u8"), ("beta", "<u8"), ("points", "<u8"),
                          ("q", "<u8"), ("num_words", "<i8"), ("n", "<i8"), ("num_points", "<i4"), ("reserved", "<i4")])
assert _MODEL_TENSOR.itemsize == 72
# qd_packed_tensor (include/qd_b200.h): one entry of the whole-model unpack
_PACKED_TENSOR = np.dtype([("packed", "<u8"), ("alpha", "<u8"), ("beta", "<u8"), ("points", "<u8"), ("q", "<u8"), ("n", "<i8"),
                           ("bits", "<i4"), ("num_points", "<i4")])
assert _PACKED_TENSOR.itemsize == 56
# qd_huffman_repack_tensor (include/qd_b200.h): one entry of the whole-model Huffman -> fixed-width transcode
_REPACK_TENSOR = np.dtype([("words", "<u8"), ("chunk_offsets", "<u8"), ("packed", "<u8"), ("num_words", "<i8"), ("n", "<i8"),
                           ("bits", "<i4"), ("limit", "<i4")])
assert _REPACK_TENSOR.itemsize == 48


def huffman_code_lengths(counts) -> dict:
    """{symbol: code length} of the reference's Huffman code for a level histogram (counts[symbol]).  A
    single-symbol histogram gives length 0.  Codes longer than HUFFMAN_MAX_LENGTH bits raise ValueError."""
    _, code = qhf.huffman_code_of_histogram(np.asarray(counts, dtype=np.int64))
    lengths = {int(sym): len(bits) for sym, bits in code}
    check_code_lengths(lengths)
    return lengths


def check_code_lengths(lengths: dict) -> None:
    """Raises ValueError unless `lengths` is a complete prefix code the stream format can carry."""
    if not lengths:
        raise ValueError("empty code")
    if any(not (0 <= int(s) < 256) for s in lengths):
        raise ValueError("symbols must be in [0, 256)")
    if len(lengths) == 1:
        if next(iter(lengths.values())) != 0:
            raise ValueError("a single-symbol code has length 0")
        return
    longest = max(lengths.values())
    if longest > HUFFMAN_MAX_LENGTH:
        raise ValueError(f"longest Huffman code is {longest} bits; the stream format supports at most {HUFFMAN_MAX_LENGTH}")
    if min(lengths.values()) < 1:
        raise ValueError("code lengths must be >= 1 when there are several symbols")
    if sum(1 << (longest - l) for l in lengths.values()) != 1 << longest:
        raise ValueError("code lengths violate Kraft equality: not a complete prefix code")


def canonical_codes(lengths: dict) -> dict:
    """{symbol: codeword}: codewords assigned in (length, symbol) order, each the previous one plus one, shifted
    to its length.  Lengths (hence the size) are those of the input."""
    codes, code, prev = {}, 0, None
    for sym, l in sorted(lengths.items(), key=lambda kv: (kv[1], kv[0])):
        if prev is not None:
            code = (code + 1) << (l - prev)
        codes[sym] = code
        prev = l
    return codes


def huffman_table(lengths: dict) -> np.ndarray:
    """The qd_huffman_table bytes (include/qd_b200.h) of a canonical code."""
    check_code_lengths(lengths)
    code = np.zeros(256, "<u8")
    first = np.zeros(64, "<u8")
    length = np.zeros(256, "<u4")
    count = np.zeros(64, "<u4")
    index = np.zeros(64, "<u4")
    symbols = np.zeros(256, "<u4")
    lut = np.zeros(1 << HUFFMAN_LUT_BITS, "<u4")
    codes = canonical_codes(lengths)
    for pos, (sym, l) in enumerate(sorted(lengths.items(), key=lambda kv: (kv[1], kv[0]))):
        code[sym], length[sym], symbols[pos] = codes[sym], l, sym
        if count[l] == 0:
            first[l], index[l] = codes[sym], pos
        count[l] += 1
        if 1 <= l <= HUFFMAN_LUT_BITS:
            lo = codes[sym] << (HUFFMAN_LUT_BITS - l)
            lut[lo:lo + (1 << (HUFFMAN_LUT_BITS - l))] = (l << 16) | sym
    tail = np.array([max(lengths.values()), 0, 0, 0], "<u4")
    out = np.concatenate([a.view(np.uint8) for a in (code, first, length, count, index, symbols, lut, tail)])
    assert out.nbytes == HUFFMAN_TABLE_BYTES
    return out


@dataclass
class HuffmanTensor:
    """One parameter of a CompressedModel: a Huffman stream + (alpha, beta) per bucket, or float32 as is."""
    name: str
    shape: tuple
    words: torch.Tensor = None          # int32 storage of the uint32 stream words
    chunk_offsets: torch.Tensor = None  # int32 storage of uint32[ceil(n / HUFFMAN_CHUNK)]
    alpha: torch.Tensor = None          # float32[rows]
    beta: torch.Tensor = None
    points: torch.Tensor = None         # non-uniform: this tensor's centroids
    raw: torch.Tensor = None            # unquantized tensor (float32)
    code_bits: int = 0                  # bits of the codes alone (no chunk padding)

    @property
    def numel(self) -> int:
        return int(math.prod(self.shape))

    @property
    def quantized(self) -> bool:
        return self.raw is None


@dataclass
class PackedEntry:
    """One parameter of a PackedModel: packed codes + (alpha, beta) per bucket, or float32 as is."""
    name: str
    shape: tuple
    bits: int = 0                       # code width of a quantized tensor: 1, 2, 4 or 8
    packed: torch.Tensor = None         # uint8[ceil(n * bits / 8)]
    alpha: torch.Tensor = None          # float32[rows]
    beta: torch.Tensor = None
    points: torch.Tensor = None         # non-uniform: this tensor's centroids
    raw: torch.Tensor = None            # unquantized tensor (float32)

    @property
    def numel(self) -> int:
        return int(math.prod(self.shape))

    @property
    def quantized(self) -> bool:
        return self.raw is None


class _Container:
    """What CompressedModel and PackedModel share: the file layout, its size accounting, the reader and the
    whole-model decode are written once (module functions below).  Each format names its sections, magic, versions,
    descriptor and native decode, and supplies its extra header and entry fields, the reading of one quantized entry
    and the descriptor of one tensor."""

    def size_breakdown(self) -> dict:
        """Bytes of the saved file by what they hold: the format's code bytes, then scales, unquantized parameters,
        stored buffers, header and alignment.  Huffman: code_bits / 8 + scale_bytes + unquantized_bytes is what
        get_size_quantized_model accounts for.  Fixed-width: code_bytes + scale_bytes is what get_size_reduction
        accounts for, up to the round-up of each tensor's codes to whole bytes.  The rest is the price of the format."""
        header, sections, data_bytes = _layout(self)
        q = [t for t in self.tensors if t.quantized]
        start = _align(_PREFIX.size + len(header))
        return {
            **self._code_sizes(q),
            "scale_bytes": sum((t.alpha.numel() + t.beta.numel()) * 4 for t in q),
            "unquantized_bytes": sum(t.raw.numel() * 4 for t in self.tensors if not t.quantized),
            "buffer_bytes": sum(b.numel() * b.element_size() for _, b in self.buffers or []),
            "header_bytes": _PREFIX.size + len(header),
            "alignment_bytes": start - _PREFIX.size - len(header) + data_bytes - sum(nb for _, nb, _ in sections),
            "file_bytes": start + data_bytes,
        }


@dataclass
class CompressedModel(_Container):
    """A model whose quantized parameters are Huffman-coded (compress_model, load_compressed)."""
    kind: str                       # "uniform" | "nonuniform"
    levels: object                  # uniform: s; non-uniform: None
    bucket_size: object
    code_lengths: dict              # symbol -> code length (canonical code)
    tensors: list
    chunk: int = HUFFMAN_CHUNK
    _tables: dict = field(default_factory=dict, repr=False)
    # persistent buffers (BatchNorm running statistics, ...) as [(name, tensor)] in state_dict() order; None: not stored
    buffers: list = None
    # a loaded file's data region: every section is a view into it, so it reaches a device in one copy
    _data: torch.Tensor = field(default=None, init=False, repr=False, compare=False)

    _SECTIONS = ("words", "chunk_offsets", "alpha", "beta")
    _MAGIC, _VERSIONS, _FILE, _WHAT = FILE_MAGIC, (FILE_VERSION, FILE_VERSION_BUFFERS), "Huffman-coded model file", "compressed model"
    _ENTRY, _DESCRIPTOR = HuffmanTensor, _MODEL_TENSOR
    _WORKSPACE, _DECODE = "qd_huffman_model_workspace_bytes", "qd_huffman_decode_dequant_model"

    def table(self, device) -> torch.Tensor:
        key = str(device)
        if key not in self._tables:
            self._tables[key] = torch.from_numpy(huffman_table(self.code_lengths)).to(device)
        return self._tables[key]

    def _code_sizes(self, q) -> dict:
        code_bits = sum(t.code_bits for t in q)
        return {"code_bits": code_bits, "padding_bits": sum(t.words.numel() for t in q) * 32 - code_bits,
                "chunk_index_bytes": sum(t.chunk_offsets.numel() * 4 for t in q)}

    def _version(self) -> int:
        # the buffers' key exists only in a version-2 header, so a file without buffers is exactly what version 1 was
        return FILE_VERSION if self.buffers is None else FILE_VERSION_BUFFERS

    def _header(self, common: dict) -> dict:
        return {"chunk": self.chunk, **common, "code": [[int(s), int(l)] for s, l in sorted(self.code_lengths.items())]}

    @staticmethod
    def _entry_fields(t) -> dict:
        return {"code_bits": int(t.code_bits)}

    @staticmethod
    def _read_header(h, version, levels, bad) -> dict:
        if ("buffers" in h) != (version == FILE_VERSION_BUFFERS):
            bad(f"a version-{version} file {'must not list' if version == FILE_VERSION else 'must list its'} buffers")
        try:
            chunk, code = h["chunk"], {int(s): int(l) for s, l in h["code"]}
        except (ValueError, KeyError, TypeError) as e:
            bad(f"unreadable header ({e})")
        if chunk != HUFFMAN_CHUNK:
            bad(f"chunk of {chunk} symbols, this reader decodes {HUFFMAN_CHUNK}")
        if len(code) != len(h["code"]):
            bad("a symbol appears twice in the code")
        try:
            check_code_lengths(code)
        except ValueError as e:
            bad(str(e))
        if levels is not None and max(code) >= levels:
            bad("a code symbol is not a level")
        return {"code_lengths": code}

    @staticmethod
    def _read_entry(e, name, n, levels, pts, section, bad) -> dict:
        # the code is model-wide: a tensor with fewer points than another never emits the higher symbols
        if pts is not None and not 1 <= pts.numel() <= 256:
            bad(f"{name}: {pts.numel()} points, expected 1 to 256")
        span = e["sections"]["words"]
        words_nb = span[1] if isinstance(span, list) and len(span) == 2 else None
        if not isinstance(words_nb, int) or words_nb < 0 or words_nb % 4:
            bad(f"{name}: section words out of range")
        words = section(e, "words", torch.int32, words_nb)
        offs = section(e, "chunk_offsets", torch.int32, 4 * -(-n // HUFFMAN_CHUNK))
        o = offs.numpy().view(np.uint32).astype(np.int64)
        if o[0] != 0 or np.any(np.diff(o) < 0) or o[-1] > words.numel():
            bad(f"{name}: chunk offsets out of range")
        return {"words": words, "chunk_offsets": offs, "code_bits": int(e.get("code_bits", 0))}

    def _descriptor(self, t, sections, points, num_points, out) -> tuple:
        words, offs, alpha, beta = sections
        return (N.ptr(words) if words.numel() else 0, N.ptr(offs), N.ptr(alpha), N.ptr(beta), points, N.ptr(out), words.numel(),
                t.numel, num_points, 0)

    def _decode_tables(self, dev) -> tuple:
        return (N.ptr(self.table(dev)),)


@dataclass
class PackedModel(_Container):
    """A model whose quantized parameters are stored fixed-width (pack_model, load_packed)."""
    kind: str                       # "uniform" | "nonuniform"
    levels: object                  # uniform: s; non-uniform: None
    bucket_size: object
    tensors: list
    # persistent buffers as [(name, tensor)] in state_dict() order; None: not stored
    buffers: list = None
    # a loaded file's data region: every section is a view into it, so it reaches a device in one copy
    _data: torch.Tensor = field(default=None, init=False, repr=False, compare=False)

    _SECTIONS = ("packed", "alpha", "beta")
    _MAGIC, _VERSIONS, _FILE, _WHAT = PACKED_MAGIC, (PACKED_VERSION,), "fixed-width model file", "packed model"
    _ENTRY, _DESCRIPTOR = PackedEntry, _PACKED_TENSOR
    _WORKSPACE, _DECODE = "qd_unpack_model_workspace_bytes", "qd_unpack_dequant_model"

    @staticmethod
    def _code_sizes(q) -> dict:
        return {"code_bytes": sum(t.packed.numel() for t in q)}

    @staticmethod
    def _version() -> int:
        return PACKED_VERSION

    @staticmethod
    def _header(common: dict) -> dict:
        return common

    @staticmethod
    def _entry_fields(t) -> dict:
        return {"bits": int(t.bits)}

    @staticmethod
    def _read_header(h, version, levels, bad) -> dict:
        if not any(isinstance(e, dict) and e.get("quantized") is True for e in h["tensors"]):
            bad("no quantized tensor")
        return {}

    @staticmethod
    def _read_entry(e, name, n, levels, pts, section, bad) -> dict:
        bits = e.get("bits")
        if bits not in (1, 2, 4, 8) or isinstance(bits, bool):
            bad(f"{name}: bits must be 1, 2, 4 or 8")
        if pts is None and levels > 1 << bits:
            bad(f"{name}: {levels} levels do not fit in {bits}-bit codes")
        if pts is not None and not 1 <= pts.numel() <= 1 << bits:
            bad(f"{name}: {pts.numel()} points do not fit in {bits}-bit codes")
        return {"bits": bits, "packed": section(e, "packed", torch.uint8, (n * bits + 7) // 8)}

    @staticmethod
    def _descriptor(t, sections, points, num_points, out) -> tuple:
        packed, alpha, beta = sections
        return (N.ptr(packed), N.ptr(alpha), N.ptr(beta), points, N.ptr(out), t.numel, t.bits, num_points)

    @staticmethod
    def _decode_tables(dev) -> tuple:
        return ()


def _align(x: int) -> int:
    return (x + _ALIGN - 1) // _ALIGN * _ALIGN


def _dtype_name(tensor) -> str:
    name = str(tensor.dtype).replace("torch.", "")
    if name not in _BUFFER_DTYPES:
        raise ValueError(f"buffers of dtype {tensor.dtype} cannot be stored (float32 and int64 can)")
    return name


def _layout(m):
    """(JSON header bytes, [(tensor, nbytes, offset)], data bytes) of a CompressedModel or PackedModel; offsets are
    relative to the first 16-byte boundary after the header, every section starts on a 16-byte boundary.  The
    buffers' sections follow the parameters', and the header lists buffers only when the model stores them."""
    sections, entries, off = [], [], 0

    def place(tensor):
        nonlocal off
        nb = tensor.numel() * tensor.element_size()
        sections.append((tensor, nb, off))
        span, off = [off, nb], _align(off + nb)
        return span

    for t in m.tensors:
        e = {"name": t.name, "shape": list(t.shape), "dtype": "float32", "quantized": t.quantized, "sections": {}}
        if t.quantized:
            e.update(m._entry_fields(t))
            if t.points is not None:
                e["points"] = [float(v) for v in t.points.detach().cpu().numpy().astype(np.float32)]
        for name in m._SECTIONS if t.quantized else ("raw",):
            e["sections"][name] = place(getattr(t, name))
        entries.append(e)
    buffers = [{"name": name, "shape": list(b.shape), "dtype": _dtype_name(b), "section": place(b)} for name, b in m.buffers or []]
    header = {**m._header({"kind": m.kind, "levels": m.levels, "bucket": m.bucket_size}), "tensors": entries, "data_bytes": off}
    if m.buffers is not None:
        header["buffers"] = buffers
    return json.dumps(header, separators=(",", ":")).encode("utf-8"), sections, off


def _write_container(m, path) -> int:
    """prefix (magic, version, 0, header length), the JSON header, then every section little-endian at its offset from
    the first 16-byte boundary after the header.  Returns the file size."""
    header, sections, data_bytes = _layout(m)
    start = _align(_PREFIX.size + len(header))
    buf = bytearray(start + data_bytes)
    buf[:_PREFIX.size] = _PREFIX.pack(m._MAGIC, m._version(), 0, len(header))
    buf[_PREFIX.size:_PREFIX.size + len(header)] = header
    little = {torch.int32: "<i4", torch.float32: "<f4", torch.int64: "<i8", torch.uint8: "u1"}
    for tensor, nb, off in sections:
        buf[start + off:start + off + nb] = tensor.detach().contiguous().cpu().numpy().astype(little[tensor.dtype], copy=False).tobytes()
    with open(path, "wb") as f:
        f.write(buf)
    return len(buf)


def _persistent_buffers(model):
    """[(name, tensor)] of the buffers model.state_dict() holds, in its order."""
    params = {id(p) for p in model.parameters()}
    return [(k, v) for k, v in model.state_dict(keep_vars=True).items() if torch.is_tensor(v) and id(v) not in params]


def _flat(p, dev):
    return p.detach().to(dev, torch.float32).contiguous().view(-1)


def _points(points, dev):
    return torch.as_tensor(points, dtype=torch.float32).detach().to(dev).contiguous().view(-1)


def _quantization_plan(model, numBits, quantize_first_and_last_layer, points, rule, include_buffers):
    """The arguments of compress_model and pack_model, checked before any device work: (named parameters,
    {index of a quantized parameter: its points, None when uniform}, s (uniform) or None, the persistent buffers copied
    to the device or None, the device).  The quantized parameters are all of them, or all but the first and the last,
    exactly as get_size_quantized_model selects them."""
    buffers = None
    if include_buffers:
        buffers = _persistent_buffers(model)
        for _, b in buffers:
            _dtype_name(b)
    if (numBits is None) == (points is None):
        raise ValueError("give numBits (uniform) or points (non-uniform), not both")
    named = list(model.named_parameters())
    order = list(range(len(named))) if quantize_first_and_last_layer is True else list(range(1, len(named) - 1))
    if not order:
        raise ValueError("no parameter is selected for quantization")
    s = None
    if points is None:
        s = 2 ** int(numBits)
        if not 2 <= s <= 256:
            raise ValueError("stored codes have at most 8 bits: numBits must be in [1, 8]")
        pts_list = [None] * len(order)
    else:
        per_tensor = len(points) > 0 and (torch.is_tensor(points[0]) or isinstance(points[0], (list, tuple, np.ndarray)))
        pts_list = list(points) if per_tensor else [points] * len(order)
        if len(pts_list) != len(order):
            raise ValueError(f"{len(pts_list)} point lists for {len(order)} quantized tensors")
        if rule not in ("nearest", "midpoint"):
            raise ValueError(f"unknown rule {rule!r}")
    N.require_cuda()
    dev = next((p.device for _, p in named if p.is_cuda), torch.device("cuda", torch.cuda.current_device()))
    if buffers is not None:
        buffers = [(name, b.detach().to(dev).clone()) for name, b in buffers]
    return named, dict(zip(order, pts_list)), s, buffers, dev


def _device_of(m, device=None):
    N.require_cuda()
    if device is not None:
        return torch.device(device)
    for t in m.tensors:
        for x in (getattr(t, m._SECTIONS[0]), t.raw):
            if x is not None and x.is_cuda:
                return x.device
    return torch.device("cuda", torch.cuda.current_device())


def _mover(m, dev):
    """tensor -> the same tensor on ``dev``.  Sections of a file loaded to the host are views into its data region,
    which goes to ``dev`` in one copy (on first use); any other tensor moves by itself (no copy when it is there)."""
    host = m._data if m._data is not None and not m._data.is_cuda else None
    region = []

    def move(x):
        if x is None:
            return None
        if host is not None and not x.is_cuda and x.untyped_storage().data_ptr() == host.untyped_storage().data_ptr():
            if not region:
                region.append(host.to(dev))
            off = x.data_ptr() - host.data_ptr()
            return region[0][off:off + x.numel() * x.element_size()].view(x.dtype).view(x.shape)
        return x.to(dev)
    return move


def _decode_args(m, items, dev, move):
    """Arguments of the format's whole-model decode (qd_huffman_decode_dequant_model / qd_unpack_dequant_model) of every
    (quantized tensor, out) of ``items`` on ``dev`` (the current device); out: contiguous float32 on ``dev``.  Also
    returns the tensors the call reads, which must outlive its enqueueing."""
    desc = np.zeros(len(items), m._DESCRIPTOR)
    keep = []
    if m.kind != "uniform":                      # every tensor's points in one upload
        src = items[0][0].points.device
        flat = move(torch.cat([t.points.reshape(-1).to(src, torch.float32) for t, _ in items]))
        keep.append(flat)
    at = 0
    for i, (t, out) in enumerate(items):
        sections = [move(getattr(t, name)) for name in m._SECTIONS]
        keep += sections
        points, k = 0, 0
        if m.kind != "uniform":
            k = t.points.numel()
            points = flat[at:at + k].data_ptr()
            at += k
        desc[i] = m._descriptor(t, sections, points, k, out)
    ws = torch.empty(int(getattr(N.lib(), m._WORKSPACE)(len(items))), dtype=torch.uint8, device=dev)
    keep += [desc, ws]
    args = (desc.ctypes.data, len(items), *m._decode_tables(dev), _bucket(m.bucket_size), int(m.levels) if m.kind == "uniform" else 0,
            N.ptr(ws), ws.numel(), N.stream_ptr(dev))
    return args, keep


def _check_target(m, model):
    """(named parameters, persistent buffers) of ``model`` once they are known to match ``m``; ValueError otherwise."""
    named = list(model.named_parameters())
    if len(named) != len(m.tensors):
        raise ValueError(f"model has {len(named)} parameters, the {m._WHAT} {len(m.tensors)}")
    for (name, p), t in zip(named, m.tensors):
        if tuple(p.shape) != tuple(t.shape):
            raise ValueError(f"{name}: shape {tuple(p.shape)} != stored {tuple(t.shape)} ({t.name})")
    bufs = []
    if m.buffers is not None:
        bufs = _persistent_buffers(model)
        if len(bufs) != len(m.buffers):
            raise ValueError(f"model has {len(bufs)} persistent buffers, the {m._WHAT} {len(m.buffers)}")
        for (name, b), (stored, s) in zip(bufs, m.buffers):
            if tuple(b.shape) != tuple(s.shape) or b.dtype != s.dtype:
                raise ValueError(f"buffer {name}: {b.dtype} {tuple(b.shape)} != stored {s.dtype} {tuple(s.shape)} ({stored})")
    return named, bufs


def _write_into(m, named, bufs, skip=()) -> None:
    """The writing half of decompress_ / unpack_: every parameter but those whose indices are in ``skip``, then the
    buffers.  Per device, the quantized tensors decode in one launch, straight into parameters that are contiguous
    float32 on that device; the others go through a temporary."""
    default = _device_of(m)
    groups = {}                                  # device -> parameter indices (host parameters decode on `default`)
    for k, (_, p) in enumerate(named):
        if k not in skip:
            groups.setdefault(p.device if p.is_cuda else default, []).append(k)
    for _, b in bufs:
        if b.is_cuda:
            groups.setdefault(b.device, [])
    with torch.no_grad():
        for dev, ks in groups.items():
            with torch.cuda.device(dev):
                move = _mover(m, dev)
                items, temps = [], []
                for k in ks:
                    t, d = m.tensors[k], named[k][1].data
                    if not t.quantized:
                        d.copy_((move(t.raw) if d.is_cuda else t.raw).view_as(d))
                    elif d.device == dev and d.dtype == torch.float32 and d.is_contiguous():
                        items.append((t, d))
                    else:
                        out = torch.empty(t.numel, dtype=torch.float32, device=dev)
                        items.append((t, out))
                        temps.append((d, out))
                if items:
                    args, keep = _decode_args(m, items, dev, move)
                    N.check(getattr(N.lib(), m._DECODE)(*args))
                for d, out in temps:
                    d.copy_(out.view_as(d))
                for (_, b), (_, s) in zip(bufs, m.buffers or []):
                    if b.is_cuda and b.device == dev:
                        b.copy_(move(s))
        for (_, b), (_, s) in zip(bufs, m.buffers or []):
            if not b.is_cuda:
                b.copy_(s)


def _read_container(cls, path, device):
    """A CompressedModel or PackedModel (``cls``) read from ``path`` and validated on the host before anything reaches a
    device: prefix, header, every tensor entry (unique names, exactly its format's sections, each in bounds, aligned and
    of the size its shape needs), buffers, and no two sections overlapping.  Every section is a view into one tensor
    holding the file's data region; a ``device`` gets that region in one copy."""
    def bad(msg):
        raise ValueError(f"not a valid {cls._FILE}: {msg}")

    with open(path, "rb") as f:
        buf = bytearray(f.read())
    if len(buf) < _PREFIX.size:
        bad("shorter than its prefix")
    magic, version, reserved, hlen = _PREFIX.unpack_from(buf)
    if magic != cls._MAGIC:
        bad("bad magic")
    if version not in cls._VERSIONS:
        bad(f"format version {version}, this reader knows {' and '.join(str(v) for v in cls._VERSIONS)}")
    if reserved != 0:
        bad("reserved prefix field is not 0")
    if _PREFIX.size + hlen > len(buf):
        bad("header runs past the end of the file")
    try:
        h = json.loads(buf[_PREFIX.size:_PREFIX.size + hlen].decode("utf-8"))
        kind, levels, bucket, entries, data_bytes = h["kind"], h["levels"], h["bucket"], h["tensors"], h["data_bytes"]
    except (ValueError, KeyError, TypeError) as e:
        bad(f"unreadable header ({e})")
    if not isinstance(data_bytes, int) or not isinstance(entries, list):
        bad("data_bytes must be an integer and tensors a list")
    start = _align(_PREFIX.size + hlen)
    if data_bytes < 0 or start + data_bytes != len(buf):
        bad(f"{len(buf)} bytes, the header describes {start + data_bytes}")
    if kind not in ("uniform", "nonuniform"):
        bad(f"unknown kind {kind!r}")
    if kind == "uniform" and not (isinstance(levels, int) and not isinstance(levels, bool) and 2 <= levels <= 256):
        bad("uniform levels must be in [2, 256]")
    if kind == "nonuniform" and levels is not None:
        bad("a non-uniform model has no levels")
    if bucket is not None and not (isinstance(bucket, int) and not isinstance(bucket, bool) and bucket > 0):
        bad("bucket must be a positive integer or null")
    extra = cls._read_header(h, version, levels, bad)
    region = torch.from_numpy(np.frombuffer(buf, np.uint8, count=data_bytes, offset=start)) if data_bytes else \
        torch.empty(0, dtype=torch.uint8)
    spans = []

    def view(off, nb, dtype, shape):
        return region[off:off + nb].view(dtype).view(shape)

    def section(e, name, dtype, nbytes):
        try:
            off, nb = (int(v) for v in e["sections"][name])
        except (KeyError, TypeError, ValueError):
            bad(f"{e.get('name')}: section {name} missing")
        if nb != nbytes:
            bad(f"{e.get('name')}: section {name} holds {nb} bytes, {nbytes} expected")
        if off < 0 or off % _ALIGN or off + nb > data_bytes:
            bad(f"{e.get('name')}: section {name} out of range")
        spans.append((off, nb))
        return view(off, nb, dtype, (nbytes // dtype.itemsize,))

    tensors, names = [], set()
    for e in entries:
        try:
            name, shape, quantized = str(e["name"]), tuple(int(d) for d in e["shape"]), e["quantized"]
        except (KeyError, TypeError, ValueError):
            bad("tensor entry without name / shape / quantized")
        if not isinstance(quantized, bool) or e.get("dtype") != "float32" or any(d < 0 for d in shape):
            bad(f"{name}: bad dtype, shape or quantized flag")
        if name in names:
            bad(f"tensor {name} appears twice")
        names.add(name)
        if not isinstance(e.get("sections"), dict) or set(e["sections"]) != (set(cls._SECTIONS) if quantized else {"raw"}):
            bad(f"{name}: unexpected sections")
        n = int(math.prod(shape))
        if not quantized:
            tensors.append(cls._ENTRY(name, shape, raw=section(e, "raw", torch.float32, 4 * n)))
            continue
        if n == 0:
            bad(f"{name}: empty quantized tensor")
        pts = None
        if kind == "uniform" and "points" in e:
            bad(f"{name}: a uniform tensor has no points")
        if kind == "nonuniform":
            try:
                pts = torch.tensor([float(v) for v in e["points"]], dtype=torch.float32)
            except (KeyError, TypeError, ValueError):
                bad(f"{name}: non-uniform tensor without points")
        fields = cls._read_entry(e, name, n, levels, pts, section, bad)
        rows = _rows(n, bucket)
        tensors.append(cls._ENTRY(name, shape, alpha=section(e, "alpha", torch.float32, 4 * rows),
                                  beta=section(e, "beta", torch.float32, 4 * rows), points=pts, **fields))
    buffers = _read_buffers(h["buffers"], view, data_bytes, bad, spans) if "buffers" in h else None
    spans.sort()
    for (o1, n1), (o2, _) in zip(spans, spans[1:]):
        if o1 + n1 > o2:
            bad(f"sections at {o1} and {o2} overlap")
    m = cls(kind=kind, levels=levels, bucket_size=bucket, tensors=tensors, buffers=buffers, **extra)
    m._data = region
    if device is not None:                       # everything is validated before anything reaches the GPU
        move = _mover(m, torch.device(device))
        pts = [t.points for t in tensors if t.points is not None]
        flat = torch.cat(pts).to(device) if pts else None          # every tensor's points in one upload too
        at = 0
        for t in tensors:
            for f_ in cls._SECTIONS + ("raw",):
                setattr(t, f_, move(getattr(t, f_)))
            if t.points is not None:
                t.points, at = flat[at:at + t.points.numel()], at + t.points.numel()
        if buffers is not None:
            m.buffers = [(name, move(b)) for name, b in buffers]
        m._data = move(region)
    return m


def _read_buffers(entries, view, data_bytes, bad, spans):
    """[(name, tensor view)] of a header's buffer entries, each checked against the data region; ``bad(msg)`` raises.
    Every buffer's (offset, bytes) is appended to ``spans``."""
    if not isinstance(entries, list):
        bad("buffers is not a list")
    buffers, names = [], set()
    for e in entries:
        try:
            name, shape, dtype = str(e["name"]), tuple(int(d) for d in e["shape"]), e["dtype"]
            off, nb = (int(v) for v in e["section"])
        except (KeyError, TypeError, ValueError):
            bad("buffer entry without name / shape / dtype / section")
        if dtype not in _BUFFER_DTYPES:
            bad(f"buffer {name}: unknown dtype {dtype!r}")
        if any(d < 0 for d in shape):
            bad(f"buffer {name}: bad shape")
        if name in names:
            bad(f"buffer {name} appears twice")
        names.add(name)
        tdtype = _BUFFER_DTYPES[dtype]
        size = int(math.prod(shape)) * tdtype.itemsize
        if nb != size:
            bad(f"buffer {name}: {nb} bytes, its shape and dtype need {size}")
        if off < 0 or off % _ALIGN or off + nb > data_bytes:
            bad(f"buffer {name}: section out of range")
        spans.append((off, nb))
        buffers.append((name, view(off, nb, tdtype, shape)))
    return buffers


def compress_model(model, numBits=None, bucket_size=256, quantize_first_and_last_layer=True, *, points=None,
                   rule="nearest", include_buffers=False) -> CompressedModel:
    """Huffman-codes a model's quantized parameters.  Uniform: ``numBits`` (s = 2**numBits levels,
    uniformQuantization).  Non-uniform: ``points`` -- one ascending list of centroids for every tensor, or one
    list per quantized tensor (the differentiable-quantization output) -- with nonUniformQuantization's
    ``rule``.  One level histogram over all quantized tensors gives the code, so the stored code bits equal
    get_huffman_encoding_mean_bit_length x the number of quantized weights.  ``include_buffers``: also store the
    persistent buffers (state_dict() order, float32 or int64, e.g. BatchNorm running statistics) as they are, so
    that decompress_ into a freshly built network gives back the whole eval-mode model."""
    named, quantized, s, buffers, dev = _quantization_plan(model, numBits, quantize_first_and_last_layer, points, rule, include_buffers)
    sp = N.stream_ptr(dev)
    tensors, idxs = [], []
    with torch.cuda.device(dev):
        for i, (name, p) in enumerate(named):
            if i not in quantized:
                tensors.append(HuffmanTensor(name, tuple(p.shape), raw=_flat(p, dev).clone()))
                continue
            pts = None if s is not None else _points(quantized[i], dev)
            idx, alpha, beta = _levels(_flat(p, dev), s, pts, bucket_size, rule, sp)
            idxs.append(idx)
            tensors.append(HuffmanTensor(name, tuple(p.shape), alpha=alpha, beta=beta, points=pts))
        return _huffman_coded("uniform" if s is not None else "nonuniform", s, bucket_size, tensors, idxs,
                              [256 if s is None else s] * len(idxs), buffers, dev)


def _huffman_coded(kind, levels, bucket_size, tensors, idxs, bins, buffers, dev) -> CompressedModel:
    """What compress_model and compress_packed run once every quantized tensor of ``tensors`` (HuffmanTensor, in order)
    has its uint8 level indices in ``idxs`` on ``dev`` (the current device): one level histogram over all of them
    gives the code, then each stream is encoded into a capacity bounded by its code bits and trimmed to its length.
    ``bins``: each tensor's number of levels; a tensor with an index >= its bins raises ValueError naming it."""
    sp = N.stream_ptr(dev)
    counts = torch.zeros(len(idxs), 256, dtype=torch.int64, device=dev)
    for k, (idx, b) in enumerate(zip(idxs, bins)):
        N.check(N.lib().qd_index_histogram(N.ptr(idx), idx.numel(), b, N.ptr(counts[k]), sp))
    counts = counts.cpu()
    quantized = [t for t in tensors if t.quantized]
    for t, idx, b, seen in zip(quantized, idxs, bins, counts.sum(1).tolist()):
        if seen != idx.numel():
            raise ValueError(f"{t.name}: {idx.numel() - seen} codes are not among its {b} levels")
    lengths = huffman_code_lengths(counts.sum(0).numpy())
    cm = CompressedModel(kind, levels, bucket_size, lengths, tensors, buffers=buffers)
    table = cm.table(dev)
    len_vec = torch.zeros(256, dtype=torch.int64)
    for sym, l in lengths.items():
        len_vec[sym] = l
    code_bits = (counts * len_vec).sum(1).tolist()
    totals, bufs = torch.zeros(len(idxs), dtype=torch.int64, device=dev), []
    for k, (t, idx) in enumerate(zip(quantized, idxs)):
        n = idx.numel()
        chunks = -(-n // HUFFMAN_CHUNK)
        capacity = -(-int(code_bits[k]) // 32) + chunks
        if capacity - chunks > 1 << 32:
            raise ValueError(f"{t.name}: its Huffman stream would exceed 2^32 words")
        capacity = min(capacity, 1 << 32)
        words = torch.empty(max(capacity, 1), dtype=torch.int32, device=dev)
        offs = torch.empty(chunks, dtype=torch.int32, device=dev)
        N.check(N.lib().qd_huffman_encode(N.ptr(idx), n, N.ptr(table), N.ptr(words), capacity, N.ptr(offs), N.ptr(totals[k:k + 1]), sp))
        t.chunk_offsets, t.code_bits = offs, int(code_bits[k])
        bufs.append((words, capacity))
    for (t, (words, capacity)), total in zip(zip(quantized, bufs), totals.cpu().tolist()):
        if total > capacity:
            raise ValueError(f"{t.name}: its Huffman stream would exceed 2^32 words")
        t.words = words[:total]
    return cm


def decompress_tensor(cm: CompressedModel, which, out: torch.Tensor = None, device=None) -> torch.Tensor:
    """Decodes one tensor (index or name) of a CompressedModel to float32 on the GPU: the fake-quantized tensor
    bit for bit, or the stored tensor when it was kept unquantized.  ``out``: contiguous float32 CUDA tensor of
    the same number of elements to decode into."""
    t = cm.tensors[which] if isinstance(which, int) else next(x for x in cm.tensors if x.name == which)
    dev = out.device if out is not None else _device_of(cm, device)
    if out is None:
        out = torch.empty(t.shape, dtype=torch.float32, device=dev)
    if out.dtype != torch.float32 or not out.is_cuda or not out.is_contiguous() or out.numel() != t.numel:
        raise ValueError("out must be a contiguous float32 CUDA tensor with as many elements as the stored one")
    with torch.cuda.device(dev):
        if not t.quantized:
            out.view(-1).copy_(t.raw.view(-1))
            return out
        words, offs = t.words.to(dev), t.chunk_offsets.to(dev)
        alpha, beta = t.alpha.to(dev), t.beta.to(dev)
        b = _bucket(cm.bucket_size)
        sp = N.stream_ptr(dev)
        args = (N.ptr(words) if words.numel() else None, words.numel(), N.ptr(offs), N.ptr(cm.table(dev)))
        if cm.kind == "uniform":
            N.check(N.lib().qd_huffman_decode_dequant_uniform(*args, N.ptr(alpha), N.ptr(beta), N.ptr(out), t.numel, b, int(cm.levels), sp))
        else:
            pts = t.points.to(dev)
            N.check(N.lib().qd_huffman_decode_dequant_nonuniform(*args, N.ptr(pts), pts.numel(), N.ptr(alpha), N.ptr(beta), N.ptr(out),
                                                                 t.numel, b, sp))
    return out


def decompress_(cm: CompressedModel, model) -> None:
    """Writes every parameter of ``model`` in place from ``cm`` (existing parameter handles stay valid), and its
    persistent buffers when ``cm`` stores them.  Everything is checked before anything is written.  Per device, the
    quantized tensors decode in one launch, straight into parameters that are contiguous float32 on that device."""
    _write_into(cm, *_check_target(cm, model))


def save_compressed(cm: CompressedModel, path) -> int:
    """Writes the Huffman-coded container: magic QDHUFF, version 1 (2 when buffers are stored), JSON header,
    16-byte-aligned little-endian sections.  Returns the file size in bytes."""
    return _write_container(cm, path)


def load_compressed(path, device=None) -> CompressedModel:
    """Reads and validates a file written by save_compressed (version 1, or 2 with buffers).  Every section is a
    view into one tensor holding the file's data region.  device=None keeps it in host memory (reading and
    validating needs no GPU; decompress_ moves it to the GPU in one copy); a device gets it in one copy here."""
    return _read_container(CompressedModel, path, device)


def pack_model(model, numBits=None, bucket_size=256, quantize_first_and_last_layer=True, *, points=None, rule="nearest",
               include_buffers=False) -> PackedModel:
    """Stores a model's quantized parameters fixed-width, one fused quantize-and-pack launch per tensor.  Parameters
    are selected as in compress_model.  Uniform: ``numBits`` (s = 2**numBits levels, uniformQuantization), codes of
    bits_for(s) bits.  Non-uniform: ``points`` -- one ascending list for every tensor, or one list per quantized tensor
    (the differentiable-quantization output) -- with nonUniformQuantization's ``rule``; tensor t gets codes of
    bits_for(K_t) bits.  ``include_buffers`` also stores the persistent buffers (float32 / int64) as they are."""
    named, quantized, s, buffers, dev = _quantization_plan(model, numBits, quantize_first_and_last_layer, points, rule, include_buffers)
    b = _bucket(bucket_size)
    tensors = []
    with torch.cuda.device(dev):
        sp = N.stream_ptr(dev)
        ws_bytes = max(int(N.lib().qd_packed_workspace_bytes(named[i][1].numel(), b)) for i in quantized)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)     # stream-ordered: free to reuse once the launches ran
        for i, (name, p) in enumerate(named):
            if i not in quantized:
                tensors.append(PackedEntry(name, tuple(p.shape), raw=_flat(p, dev).clone()))
                continue
            x = _flat(p, dev)
            n = x.numel()
            rows = _rows(n, bucket_size)
            alpha = torch.empty(rows, device=dev)
            beta = torch.empty(rows, device=dev)
            if s is not None:
                bits, pts = bits_for(s), None
                packed = torch.empty((n * bits + 7) // 8, dtype=torch.uint8, device=dev)
                N.check(N.lib().qd_uniform_fwd_packed(N.ptr(x), N.ptr(packed), bits, N.ptr(alpha), N.ptr(beta), n, b, s, N.ptr(ws),
                                                      ws.numel(), sp))
            else:
                pts = _points(quantized[i], dev)
                if not 1 <= pts.numel() <= 256:
                    raise ValueError(f"{name}: {pts.numel()} points, the packed codec stores 1 to 256")
                bits = bits_for(pts.numel())
                packed = torch.empty((n * bits + 7) // 8, dtype=torch.uint8, device=dev)
                N.check(N.lib().qd_nonuniform_fwd_packed(N.ptr(x), N.ptr(pts), pts.numel(),
                                                         N.RULE_MIDPOINT if rule == "midpoint" else N.RULE_NEAREST, N.ptr(packed), bits,
                                                         N.ptr(alpha), N.ptr(beta), n, b, N.ptr(ws), ws.numel(), sp))
            tensors.append(PackedEntry(name, tuple(p.shape), bits=bits, packed=packed, alpha=alpha, beta=beta, points=pts))
    return PackedModel("uniform" if s is not None else "nonuniform", s, bucket_size, tensors, buffers=buffers)


def unpack_(pm: PackedModel, model) -> None:
    """Writes every parameter of ``model`` in place from ``pm`` (existing parameter handles stay valid), and its
    persistent buffers when ``pm`` stores them.  Everything is checked before anything is written.  Per device, the
    quantized tensors decode in one launch, straight into parameters that are contiguous float32 on that device."""
    _write_into(pm, *_check_target(pm, model))


def _hold_sections(layer, entry: PackedEntry, kind: str, levels, bucket_size, bias, out: int) -> None:
    """Registers one quantized tensor's packed sections (and the layer's bias of ``out`` elements) as non-persistent
    buffers of ``layer`` on the sections' CUDA device: what PackedLinear and PackedConv2d hold in place of a float32
    weight."""
    if kind not in ("uniform", "nonuniform"):
        raise ValueError(f"unknown kind {kind!r}")
    layer.kind, layer.bits, layer.bucket_size = kind, int(entry.bits), bucket_size
    layer.levels = int(levels) if kind == "uniform" else 0
    dev = entry.packed.device
    if not dev.type == "cuda":
        raise ValueError(f"{entry.name}: the packed sections must be on a CUDA device")

    def own(t):                                  # a view into a loaded file's region is copied out of it
        t = t.to(dev).contiguous()
        return t.clone() if t.untyped_storage().nbytes() > t.numel() * t.element_size() else t
    layer.register_buffer("packed", own(entry.packed), persistent=False)
    layer.register_buffer("alpha", own(entry.alpha.to(torch.float32)), persistent=False)
    layer.register_buffer("beta", own(entry.beta.to(torch.float32)), persistent=False)
    layer.register_buffer("points", None if kind == "uniform" else own(entry.points.reshape(-1).to(torch.float32)), persistent=False)
    if bias is not None:
        if tuple(bias.shape) != (out,):
            raise ValueError(f"{entry.name}: bias of shape {tuple(bias.shape)}, expected ({out},)")
        bias = bias.detach().to(dev, torch.float32).contiguous()
    layer.register_buffer("bias", bias, persistent=False)


def _check_input(layer, x, what: str) -> None:
    if not torch.is_tensor(x) or not x.is_cuda or x.dtype != torch.float32:
        raise ValueError(f"{what} takes a float32 CUDA tensor")
    if x.device != layer.packed.device:
        raise ValueError(f"input on {x.device}, the packed weight on {layer.packed.device}")


def _check_state(layer, x, what: str) -> None:
    """Refusals after the input's shape: sections cast away from uint8 / float32, an input that needs a gradient in
    grad mode."""
    if layer.packed.dtype != torch.uint8 or any(t is not None and t.dtype != torch.float32 for t in (layer.alpha, layer.beta, layer.points, layer.bias)):
        raise RuntimeError(f"{what}'s sections must stay uint8 codes and float32 scales, points and bias "
                           "(the module was cast, e.g. by .half() or .double())")
    if torch.is_grad_enabled() and x.requires_grad:
        raise RuntimeError(f"{what} is forward only: it cannot propagate a gradient to its input "
                           "(run it under torch.no_grad() or torch.inference_mode())")


def _decoded(layer, shape) -> torch.Tensor:
    w = torch.empty(*shape, dtype=torch.float32, device=layer.packed.device)
    return _unpack(layer.packed, layer.bits, layer.alpha, layer.beta, layer.points, layer.levels, layer.bucket_size, w)


class PackedLinear(torch.nn.Module):
    """Inference replacement of an ``nn.Linear`` whose weight stays in its fixed-width stored form (one PackedEntry of
    a PackedModel: codes, alpha and beta per bucket, points) on the device.  For batches of at most CROSSOVER_ROWS
    rows, forward runs qd_packed_linear, which reads the codes and never materialises the float32 weight; its weights
    are the decoded ones bit for bit, the sum is float32 in a fixed order.  Larger batches decode the weight into a
    scratch tensor (qd_unpack_dequant_*) and call F.linear: exactly what an unpack_-loaded model computes.  Forward
    only: an input that needs a gradient in grad mode is refused.  No host synchronisation, so it can be captured in
    a CUDA graph."""
    # largest batch (rows of x after flattening) that runs on the packed kernel.  Measured (DESIGN.md section 3.7.2):
    # up to 4 rows the kernel beats decode + F.linear on the AlexNet heads (37.7 M and 16.8 M weights) at every width,
    # from 16 rows on it loses there; on layers of under a million weights it loses at every batch size.
    CROSSOVER_ROWS = 4

    def __init__(self, entry: PackedEntry, kind: str, levels, bucket_size, bias: torch.Tensor = None):
        super().__init__()
        if not entry.quantized or len(entry.shape) != 2:
            raise ValueError(f"{entry.name}: a PackedLinear needs a quantized two-dimensional weight")
        self.out_features, self.in_features = (int(d) for d in entry.shape)
        _hold_sections(self, entry, kind, levels, bucket_size, bias, self.out_features)

    def extra_repr(self) -> str:
        return (f"in_features={self.in_features}, out_features={self.out_features}, bias={self.bias is not None}, "
                f"{self.kind}, bits={self.bits}, bucket_size={self.bucket_size}")

    def decoded_weight(self) -> torch.Tensor:
        """The decoded float32 weight [out_features, in_features], bit for bit what unpack_ writes."""
        return _decoded(self, (self.out_features, self.in_features))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        _check_input(self, x, "PackedLinear")
        if x.dim() < 1 or x.shape[-1] != self.in_features:
            raise ValueError(f"input of shape {tuple(x.shape)}, expected (..., {self.in_features})")
        _check_state(self, x, "PackedLinear")
        lead = x.shape[:-1]
        x2 = x.reshape(-1, self.in_features).contiguous()
        m = x2.shape[0]
        with torch.cuda.device(x.device):
            if m > self.CROSSOVER_ROWS:
                return torch.nn.functional.linear(x2, self.decoded_weight(), self.bias).view(*lead, self.out_features)
            y = torch.empty(m, self.out_features, dtype=torch.float32, device=x.device)
            if m:
                b = 0 if self.bucket_size is None else int(self.bucket_size)
                N.check(N.lib().qd_packed_linear(N.ptr(x2), m, self.in_features, self.out_features, N.ptr(self.packed), self.bits,
                                                 N.ptr(self.alpha), N.ptr(self.beta), N.ptr(self.points),
                                                 0 if self.points is None else self.points.numel(), self.levels, b, N.ptr(self.bias),
                                                 N.ptr(y), N.stream_ptr(x.device)))
        return y.view(*lead, self.out_features)


def _pair(v, what: str) -> tuple:
    p = (v, v) if isinstance(v, int) else tuple(v)
    if len(p) != 2 or not all(isinstance(i, int) and not isinstance(i, bool) for i in p):
        raise ValueError(f"{what} must be an int or a pair of ints, got {v!r}")
    return p


class PackedConv2d(torch.nn.Module):
    """Inference replacement of an ``nn.Conv2d`` (groups 1, dilation 1, symmetric zero padding) whose weight stays in
    its fixed-width stored form (one PackedEntry of a PackedModel with a [O, C, kh, kw] shape) on the device.  Takes
    NCHW float32 input, or one CHW image.  When the layer has K = C*kh*kw <= KERNEL_MAX_TAPS and a call's work,
    N*Ho*Wo*O*K multiply-adds, is at most CROSSOVER_MACS (runs_kernel), forward runs qd_packed_conv2d, which reads the codes and never materialises the float32 weight; its
    weights are the decoded ones bit for bit, each output is one float32 fmaf chain in a fixed order.  Above it, the
    weight is decoded into a scratch tensor (qd_unpack_dequant_*), F.conv2d is called and the scratch is freed: exactly
    what an unpack_-loaded nn.Conv2d computes, TF32 setting and input strides included (the kernel path reads a
    contiguous copy of a non-contiguous input).  Forward only: an input that needs a gradient in
    grad mode is refused.  No host synchronisation, so it can be captured in a CUDA graph."""
    # Measured (DESIGN.md section 3.7.3): the kernel beats decode + F.conv2d (TF32 on) by 5-25 % on layers of 16 and
    # 27 taps up to 8.4 M multiply-adds (WRN's 16->352 shortcut at batch 1, its stem up to batch 8); on every layer of
    # 144 taps or more it loses at every batch, by up to 10x, since one CTA walks the whole K chain.
    KERNEL_MAX_TAPS = 32
    CROSSOVER_MACS = 1 << 23

    def __init__(self, entry: PackedEntry, kind: str, levels, bucket_size, stride=1, padding=0, bias: torch.Tensor = None):
        super().__init__()
        if not entry.quantized or len(entry.shape) != 4:
            raise ValueError(f"{entry.name}: a PackedConv2d needs a quantized four-dimensional weight")
        self.out_channels, self.in_channels, kh, kw = (int(d) for d in entry.shape)
        self.kernel_size = (kh, kw)
        self.stride, self.padding = _pair(stride, "stride"), _pair(padding, "padding")
        if min(self.stride) < 1 or min(self.padding) < 0:
            raise ValueError(f"{entry.name}: stride must be >= 1 and padding >= 0")
        _hold_sections(self, entry, kind, levels, bucket_size, bias, self.out_channels)

    def extra_repr(self) -> str:
        return (f"{self.in_channels}, {self.out_channels}, kernel_size={self.kernel_size}, stride={self.stride}, "
                f"padding={self.padding}, bias={self.bias is not None}, {self.kind}, bits={self.bits}, bucket_size={self.bucket_size}")

    def decoded_weight(self) -> torch.Tensor:
        """The decoded float32 weight [out_channels, in_channels, kh, kw], bit for bit what unpack_ writes."""
        return _decoded(self, (self.out_channels, self.in_channels, *self.kernel_size))

    def runs_kernel(self, n: int, ho: int, wo: int) -> bool:
        """True when a call with batch n and output Ho x Wo runs qd_packed_conv2d, False when it decodes."""
        k = self.in_channels * self.kernel_size[0] * self.kernel_size[1]
        return k <= self.KERNEL_MAX_TAPS and n * ho * wo * self.out_channels * k <= self.CROSSOVER_MACS

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        _check_input(self, x, "PackedConv2d")
        if x.dim() not in (3, 4) or x.shape[-3] != self.in_channels:
            raise ValueError(f"input of shape {tuple(x.shape)}, expected (N, {self.in_channels}, H, W) or ({self.in_channels}, H, W)")
        _check_state(self, x, "PackedConv2d")
        (kh, kw), (sh, sw), (ph, pw) = self.kernel_size, self.stride, self.padding
        n, (h, w) = (x.shape[0] if x.dim() == 4 else 1), x.shape[-2:]
        if h + 2 * ph < kh or w + 2 * pw < kw:
            raise ValueError(f"input of shape {tuple(x.shape)} is smaller than the {kh}x{kw} kernel after padding {self.padding}")
        ho, wo = (h + 2 * ph - kh) // sh + 1, (w + 2 * pw - kw) // sw + 1
        with torch.cuda.device(x.device):
            if not self.runs_kernel(n, ho, wo):
                return torch.nn.functional.conv2d(x, self.decoded_weight(), self.bias, self.stride, self.padding)
            xc = x.contiguous()
            y = torch.empty(n, self.out_channels, ho, wo, dtype=torch.float32, device=x.device)
            if n:
                b = 0 if self.bucket_size is None else int(self.bucket_size)
                N.check(N.lib().qd_packed_conv2d(N.ptr(xc), n, self.in_channels, h, w, self.out_channels, kh, kw, sh, sw, ph, pw,
                                                 N.ptr(self.packed), self.bits, N.ptr(self.alpha), N.ptr(self.beta), N.ptr(self.points),
                                                 0 if self.points is None else self.points.numel(), self.levels, b, N.ptr(self.bias),
                                                 N.ptr(y), N.stream_ptr(x.device)))
        return y if x.dim() == 4 else y[0]


class PackedEmbedding(torch.nn.Module):
    """Inference replacement of an ``nn.Embedding`` whose weight stays in its fixed-width stored form (one PackedEntry
    of a PackedModel with a [num_embeddings, embedding_dim] shape) on the device.  Forward takes int32 or int64 CUDA
    indices of any shape and returns ``input.shape + (embedding_dim,)`` float32 rows gathered by qd_packed_embedding,
    which reads only the codes of those rows: every value is bit for bit what unpack_ writes for it.  The row of
    ``padding_idx`` is returned as stored, as an unpack_-loaded nn.Embedding returns it.  Unlike torch, an index outside
    [0, num_embeddings) does not raise a device-side assert: its output row is NaN and it is counted on the device,
    which invalid_index_count() reads.  Forward never synchronises, so it can be captured in a CUDA graph."""

    def __init__(self, entry: PackedEntry, kind: str, levels, bucket_size, padding_idx=None):
        super().__init__()
        if not entry.quantized or len(entry.shape) != 2:
            raise ValueError(f"{entry.name}: a PackedEmbedding needs a quantized two-dimensional weight")
        self.num_embeddings, self.embedding_dim = (int(d) for d in entry.shape)
        if padding_idx is not None:
            if not -self.num_embeddings <= padding_idx < self.num_embeddings:
                raise ValueError(f"{entry.name}: padding_idx {padding_idx} outside the {self.num_embeddings} embeddings")
            padding_idx = padding_idx % self.num_embeddings
        self.padding_idx = padding_idx
        _hold_sections(self, entry, kind, levels, bucket_size, None, 0)
        self.register_buffer("invalid", torch.zeros(1, dtype=torch.int32, device=self.packed.device), persistent=False)

    def extra_repr(self) -> str:
        return (f"{self.num_embeddings}, {self.embedding_dim}, padding_idx={self.padding_idx}, {self.kind}, bits={self.bits}, "
                f"bucket_size={self.bucket_size}")

    def decoded_weight(self) -> torch.Tensor:
        """The decoded float32 weight [num_embeddings, embedding_dim], bit for bit what unpack_ writes."""
        return _decoded(self, (self.num_embeddings, self.embedding_dim))

    def invalid_index_count(self) -> int:
        """Number of out-of-range indices forward has met since the last call, read with one device synchronise, then
        reset to 0."""
        torch.cuda.synchronize(self.invalid.device)
        n = int(self.invalid.item())
        self.invalid.zero_()
        return n

    def forward(self, input: torch.Tensor) -> torch.Tensor:
        if not torch.is_tensor(input) or not input.is_cuda or input.dtype not in (torch.int32, torch.int64):
            raise ValueError("PackedEmbedding takes an int32 or int64 CUDA tensor of indices")
        if input.device != self.packed.device:
            raise ValueError(f"input on {input.device}, the packed weight on {self.packed.device}")
        _check_state(self, input, "PackedEmbedding")
        out = torch.empty(*input.shape, self.embedding_dim, dtype=torch.float32, device=input.device)
        if input.numel():
            idx = input.contiguous()
            b = 0 if self.bucket_size is None else int(self.bucket_size)
            with torch.cuda.device(input.device):
                N.check(N.lib().qd_packed_embedding(N.ptr(idx), idx.element_size(), idx.numel(), self.num_embeddings,
                                                    self.embedding_dim, N.ptr(self.packed), self.bits, N.ptr(self.alpha),
                                                    N.ptr(self.beta), N.ptr(self.points), 0 if self.points is None else self.points.numel(),
                                                    self.levels, b, N.ptr(out), N.ptr(self.invalid), N.stream_ptr(input.device)))
        return out


class _PackedWeight(torch.nn.Module):
    """One packed [rows, cols] weight matrix of a recurrent module and the bias that goes with it, held as the sections
    _hold_sections registers (packed, alpha, beta, points, bias)."""

    def __init__(self, entry: PackedEntry, kind: str, levels, bucket_size, bias, rows: int, cols: int):
        super().__init__()
        if not entry.quantized or tuple(entry.shape) != (rows, cols):
            raise ValueError(f"{entry.name}: expected a quantized [{rows}, {cols}] weight, got {tuple(entry.shape)}"
                             f"{'' if entry.quantized else ' kept float32'}")
        self.shape = (rows, cols)
        _hold_sections(self, entry, kind, levels, bucket_size, bias, rows)

    def decoded(self) -> torch.Tensor:
        return _decoded(self, self.shape)

    def descriptor(self) -> np.ndarray:
        """The host qd_packed_tensor of the weight (q NULL: the LSTM entry points do not write one)."""
        d = np.zeros(1, _PACKED_TENSOR)
        d[0] = (N.ptr(self.packed), N.ptr(self.alpha), N.ptr(self.beta), 0 if self.points is None else N.ptr(self.points), 0,
                self.shape[0] * self.shape[1], self.bits, 0 if self.points is None else self.points.numel())
        return d


def _check_weights(weights, x, what: str) -> None:
    for w in weights:
        _check_input(w, x, what)
        _check_state(w, x, what)


def _gate_sizes(entry, gates: int, what: str) -> tuple:
    """(hidden_size, input_size) of a recurrent input weight [gates * hidden_size, input_size]; ``what`` names the layer
    with its article ("an LSTM")."""
    if len(entry.shape) != 2 or entry.shape[0] % gates or entry.shape[0] < gates:
        raise ValueError(f"{entry.name}: {what} input weight is [{gates} * hidden_size, input_size], got {tuple(entry.shape)}")
    return int(entry.shape[0]) // gates, int(entry.shape[1])


def _cell_pair(entry_ih, entry_hh, kind, levels, bucket_size, bias_ih, bias_hh, gates, hidden_size, input_size) -> torch.nn.ModuleList:
    return torch.nn.ModuleList([_PackedWeight(entry_ih, kind, levels, bucket_size, bias_ih, gates * hidden_size, input_size),
                                _PackedWeight(entry_hh, kind, levels, bucket_size, bias_hh, gates * hidden_size, hidden_size)])


class PackedLSTMCell(torch.nn.Module):
    """Inference replacement of an ``nn.LSTMCell`` whose two weight matrices stay in their fixed-width stored form (two
    PackedEntry of a PackedModel, [4H, I] and [4H, H]) on the device.  Takes input [B, I] or [I] and ``hx`` = (h, c) or
    None (zeros), returns (h', c') in nn.LSTMCell's shapes.  Up to CROSSOVER_ROWS rows (none by default), forward runs
    qd_packed_lstm_cell: one launch that reads the codes of both weights and applies the cell update in registers,
    every weight bit for bit the decoded one, each gate's sum in qd_packed_linear's fixed float32 order (include/qd_b200.h
    states the contract).  Larger batches decode both weights into scratch tensors and call torch's LSTM cell: exactly
    what an unpack_-loaded nn.LSTMCell computes.  Forward only, no host synchronisation (graph-capturable)."""
    # largest batch that runs on the packed kernel (at most N.PACKED_LSTM_MAX_ROWS).  Measured (DESIGN.md section
    # 3.7.6): on the NMT decoder cells the kernel loses to decode + torch at batch 1, 5, 30 and 64 (35.7 against
    # 21.7 us per step at batch 1, 1000 -> 500), so by default every batch decodes.
    CROSSOVER_ROWS = 0

    def __init__(self, entry_ih: PackedEntry, entry_hh: PackedEntry, kind: str, levels, bucket_size, bias_ih: torch.Tensor = None,
                 bias_hh: torch.Tensor = None):
        super().__init__()
        self.hidden_size, self.input_size = _gate_sizes(entry_ih, 4, "an LSTM")
        self.bias = bias_ih is not None or bias_hh is not None
        self.weights = _cell_pair(entry_ih, entry_hh, kind, levels, bucket_size, bias_ih, bias_hh, 4, self.hidden_size, self.input_size)

    def extra_repr(self) -> str:
        ih = self.weights[0]
        return f"{self.input_size}, {self.hidden_size}, bias={self.bias}, {ih.kind}, bits={ih.bits}/{self.weights[1].bits}, bucket_size={ih.bucket_size}"

    def decoded_weights(self) -> tuple:
        """(weight_ih, weight_hh) decoded to float32, bit for bit what unpack_ writes."""
        return self.weights[0].decoded(), self.weights[1].decoded()

    def forward(self, input: torch.Tensor, hx=None) -> tuple:
        _check_weights(self.weights, input, "PackedLSTMCell")
        if input.dim() not in (1, 2) or input.shape[-1] != self.input_size:
            raise ValueError(f"input of shape {tuple(input.shape)}, expected (B, {self.input_size}) or ({self.input_size},)")
        batched = input.dim() == 2
        x = input if batched else input.unsqueeze(0)
        B, H = x.shape[0], self.hidden_size
        if hx is None:
            h = c = torch.zeros(B, H, dtype=torch.float32, device=x.device)
        else:
            h, c = hx
            for t in (h, c):
                _check_weights(self.weights, t, "PackedLSTMCell")
                if tuple(t.shape) != ((B, H) if batched else (H,)):
                    raise ValueError(f"hidden state of shape {tuple(t.shape)}, expected {(B, H) if batched else (H,)}")
            h, c = (h, c) if batched else (h.unsqueeze(0), c.unsqueeze(0))
        ih, hh = self.weights
        with torch.cuda.device(x.device):
            if B == 0 or B > self.CROSSOVER_ROWS:
                w_ih, w_hh = self.decoded_weights()
                h1, c1 = torch._VF.lstm_cell(x, (h, c), w_ih, w_hh, ih.bias, hh.bias)
            else:
                x, h = (t if t.stride(-1) == 1 and t.stride(0) >= t.shape[1] else t.contiguous() for t in (x, h))
                c = c.contiguous()
                h1 = torch.empty(B, H, dtype=torch.float32, device=x.device)
                c1 = torch.empty(B, H, dtype=torch.float32, device=x.device)
                d_ih, d_hh = ih.descriptor(), hh.descriptor()
                N.check(N.lib().qd_packed_lstm_cell(N.ptr(x), x.stride(0), N.ptr(h), h.stride(0), N.ptr(c), B, self.input_size, H,
                                                    d_ih.ctypes.data, d_hh.ctypes.data, ih.levels,
                                                    _bucket(ih.bucket_size), N.ptr(ih.bias), N.ptr(hh.bias), N.ptr(h1), H, N.ptr(c1),
                                                    N.stream_ptr(x.device)))
        return (h1, c1) if batched else (h1[0], c1[0])


class _PackedRNN(torch.nn.Module):
    """The sequence plumbing PackedLSTM and PackedGRU share: the weight pairs per layer and direction, the input layouts
    (padded 3-D, batch_first or not, unbatched 2-D, PackedSequence sorted or not), the state checks and the
    PackedSequence permutation, and the choice between the packed layer kernel and decode + torch.  A subclass names
    its gates per hidden unit, its state tensors, its layer entry point and its torch function."""
    _gates = _states = None                      # weight rows per hidden unit; state tensors per layer (h or h, c)
    _what = _article = _layer_fn = _vf = None    # module name, "an LSTM" / "a GRU", qd_packed_*_layer, torch._VF function

    def __init__(self, weights, kind: str, levels, bucket_size, *, num_layers=1, batch_first=False, dropout=0.0, bidirectional=False,
                 biases=None):
        super().__init__()
        dirs = 2 if bidirectional else 1
        if num_layers < 1 or len(weights) != num_layers * dirs:
            raise ValueError(f"{len(weights)} weight pairs for {num_layers} layers x {dirs} directions")
        if biases is not None and len(biases) != len(weights):
            raise ValueError(f"{len(biases)} bias pairs for {len(weights)} weight pairs")
        self.hidden_size, self.input_size = _gate_sizes(weights[0][0], self._gates, self._article)
        self.num_layers, self.batch_first, self.dropout, self.bidirectional = num_layers, batch_first, float(dropout), bidirectional
        self.bias = biases is not None
        self.cells = torch.nn.ModuleList()
        for k, (e_ih, e_hh) in enumerate(weights):
            b_ih, b_hh = biases[k] if biases is not None else (None, None)
            in_size = self.input_size if k < dirs else dirs * self.hidden_size
            self.cells.append(_cell_pair(e_ih, e_hh, kind, levels, bucket_size, b_ih, b_hh, self._gates, self.hidden_size, in_size))

    def extra_repr(self) -> str:
        ih = self.cells[0][0]
        return (f"{self.input_size}, {self.hidden_size}, num_layers={self.num_layers}, bias={self.bias}, batch_first={self.batch_first}, "
                f"dropout={self.dropout}, bidirectional={self.bidirectional}, {ih.kind}, bucket_size={ih.bucket_size}")

    def decoded_weights(self) -> list:
        """torch's flat weight list (w_ih, w_hh[, b_ih, b_hh] per layer and direction), the matrices decoded to float32
        bit for bit as unpack_ writes them."""
        flat = []
        for ih, hh in self.cells:
            flat += [ih.decoded(), hh.decoded()] + ([ih.bias, hh.bias] if self.bias else [])
        return flat

    def _run(self, input, hx) -> tuple:
        """(output, final states) for ``hx`` = the initial state tensors (a tuple of _states) or None (zeros), in the
        input's layout."""
        packed_in = isinstance(input, torch.nn.utils.rnn.PackedSequence)
        weights = [w for pair in self.cells for w in pair]
        x = input.data if packed_in else input
        _check_weights(weights, x, self._what)
        if self.training and self.dropout > 0 and self.num_layers > 1:
            raise RuntimeError(f"{self._what} does not apply inter-layer dropout: call eval(), or set dropout to 0")
        dirs, H, L = 2 if self.bidirectional else 1, self.hidden_size, self.num_layers
        if packed_in:
            if x.dim() != 2 or x.shape[1] != self.input_size:
                raise ValueError(f"PackedSequence data of shape {tuple(x.shape)}, expected (N, {self.input_size})")
            batch_sizes = input.batch_sizes
            B, batched = int(batch_sizes[0]), True
        else:
            if x.dim() not in (2, 3) or x.shape[-1] != self.input_size:
                raise ValueError(f"input of shape {tuple(x.shape)}, expected 3-D or 2-D with {self.input_size} features")
            batched = x.dim() == 3
            batch_dim = 0 if self.batch_first else 1
            if not batched:
                x = x.unsqueeze(batch_dim)
            B = x.shape[batch_dim]
        if hx is None:
            states = [torch.zeros(L * dirs, B, H, dtype=torch.float32, device=x.device) for _ in range(self._states)]
        else:
            states = list(hx)
            if len(states) != self._states:
                raise ValueError(f"{len(states)} state tensors, expected {self._states}")
            for t in states:
                _check_weights(weights, t, self._what)
                if tuple(t.shape) != ((L * dirs, B, H) if batched else (L * dirs, H)):
                    raise ValueError(f"hidden state of shape {tuple(t.shape)}, expected {(L * dirs, B, H) if batched else (L * dirs, H)}")
            if not batched:
                states = [t.unsqueeze(1) for t in states]
            if packed_in and input.sorted_indices is not None:         # torch's permute_hidden
                states = [t.index_select(1, input.sorted_indices) for t in states]
        with torch.cuda.device(x.device):
            if B == 0 or x.numel() == 0 or B > self.CROSSOVER_ROWS:
                out, finals = self._decoded_forward(x, batch_sizes if packed_in else None, states)
            else:
                out, finals = self._packed_forward(x, batch_sizes if packed_in else None, states)
        if packed_in:
            if input.unsorted_indices is not None:
                finals = [t.index_select(1, input.unsorted_indices) for t in finals]
            return torch.nn.utils.rnn.PackedSequence(out, batch_sizes, input.sorted_indices, input.unsorted_indices), tuple(finals)
        if not batched:
            out, finals = out.squeeze(batch_dim), [t.squeeze(1) for t in finals]
        return out, tuple(finals)

    def _decoded_forward(self, x, batch_sizes, states):
        import warnings
        flat = self.decoded_weights()
        hx = tuple(states) if len(states) > 1 else states[0]
        rnn = getattr(torch._VF, self._vf)
        with warnings.catch_warnings():       # the decoded weights are not one flattened buffer; cuDNN copies them into one
            warnings.filterwarnings("ignore", message="RNN module weights are not part of single contiguous chunk")
            if batch_sizes is not None:
                res = rnn(x, batch_sizes, hx, flat, self.bias, self.num_layers, self.dropout, self.training, self.bidirectional)
            else:
                res = rnn(x, hx, flat, self.bias, self.num_layers, self.dropout, self.training, self.bidirectional, self.batch_first)
        return res[0], list(res[1:])

    def _packed_forward(self, x, batch_sizes, states):
        dirs, H = 2 if self.bidirectional else 1, self.hidden_size
        if batch_sizes is not None:
            bs = np.ascontiguousarray(batch_sizes.cpu().numpy(), dtype=np.int64)
            data = x
        else:
            seq = x.transpose(0, 1) if self.batch_first else x               # (T, B, I)
            bs = np.full(seq.shape[0], seq.shape[1], dtype=np.int64)
            data = seq.reshape(-1, self.input_size)
        if data.stride(-1) != 1:
            data = data.contiguous()
        states = [t.contiguous() for t in states]
        finals = [torch.empty_like(t) for t in states]
        rows, sp = data.shape[0], N.stream_ptr(data.device)
        layer_fn = getattr(N.lib(), self._layer_fn)
        for layer in range(self.num_layers):
            out = torch.empty(rows, dirs * H, dtype=torch.float32, device=data.device)
            for d in range(dirs):
                k = layer * dirs + d
                ih, hh = self.cells[k]
                d_ih, d_hh = ih.descriptor(), hh.descriptor()
                # (x, ldx, batch_sizes, steps, reverse, I, H, w_ih, w_hh, levels, bucket, b_ih, b_hh, initial states, out,
                # ldo, final states, stream)
                N.check(layer_fn(N.ptr(data), data.stride(0), bs.ctypes.data, len(bs), d, ih.shape[1], H, d_ih.ctypes.data, d_hh.ctypes.data,
                                 ih.levels, _bucket(ih.bucket_size), N.ptr(ih.bias), N.ptr(hh.bias), *(N.ptr(t[k]) for t in states),
                                 N.ptr(out) + 4 * d * H, dirs * H, *(N.ptr(t[k]) for t in finals), sp))
            data = out
        if batch_sizes is None:
            data = data.view(len(bs), -1, dirs * H)
            if self.batch_first:
                data = data.transpose(0, 1).contiguous()
        return data, finals


class PackedLSTM(_PackedRNN):
    """Inference replacement of an ``nn.LSTM`` (no projection) whose weight matrices stay in their fixed-width stored
    form on the device: ``weights`` is one (entry_ih, entry_hh) pair per layer and direction in nn.LSTM's order (l0,
    l0_reverse, l1, ...), ``biases`` the matching (bias_ih, bias_hh) pairs or None.  Takes what nn.LSTM takes -- padded
    3-D input (batch_first or not), unbatched 2-D input, or a PackedSequence (sorted or not), with ``hx`` = (h_0, c_0)
    or None -- and returns (output, (h_n, c_n)) in nn.LSTM's shapes.  For batches of up to CROSSOVER_ROWS rows (none by
    default), every
    layer and direction is one qd_packed_lstm_layer call (one fused cell launch per step, no host synchronisation, so
    the forward can be captured in a CUDA graph); the arithmetic is qd_packed_lstm_cell's, so a sequence gives the same
    bits alone, inside any batch and at any position of a PackedSequence.  Larger batches decode every weight and call
    torch's LSTM: exactly what an unpack_-loaded nn.LSTM computes.  Inter-layer dropout is not applied: in training
    mode with dropout > 0 and several layers forward raises, since the result would differ from nn.LSTM's."""
    # largest batch that runs on qd_packed_lstm_layer (at most N.PACKED_LSTM_MAX_ROWS).  Measured (DESIGN.md section
    # 3.7.6): on the NMT encoder layer the kernel loses to decode + torch at batch 1, 5, 30 and 64, so by default every
    # batch decodes.
    CROSSOVER_ROWS = 0
    _gates, _states, _what, _article, _layer_fn, _vf = 4, 2, "PackedLSTM", "an LSTM", "qd_packed_lstm_layer", "lstm"

    def forward(self, input, hx=None):
        out, (h_n, c_n) = self._run(input, hx)
        return out, (h_n, c_n)


class PackedGRU(_PackedRNN):
    """Inference replacement of an ``nn.GRU`` whose weight matrices stay in their fixed-width stored form on the device:
    ``weights`` is one (entry_ih, entry_hh) pair per layer and direction in nn.GRU's order (l0, l0_reverse, l1, ...),
    ``biases`` the matching (bias_ih, bias_hh) pairs or None.  Takes what nn.GRU takes -- padded 3-D input
    (batch_first or not), unbatched 2-D input, or a PackedSequence (sorted or not), with ``hx`` = h_0 or None -- and
    returns (output, h_n) in nn.GRU's shapes.  For batches of up to CROSSOVER_ROWS rows (none by default), every layer
    and direction is one qd_packed_gru_layer call (one fused cell launch per step, no host synchronisation, so the
    forward can be captured in a CUDA graph); the arithmetic is qd_packed_gru_cell's, so a sequence gives the same bits
    alone, inside any batch and at any position of a PackedSequence.  Larger batches decode every weight and call
    torch's GRU: exactly what an unpack_-loaded nn.GRU computes.  Inter-layer dropout is not applied: in training mode
    with dropout > 0 and several layers forward raises, since the result would differ from nn.GRU's."""
    # largest batch that runs on qd_packed_gru_layer (at most N.PACKED_GRU_MAX_ROWS).  Measured (DESIGN.md section
    # 3.7.7): on the NMT encoder layer the kernel loses to decode + torch at batch 1, 5, 30 and 64 (28.6 against 8.7 us
    # per step at batch 1), so by default every batch decodes.
    CROSSOVER_ROWS = 0
    _gates, _states, _what, _article, _layer_fn, _vf = 3, 1, "PackedGRU", "a GRU", "qd_packed_gru_layer", "gru"

    def forward(self, input, hx=None):
        out, (h_n,) = self._run(input, None if hx is None else (hx,))
        return out, h_n


class PackedGRUCell(torch.nn.Module):
    """Inference replacement of an ``nn.GRUCell`` whose two weight matrices stay in their fixed-width stored form (two
    PackedEntry of a PackedModel, [3H, I] and [3H, H]) on the device.  Takes input [B, I] or [I] and ``hx`` = h or None
    (zeros), returns h' in nn.GRUCell's shape.  Up to CROSSOVER_ROWS rows (none by default), forward runs
    qd_packed_gru_cell: one launch that reads the codes of both weights and applies the cell update in registers, every
    weight bit for bit the decoded one, each gate's linear output in qd_packed_linear's fixed float32 order
    (include/qd_b200.h states the contract).  Larger batches decode both weights into scratch tensors and call torch's
    GRU cell: exactly what an unpack_-loaded nn.GRUCell computes.  Forward only, no host synchronisation
    (graph-capturable)."""
    # largest batch that runs on the packed kernel (at most N.PACKED_GRU_MAX_ROWS).  Measured (DESIGN.md section
    # 3.7.7): on the NMT decoder cells the kernel loses to decode + torch at batch 1, 5, 30 and 64 (28.9 against
    # 19.7 us per step at batch 1, 1000 -> 500), so by default every batch decodes.
    CROSSOVER_ROWS = 0

    def __init__(self, entry_ih: PackedEntry, entry_hh: PackedEntry, kind: str, levels, bucket_size, bias_ih: torch.Tensor = None,
                 bias_hh: torch.Tensor = None):
        super().__init__()
        self.hidden_size, self.input_size = _gate_sizes(entry_ih, 3, "a GRU")
        self.bias = bias_ih is not None or bias_hh is not None
        self.weights = _cell_pair(entry_ih, entry_hh, kind, levels, bucket_size, bias_ih, bias_hh, 3, self.hidden_size, self.input_size)

    def extra_repr(self) -> str:
        ih = self.weights[0]
        return f"{self.input_size}, {self.hidden_size}, bias={self.bias}, {ih.kind}, bits={ih.bits}/{self.weights[1].bits}, bucket_size={ih.bucket_size}"

    def decoded_weights(self) -> tuple:
        """(weight_ih, weight_hh) decoded to float32, bit for bit what unpack_ writes."""
        return self.weights[0].decoded(), self.weights[1].decoded()

    def forward(self, input: torch.Tensor, hx=None) -> torch.Tensor:
        _check_weights(self.weights, input, "PackedGRUCell")
        if input.dim() not in (1, 2) or input.shape[-1] != self.input_size:
            raise ValueError(f"input of shape {tuple(input.shape)}, expected (B, {self.input_size}) or ({self.input_size},)")
        batched = input.dim() == 2
        x = input if batched else input.unsqueeze(0)
        B, H = x.shape[0], self.hidden_size
        if hx is None:
            h = torch.zeros(B, H, dtype=torch.float32, device=x.device)
        else:
            _check_weights(self.weights, hx, "PackedGRUCell")
            if tuple(hx.shape) != ((B, H) if batched else (H,)):
                raise ValueError(f"hidden state of shape {tuple(hx.shape)}, expected {(B, H) if batched else (H,)}")
            h = hx if batched else hx.unsqueeze(0)
        ih, hh = self.weights
        with torch.cuda.device(x.device):
            if B == 0 or B > self.CROSSOVER_ROWS:
                w_ih, w_hh = self.decoded_weights()
                h1 = torch._VF.gru_cell(x, h, w_ih, w_hh, ih.bias, hh.bias)
            else:
                x, h = (t if t.stride(-1) == 1 and t.stride(0) >= t.shape[1] else t.contiguous() for t in (x, h))
                h1 = torch.empty(B, H, dtype=torch.float32, device=x.device)
                d_ih, d_hh = ih.descriptor(), hh.descriptor()
                N.check(N.lib().qd_packed_gru_cell(N.ptr(x), x.stride(0), N.ptr(h), h.stride(0), B, self.input_size, H, d_ih.ctypes.data,
                                                   d_hh.ctypes.data, ih.levels, _bucket(ih.bucket_size), N.ptr(ih.bias), N.ptr(hh.bias),
                                                   N.ptr(h1), H, N.stream_ptr(x.device)))
        return h1 if batched else h1[0]


def _conv_padding(conv) -> tuple:
    """(pad_h, pad_w) of an nn.Conv2d's padding when it is symmetric: an int pair, "valid", or "same" whose total
    padding per side is even; None otherwise."""
    p = conv.padding
    if p == "valid":
        return (0, 0)
    if p == "same":
        total = [d * (k - 1) for k, d in zip(conv.kernel_size, conv.dilation)]
        return None if any(t % 2 for t in total) else tuple(t // 2 for t in total)
    if isinstance(p, tuple) and len(p) == 2 and all(isinstance(v, int) for v in p):
        return p
    return None


def _linear_target(mod) -> bool:
    return isinstance(mod, torch.nn.Linear)


def _conv_target(mod) -> bool:
    # type, not isinstance: a subclass may override forward
    return (type(mod) is torch.nn.Conv2d and mod.groups == 1 and tuple(mod.dilation) == (1, 1) and mod.padding_mode == "zeros"
            and _conv_padding(mod) is not None)


def _embedding_target(mod) -> bool:
    # type, not isinstance: a subclass may override forward; max_norm renormalises the weight in place during forward
    return type(mod) is torch.nn.Embedding and mod.max_norm is None


def _packed_linear(entries, pm, lin):
    return PackedLinear(entries[0], pm.kind, pm.levels, pm.bucket_size, None if lin.bias is None else lin.bias.data)


def _packed_conv(entries, pm, conv):
    return PackedConv2d(entries[0], pm.kind, pm.levels, pm.bucket_size, conv.stride, _conv_padding(conv),
                        None if conv.bias is None else conv.bias.data)


def _packed_embedding(entries, pm, emb):
    return PackedEmbedding(entries[0], pm.kind, pm.levels, pm.bucket_size, emb.padding_idx)


def _lstm_target(mod) -> bool:
    return type(mod) is torch.nn.LSTM and mod.proj_size == 0


def _lstm_cell_target(mod) -> bool:
    return type(mod) is torch.nn.LSTMCell


def _gru_target(mod) -> bool:
    return type(mod) is torch.nn.GRU


def _gru_cell_target(mod) -> bool:
    return type(mod) is torch.nn.GRUCell


def _own_bias(b):
    # a copy: on CUDA an nn.LSTM's or nn.GRU's parameters are views into one flattened buffer, which must not outlive
    # the module
    return None if b is None else b.data.clone()


def _packed_rnn(cls, entries, pm, rnn):
    biases = None
    if rnn.bias:
        names = [n for n in rnn._flat_weights_names if n.startswith("bias")]
        biases = [(_own_bias(getattr(rnn, a)), _own_bias(getattr(rnn, b))) for a, b in zip(names[0::2], names[1::2])]
    return cls(list(zip(entries[0::2], entries[1::2])), pm.kind, pm.levels, pm.bucket_size, num_layers=rnn.num_layers,
               batch_first=rnn.batch_first, dropout=rnn.dropout, bidirectional=rnn.bidirectional, biases=biases)


def _packed_lstm(entries, pm, lstm):
    return _packed_rnn(PackedLSTM, entries, pm, lstm)


def _packed_gru(entries, pm, gru):
    return _packed_rnn(PackedGRU, entries, pm, gru)


def _packed_lstm_cell(entries, pm, cell):
    return PackedLSTMCell(entries[0], entries[1], pm.kind, pm.levels, pm.bucket_size, _own_bias(cell.bias_ih), _own_bias(cell.bias_hh))


def _packed_gru_cell(entries, pm, cell):
    return PackedGRUCell(entries[0], entries[1], pm.kind, pm.levels, pm.bucket_size, _own_bias(cell.bias_ih), _own_bias(cell.bias_hh))


def _weight_matrices(mod) -> list:
    """The weights a packed replacement of ``mod`` holds: an LSTM's or GRU's (ih, hh) per layer and direction in torch's
    order, an LSTMCell's or GRUCell's (ih, hh), else the module's one weight."""
    if isinstance(mod, (torch.nn.LSTM, torch.nn.GRU)):
        return [getattr(mod, n) for n in mod._flat_weights_names if n.startswith("weight")]
    if isinstance(mod, (torch.nn.LSTMCell, torch.nn.GRUCell)):
        return [mod.weight_ih, mod.weight_hh]
    return [mod.weight]


def _tied_pair(mods) -> bool:
    """True when a weight's registrations are exactly one eligible nn.Embedding and one nn.Linear: a generator tied to
    an embedding, whose [V, D] weight reads row v the same way in both."""
    return len(mods) == 2 and mods[0] is not mods[1] and any(_embedding_target(m) for m in mods) \
        and any(_linear_target(m) for m in mods)


def _attach(pm: PackedModel, model, kinds, tied=False) -> list:
    """unpack_, except that every module accepted by the ``accept`` of one of ``kinds`` -- (accept, make, what) -- whose
    weight matrices (_weight_matrices) ``pm`` all stores quantized and which is each one's only holder is replaced in
    its parent by make(entries, pm, module), one entry per matrix; the float32 matrices are released.  With ``tied``,
    so are both modules of a tied embedding / generator pair (_tied_pair), and the two share one set of device sections.
    Returns the names of the replaced modules."""
    named, bufs = _check_target(pm, model)
    index = {id(p): k for k, (_, p) in enumerate(named)}
    holders = {}                                 # parameter -> its registrations in the module tree, every path counted
    for _, mod in model.named_modules(remove_duplicate=False):
        for p in mod._parameters.values():
            if p is not None:
                holders.setdefault(id(p), []).append(mod)

    def eligible(ws):
        return all(id(w) in index and pm.tensors[index[id(w)]].quantized for w in ws) and \
            (all(len(holders[id(w)]) == 1 for w in ws) or tied and len(ws) == 1 and _tied_pair(holders[id(ws[0])]))
    targets = []                                 # (module name, parent, attribute, module, weight indices, make)
    for mname, mod in model.named_modules():
        for accept, make, what in kinds:
            if accept(mod) and eligible(ws := _weight_matrices(mod)):
                if not ws[0].is_cuda:
                    raise ValueError(f"{mname}: a Packed{what} runs on a CUDA device, the {what} is on {ws[0].device}")
                parent_name, _, attr = mname.rpartition(".")
                targets.append((mname, model.get_submodule(parent_name) if parent_name else model, attr, mod,
                                [index[id(w)] for w in ws], make))
                break
    _write_into(pm, named, bufs, skip={k for t in targets for k in t[4]})
    movers = {}
    held = {}                                    # weight index -> the sections its first replacement holds
    for mname, parent, attr, mod, ks, make in targets:
        dev = _weight_matrices(mod)[0].device
        with torch.cuda.device(dev):
            move = movers.setdefault(dev, _mover(pm, dev))
            entries = [held.get(k) or PackedEntry(t.name, t.shape, bits=t.bits, packed=move(t.packed), alpha=move(t.alpha),
                                                  beta=move(t.beta), points=None if t.points is None else t.points.to(dev))
                       for k, t in ((k, pm.tensors[k]) for k in ks)]
            layer = make(entries, pm, mod)
        if len(ks) == 1:
            t = pm.tensors[ks[0]]
            held[ks[0]] = PackedEntry(t.name, t.shape, bits=t.bits, packed=layer.packed, alpha=layer.alpha, beta=layer.beta,
                                      points=layer.points)
        setattr(parent, attr, layer)
    return [t[0] for t in targets]


def attach_packed_linear_(pm: PackedModel, model) -> list:
    """unpack_, except that every ``nn.Linear`` whose weight ``pm`` stores quantized is replaced in its parent module
    by a PackedLinear holding that weight's packed sections (and the Linear's bias, decoded as unpack_ decodes it);
    the float32 weight is released.  Everything else -- the other parameters, Linear layers kept float32, the stored
    buffers -- is written exactly as unpack_ writes it, quantized tensors in one launch per device.  Everything is
    checked before anything is written.  A Linear whose weight is also held elsewhere -- tied to another module (a
    generator sharing the embedding's matrix) or the Linear itself registered under two parents -- stays an nn.Linear
    and its weight is decoded as unpack_ decodes it: replacing it in one place would leave the other holder with a
    weight that was never written.  Returns the names of the replaced modules."""
    return _attach(pm, model, [(_linear_target, _packed_linear, "Linear")])


def attach_packed_(pm: PackedModel, model, *, embeddings=False, recurrent=False, gru=False) -> list:
    """attach_packed_linear_ for Linear and convolution layers: every nn.Linear it would replace becomes a
    PackedLinear, and every ``nn.Conv2d`` (the class itself, not a subclass) with groups 1, dilation 1, zero padding
    that is symmetric (int padding, "valid", or "same" that resolves to equal sides) and a weight ``pm`` stores
    quantized and it alone holds becomes a PackedConv2d with that weight's packed sections, its stride, padding and
    bias.  With ``embeddings=True``, also every ``nn.Embedding`` (the class itself) without max_norm whose weight ``pm``
    stores quantized and it alone holds becomes a PackedEmbedding; and a weight held by exactly one such embedding and
    one nn.Linear -- a generator tied to an embedding -- replaces both, by a PackedEmbedding and a PackedLinear (with the
    Linear's bias) that share one copy of the sections on the device.  Any other weight with several holders is
    decoded as unpack_ decodes it.  The replaced float32 weights are released; every other parameter and layer, and the
    stored buffers, are written exactly as unpack_ writes them, quantized tensors in one launch per device.  Everything
    is checked before anything is written.  With ``recurrent=True``, also every ``nn.LSTM`` (the class itself) without
    projection becomes a PackedLSTM, and every ``nn.LSTMCell`` a PackedLSTMCell, when ``pm`` stores all of its weight
    matrices quantized and it alone holds each of them; its biases are written as unpack_ writes them and handed to the
    packed module (as copies: nothing keeps an LSTM's flattened weight buffer alive).  With ``gru=True``, likewise
    every ``nn.GRU`` becomes a PackedGRU and every ``nn.GRUCell`` a PackedGRUCell.  Every other recurrent module -- a
    GRU without ``gru=True``, an LSTM without ``recurrent=True``, a subclass, one with a projection or a shared or
    float32 matrix -- is decoded as unpack_ decodes it.  Returns the names of the replaced modules, in module order."""
    kinds = [(_linear_target, _packed_linear, "Linear"), (_conv_target, _packed_conv, "Conv2d")]
    if embeddings:
        kinds.append((_embedding_target, _packed_embedding, "Embedding"))
    if recurrent:
        kinds += [(_lstm_target, _packed_lstm, "LSTM"), (_lstm_cell_target, _packed_lstm_cell, "LSTMCell")]
    if gru:
        kinds += [(_gru_target, _packed_gru, "GRU"), (_gru_cell_target, _packed_gru_cell, "GRUCell")]
    return _attach(pm, model, kinds, tied=embeddings)


def save_packed(pm: PackedModel, path) -> int:
    """Writes the fixed-width container: magic QDPACK, version 1, JSON header, 16-byte-aligned little-endian sections
    (packed codes as bytes).  Returns the file size in bytes."""
    return _write_container(pm, path)


def load_packed(path, device=None) -> PackedModel:
    """Reads and validates a file written by save_packed; everything is checked on the host before anything reaches a
    device.  Every section is a view into one tensor holding the file's data region.  device=None keeps it in host
    memory (unpack_ moves it to the GPU in one copy); a device gets it in one copy here."""
    return _read_container(PackedModel, path, device)


def _transcode_limits(m) -> list:
    """Host-side checks of a model about to change container (pack_compressed, compress_packed), before any device
    work: [(quantized entry, number of levels it may use: uniform s, non-uniform K_t)]; ValueError otherwise."""
    if m.kind not in ("uniform", "nonuniform"):
        raise ValueError(f"unknown kind {m.kind!r}")
    if m.kind == "uniform" and not (isinstance(m.levels, int) and 2 <= m.levels <= 256):
        raise ValueError("uniform levels must be in [2, 256]")
    q = [t for t in m.tensors if t.quantized]
    if not q:
        raise ValueError(f"the {m._WHAT} has no quantized tensor")
    out = []
    for t in q:
        limit = int(m.levels) if m.kind == "uniform" else (0 if t.points is None else t.points.numel())
        if not 1 <= limit <= 256:
            raise ValueError(f"{t.name}: {limit} points, expected 1 to 256")
        out.append((t, limit))
    return out


def _own_points(limits, dev) -> list:
    """Every non-uniform entry's points on ``dev`` in one upload, in new storage; None for a uniform model."""
    pts = [t.points for t, _ in limits if t.points is not None]
    if not pts:
        return [None] * len(limits)
    flat = torch.cat([p.reshape(-1).to(pts[0].device, torch.float32) for p in pts]).to(dev)
    return list(flat.split([p.numel() for p in pts]))


def pack_compressed(cm: CompressedModel, device=None) -> PackedModel:
    """The fixed-width model holding exactly what the Huffman-coded ``cm`` holds: same kind, levels, bucket, names,
    shapes, points, (alpha, beta), unquantized tensors and buffers, each tensor's codes at pack_model's width
    (bits_for(levels), or bits_for(K_t) for tensor t of a non-uniform model).  Every stream is decoded straight to
    packed codes in one launch (qd_huffman_decode_packed_model); nothing is re-quantized, so unpack_ of the result
    writes the parameters decompress_ of ``cm`` writes, bit for bit.  A host-loaded file reaches the device in one
    copy of its data region; the result shares no storage with ``cm``.  One synchronise reads the count of
    out-of-range symbols: a stream that emits a symbol >= s or >= K_t raises ValueError naming its tensor.  Runs
    attach_packed_ on a Huffman-coded file: attach_packed_(pack_compressed(load_compressed(path, "cuda")), net)."""
    limits = _transcode_limits(cm)
    for t, _ in limits:
        if t.chunk_offsets.numel() != -(-t.numel // HUFFMAN_CHUNK):
            raise ValueError(f"{t.name}: {t.chunk_offsets.numel()} chunk offsets for {t.numel} symbols")
    dev = _device_of(cm, device)
    with torch.cuda.device(dev):
        move = _mover(cm, dev)
        points = iter(_own_points(limits, dev))
        tensors, desc, keep = [], np.zeros(len(limits), _REPACK_TENSOR), []
        for t in cm.tensors:
            if not t.quantized:
                tensors.append(PackedEntry(t.name, tuple(t.shape), raw=move(t.raw).clone()))
                continue
            k = len(keep) // 2
            limit = limits[k][1]
            bits = bits_for(limit)
            words, offs = move(t.words).contiguous(), move(t.chunk_offsets).contiguous()
            packed = torch.empty((t.numel * bits + 7) // 8, dtype=torch.uint8, device=dev)
            desc[k] = (N.ptr(words) if words.numel() else 0, N.ptr(offs), N.ptr(packed), words.numel(), t.numel, bits, limit)
            keep += [words, offs]
            tensors.append(PackedEntry(t.name, tuple(t.shape), bits=bits, packed=packed, alpha=move(t.alpha).clone(),
                                       beta=move(t.beta).clone(), points=next(points)))
        buffers = None if cm.buffers is None else [(name, move(b).clone()) for name, b in cm.buffers]
        ws = torch.empty(int(N.lib().qd_huffman_repack_model_workspace_bytes(len(limits))), dtype=torch.uint8, device=dev)
        bad = torch.zeros(len(limits), dtype=torch.int64, device=dev)
        N.check(N.lib().qd_huffman_decode_packed_model(desc.ctypes.data, len(limits), N.ptr(cm.table(dev)), N.ptr(bad), N.ptr(ws),
                                                       ws.numel(), N.stream_ptr(dev)))
        for (t, limit), count in zip(limits, bad.cpu().tolist()):
            if count:
                raise ValueError(f"{t.name}: its Huffman stream emits {count} symbols that are not among its {limit} levels")
    return PackedModel(cm.kind, cm.levels, cm.bucket_size, tensors, buffers=buffers)


def compress_packed(pm: PackedModel, device=None) -> CompressedModel:
    """The Huffman-coded model holding exactly what the fixed-width ``pm`` holds: every tensor's codes are unpacked to
    levels (qd_unpack_indices), then compress_model's histogram, code and encoder run on them, so that for a model
    compress_packed(pack_model(model, ...)) saves to the bytes compress_model(model, ...) saves to.  (alpha, beta),
    points, unquantized tensors and buffers are carried over.  A code >= s (uniform) or >= K_t (non-uniform tensor t)
    raises ValueError naming its tensor, as does a code longer than HUFFMAN_MAX_LENGTH bits."""
    limits = _transcode_limits(pm)
    for t, limit in limits:
        if t.bits not in (1, 2, 4, 8) or limit > 1 << t.bits or t.packed.numel() != (t.numel * t.bits + 7) // 8:
            raise ValueError(f"{t.name}: {t.packed.numel()} bytes of {t.bits}-bit codes cannot hold {t.numel} codes of {limit} levels")
    dev = _device_of(pm, device)
    with torch.cuda.device(dev):
        move, sp = _mover(pm, dev), N.stream_ptr(dev)
        points = iter(_own_points(limits, dev))
        tensors, idxs = [], []
        for t in pm.tensors:
            if not t.quantized:
                tensors.append(HuffmanTensor(t.name, tuple(t.shape), raw=move(t.raw).clone()))
                continue
            idx = torch.empty(t.numel, dtype=torch.uint8, device=dev)
            N.check(N.lib().qd_unpack_indices(N.ptr(move(t.packed).contiguous()), t.bits, N.ptr(idx), t.numel, sp))
            idxs.append(idx)
            tensors.append(HuffmanTensor(t.name, tuple(t.shape), alpha=move(t.alpha).clone(), beta=move(t.beta).clone(),
                                         points=next(points)))
        buffers = None if pm.buffers is None else [(name, move(b).clone()) for name, b in pm.buffers]
        return _huffman_coded(pm.kind, pm.levels, pm.bucket_size, tensors, idxs, [limit for _, limit in limits], buffers, dev)


def get_size_reduction(effective_number_bits, bucket_size=256, full_precision_bits=32):
    """Compression factor of b-bit weights with two full-precision scalars per bucket
    (reference: helpers/functions.py:216-224)."""
    if bucket_size is None:
        return full_precision_bits / effective_number_bits
    f, k, b = full_precision_bits, bucket_size, effective_number_bits
    return (k * f) / (k * b + 2 * f)


def get_size_quantized_model(model, numBits, quantization_functions, bucket_size=256, type_quantization="uniform",
                             quantizeFirstLastLayer=True):
    """Model size in MB with Huffman-coded indices (reference: helpers/functions.py:226-262)."""
    params = list(model.parameters())
    if numBits is None:
        return sum(p.numel() for p in params) * 4 / 1000000
    quantized = params if quantizeFirstLastLayer is True else params[1:-1]
    unquantized = [] if quantizeFirstLastLayer is True else [params[0], params[-1]]
    count_q = sum(p.numel() for p in quantized)
    count_u = sum(p.numel() for p in unquantized)
    mean_bits = qhf.get_huffman_encoding_mean_bit_length(iter(quantized), quantization_functions, type_quantization,
                                                         s=2 ** numBits)
    size = count_u * 4 + mean_bits * count_q / 8
    if bucket_size is not None:
        size += count_q / bucket_size * 8
    return size / 1000000
