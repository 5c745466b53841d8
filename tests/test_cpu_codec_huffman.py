"""Huffman-coded model container, host side (no GPU): the canonical code against the reference's pinned Huffman
code, the stream format through its NumPy restatement (oracle/huffman_oracle.py), the file format and its
validation, and the refusal of codes longer than the decoder's 64-bit window allows."""
import json
import os
import struct

import numpy as np
import pytest
import torch

from oracle import huffman_oracle as HO
from quantized_distillation_b200 import codec
from quantized_distillation_b200.quantization import help_functions as H

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _prefix_free(codes, lengths):
    words = sorted(format(c, f"0{lengths[s]}b") for s, c in codes.items())
    return all(not b.startswith(a) for a, b in zip(words, words[1:]))


def test_canonical_code_keeps_the_reference_code_lengths():
    with open(os.path.join(ROOT, "tests", "golden", "reference_host_logic.json")) as f:
        cases = json.load(f)["huffman_encode"]
    assert cases
    for c in cases:
        freq = {int(s): f for s, f in c["freq"]}
        ref_lengths = {int(s): len(bits) for s, bits in c["code"]}
        lengths = {s: len(bits) for s, bits in H.huffman_encode(freq)}
        assert lengths == ref_lengths
        codes = codec.canonical_codes(lengths)
        assert codes == HO.canonical_codes(lengths)
        if len(lengths) > 1:
            longest = max(lengths.values())
            assert sum(1 << (longest - l) for l in lengths.values()) == 1 << longest      # Kraft equality
            assert all(codes[s] < (1 << lengths[s]) for s in codes) and _prefix_free(codes, lengths)
        assert codec.huffman_table(lengths).nbytes == codec.HUFFMAN_TABLE_BYTES


def test_code_of_a_histogram_is_the_size_accounting_code():
    counts = np.zeros(256, np.int64)
    counts[[0, 1, 2, 3, 7]] = [500, 250, 125, 124, 1]
    freq, code = H.huffman_code_of_histogram(counts)
    mean = sum(freq[s] * len(b) for s, b in code)
    lengths = codec.huffman_code_lengths(counts)
    assert sum(counts[s] * l for s, l in lengths.items()) / counts.sum() == pytest.approx(mean, rel=1e-15)
    assert codec.huffman_code_lengths(np.eye(1, 256, 9, dtype=np.int64)[0] * 77) == {9: 0}     # one symbol: length 0


def _fibonacci_counts(symbols):
    a, b, out = 1, 1, []
    for _ in range(symbols):
        out.append(a)
        a, b = b, a + b
    counts = np.zeros(256, np.int64)
    counts[:symbols] = out
    return counts


def test_codes_longer_than_57_bits_are_refused():
    ok = codec.huffman_code_lengths(_fibonacci_counts(58))        # longest code: 57 bits
    assert max(ok.values()) == codec.HUFFMAN_MAX_LENGTH
    with pytest.raises(ValueError, match="57"):
        codec.huffman_code_lengths(_fibonacci_counts(59))
    with pytest.raises(ValueError):
        codec.huffman_table({0: 1, 1: 2})                          # not complete (Kraft sum 3/4)


@pytest.mark.parametrize("case", ["single", "two", "all256", "long", "skewed"])
@pytest.mark.parametrize("n", [1, 10, 1023, 1024, 1025, 2049, 3000])
def test_oracle_stream_round_trip(case, n):
    rng = np.random.default_rng(n)
    if case == "single":
        sym = np.full(n, 5, np.uint8)
    elif case == "two":
        sym = rng.integers(0, 2, n).astype(np.uint8)
    elif case == "all256":
        sym = rng.integers(0, 256, n).astype(np.uint8)
    elif case == "long":
        sym = np.minimum(rng.geometric(0.5, n) - 1, 40).astype(np.uint8)
    else:
        sym = (rng.integers(0, 16, n) * (rng.random(n) < 0.1)).astype(np.uint8)
    counts = np.bincount(sym, minlength=256)
    if case == "long":                                  # a code of Fibonacci-histogram lengths: up to 44 bits
        lengths = codec.huffman_code_lengths(_fibonacci_counts(45))
        assert max(lengths.values()) == 44
        sym = (44 - sym).astype(np.uint8)               # the rare symbols get the long codes
    else:
        lengths = codec.huffman_code_lengths(counts)
    words, offs = HO.encode(sym, lengths)
    assert offs.size == -(-n // HO.CHUNK) and offs[0] == 0
    bits = sum(lengths[s] for s in sym.tolist())
    assert words.size * 32 - bits < 32 * offs.size                # at most 31 padding bits per chunk
    assert np.array_equal(HO.decode(words, offs, lengths, n), sym)


def _oracle_model(kind="uniform", bucket=256):
    """A CompressedModel assembled on the host from oracle-encoded streams."""
    rng = np.random.default_rng(1)
    shapes = [(3, 5), (2000,), (7, 300), (4,)]
    sym = [rng.integers(0, 16, int(np.prod(s))).astype(np.uint8) for s in shapes[1:3]]
    counts = np.bincount(np.concatenate(sym), minlength=256)
    lengths = codec.huffman_code_lengths(counts)
    tensors = [codec.HuffmanTensor("first", shapes[0], raw=torch.randn(15))]
    for k, (shape, s) in enumerate(zip(shapes[1:3], sym)):
        words, offs = HO.encode(s, lengths)
        rows = codec._rows(s.size, bucket)
        pts = torch.linspace(0, 1, 16) if kind == "nonuniform" else None
        tensors.append(codec.HuffmanTensor(f"t{k}", shape, words=torch.from_numpy(words.view(np.int32)),
                                           chunk_offsets=torch.from_numpy(offs.view(np.int32)), alpha=torch.rand(rows),
                                           beta=torch.randn(rows), points=pts, code_bits=int(sum(lengths[v] for v in s.tolist()))))
    tensors.append(codec.HuffmanTensor("last", shapes[3], raw=torch.randn(4)))
    return codec.CompressedModel(kind, 16 if kind == "uniform" else None, bucket, lengths, tensors)


@pytest.mark.parametrize("kind,bucket", [("uniform", 256), ("nonuniform", None)])
def test_container_round_trip(tmp_path, kind, bucket):
    cm = _oracle_model(kind, bucket)
    path = tmp_path / "m.qdh"
    size = codec.save_compressed(cm, path)
    assert size == os.path.getsize(path) == cm.size_breakdown()["file_bytes"]
    back = codec.load_compressed(path)
    assert (back.kind, back.levels, back.bucket_size, back.code_lengths) == (cm.kind, cm.levels, cm.bucket_size, cm.code_lengths)
    for a, b in zip(cm.tensors, back.tensors):
        assert (a.name, a.shape, a.quantized, a.code_bits) == (b.name, b.shape, b.quantized, b.code_bits)
        for f in ("words", "chunk_offsets", "alpha", "beta", "points", "raw"):
            x, y = getattr(a, f), getattr(b, f)
            assert (x is None) == (y is None), f
            if x is not None:
                assert not y.is_cuda and torch.equal(x.view(-1), y.view(-1)), f
    assert back.size_breakdown() == cm.size_breakdown()
    sb = cm.size_breakdown()
    assert sb["file_bytes"] == (sb["code_bits"] + sb["padding_bits"]) // 8 + sb["chunk_index_bytes"] + sb["scale_bytes"] + \
        sb["unquantized_bytes"] + sb["header_bytes"] + sb["alignment_bytes"]
    for t in back.tensors[1:3]:
        assert np.array_equal(HO.decode(t.words.numpy().view(np.uint32), t.chunk_offsets.numpy().view(np.uint32), back.code_lengths,
                                        t.numel), HO.decode(t.words.numpy().view(np.uint32), t.chunk_offsets.numpy().view(np.uint32),
                                                            cm.code_lengths, t.numel))


def _rewrite_header(raw, fn):
    magic, version, res, hlen = struct.unpack_from("<8sIIQ", raw)
    h = json.loads(raw[24:24 + hlen])
    fn(h)
    start = (24 + hlen + 15) // 16 * 16
    data = raw[start:]
    hb = json.dumps(h).encode()
    new_start = (24 + len(hb) + 15) // 16 * 16
    return struct.pack("<8sIIQ", magic, version, res, len(hb)) + hb + b"\0" * (new_start - 24 - len(hb)) + data


def test_malformed_files_are_rejected(tmp_path):
    path = tmp_path / "m.qdh"
    codec.save_compressed(_oracle_model(), path)
    good = path.read_bytes()
    bad = tmp_path / "bad.qdh"

    def rejected(raw, match=None):
        bad.write_bytes(raw)
        with pytest.raises(ValueError, match=match):
            codec.load_compressed(bad)

    rejected(b"XXHUFF\0\0" + good[8:], "magic")
    rejected(good[:8] + struct.pack("<I", 99) + good[12:], "version")
    rejected(good[:-20], None)                                                     # truncated last section
    rejected(good[:30], None)                                                      # truncated header

    def far_section(h):
        h["tensors"][1]["sections"]["alpha"][0] = h["data_bytes"] + 4096
    rejected(_rewrite_header(good, far_section), "out of range")

    def odd_section(h):
        h["tensors"][1]["sections"]["words"][0] += 4
    rejected(_rewrite_header(good, odd_section), "out of range")

    def bad_offsets(h):                                                            # chunk offsets beyond the stream
        h["tensors"][1]["sections"]["words"][1] = 4
    rejected(_rewrite_header(good, bad_offsets), "out of range")

    def long_code(h):
        h["code"] = [[0, 1], [1, 58], [2, 58]]
    rejected(_rewrite_header(good, long_code), "57")

    def incomplete(h):
        h["code"] = [[0, 1], [1, 3]]
    rejected(_rewrite_header(good, incomplete), "Kraft")

    # the checks both containers share: the Huffman reader refuses what the fixed-width reader refuses
    def edit(fn):
        return _rewrite_header(good, fn)
    rejected(good[:12] + struct.pack("<I", 1) + good[16:], "reserved")
    rejected(edit(lambda h: h.__setitem__("data_bytes", float(h["data_bytes"]))), "data_bytes")
    rejected(edit(lambda h: h["tensors"][2].__setitem__("name", "t0")), "twice")                     # duplicate tensor name
    rejected(edit(lambda h: h["tensors"][0].__setitem__("quantized", 0)), "quantized flag")
    rejected(edit(lambda h: h["tensors"][1]["sections"].__setitem__("packed", [0, 0])), "sections")  # unexpected section
    rejected(edit(lambda h: h["tensors"][1].__setitem__("points", [0.0, 1.0])), "no points")        # points on a uniform model
    rejected(edit(lambda h: h["tensors"][2]["sections"].__setitem__(
        "alpha", [h["tensors"][1]["sections"]["words"][0], h["tensors"][2]["sections"]["alpha"][1]])), "overlap")
    codec.save_compressed(_oracle_model("nonuniform", None), path)
    rejected(_rewrite_header(path.read_bytes(), lambda h: h.__setitem__("levels", 16)), "no levels")
    codec.save_compressed(_oracle_model(bucket=1), path)       # bucket true would read as 1
    rejected(_rewrite_header(path.read_bytes(), lambda h: h.__setitem__("bucket", True)), "bucket")
    codec.save_compressed(_oracle_model(), path)
    assert codec.load_compressed(path).tensors[1].numel == 2000


def test_compress_model_refuses_an_unknown_rule_before_device_work():
    with pytest.raises(ValueError, match="rule"):
        codec.compress_model(torch.nn.Linear(4, 4), points=[0.0, 0.5, 1.0], rule="midpiont")


def test_decoding_needs_a_gpu(tmp_path):
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    cm = _oracle_model()
    with pytest.raises(RuntimeError):
        codec.decompress_tensor(cm, 1)
    with pytest.raises(RuntimeError):
        codec.compress_model(torch.nn.Linear(4, 4), 4)
