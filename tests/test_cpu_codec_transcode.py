"""Container transcoding without a GPU: pack_compressed and compress_packed refuse to run without a CUDA device (no CPU
fallback) and refuse a model with no quantized tensor; and the NumPy restatement the GPU tests check them against --
oracle/huffman_oracle.py decode and encode, plus the qd_pack_indices layout -- takes every Huffman-coded golden
container to fixed-width codes and back to the golden file's exact bytes."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from oracle import huffman_oracle as HO
from quantized_distillation_b200 import codec

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location("make_golden_containers", os.path.join(HERE, "golden", "make_golden_containers.py"))
G = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(G)

GOLDEN = np.load(os.path.join(HERE, "golden", "containers.npz"))
MODELS = G.models()
HUFFMAN_CASES = sorted(k for k, (_, fmt) in MODELS.items() if fmt == "huffman")
PACKED_CASES = sorted(k for k, (_, fmt) in MODELS.items() if fmt == "packed")


def np_pack(codes, bits):
    """The qd_pack_indices layout, vectorised: code of element e in byte e*bits/8 at bit (e*bits)%8."""
    per = 8 // bits
    c = np.zeros(-(-codes.size // per) * per, np.uint32)
    c[:codes.size] = codes
    return (c.reshape(-1, per) << (np.arange(per, dtype=np.uint32) * bits)).sum(1).astype(np.uint8)


def np_unpack(packed, bits, n):
    per = 8 // bits
    b = np.asarray(packed, np.uint32)[:, None] >> (np.arange(per, dtype=np.uint32) * bits)
    return (b & ((1 << bits) - 1)).reshape(-1)[:n].astype(np.uint8)


def _load(case, tmp_path):
    path = tmp_path / "m"
    path.write_bytes(GOLDEN[case].tobytes())
    return codec.load_compressed(path) if MODELS[case][1] == "huffman" else codec.load_packed(path)


@pytest.mark.parametrize("case", sorted(MODELS))
def test_transcoders_need_a_cuda_device(case, tmp_path, monkeypatch):
    m = _load(case, tmp_path)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RuntimeError, match="CUDA device"):
        (codec.pack_compressed if MODELS[case][1] == "huffman" else codec.compress_packed)(m)


def test_transcoders_refuse_a_model_without_quantized_tensors():
    raw = torch.zeros(3)
    cm = codec.CompressedModel("uniform", 4, 256, {0: 1, 1: 1}, [codec.HuffmanTensor("w", (3,), raw=raw)])
    pm = codec.PackedModel("uniform", 4, 256, [codec.PackedEntry("w", (3,), raw=raw)])
    with pytest.raises(ValueError, match="no quantized tensor"):
        codec.pack_compressed(cm)
    with pytest.raises(ValueError, match="no quantized tensor"):
        codec.compress_packed(pm)


def test_compress_packed_checks_code_widths_on_the_host():
    t = codec.PackedEntry("w", (10,), bits=1, packed=torch.zeros(2, dtype=torch.uint8), alpha=torch.ones(1), beta=torch.zeros(1))
    with pytest.raises(ValueError, match="w:"):
        codec.compress_packed(codec.PackedModel("uniform", 4, 256, [t]))      # 4 levels do not fit in 1-bit codes


def _limits(m):
    return [int(m.levels) if m.kind == "uniform" else t.points.numel() for t in m.tensors if t.quantized]


def _oracle_pack_compressed(cm):
    """[(packed bytes, bits)] of every quantized tensor: decode each stream, pack at pack_model's width."""
    out = []
    for t, limit in zip([t for t in cm.tensors if t.quantized], _limits(cm)):
        sym = HO.decode(t.words.numpy().view(np.uint32), t.chunk_offsets.numpy().view(np.uint32), cm.code_lengths, t.numel)
        assert sym.max() < limit
        bits = codec.bits_for(limit)
        out.append((np_pack(sym, bits), bits))
    return out


def _oracle_compress_packed(pm, packed):
    """A CompressedModel from each tensor's codes: unpack, one histogram over all tensors, the code, encode."""
    q = [t for t in pm.tensors if t.quantized]
    syms = [np_unpack(p, bits, t.numel) for t, (p, bits) in zip(q, packed)]
    counts = np.bincount(np.concatenate(syms), minlength=256)
    lengths = codec.huffman_code_lengths(counts)
    tensors, it = [], iter(zip(q, syms))
    for t in pm.tensors:
        if not t.quantized:
            tensors.append(codec.HuffmanTensor(t.name, t.shape, raw=t.raw))
            continue
        e, sym = next(it)
        words, offs = HO.encode(sym, lengths)
        tensors.append(codec.HuffmanTensor(e.name, e.shape, words=torch.from_numpy(words.view(np.int32)),
                                           chunk_offsets=torch.from_numpy(offs.view(np.int32)), alpha=e.alpha, beta=e.beta,
                                           points=e.points, code_bits=int(sum(lengths[int(v)] for v in sym))))
    return codec.CompressedModel(pm.kind, pm.levels, pm.bucket_size, lengths, tensors, buffers=pm.buffers)


@pytest.mark.parametrize("case", HUFFMAN_CASES)
def test_oracle_round_trip_reproduces_the_golden_huffman_file(case, tmp_path):
    cm = _load(case, tmp_path)
    packed = _oracle_pack_compressed(cm)
    assert G.file_bytes(_oracle_compress_packed(cm, packed), "huffman") == GOLDEN[case].tobytes()


@pytest.mark.parametrize("bits", [1, 2, 4, 8])
def test_numpy_pack_is_the_golden_layout(bits):
    rng = np.random.default_rng(bits)
    for n in (1, 7, 8, 9, 100, 1031):
        codes = rng.integers(0, 1 << bits, n)
        assert np.array_equal(np_pack(codes, bits), G._pack(codes, bits))
        assert np.array_equal(np_unpack(np_pack(codes, bits), bits, n), codes)
