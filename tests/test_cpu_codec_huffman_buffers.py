"""Huffman-coded model files with persistent buffers, host side (no GPU): version 2 exactly when buffers are stored,
the buffer sections and their validation, one data region behind every section of a loaded file, and decompress_
refusing a model whose buffers do not match before it writes anything."""
import json
import struct

import numpy as np
import pytest
import torch

from oracle import huffman_oracle as HO
from quantized_distillation_b200 import codec

V1_KEYS = {"chunk", "kind", "levels", "bucket", "code", "tensors", "data_bytes"}


def _cm(buffers=None):
    """Two quantized tensors (oracle-encoded streams) between two unquantized ones, optionally with buffers."""
    rng = np.random.default_rng(2)
    sym = [rng.integers(0, 16, n).astype(np.uint8) for n in (2000, 1500)]
    lengths = codec.huffman_code_lengths(np.bincount(np.concatenate(sym), minlength=256))
    tensors = [codec.HuffmanTensor("first", (3, 5), raw=torch.randn(15))]
    for k, s in enumerate(sym):
        words, offs = HO.encode(s, lengths)
        rows = codec._rows(s.size, 256)
        tensors.append(codec.HuffmanTensor(f"t{k}", (s.size,), words=torch.from_numpy(words.view(np.int32)),
                                           chunk_offsets=torch.from_numpy(offs.view(np.int32)), alpha=torch.rand(rows),
                                           beta=torch.randn(rows), code_bits=int(sum(lengths[v] for v in s.tolist()))))
    tensors.append(codec.HuffmanTensor("last", (4,), raw=torch.randn(4)))
    return codec.CompressedModel("uniform", 16, 256, lengths, tensors, buffers=buffers)


def _buffers():
    return [("bn.running_mean", torch.randn(7)), ("bn.running_var", torch.rand(3, 2)),
            ("bn.num_batches_tracked", torch.tensor(5, dtype=torch.int64)), ("scale", torch.tensor(1.5)),
            ("steps", torch.arange(-3, 6, dtype=torch.int64).view(3, 3)), ("empty", torch.zeros(0))]


def _header(raw):
    magic, version, _, hlen = struct.unpack_from("<8sIIQ", raw)
    return version, json.loads(raw[24:24 + hlen])


def _rewrite(raw, fn, version=None):
    magic, v, res, hlen = struct.unpack_from("<8sIIQ", raw)
    h = json.loads(raw[24:24 + hlen])
    fn(h)
    data = raw[(24 + hlen + 15) // 16 * 16:]
    hb = json.dumps(h).encode()
    pad = (24 + len(hb) + 15) // 16 * 16 - 24 - len(hb)
    return struct.pack("<8sIIQ", magic, v if version is None else version, res, len(hb)) + hb + b"\0" * pad + data


def test_version_2_round_trip_with_float32_and_int64_buffers(tmp_path):
    cm = _cm(_buffers())
    path = tmp_path / "m.qdh"
    size = codec.save_compressed(cm, path)
    raw = path.read_bytes()
    version, h = _header(raw)
    assert version == 2 and [b["name"] for b in h["buffers"]] == [n for n, _ in _buffers()]
    assert all(b["section"][0] % 16 == 0 for b in h["buffers"])
    back = codec.load_compressed(path)
    assert [n for n, _ in back.buffers] == [n for n, _ in cm.buffers]
    for (_, a), (_, b) in zip(cm.buffers, back.buffers):
        assert a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b) and not b.is_cuda
    assert back.buffers[2][1].dim() == 0 and int(back.buffers[2][1]) == 5
    sb = cm.size_breakdown()
    assert back.size_breakdown() == sb and sb["file_bytes"] == size
    assert sb["buffer_bytes"] == 7 * 4 + 6 * 4 + 8 + 4 + 9 * 8
    assert sb["file_bytes"] == (sb["code_bits"] + sb["padding_bits"]) // 8 + sb["chunk_index_bytes"] + sb["scale_bytes"] + \
        sb["unquantized_bytes"] + sb["buffer_bytes"] + sb["header_bytes"] + sb["alignment_bytes"]
    # every section of the loaded file is a view into one host tensor holding the data region
    base = back._data.untyped_storage().data_ptr()
    views = [x for t in back.tensors for x in (t.words, t.chunk_offsets, t.alpha, t.beta, t.raw) if x is not None]
    assert all(x.untyped_storage().data_ptr() == base for x in views + [b for _, b in back.buffers])
    for a, b in zip(cm.tensors, back.tensors):
        for f in ("words", "chunk_offsets", "alpha", "beta", "raw"):
            if getattr(a, f) is not None:
                assert torch.equal(getattr(a, f).view(-1), getattr(b, f).view(-1)), f


def test_file_without_buffers_is_version_1(tmp_path):
    for cm in (_cm(), codec.CompressedModel(*[getattr(_cm(), f) for f in ("kind", "levels", "bucket_size", "code_lengths", "tensors")])):
        path = tmp_path / "m.qdh"
        codec.save_compressed(cm, path)
        version, h = _header(path.read_bytes())
        assert version == 1 and set(h) == V1_KEYS
        back = codec.load_compressed(path)
        assert back.buffers is None and back.size_breakdown()["buffer_bytes"] == 0
    # an empty list still records that the model has no buffers
    codec.save_compressed(_cm([]), path)
    version, h = _header(path.read_bytes())
    assert version == 2 and h["buffers"] == [] and codec.load_compressed(path).buffers == []


def test_malformed_buffer_entries_are_rejected(tmp_path):
    path = tmp_path / "m.qdh"
    codec.save_compressed(_cm(_buffers()), path)
    good = path.read_bytes()
    codec.save_compressed(_cm(), path)
    good_v1 = path.read_bytes()
    bad = tmp_path / "bad.qdh"

    def rejected(raw, match):
        bad.write_bytes(raw)
        with pytest.raises(ValueError, match=match):
            codec.load_compressed(bad)

    def edit(k, key, value):
        def fn(h):
            h["buffers"][k][key] = value
        return fn

    rejected(_rewrite(good, lambda h: h["buffers"][0]["section"].__setitem__(0, h["data_bytes"])), "out of range")
    rejected(_rewrite(good, lambda h: h["buffers"][0]["section"].__setitem__(0, h["buffers"][0]["section"][0] + 4)), "out of range")
    rejected(_rewrite(good, lambda h: h["buffers"][0]["section"].__setitem__(0, -16)), "out of range")
    rejected(_rewrite(good, edit(1, "dtype", "float16")), "dtype")
    rejected(_rewrite(good, edit(2, "dtype", "float32")), "bytes")                 # int64 scalar: 8 bytes, not 4
    rejected(_rewrite(good, edit(0, "shape", [8])), "bytes")
    rejected(_rewrite(good, edit(1, "name", "bn.running_mean")), "twice")
    rejected(_rewrite(good, lambda h: h["buffers"][0].pop("section")), "buffer entry")
    rejected(_rewrite(good, lambda h: h.__setitem__("buffers", {})), "not a list")
    rejected(_rewrite(good, lambda h: None, version=1), "version-1")                # buffers in a version-1 file
    rejected(_rewrite(good_v1, lambda h: None, version=2), "version-2")             # no buffers in a version-2 file
    rejected(_rewrite(good_v1, lambda h: None, version=3), "version")
    assert len(codec.load_compressed(bad.parent / "m.qdh").tensors) == 4


class _Net(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.fc = torch.nn.Linear(4, 3)
        self.bn = torch.nn.BatchNorm1d(3)
        self.register_buffer("scratch", torch.zeros(2, dtype=torch.bool), persistent=False)


def _raw_cm(net, buffers):
    tensors = [codec.HuffmanTensor(n, tuple(p.shape), raw=torch.randn(p.numel())) for n, p in net.named_parameters()]
    return codec.CompressedModel("uniform", 16, 256, {0: 1, 1: 1}, tensors, buffers=buffers)


def test_persistent_buffers_follow_state_dict():
    net = _Net()
    assert [n for n, _ in codec._persistent_buffers(net)] == ["bn.running_mean", "bn.running_var", "bn.num_batches_tracked"]


def test_decompress_with_mismatched_buffers_raises_before_writing():
    net = _Net()
    state = {k: v.clone() for k, v in net.state_dict().items()}
    good = [(n, b.clone() + 1) for n, b in codec._persistent_buffers(net)]
    cases = [good[:2],                                                             # count
             [good[0], ("bn.running_var", torch.ones(4)), good[2]],                # shape
             [good[0], good[1], ("bn.num_batches_tracked", torch.tensor(1.0))]]    # dtype
    for buffers in cases:
        with pytest.raises(ValueError, match="buffer"):
            codec.decompress_(_raw_cm(net, buffers), net)
        assert all(torch.equal(v, net.state_dict()[k]) for k, v in state.items())


def test_unsupported_buffer_dtype_is_refused_at_compress_time():
    net = _Net()
    net.register_buffer("mask", torch.ones(3, dtype=torch.bool))
    with pytest.raises(ValueError, match="bool"):
        codec.compress_model(net, 4, include_buffers=True)


def test_decompress_with_buffers_needs_a_gpu():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    net = _Net()
    state = {k: v.clone() for k, v in net.state_dict().items()}
    with pytest.raises(RuntimeError):
        codec.decompress_(_raw_cm(net, [(n, b.clone() + 1) for n, b in codec._persistent_buffers(net)]), net)
    assert all(torch.equal(v, net.state_dict()[k]) for k, v in state.items())
