"""Fixed-width model files, host side (no GPU): the layout and its size accounting against get_size_reduction, a
save / load round trip into one data region, every malformed header or section refused while reading, and unpack_
refusing a mismatched model before it writes anything."""
import json
import struct

import numpy as np
import pytest
import torch

from quantized_distillation_b200 import codec


def _pack(codes, bits):
    """The qd_pack_indices layout: code of element e in byte e*bits/8 at bit (e*bits)%8, little endian."""
    out = np.zeros((codes.size * bits + 7) // 8, np.uint8)
    for e, c in enumerate(codes.tolist()):
        out[e * bits // 8] |= (c << (e * bits % 8)) & 0xFF
    return out


def test_pack_layout_of_the_helper():
    assert _pack(np.array([1, 0, 1, 1, 0, 0, 0, 1, 1]), 1).tolist() == [0b10001101, 1]
    assert _pack(np.array([3, 2, 1]), 2).tolist() == [0b011011]
    assert _pack(np.array([0xA, 0x5, 0xF]), 4).tolist() == [0x5A, 0x0F]


def _pm(bits=(4, 2), ns=(2048, 1500), s=4, bucket=256, buffers=None, kind="uniform", points=None):
    rng = np.random.default_rng(2)
    tensors = [codec.PackedEntry("first", (3, 5), raw=torch.randn(15))]
    for k, (b, n) in enumerate(zip(bits, ns)):
        levels = s if kind == "uniform" else len(points[k])
        codes = rng.integers(0, levels, n)
        rows = codec._rows(n, bucket)
        tensors.append(codec.PackedEntry(f"t{k}", (n,), bits=b, packed=torch.from_numpy(_pack(codes, b)), alpha=torch.rand(rows),
                                         beta=torch.randn(rows), points=None if points is None else torch.tensor(points[k])))
    tensors.append(codec.PackedEntry("last", (4,), raw=torch.randn(4)))
    return codec.PackedModel(kind, s if kind == "uniform" else None, bucket, tensors, buffers=buffers)


def _buffers():
    return [("bn.running_mean", torch.randn(7)), ("bn.num_batches_tracked", torch.tensor(5, dtype=torch.int64)),
            ("empty", torch.zeros(0))]


def _split(raw):
    magic, version, res, hlen = struct.unpack_from("<8sIIQ", raw)
    return magic, version, json.loads(raw[24:24 + hlen]), raw[(24 + hlen + 15) // 16 * 16:]


def _rewrite(raw, fn=None, version=None, magic=None):
    m, v, h, data = _split(raw)
    if fn is not None:
        fn(h)
    hb = json.dumps(h).encode()
    pad = (24 + len(hb) + 15) // 16 * 16 - 24 - len(hb)
    return struct.pack("<8sIIQ", magic or m, v if version is None else version, 0, len(hb)) + hb + b"\0" * pad + data


def test_round_trip_layout_and_size_accounting(tmp_path):
    pm = _pm(buffers=_buffers())
    path = tmp_path / "m.qdp"
    size = codec.save_packed(pm, path)
    raw = path.read_bytes()
    magic, version, h, _ = _split(raw)
    assert magic == b"QDPACK\0\0" and version == 1
    assert [t["bits"] for t in h["tensors"] if t["quantized"]] == [4, 2]
    for t in h["tensors"]:
        for off, nb in t["sections"].values():
            assert off % 16 == 0
    back = codec.load_packed(path)
    sb = back.size_breakdown()
    assert sb == pm.size_breakdown() and sb["file_bytes"] == size == len(raw)
    assert sb["code_bytes"] == 2048 * 4 // 8 + 1500 * 2 // 8
    assert sb["scale_bytes"] == 8 * (8 + 6)
    assert sb["unquantized_bytes"] == 19 * 4 and sb["buffer_bytes"] == 7 * 4 + 8
    assert sb["file_bytes"] == sum(v for k, v in sb.items() if k != "file_bytes")
    # every section of the loaded file is a view into one host tensor holding the data region
    base = back._data.untyped_storage().data_ptr()
    views = [x for t in back.tensors for x in (t.packed, t.alpha, t.beta, t.raw) if x is not None]
    assert all(x.untyped_storage().data_ptr() == base and not x.is_cuda for x in views + [b for _, b in back.buffers])
    for a, b in zip(pm.tensors, back.tensors):
        assert a.name == b.name and a.shape == b.shape and a.bits == b.bits
        for f in ("packed", "alpha", "beta", "raw"):
            if getattr(a, f) is not None:
                assert torch.equal(getattr(a, f).view(-1), getattr(b, f).view(-1)), f
    for (na, a), (nb_, b) in zip(pm.buffers, back.buffers):
        assert na == nb_ and a.dtype == b.dtype and torch.equal(a, b)


def test_file_without_buffers_has_no_buffer_key(tmp_path):
    codec.save_packed(_pm(), tmp_path / "m.qdp")
    _, _, h, _ = _split((tmp_path / "m.qdp").read_bytes())
    assert "buffers" not in h and codec.load_packed(tmp_path / "m.qdp").buffers is None


@pytest.mark.parametrize("bits,bucket", [(1, 256), (2, 256), (4, 512), (8, 1024), (2, None)])
def test_code_and_scale_bytes_are_what_get_size_reduction_counts(bits, bucket):
    """Tensors whose codes fill whole bytes and whole buckets: code + scale bytes are exactly the float32 size over
    get_size_reduction(bits, bucket)."""
    ns = (4096, 1024 * 3, 8192)
    pm = _pm(bits=(bits,) * 3, ns=ns, s=2, bucket=bucket)
    sb = pm.size_breakdown()
    count = sum(ns)
    if bucket is None:                        # one bucket per tensor: 8 bytes each on top of the codes
        assert sb["code_bytes"] == count * 32 / codec.get_size_reduction(bits, None) / 8
        assert sb["scale_bytes"] == 8 * len(ns)
    else:
        assert sb["code_bytes"] + sb["scale_bytes"] == count * 4 / codec.get_size_reduction(bits, bucket)


def test_nonuniform_points_round_trip(tmp_path):
    pts = [[0.0, 0.25, 1.0], [-1.0, 0.1, 0.1, 0.3, 0.5, 0.7, 0.9, 1.0, 2.0]]
    pm = _pm(bits=(2, 4), kind="nonuniform", points=pts)
    codec.save_packed(pm, tmp_path / "m.qdp")
    back = codec.load_packed(tmp_path / "m.qdp")
    assert back.kind == "nonuniform" and back.levels is None
    for t, p in zip([t for t in back.tensors if t.quantized], pts):
        assert torch.equal(t.points, torch.tensor(p, dtype=torch.float32))


def test_malformed_files_are_refused(tmp_path):
    path = tmp_path / "m.qdp"
    codec.save_packed(_pm(buffers=_buffers()), path)
    good = path.read_bytes()
    codec.save_packed(_pm(bits=(2, 4), kind="nonuniform", points=[[0.0, 0.5, 1.0], [0.0, 1.0]]), path)
    good_nu = path.read_bytes()
    bad = tmp_path / "bad.qdp"

    def rejected(raw, match):
        bad.write_bytes(raw)
        with pytest.raises(ValueError, match=match):
            codec.load_packed(bad)

    def tensor(k, key, value):
        def fn(h):
            h["tensors"][k][key] = value
        return fn

    def sec(k, name, i, value):
        def fn(h):
            h["tensors"][k]["sections"][name][i] = value
        return fn

    rejected(b"QDPACK", "prefix")
    rejected(_rewrite(good, magic=b"QDHUFF\0\0"), "magic")
    rejected(_rewrite(good, version=2), "version")
    rejected(_rewrite(good, version=0), "version")
    rejected(good[:-1], "bytes")                                                  # truncated data region
    rejected(good + b"\0" * 16, "bytes")
    rejected(_rewrite(good, lambda h: h.pop("kind")), "header")
    rejected(_rewrite(good, lambda h: h.__setitem__("kind", "huffman")), "kind")
    rejected(_rewrite(good, lambda h: h.__setitem__("levels", 300)), "levels")
    rejected(_rewrite(good, lambda h: h.__setitem__("bucket", 0)), "bucket")
    rejected(_rewrite(good, tensor(1, "bits", 3)), "bits")
    rejected(_rewrite(good, tensor(2, "bits", 1)), "4 levels do not fit in 1-bit")    # bits against levels
    rejected(_rewrite(good_nu, tensor(1, "bits", 1)), "3 points do not fit in 1-bit")  # bits against points
    rejected(_rewrite(good_nu, lambda h: h["tensors"][1].pop("points")), "points")
    rejected(_rewrite(good, tensor(1, "points", [0.0, 1.0])), "no points")
    rejected(_rewrite(good, sec(1, "packed", 1, 1023)), "1023 bytes")            # short section
    rejected(_rewrite(good, sec(1, "alpha", 1, 28)), "28 bytes")
    rejected(_rewrite(good, sec(0, "raw", 1, 64)), "64 bytes")
    rejected(_rewrite(good, sec(1, "alpha", 0, 8)), "out of range")               # misaligned
    rejected(_rewrite(good, sec(1, "beta", 0, -16)), "out of range")
    rejected(_rewrite(good, lambda h: h["tensors"][1]["sections"]["beta"].__setitem__(0, h["data_bytes"])), "out of range")
    rejected(_rewrite(good, lambda h: h["tensors"][2]["sections"]["alpha"].__setitem__(
        0, h["tensors"][1]["sections"]["packed"][0])), "overlap")                 # overlapping sections
    rejected(_rewrite(good, lambda h: h["buffers"][0]["section"].__setitem__(0, 0)), "overlap")
    rejected(_rewrite(good, lambda h: h["tensors"][1]["sections"].pop("beta")), "sections")
    rejected(_rewrite(good, lambda h: h["tensors"][1]["sections"].__setitem__("words", [0, 0])), "sections")
    rejected(_rewrite(good, tensor(2, "name", "t0")), "twice")                    # duplicate tensor name
    rejected(_rewrite(good, lambda h: h["buffers"][1].__setitem__("name", "bn.running_mean")), "twice")
    rejected(_rewrite(good, lambda h: h["buffers"][0].__setitem__("dtype", "float16")), "dtype")
    rejected(_rewrite(good, lambda h: h.__setitem__("buffers", {})), "not a list")
    rejected(_rewrite(good, tensor(1, "shape", [0])), "empty")
    rejected(_rewrite(good, tensor(1, "dtype", "float16")), "dtype")
    assert len(codec.load_packed(tmp_path / "m.qdp").tensors) == 4


def test_the_two_containers_refuse_each_other(tmp_path):
    codec.save_packed(_pm(), tmp_path / "m.qdp")
    with pytest.raises(ValueError, match="magic"):
        codec.load_compressed(tmp_path / "m.qdp")
    cm = codec.CompressedModel("uniform", 16, 256, {0: 1, 1: 1}, [codec.HuffmanTensor("w", (4,), raw=torch.randn(4))])
    codec.save_compressed(cm, tmp_path / "m.qdh")
    with pytest.raises(ValueError, match="magic"):
        codec.load_packed(tmp_path / "m.qdh")


class _Net(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.fc = torch.nn.Linear(4, 3)
        self.bn = torch.nn.BatchNorm1d(3)


def _net_pm(net, buffers, shapes=None):
    tensors = [codec.PackedEntry(n, tuple(p.shape) if shapes is None else shapes[i], raw=torch.randn(p.numel()))
               for i, (n, p) in enumerate(net.named_parameters())]
    return codec.PackedModel("uniform", 16, 256, tensors, buffers=buffers)


def test_unpack_with_a_mismatched_model_raises_before_writing():
    net = _Net()
    state = {k: v.clone() for k, v in net.state_dict().items()}
    good = [(n, b.clone() + 1) for n, b in codec._persistent_buffers(net)]
    cases = [(_net_pm(net, good[:2]), "buffer"),                                                       # missing buffer
             (_net_pm(net, good + [("extra", torch.ones(1))]), "buffer"),                              # extra buffer
             (_net_pm(net, [good[0], ("bn.running_var", torch.ones(4)), good[2]]), "buffer"),          # buffer shape
             (_net_pm(net, [good[0], good[1], ("bn.num_batches_tracked", torch.tensor(1.0))]), "buffer"),   # dtype
             (_net_pm(net, good, shapes=[(4, 3), (3,), (3,), (3,)]), "shape"),
             (codec.PackedModel("uniform", 16, 256, _net_pm(net, good).tensors[:3], buffers=good), "parameters")]
    for pm, match in cases:
        with pytest.raises(ValueError, match=match):
            codec.unpack_(pm, net)
        assert all(torch.equal(v, net.state_dict()[k]) for k, v in state.items())


def test_pack_model_refuses_bad_buffers_before_device_work():
    net = _Net()
    net.register_buffer("mask", torch.ones(3, dtype=torch.bool))
    with pytest.raises(ValueError, match="bool"):
        codec.pack_model(net, 4, include_buffers=True)


def test_unpack_needs_a_gpu():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    net = _Net()
    state = {k: v.clone() for k, v in net.state_dict().items()}
    with pytest.raises(RuntimeError):
        codec.unpack_(_net_pm(net, [(n, b.clone() + 1) for n, b in codec._persistent_buffers(net)]), net)
    assert all(torch.equal(v, net.state_dict()[k]) for k, v in state.items())
