"""Transcoding between the Huffman-coded and the fixed-width model containers on the GPU.

pack_compressed (qd_huffman_decode_packed_model: every stream of a model straight to fixed-width codes in one launch)
is checked byte for byte against the NumPy oracle's decode-then-pack; compress_packed (qd_unpack_indices, then
compress_model's histogram, code and encoder) and both directions are checked as whole files against compress_model and
pack_model; whole networks loaded through the transcoder compute the logits of networks loaded from the original."""
import threading

import numpy as np
import pytest
import torch

from oracle import huffman_oracle as HO

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from quantized_distillation_b200 import _native as N
    from quantized_distillation_b200 import codec
    return N, codec


def np_pack(codes, bits):
    """The qd_pack_indices layout, vectorised: code of element e in byte e*bits/8 at bit (e*bits)%8."""
    per = 8 // bits
    c = np.zeros(-(-codes.size // per) * per, np.uint32)
    c[:codes.size] = codes
    return (c.reshape(-1, per) << (np.arange(per, dtype=np.uint32) * bits)).sum(1).astype(np.uint8)


def _symbols(rng, n, limit):
    """Skewed draws in [0, limit): rare symbols get long codes, so codes of every length cross word and chunk edges."""
    if limit == 1:
        return np.zeros(n, np.uint8)
    p = 0.6 ** np.arange(limit)
    return rng.choice(limit, size=n, p=p / p.sum()).astype(np.uint8)


def _huffman_model(codec, kind, levels, bucket, sizes, limits, seed=0, lengths=None, syms=None):
    """A host CompressedModel (float32 first and last tensors around quantized ones) whose tensor t holds symbols in
    [0, limits[t]) (or ``syms``) under one model-wide code, and the symbols."""
    rng = np.random.default_rng(seed)
    if syms is None:
        syms = [_symbols(rng, n, k) for n, k in zip(sizes, limits)]
    if lengths is None:
        counts = np.bincount(np.concatenate(syms), minlength=256)
        lengths = codec.huffman_code_lengths(counts)
    tensors = [codec.HuffmanTensor("first", (3,), raw=torch.from_numpy(rng.standard_normal(3).astype(np.float32)))]
    for k, (n, s) in enumerate(zip(sizes, syms)):
        rows = codec._rows(n, bucket)
        words, offs = HO.encode(s, lengths)
        pts = None if kind == "uniform" else torch.from_numpy(np.sort(rng.standard_normal(limits[k])).astype(np.float32))
        tensors.append(codec.HuffmanTensor(f"t{k}", (n,), words=torch.from_numpy(words.view(np.int32)),
                                           chunk_offsets=torch.from_numpy(offs.view(np.int32)),
                                           alpha=torch.from_numpy(rng.random(rows).astype(np.float32)),
                                           beta=torch.from_numpy(rng.standard_normal(rows).astype(np.float32)), points=pts,
                                           code_bits=int(sum(lengths[int(v)] * int(c) for v, c in zip(*np.unique(s, return_counts=True))))))
    tensors.append(codec.HuffmanTensor("last", (2,), raw=torch.from_numpy(rng.standard_normal(2).astype(np.float32))))
    return codec.CompressedModel(kind, levels, bucket, lengths, tensors), syms


def _check_against_oracle(codec, cm, syms, limits, device="cuda"):
    pm = codec.pack_compressed(cm, device)
    q = [t for t in pm.tensors if t.quantized]
    assert len(q) == len(syms)
    for t, src, s, k in zip(q, [t for t in cm.tensors if t.quantized], syms, limits):
        bits = codec.bits_for(k)
        assert t.bits == bits and t.packed.is_cuda
        assert np.array_equal(t.packed.cpu().numpy(), np_pack(s, bits)), t.name
        assert torch.equal(t.alpha.cpu(), src.alpha.cpu().reshape(-1)) and torch.equal(t.beta.cpu(), src.beta.cpu().reshape(-1))
        assert (t.points is None) == (src.points is None)
        if t.points is not None:
            assert torch.equal(t.points.cpu(), src.points.cpu())
    assert [t.name for t in pm.tensors] == [t.name for t in cm.tensors]
    assert (pm.kind, pm.levels, pm.bucket_size) == (cm.kind, cm.levels, cm.bucket_size)
    return pm


SIZES = [1, 1023, 1024, 1025, 3 * 1024 * 128 + 1, 5000]


@pytest.mark.parametrize("bucket", [256, 1024, 100, None])
@pytest.mark.parametrize("s", [2, 3, 4, 16, 256])
def test_uniform_matches_oracle(env, s, bucket):
    N, codec = env
    sizes = SIZES + ([(1 << 20) + 3] if bucket in (256, None) else [])
    cm, syms = _huffman_model(codec, "uniform", s, bucket, sizes, [s] * len(sizes), seed=s)
    _check_against_oracle(codec, cm, syms, [s] * len(sizes))


@pytest.mark.parametrize("bucket", [256, None])
def test_nonuniform_per_tensor_widths_match_oracle(env, bucket):
    N, codec = env
    limits = [1, 2, 3, 5, 16, 17, 256]
    sizes = [1025, 1, 4097, 1024, 131073, 1023, 70000]
    cm, syms = _huffman_model(codec, "nonuniform", None, bucket, sizes, limits, seed=3)
    _check_against_oracle(codec, cm, syms, limits)


def test_single_symbol_code_has_no_stream(env):
    N, codec = env
    cm, syms = _huffman_model(codec, "nonuniform", None, 256, [1, 1025, 3000], [1, 3, 1], lengths={0: 0},
                              syms=[np.zeros(n, np.uint8) for n in (1, 1025, 3000)])
    assert all(t.words.numel() == 0 for t in cm.tensors if t.quantized)
    _check_against_oracle(codec, cm, syms, [1, 3, 1])


def test_thousands_of_tensors_in_one_launch(env):
    N, codec = env
    rng = np.random.default_rng(11)
    sizes = [int(v) for v in rng.integers(1, 3000, 3000)]
    cm, syms = _huffman_model(codec, "uniform", 16, 64, sizes, [16] * len(sizes), seed=12)
    _check_against_oracle(codec, cm, syms, [16] * len(sizes))


def test_device_resident_input_and_no_shared_storage(env):
    N, codec = env
    cm, syms = _huffman_model(codec, "uniform", 4, 256, [5000, 70], [4, 4], seed=5)
    cm.buffers = [("bn.running_mean", torch.arange(3, dtype=torch.float32)), ("steps", torch.tensor(7))]
    for t in cm.tensors:
        for f in ("words", "chunk_offsets", "alpha", "beta", "raw"):
            if getattr(t, f) is not None:
                setattr(t, f, getattr(t, f).cuda())
    pm = _check_against_oracle(codec, cm, syms, [4, 4])
    ptrs = {x.untyped_storage().data_ptr() for t in cm.tensors for x in (t.words, t.chunk_offsets, t.alpha, t.beta, t.raw)
            if x is not None}
    assert not any(x.untyped_storage().data_ptr() in ptrs for t in pm.tensors for x in (t.packed, t.alpha, t.beta, t.raw)
                   if x is not None)
    assert [(n, b.tolist()) for n, b in pm.buffers] == [(n, b.tolist()) for n, b in cm.buffers]


# ---- whole files against compress_model / pack_model ---------------------------------------------------------------
def _net(seed):
    torch.manual_seed(seed)
    net = torch.nn.Sequential(torch.nn.Conv2d(3, 8, 3, padding=1), torch.nn.BatchNorm2d(8), torch.nn.ReLU(),
                              torch.nn.Conv2d(8, 16, 3), torch.nn.Flatten(), torch.nn.Linear(16 * 6 * 6, 300), torch.nn.ReLU(),
                              torch.nn.Linear(300, 10)).cuda()
    with torch.no_grad():
        net(torch.randn(4, 3, 8, 8, device="cuda"))           # moves the BatchNorm statistics
    return net


def _file(codec, m, tmp_path, name):
    path = tmp_path / name
    (codec.save_compressed if isinstance(m, codec.CompressedModel) else codec.save_packed)(m, path)
    return path.read_bytes()


ENCODINGS = {
    "uniform2": dict(numBits=2), "uniform4-b100": dict(numBits=4, bucket_size=100), "uniform8-none": dict(numBits=8, bucket_size=None),
    "uniform1-keep-ends": dict(numBits=1, quantize_first_and_last_layer=False),
    "nearest-shared": dict(points=[-1.0, -0.2, 0.0, 0.3, 1.0]),
    "midpoint-per-tensor": dict(points=[[-1.0, 1.0], [0.0], [-0.5, 0.0, 0.5], [-2.0, -1.0, 0.0, 0.5, 1.0, 1.5, 2.0, 3.0, 4.0],
                                        [float(v) for v in np.linspace(-1, 1, 17)], [0.1, 0.2, 0.3],
                                        [float(v) for v in np.linspace(-1, 1, 200)], [-0.1, 0.1], [0.5], [-3.0, 0.0, 3.0, 4.0]],
                                rule="midpoint"),
}


@pytest.mark.parametrize("buffers", [False, True])
@pytest.mark.parametrize("enc", sorted(ENCODINGS))
def test_files_equal_the_direct_encoders(env, enc, buffers, tmp_path):
    N, codec = env
    net = _net(1)
    kw = dict(ENCODINGS[enc], include_buffers=buffers)
    cm = codec.compress_model(net, **kw)
    pm = codec.pack_model(net, **kw)
    cm_file, pm_file = _file(codec, cm, tmp_path, "cm"), _file(codec, pm, tmp_path, "pm")
    assert _file(codec, codec.pack_compressed(cm), tmp_path, "a") == pm_file
    assert _file(codec, codec.compress_packed(pm), tmp_path, "b") == cm_file
    assert _file(codec, codec.pack_compressed(codec.compress_packed(pm)), tmp_path, "c") == pm_file
    assert _file(codec, codec.compress_packed(codec.pack_compressed(cm)), tmp_path, "d") == cm_file
    # from host-loaded files: one copy of the data region each
    assert _file(codec, codec.pack_compressed(codec.load_compressed(tmp_path / "cm")), tmp_path, "e") == pm_file
    assert _file(codec, codec.compress_packed(codec.load_packed(tmp_path / "pm")), tmp_path, "f") == cm_file


# ---- refusals ---------------------------------------------------------------------------------------------------------
def test_stream_symbol_beyond_a_tensors_points_is_refused(env):
    N, codec = env
    # one model-wide code over symbols 0..5; tensor t1 has K_t = 3 points but its stream emits symbol 5
    lengths = codec.huffman_code_lengths(np.bincount([0, 1, 2, 3, 4, 5, 5, 5], minlength=256))
    cm, _ = _huffman_model(codec, "nonuniform", None, 256, [2000, 2000], [6, 3], lengths=lengths)
    bad = np.zeros(2000, np.uint8)
    bad[1500] = 5
    words, offs = HO.encode(bad, lengths)
    cm.tensors[2].words, cm.tensors[2].chunk_offsets = torch.from_numpy(words.view(np.int32)), torch.from_numpy(offs.view(np.int32))
    with pytest.raises(ValueError, match="t1"):
        codec.pack_compressed(cm)


def test_stream_symbol_beyond_the_levels_is_refused(env):
    N, codec = env
    lengths = codec.huffman_code_lengths(np.bincount([0, 1, 2, 3], minlength=256))
    cm, _ = _huffman_model(codec, "uniform", 3, None, [10, 5000], [3, 3], lengths=lengths)
    sym = np.zeros(5000, np.uint8)
    sym[4999] = 3
    words, offs = HO.encode(sym, lengths)
    cm.tensors[2].words, cm.tensors[2].chunk_offsets = torch.from_numpy(words.view(np.int32)), torch.from_numpy(offs.view(np.int32))
    with pytest.raises(ValueError, match="t1"):
        codec.pack_compressed(cm)


def _packed_model(codec, kind, levels, codes, bits, points=None):
    tensors = []
    for k, (c, b) in enumerate(zip(codes, bits)):
        tensors.append(codec.PackedEntry(f"w{k}", (c.size,), bits=b, packed=torch.from_numpy(np_pack(c, b)), alpha=torch.ones(1),
                                         beta=torch.zeros(1), points=None if points is None else torch.tensor(points[k])))
    return codec.PackedModel(kind, levels, None, tensors)


def test_packed_code_beyond_the_levels_or_points_is_refused(env):
    N, codec = env
    ok = np.zeros(100, np.uint8)
    bad = ok.copy()
    bad[77] = 3
    with pytest.raises(ValueError, match="w1"):
        codec.compress_packed(_packed_model(codec, "uniform", 3, [ok, bad], [2, 2]))
    with pytest.raises(ValueError, match="w1"):
        codec.compress_packed(_packed_model(codec, "nonuniform", None, [ok, bad], [2, 4], points=[[0.0, 1.0, 2.0, 3.0], [0.0, 1.0, 2.0]]))
    codec.compress_packed(_packed_model(codec, "nonuniform", None, [ok, bad], [2, 2], points=[[0.0, 1.0], [0.0, 1.0, 2.0, 3.0]]))


def test_c_entry_point_refusals(env):
    N, codec = env
    cm, _ = _huffman_model(codec, "uniform", 4, 256, [3000], [4])
    t = cm.tensors[1]
    words, offs = t.words.cuda(), t.chunk_offsets.cuda()
    packed = torch.empty(750, dtype=torch.uint8, device="cuda")
    table = cm.table("cuda")
    oor = torch.zeros(2, dtype=torch.int64, device="cuda")
    ws = torch.empty(int(N.lib().qd_huffman_repack_model_workspace_bytes(1)), dtype=torch.uint8, device="cuda")
    good = (N.ptr(words), N.ptr(offs), N.ptr(packed), words.numel(), 3000, 2, 4)

    def call(fields=good, count=1, tab=N.ptr(table), out=N.ptr(oor), w=N.ptr(ws), wb=ws.numel(), desc=True):
        d = np.zeros(max(count, 1), codec._REPACK_TENSOR)
        d[:] = fields
        return N.lib().qd_huffman_decode_packed_model(d.ctypes.data if desc else None, count, tab, out, w, wb, N.stream_ptr())

    assert call() == N.QD_OK
    torch.cuda.synchronize()
    assert oor.tolist() == [0, 0]
    bad = [dict(count=0), dict(desc=False), dict(tab=None), dict(out=None)]
    for i in range(3):                          # words NULL with num_words > 0, chunk_offsets NULL, packed NULL
        f = list(good)
        f[i] = 0
        bad.append(dict(fields=tuple(f)))
    for i, v in [(3, -1), (4, 0), (5, 3), (5, 16), (6, 0), (6, 5)]:   # num_words < 0, n < 1, bits, limit outside [1, 2^bits]
        f = list(good)
        f[i] = v
        bad.append(dict(fields=tuple(f)))
    for kw in bad:
        assert call(**kw) == N.QD_ERR_INVALID_ARG, kw
    assert call(wb=ws.numel() - 1) == N.QD_ERR_WORKSPACE
    assert call(w=None) == N.QD_ERR_WORKSPACE
    # one-symbol stream: words may be NULL when num_words is 0
    f = list(good)
    f[0], f[3] = 0, 0
    assert call(fields=tuple(f)) == N.QD_OK
    torch.cuda.synchronize()


@pytest.mark.parametrize("bits", [1, 2, 4, 8])
def test_unpack_indices_inverts_pack_indices(env, bits):
    N, codec = env
    g = torch.Generator(device="cuda").manual_seed(bits)
    for n in (1, 5, 13, 16, 17, 1000, 4099, (1 << 20) + 7):
        for off_in, off_out in ((0, 0), (1, 3), (3, 1), (2, 15)):
            idx = torch.randint(0, 1 << bits, (n + off_in,), generator=g, device="cuda", dtype=torch.int32).to(torch.uint8)[off_in:]
            pbuf = torch.zeros((n * bits + 7) // 8 + off_in, dtype=torch.uint8, device="cuda")
            packed = pbuf[off_in:]
            N.check(N.lib().qd_pack_indices(N.ptr(idx), N.ptr(packed), n, bits, N.stream_ptr()))
            obuf = torch.full((n + off_out + 16,), 0xAB, dtype=torch.uint8, device="cuda")
            out = obuf[off_out:off_out + n]
            N.check(N.lib().qd_unpack_indices(N.ptr(packed), bits, N.ptr(out), n, N.stream_ptr()))
            assert torch.equal(out, idx), (n, off_in, off_out)
            assert torch.all(obuf[:off_out] == 0xAB) and torch.all(obuf[off_out + n:] == 0xAB)
    x = torch.zeros(4, dtype=torch.uint8, device="cuda")
    assert N.lib().qd_unpack_indices(None, bits, N.ptr(x), 4, N.stream_ptr()) == N.QD_ERR_INVALID_ARG
    assert N.lib().qd_unpack_indices(N.ptr(x), bits, None, 4, N.stream_ptr()) == N.QD_ERR_INVALID_ARG
    assert N.lib().qd_unpack_indices(N.ptr(x), bits, N.ptr(x), 0, N.stream_ptr()) == N.QD_ERR_INVALID_ARG
    assert N.lib().qd_unpack_indices(N.ptr(x), 3, N.ptr(x), 4, N.stream_ptr()) == N.QD_ERR_INVALID_ARG


# ---- end to end ---------------------------------------------------------------------------------------------------------
def _student(seed):
    from quantized_distillation_b200.cnn_models import conv_forward_model as cfm
    torch.manual_seed(seed)
    return cfm.ConvolForwardNet(**cfm.smallerModelSpec, useBatchNorm=True, useAffineTransformInBatchNorm=True).cuda()


def _wrn(seed):
    from quantized_distillation_b200.cnn_models.wide_resnet import Wide_ResNet
    torch.manual_seed(seed)
    return Wide_ResNet(depth=16, widen_factor=22, dropout_rate=0.3, num_classes=10).cuda()


@pytest.mark.parametrize("which,numBits", [("student", 4), ("wrn16_22", 2)])
def test_huffman_file_runs_from_packed_codes(env, which, numBits, tmp_path):
    N, codec = env
    make = _student if which == "student" else _wrn
    net = make(0)
    with torch.no_grad():
        net(torch.randn(8, 3, 32, 32, device="cuda"))               # training-mode forward: running statistics move
    cm = codec.compress_model(net, numBits, bucket_size=256, quantize_first_and_last_layer=False, include_buffers=True)
    codec.save_compressed(cm, tmp_path / "m.qdh")
    del cm
    host = codec.load_compressed(tmp_path / "m.qdh")
    a = make(1)
    replaced = codec.attach_packed_(codec.pack_compressed(host), a)
    b = make(2)
    assert codec.attach_packed_(codec.pack_model(net, numBits, bucket_size=256, quantize_first_and_last_layer=False,
                                                 include_buffers=True), b) == replaced and replaced
    a.eval(), b.eval()
    x = torch.randn(4, 3, 32, 32, device="cuda")
    with torch.no_grad():
        assert torch.equal(a(x), b(x))
    c, d = make(3), make(4)
    codec.unpack_(codec.pack_compressed(host), c)
    codec.decompress_(host, d)
    for (name, p), q in zip(c.state_dict().items(), d.state_dict().values()):
        assert torch.equal(p, q), name


def test_concurrent_streams_give_identical_bytes(env, tmp_path):
    N, codec = env
    net = _student(0)
    cm = codec.compress_model(net, 4, bucket_size=256, include_buffers=True)
    pm = codec.pack_model(net, 4, bucket_size=256, include_buffers=True)
    want_pm, want_cm = _file(codec, pm, tmp_path, "pm"), _file(codec, cm, tmp_path, "cm")
    results, errors = {}, []

    def work(k):
        try:
            with torch.cuda.stream(torch.cuda.Stream()):
                for r in range(3):
                    results[(k, r, "p")] = _file(codec, codec.pack_compressed(cm), tmp_path, f"p{k}")
                    results[(k, r, "c")] = _file(codec, codec.compress_packed(pm), tmp_path, f"c{k}")
        except Exception as e:  # noqa: BLE001 - reported below
            errors.append(e)

    threads = [threading.Thread(target=work, args=(k,)) for k in range(4)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    assert len(results) == 24
    assert all(v == (want_pm if key[2] == "p" else want_cm) for key, v in results.items())
