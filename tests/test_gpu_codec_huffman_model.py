"""Whole-model Huffman decode on the GPU: qd_huffman_decode_dequant_model (every chunk of every tensor in one launch)
against the per-tensor entry points and the fake-quantization ops, bit for bit; and complete models -- parameters and
BatchNorm buffers -- through compress_model(include_buffers=True) -> save -> load -> decompress_ into a network
built with another seed."""
import numpy as np
import pytest
import torch

from oracle import huffman_oracle as HO

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FC0DEAD           # a NaN payload no decode produces


@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import quantized_distillation_b200.quantization as Q
    from quantized_distillation_b200 import _native as N
    from quantized_distillation_b200 import codec
    return Q, N, codec


def _levels(N, x, bucket, s=None, pts=None):
    """(uint8 levels, alpha, beta) of uniformQuantization (s) or nonUniformQuantization, nearest rule (pts)."""
    n, b = x.numel(), bucket or 0
    rows = N.geometry(n, b)[0]
    alpha, beta = torch.empty(rows, device="cuda"), torch.empty(rows, device="cuda")
    idx = torch.empty(n, dtype=torch.uint8, device="cuda")
    ws = N.workspace(n, b, x.device)
    if pts is None:
        N.check(N.lib().qd_uniform_fwd(N.ptr(x), None, N.ptr(idx), N.ptr(alpha), N.ptr(beta), None, None, n, b, s, None, 0.0, 0, 0, 0,
                                       N.ptr(ws), ws.numel(), N.stream_ptr()))
    else:
        N.check(N.lib().qd_nonuniform_fwd(N.ptr(x), N.ptr(pts), pts.numel(), N.RULE_NEAREST, None, N.ptr(idx), None, N.ptr(alpha),
                                          N.ptr(beta), n, b, None, 0.0, N.ptr(ws), ws.numel(), N.stream_ptr()))
    return idx, alpha, beta


def _model(env, ns, bucket, s=None, point_counts=None, seed=0, constant=False):
    """Tensors of a model with one code over all their levels: [dict(words, offs, alpha, beta, points, n, ref)] and the table.
    ref is the fake-quantized tensor from the public op."""
    Q, N, codec = env
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = []
    for i, n in enumerate(ns):
        x = torch.full((n,), 0.25, device="cuda") if constant else torch.randn(n, generator=g, device="cuda") * 0.05
        pts = None
        if point_counts is not None:
            pts = torch.sort(torch.rand(point_counts[i % len(point_counts)], generator=g, device="cuda"))[0]
            idx, alpha, beta = _levels(N, x, bucket, pts=pts)
            ref = Q.nonUniformQuantization(x.clone(), pts, bucket_size=bucket)[0].reshape(-1)
        else:
            idx, alpha, beta = _levels(N, x, bucket, s=s)
            ref = Q.uniformQuantization(x.clone(), s, bucket_size=bucket)[0].reshape(-1)
        out.append(dict(idx=idx, alpha=alpha, beta=beta, points=pts, n=n, ref=ref))
    sym = torch.cat([t["idx"] for t in out]).cpu().numpy()
    lengths = codec.huffman_code_lengths(np.bincount(sym, minlength=256))
    at = 0
    for t in out:
        words, offs = HO.encode(sym[at:at + t["n"]], lengths)
        at += t["n"]
        t["words"] = torch.from_numpy(words.view(np.int32)).cuda()
        t["offs"] = torch.from_numpy(offs.view(np.int32)).cuda()
    return out, lengths, torch.from_numpy(codec.huffman_table(lengths)).cuda()


def _per_tensor(N, t, table, bucket, s):
    q = torch.empty(t["n"], device="cuda")
    w = t["words"]
    args = (N.ptr(w) if w.numel() else None, w.numel(), N.ptr(t["offs"]), N.ptr(table))
    if t["points"] is None:
        N.check(N.lib().qd_huffman_decode_dequant_uniform(*args, N.ptr(t["alpha"]), N.ptr(t["beta"]), N.ptr(q), t["n"], bucket or 0, s,
                                                          N.stream_ptr()))
    else:
        N.check(N.lib().qd_huffman_decode_dequant_nonuniform(*args, N.ptr(t["points"]), t["points"].numel(), N.ptr(t["alpha"]),
                                                             N.ptr(t["beta"]), N.ptr(q), t["n"], bucket or 0, N.stream_ptr()))
    return q


def _arena(ns):
    """One int32-filled float buffer holding every output, with at least one sentinel element before, between and
    after the outputs; outputs alternate between 16-byte-aligned and only 4-byte-aligned starts."""
    starts, pos = [], 1
    for i, n in enumerate(ns):
        while (pos % 4 == 0) != (i % 2 == 1):
            pos += 1
        starts.append(pos)
        pos += n + 1
    arena = torch.full((pos + 1,), SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)
    assert arena.data_ptr() % 16 == 0
    return arena, starts


def _decode_model(env, tensors, table, bucket, s, arena, starts, workspace_bytes=None):
    Q, N, codec = env
    desc = np.zeros(len(tensors), codec._MODEL_TENSOR)
    for i, (t, st) in enumerate(zip(tensors, starts)):
        w = t["words"]
        desc[i] = (N.ptr(w) if w.numel() else 0, N.ptr(t["offs"]), N.ptr(t["alpha"]), N.ptr(t["beta"]),
                   0 if t["points"] is None else N.ptr(t["points"]), arena[st:].data_ptr(), w.numel(), t["n"],
                   0 if t["points"] is None else t["points"].numel(), 0)
    need = int(N.lib().qd_huffman_model_workspace_bytes(len(tensors)))
    assert need == len(tensors) * 72 + (len(tensors) + 1) * 4
    ws = torch.empty(need if workspace_bytes is None else workspace_bytes, dtype=torch.uint8, device="cuda")
    N.check(N.lib().qd_huffman_decode_dequant_model(desc.ctypes.data, len(tensors), N.ptr(table), bucket or 0, s or 0, N.ptr(ws),
                                                    ws.numel(), N.stream_ptr()))
    desc[:] = 0                 # the host array may be reused as soon as the call returns


def _check(env, tensors, table, bucket, s):
    Q, N, codec = env
    ns = [t["n"] for t in tensors]
    arena, starts = _arena(ns)
    _decode_model(env, tensors, table, bucket, s, arena, starts)
    bits = arena.view(torch.int32)
    covered = torch.zeros(arena.numel(), dtype=torch.bool, device="cuda")
    for t, st in zip(tensors, starts):
        got = bits[st:st + t["n"]]
        assert torch.equal(got, _per_tensor(N, t, table, bucket, s).view(torch.int32)), (t["n"], st)
        assert torch.equal(got, t["ref"].view(torch.int32)), (t["n"], st)
        covered[st:st + t["n"]] = True
    assert torch.all(bits[~covered] == SENTINEL)


NS = [1, 10, 255, 1024, 1025, 1_000_003]


@pytest.mark.parametrize("bucket", [256, 1024, None])
@pytest.mark.parametrize("s", [2, 4, 16, 256])
def test_uniform_model_decode_matches_per_tensor_and_op(env, s, bucket):
    tensors, _, table = _model(env, NS + NS[::-1], bucket, s=s, seed=s)
    _check(env, tensors, table, bucket, s)


@pytest.mark.parametrize("bucket", [256, 1024, None])
def test_nonuniform_model_decode_with_points_per_tensor(env, bucket):
    """One model, tensors with 1, 3, 16, 33 and 256 points: a CTA loads its own tensor's unit table."""
    tensors, _, table = _model(env, NS + [7, 300, 4097, 65_537], bucket, point_counts=[1, 3, 16, 33, 256], seed=11)
    assert len({t["points"].numel() for t in tensors}) == 5
    _check(env, tensors, table, bucket, None)


def test_single_symbol_code_model(env):
    tensors, lengths, table = _model(env, NS, 256, s=16, constant=True)
    assert list(lengths.values()) == [0] and all(t["words"].numel() == 0 for t in tensors)
    _check(env, tensors, table, 256, 16)


def test_thousands_of_tensors_in_one_launch(env):
    Q, N, codec = env
    rng = np.random.default_rng(5)
    ns = [int(v) for v in rng.integers(1, 300, 3000)] + [1_000_003]
    tensors, _, table = _model(env, ns, 256, s=4, seed=5)
    arena, starts = _arena(ns)
    _decode_model(env, tensors, table, 256, 4, arena, starts, workspace_bytes=int(N.lib().qd_huffman_model_workspace_bytes(len(ns))))
    bits = arena.view(torch.int32)
    ref = torch.full_like(bits, SENTINEL)
    for t, st in zip(tensors, starts):
        ref[st:st + t["n"]] = t["ref"].view(torch.int32)
    assert torch.equal(bits, ref)
    for t, st in zip(tensors[::97] + tensors[-1:], starts[::97] + starts[-1:]):
        assert torch.equal(bits[st:st + t["n"]], _per_tensor(N, t, table, 256, 4).view(torch.int32))


def test_invalid_model_arguments_are_refused(env):
    Q, N, codec = env
    tensors, _, table = _model(env, [1000, 3000], 256, s=16)
    arena, starts = _arena([1000, 3000])
    with pytest.raises(RuntimeError, match="workspace"):
        _decode_model(env, tensors, table, 256, 16, arena, starts, workspace_bytes=int(N.lib().qd_huffman_model_workspace_bytes(2)) - 1)
    with pytest.raises(ValueError, match="levels"):
        _decode_model(env, tensors, table, 256, 1, arena, starts)
    bad = dict(tensors[1], n=0)
    with pytest.raises(ValueError, match="tensor 1"):
        _decode_model(env, [tensors[0], bad], table, 256, 16, arena, starts)
    with pytest.raises(ValueError, match="points"):                  # a non-uniform call needs points
        _decode_model(env, tensors, table, 256, None, arena, starts)
    assert torch.all(arena.view(torch.int32) == SENTINEL)             # nothing was launched


# ---------------------------------------------------------------------------------------------------- models
def _student():
    from quantized_distillation_b200.cnn_models import conv_forward_model as cfm
    return cfm.ConvolForwardNet(**cfm.smallerModelSpec, useBatchNorm=True, useAffineTransformInBatchNorm=True).cuda()


def _wrn():
    from quantized_distillation_b200.cnn_models.wide_resnet import Wide_ResNet
    return Wide_ResNet(depth=16, widen_factor=22, dropout_rate=0.3, num_classes=10).cuda()


@pytest.mark.parametrize("make,numBits", [(_student, 4), (_wrn, 2)], ids=["student_4bit", "wrn_16_22_2bit"])
def test_complete_model_round_trip_with_buffers(env, tmp_path, make, numBits):
    Q, N, codec = env
    torch.manual_seed(0)
    model = make()
    with torch.no_grad():
        for p in model.parameters():
            p.normal_(0, 0.05)
        model.train()
        for _ in range(3):                        # BatchNorm statistics away from their defaults
            model(torch.randn(16, 3, 32, 32, device="cuda"))
    bufs = codec._persistent_buffers(model)
    assert any(name.endswith("num_batches_tracked") for name, _ in bufs)
    assert all(int(b) == 3 for name, b in bufs if name.endswith("num_batches_tracked"))
    cm = codec.compress_model(model, numBits, bucket_size=256, quantize_first_and_last_layer=False, include_buffers=True)
    path = tmp_path / "model.qdh"
    size = codec.save_compressed(cm, path)
    assert int.from_bytes(path.read_bytes()[8:12], "little") == 2
    back = codec.load_compressed(path)
    sb = back.size_breakdown()
    assert sb == cm.size_breakdown() and sb["file_bytes"] == size
    assert sb["buffer_bytes"] == sum(b.numel() * b.element_size() for _, b in bufs) > 0

    torch.manual_seed(123)
    fresh = make()
    handles = list(fresh.parameters())
    codec.decompress_(back, fresh)                # parameters and buffers: nothing copied by hand
    assert all(a is b for a, b in zip(handles, fresh.parameters()))
    for (name, b), (_, r) in zip(bufs, codec._persistent_buffers(fresh)):
        assert b.dtype == r.dtype and torch.equal(b, r), name

    params = list(model.parameters())
    with torch.no_grad():                         # the fake-quantized original
        for p in params[1:-1]:
            p.copy_(Q.uniformQuantization(p.data.clone(), 2 ** numBits, bucket_size=256)[0].view_as(p))
    for p, r in zip(model.parameters(), fresh.parameters()):
        assert torch.equal(p.data.view(torch.int32), r.data.view(torch.int32))
    model.eval(), fresh.eval()
    x = torch.randn(8, 3, 32, 32, device="cuda")
    with torch.no_grad():
        assert torch.equal(model(x), fresh(x))

    # the same file straight to the device: one allocation, every section a view into it
    dev = codec.load_compressed(path, device="cuda")
    base = dev._data.untyped_storage().data_ptr()
    assert dev._data.is_cuda and all(x.untyped_storage().data_ptr() == base for t in dev.tensors
                                     for x in (t.words, t.chunk_offsets, t.alpha, t.beta, t.raw) if x is not None)
    assert all(b.untyped_storage().data_ptr() == base for _, b in dev.buffers)
    again = make()
    codec.decompress_(dev, again)
    again.eval()
    with torch.no_grad():
        assert torch.equal(again(x), fresh(x))


@pytest.mark.parametrize("where", ["cuda", "cpu"])
def test_decompress_matches_decompress_tensor(env, tmp_path, where):
    """Without buffers, decompress_ (one launch per device) writes the bits decompress_tensor gives for every tensor,
    also into host parameters (decoded into a temporary, then copied); points per tensor take the non-uniform path."""
    Q, N, codec = env
    torch.manual_seed(0)
    model = _student()
    with torch.no_grad():
        for p in model.parameters():
            p.normal_(0, 0.05)
    gen = torch.Generator().manual_seed(3)
    npar = len(list(model.parameters()))
    points = [torch.sort(torch.rand(int(k), generator=gen))[0].cuda() for k in np.resize([3, 16, 33, 256], npar)]
    cm = codec.compress_model(model, None, bucket_size=256, points=points)
    codec.save_compressed(cm, tmp_path / "m.qdh")
    assert int.from_bytes((tmp_path / "m.qdh").read_bytes()[8:12], "little") == 1
    back = codec.load_compressed(tmp_path / "m.qdh")
    assert back.buffers is None
    fresh = _student() if where == "cuda" else _student().cpu()
    before = [b.clone() for _, b in codec._persistent_buffers(fresh)]
    codec.decompress_(back, fresh)
    for k, p in enumerate(fresh.parameters()):
        want = codec.decompress_tensor(cm, k).cpu()
        assert torch.equal(p.data.cpu().view(-1).view(torch.int32), want.view(-1).view(torch.int32)), k
    assert all(torch.equal(a, b) for a, (_, b) in zip(before, codec._persistent_buffers(fresh)))   # buffers untouched
