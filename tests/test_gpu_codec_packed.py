"""Fixed-width storage on the GPU: the fused quantize-and-pack encoders (qd_uniform_fwd_packed /
qd_nonuniform_fwd_packed) against the level op followed by qd_pack_indices, byte for byte; the whole-model unpack
(qd_unpack_dequant_model) against the per-tensor unpack and the fake-quantization ops, bit for bit; and complete
models through pack_model -> save_packed -> load_packed -> unpack_ into a network built with another seed."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FC0DEAD           # a NaN payload no decode produces
BYTE_SENTINEL = 0xA5


@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import quantized_distillation_b200.quantization as Q
    from quantized_distillation_b200 import _native as N
    from quantized_distillation_b200 import codec
    return Q, N, codec


def _scales(N, n, b):
    rows = N.geometry(n, b)[0]
    return torch.empty(rows, device="cuda"), torch.empty(rows, device="cuda")


def _two_step(N, x, bits, b, s=None, pts=None, rule=0):
    """(packed, alpha, beta, q) of the level op (uint8 levels) followed by qd_pack_indices; q is the op's own
    fake-quantized output."""
    n = x.numel()
    alpha, beta = _scales(N, n, b)
    idx = torch.empty(n, dtype=torch.uint8, device="cuda")
    q = torch.empty(n, device="cuda")
    ws = N.workspace(n, b, x.device)
    if pts is None:
        N.check(N.lib().qd_uniform_fwd(N.ptr(x), N.ptr(q), N.ptr(idx), N.ptr(alpha), N.ptr(beta), None, None, n, b, s, None, 0.0, 0, 0, 0,
                                       N.ptr(ws), ws.numel(), N.stream_ptr()))
    else:
        N.check(N.lib().qd_nonuniform_fwd(N.ptr(x), N.ptr(pts), pts.numel(), rule, N.ptr(q), N.ptr(idx), None, N.ptr(alpha), N.ptr(beta),
                                          n, b, None, 0.0, N.ptr(ws), ws.numel(), N.stream_ptr()))
    packed = torch.empty((n * bits + 7) // 8, dtype=torch.uint8, device="cuda")
    N.check(N.lib().qd_pack_indices(N.ptr(idx), N.ptr(packed), n, bits, N.stream_ptr()))
    return packed, alpha, beta, q


def _fused(N, x, bits, b, s=None, pts=None, rule=0, offset=0):
    """(packed, alpha, beta, arena) of the fused encoder; packed starts `offset` bytes into an arena of sentinel bytes
    that extends 16 bytes past its end."""
    n = x.numel()
    nbytes = (n * bits + 7) // 8
    arena = torch.full((offset + nbytes + 16,), BYTE_SENTINEL, dtype=torch.uint8, device="cuda")
    packed = arena[offset:offset + nbytes]
    alpha, beta = _scales(N, n, b)
    ws = torch.empty(int(N.lib().qd_packed_workspace_bytes(n, b)), dtype=torch.uint8, device="cuda")
    if pts is None:
        N.check(N.lib().qd_uniform_fwd_packed(N.ptr(x), N.ptr(packed), bits, N.ptr(alpha), N.ptr(beta), n, b, s, N.ptr(ws), ws.numel(),
                                              N.stream_ptr()))
    else:
        N.check(N.lib().qd_nonuniform_fwd_packed(N.ptr(x), N.ptr(pts), pts.numel(), rule, N.ptr(packed), bits, N.ptr(alpha), N.ptr(beta),
                                                 n, b, N.ptr(ws), ws.numel(), N.stream_ptr()))
    return packed, alpha, beta, arena


def _unpack(N, packed, bits, alpha, beta, n, b, s=None, pts=None):
    q = torch.empty(n, device="cuda")
    if pts is None:
        N.check(N.lib().qd_unpack_dequant_uniform(N.ptr(packed), bits, N.ptr(alpha), N.ptr(beta), N.ptr(q), n, b, s, N.stream_ptr()))
    else:
        N.check(N.lib().qd_unpack_dequant_nonuniform(N.ptr(packed), bits, N.ptr(pts), pts.numel(), N.ptr(alpha), N.ptr(beta), N.ptr(q),
                                                     n, b, N.stream_ptr()))
    return q


def _check_encoder(N, x, bits, b, s=None, pts=None, rule=0, offset=0):
    n = x.numel()
    want = _two_step(N, x, bits, b, s, pts, rule)
    packed, alpha, beta, arena = _fused(N, x, bits, b, s, pts, rule, offset)
    case = (n, bits, b, s, None if pts is None else pts.numel(), rule, offset)
    assert torch.equal(packed, want[0]), case
    assert torch.equal(alpha.view(torch.int32), want[1].view(torch.int32)), case
    assert torch.equal(beta.view(torch.int32), want[2].view(torch.int32)), case
    assert torch.all(arena[:offset] == BYTE_SENTINEL) and torch.all(arena[offset + packed.numel():] == BYTE_SENTINEL), case
    q = _unpack(N, packed, bits, alpha, beta, n, b, s, pts)
    assert torch.equal(q.view(torch.int32), want[3].view(torch.int32)), case


# (bits, s) with s <= 2^bits
UNIFORM_CASES = [(bits, s) for bits in (1, 2, 4, 8) for s in (2, 3, 4, 16, 256) if s <= 1 << bits]
NS = [1, 255, 256, 257, 1_000_003]


@pytest.mark.parametrize("bucket", [256, 512, 1024, 100, None])
@pytest.mark.parametrize("bits,s", UNIFORM_CASES)
def test_uniform_packed_encoder_matches_levels_then_pack(env, bits, s, bucket):
    Q, N, codec = env
    g = torch.Generator(device="cuda").manual_seed(bits * 1000 + s)
    for n in NS:
        x = torch.randn(n, generator=g, device="cuda") * 0.05
        _check_encoder(N, x, bits, bucket or 0, s=s)


@pytest.mark.parametrize("bits,s", [(2, 4), (4, 16), (1, 2), (8, 256)])
def test_uniform_packed_encoder_at_2_26(env, bits, s):
    Q, N, codec = env
    x = torch.randn(1 << 26, generator=torch.Generator(device="cuda").manual_seed(7), device="cuda")
    _check_encoder(N, x, bits, 256, s=s)


@pytest.mark.parametrize("bits,s", [(1, 2), (2, 3), (4, 16), (8, 256)])
def test_rows_off_byte_boundaries_and_unaligned_views(env, bits, s):
    """Buckets whose packed rows start inside a byte (4, 12, 100 and 260 at one bit; 6 and 10 at 2 / 4 bits), an
    input view 4 bytes past an aligned start (the scalar lane layout) and packed streams at odd addresses."""
    Q, N, codec = env
    g = torch.Generator(device="cuda").manual_seed(bits + s)
    base = torch.randn(70_001, generator=g, device="cuda")
    for b in (4, 6, 10, 12, 100, 260, 256):
        for x in (base[:70_000], base[1:], base[3:1003]):
            for offset in (0, 1, 3, 8):
                _check_encoder(N, x, bits, b, s=s, offset=offset)


@pytest.mark.parametrize("rule", [0, 1], ids=["nearest", "midpoint"])
@pytest.mark.parametrize("K", [1, 3, 4, 16, 33, 256])
def test_nonuniform_packed_encoder_matches_levels_then_pack(env, K, rule):
    Q, N, codec = env
    from quantized_distillation_b200.codec import bits_for
    g = torch.Generator(device="cuda").manual_seed(K * 10 + rule)
    pts = torch.sort(torch.rand(K, generator=g, device="cuda"))[0]
    if K >= 4:
        pts[1] = pts[2]                              # duplicate points
    for bits in (b for b in (1, 2, 4, 8) if b >= bits_for(K)):
        for bucket in (256, 1024, 100, None):
            for n in NS:
                x = torch.randn(n, generator=g, device="cuda") * 0.05
                _check_encoder(N, x, bits, bucket or 0, pts=pts, rule=rule)
        _check_encoder(N, torch.randn(10_001, generator=g, device="cuda")[1:], bits, 256, pts=pts, rule=rule, offset=1)


def test_encoder_refuses_bad_widths_and_workspace(env):
    Q, N, codec = env
    x = torch.randn(1000, device="cuda")
    alpha, beta = _scales(N, 1000, 256)
    packed = torch.empty(1000, dtype=torch.uint8, device="cuda")
    ws = torch.empty(int(N.lib().qd_packed_workspace_bytes(1000, 256)), dtype=torch.uint8, device="cuda")
    lib, sp = N.lib(), N.stream_ptr()
    for bits, s in ((3, 4), (1, 3), (2, 5), (4, 17), (8, 257), (0, 2)):
        with pytest.raises(ValueError):
            N.check(lib.qd_uniform_fwd_packed(N.ptr(x), N.ptr(packed), bits, N.ptr(alpha), N.ptr(beta), 1000, 256, s, N.ptr(ws), ws.numel(), sp))
    pts = torch.linspace(0, 1, 5, device="cuda")
    with pytest.raises(ValueError, match="num_points"):
        N.check(lib.qd_nonuniform_fwd_packed(N.ptr(x), N.ptr(pts), 5, 0, N.ptr(packed), 2, N.ptr(alpha), N.ptr(beta), 1000, 256, N.ptr(ws),
                                             ws.numel(), sp))
    with pytest.raises(RuntimeError, match="workspace"):
        N.check(lib.qd_uniform_fwd_packed(N.ptr(x), N.ptr(packed), 4, N.ptr(alpha), N.ptr(beta), 1000, 256, 16, N.ptr(ws), ws.numel() - 1, sp))


# ---------------------------------------------------------------------------------------------- whole-model unpack
def _model_tensors(env, ns, bucket, s=None, point_counts=None, seed=0):
    """[dict(packed, alpha, beta, points, bits, n, ref)] with a width per tensor: uniform tensors cycle through every
    width that holds s, non-uniform ones use bits_for(K); ref is the fake-quantized tensor from the public op."""
    Q, N, codec = env
    g = torch.Generator(device="cuda").manual_seed(seed)
    widths = [b for b in (1, 2, 4, 8) if s is None or s <= 1 << b]
    out = []
    for i, n in enumerate(ns):
        x = torch.randn(n, generator=g, device="cuda") * 0.05
        pts = None
        if point_counts is not None:
            pts = torch.sort(torch.rand(point_counts[i % len(point_counts)], generator=g, device="cuda"))[0]
            bits = codec.bits_for(pts.numel())
            ref = Q.nonUniformQuantization(x.clone(), pts, bucket_size=bucket)[0].reshape(-1)
        else:
            bits = widths[i % len(widths)]
            ref = Q.uniformQuantization(x.clone(), s, bucket_size=bucket)[0].reshape(-1)
        packed, alpha, beta, _ = _fused(N, x, bits, bucket or 0, s=s, pts=pts)
        out.append(dict(packed=packed, alpha=alpha, beta=beta, points=pts, bits=bits, n=n, ref=ref))
    return out


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


def _decode_model(env, tensors, bucket, s, arena, starts, workspace_bytes=None):
    Q, N, codec = env
    desc = np.zeros(len(tensors), codec._PACKED_TENSOR)
    for i, (t, st) in enumerate(zip(tensors, starts)):
        desc[i] = (N.ptr(t["packed"]), N.ptr(t["alpha"]), N.ptr(t["beta"]), 0 if t["points"] is None else N.ptr(t["points"]),
                   arena[st:].data_ptr(), t["n"], t["bits"], 0 if t["points"] is None else t["points"].numel())
    need = int(N.lib().qd_unpack_model_workspace_bytes(len(tensors)))
    assert need == len(tensors) * 56 + (len(tensors) + 1) * 4
    ws = torch.empty(need if workspace_bytes is None else workspace_bytes, dtype=torch.uint8, device="cuda")
    N.check(N.lib().qd_unpack_dequant_model(desc.ctypes.data, len(tensors), bucket or 0, s or 0, N.ptr(ws), ws.numel(), N.stream_ptr()))
    desc[:] = 0                 # the host array may be reused as soon as the call returns


def _check_model(env, tensors, bucket, s):
    Q, N, codec = env
    arena, starts = _arena([t["n"] for t in tensors])
    _decode_model(env, tensors, bucket, s, arena, starts)
    bits = arena.view(torch.int32)
    covered = torch.zeros(arena.numel(), dtype=torch.bool, device="cuda")
    for t, st in zip(tensors, starts):
        got = bits[st:st + t["n"]]
        per = _unpack(N, t["packed"], t["bits"], t["alpha"], t["beta"], t["n"], bucket or 0, s, t["points"])
        assert torch.equal(got, per.view(torch.int32)), (t["n"], t["bits"], st)
        assert torch.equal(got, t["ref"].view(torch.int32)), (t["n"], t["bits"], st)
        covered[st:st + t["n"]] = True
    assert torch.all(bits[~covered] == SENTINEL)


MODEL_NS = [1, 10, 255, 1024, 1025, 4099, 1_000_003]


@pytest.mark.parametrize("bucket", [256, 1024, 100, None])
@pytest.mark.parametrize("s", [2, 4, 16, 256])
def test_uniform_model_unpack_with_mixed_widths(env, s, bucket):
    tensors = _model_tensors(env, MODEL_NS + MODEL_NS[::-1], bucket, s=s, seed=s)
    _check_model(env, tensors, bucket, s)


@pytest.mark.parametrize("bucket", [256, 1024, None])
def test_nonuniform_model_unpack_with_points_per_tensor(env, bucket):
    tensors = _model_tensors(env, MODEL_NS + [7, 300, 65_537], bucket, point_counts=[1, 3, 16, 33, 256, 4, 9], seed=11)
    assert {t["bits"] for t in tensors} == {1, 2, 4, 8}
    _check_model(env, tensors, bucket, None)


def test_thousands_of_tensors_in_one_launch(env):
    Q, N, codec = env
    rng = np.random.default_rng(5)
    ns = [1] * 50 + [int(v) for v in rng.integers(1, 300, 2950)] + [1_000_003]
    tensors = _model_tensors(env, ns, 256, s=4, seed=5)
    arena, starts = _arena(ns)
    _decode_model(env, tensors, 256, 4, arena, starts)
    bits = arena.view(torch.int32)
    ref = torch.full_like(bits, SENTINEL)
    for t, st in zip(tensors, starts):
        ref[st:st + t["n"]] = t["ref"].view(torch.int32)
    assert torch.equal(bits, ref)


def test_invalid_model_arguments_are_refused(env):
    Q, N, codec = env
    tensors = _model_tensors(env, [1000, 3000], 256, s=16)
    arena, starts = _arena([1000, 3000])
    with pytest.raises(RuntimeError, match="workspace"):
        _decode_model(env, tensors, 256, 16, arena, starts, workspace_bytes=int(N.lib().qd_unpack_model_workspace_bytes(2)) - 1)
    with pytest.raises(ValueError, match="levels"):
        _decode_model(env, tensors, 256, 1, arena, starts)
    with pytest.raises(ValueError, match="tensor 1"):
        _decode_model(env, [tensors[0], dict(tensors[1], n=0)], 256, 16, arena, starts)
    with pytest.raises(ValueError, match="tensor 0"):                # 16 levels in 2-bit codes
        _decode_model(env, [dict(tensors[0], bits=2), tensors[1]], 256, 16, arena, starts)
    with pytest.raises(ValueError, match="tensor 1"):
        _decode_model(env, [tensors[0], dict(tensors[1], bits=3)], 256, 16, arena, starts)
    with pytest.raises(ValueError, match="points"):                  # a non-uniform call needs points
        _decode_model(env, tensors, 256, None, arena, starts)
    assert torch.all(arena.view(torch.int32) == SENTINEL)             # nothing was launched


# ---------------------------------------------------------------------------------------------------- models
def _student():
    from quantized_distillation_b200.cnn_models import conv_forward_model as cfm
    return cfm.ConvolForwardNet(**cfm.smallerModelSpec, useBatchNorm=True, useAffineTransformInBatchNorm=True).cuda()


def _wrn():
    from quantized_distillation_b200.cnn_models.wide_resnet import Wide_ResNet
    return Wide_ResNet(depth=16, widen_factor=22, dropout_rate=0.3, num_classes=10).cuda()


def _trained(make):
    torch.manual_seed(0)
    model = make()
    with torch.no_grad():
        for p in model.parameters():
            p.normal_(0, 0.05)
        model.train()
        for _ in range(3):                        # BatchNorm statistics away from their defaults
            model(torch.randn(16, 3, 32, 32, device="cuda"))
    return model


@pytest.mark.parametrize("make,numBits", [(_student, 4), (_wrn, 2)], ids=["student_4bit", "wrn_16_22_2bit"])
def test_complete_model_round_trip_with_buffers(env, tmp_path, make, numBits):
    Q, N, codec = env
    model = _trained(make)
    bufs = codec._persistent_buffers(model)
    pm = codec.pack_model(model, numBits, bucket_size=256, quantize_first_and_last_layer=False, include_buffers=True)
    path = tmp_path / "model.qdp"
    size = codec.save_packed(pm, path)
    assert path.read_bytes()[:8] == codec.PACKED_MAGIC
    back = codec.load_packed(path)
    sb = back.size_breakdown()
    assert sb == pm.size_breakdown() and sb["file_bytes"] == size
    q = [p for p in model.parameters()][1:-1]
    assert sb["code_bytes"] == sum((p.numel() * codec.bits_for(2 ** numBits) + 7) // 8 for p in q)

    torch.manual_seed(123)
    fresh = make()
    handles = list(fresh.parameters())
    codec.unpack_(back, fresh)
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
    dev = codec.load_packed(path, device="cuda")
    base = dev._data.untyped_storage().data_ptr()
    assert dev._data.is_cuda and all(x.untyped_storage().data_ptr() == base for t in dev.tensors
                                     for x in (t.packed, t.alpha, t.beta, t.raw) if x is not None)
    assert all(b.untyped_storage().data_ptr() == base for _, b in dev.buffers)
    again = make()
    codec.unpack_(dev, again)
    again.eval()
    with torch.no_grad():
        assert torch.equal(again(x), fresh(x))


@pytest.mark.parametrize("where", ["cuda", "cpu"])
def test_differentiable_quantization_model_with_point_counts_per_tensor(env, tmp_path, where):
    """A different number of points per tensor (3, 4, 9, 37, 2, 256, ...): each tensor gets codes of bits_for(K_t)
    bits, and unpack_ gives back nonUniformQuantization of every tensor with its own points, also into host
    parameters (decoded into a temporary, then copied)."""
    Q, N, codec = env
    model = _trained(_student)
    gen = torch.Generator().manual_seed(3)
    params = list(model.parameters())
    counts = np.resize([3, 4, 9, 37, 2, 256, 1], len(params))
    points = [torch.sort(torch.rand(int(k), generator=gen))[0].cuda() for k in counts]
    pm = codec.pack_model(model, None, bucket_size=256, points=points, rule="midpoint")
    assert [t.bits for t in pm.tensors] == [codec.bits_for(int(k)) for k in counts]
    codec.save_packed(pm, tmp_path / "m.qdp")
    back = codec.load_packed(tmp_path / "m.qdp")
    assert back.buffers is None
    fresh = _student() if where == "cuda" else _student().cpu()
    codec.unpack_(back, fresh)
    for k, (p, r) in enumerate(zip(params, fresh.parameters())):
        want = _nonuniform_ref(N, p.data.view(-1), points[k], 256)    # the midpoint-rule op on the original tensor
        assert torch.equal(r.data.cpu().view(-1).view(torch.int32), want.cpu().view(torch.int32)), k


def _nonuniform_ref(N, x, pts, b):
    x = x.contiguous()
    n = x.numel()
    q = torch.empty(n, device="cuda")
    ws = N.workspace(n, b, x.device)
    N.check(N.lib().qd_nonuniform_fwd(N.ptr(x), N.ptr(pts), pts.numel(), N.RULE_MIDPOINT, N.ptr(q), None, None, None, None, n, b, None, 0.0,
                                      N.ptr(ws), ws.numel(), N.stream_ptr()))
    return q
