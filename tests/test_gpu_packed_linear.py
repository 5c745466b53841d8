"""Fully-connected layers run from their packed codes: qd_packed_linear against the float64 oracle over every code
width, level / point count, bucket (straddling output rows, ragged, None), shape and batch size; its weights against
qd_unpack_dequant_* bit for bit; determinism across calls, batch sizes and streams; refusals at the C ABI and in the
module; PackedLinear on both sides of its crossover and in a CUDA graph; and attach_packed_linear_ on the student,
a non-uniform student and WRN-16-22 against unpack_."""
import threading

import numpy as np
import pytest
import torch

from oracle import packed_linear_oracle as P

pytestmark = pytest.mark.gpu

MAX = 64                                 # QD_PACKED_LINEAR_MAX_ROWS
MS = [1, 2, 3, 7, 8, 15, 16, 17, MAX - 1, MAX]
UNIFORM = [(bits, s, None) for bits in (1, 2, 4, 8) for s in (2, 3, 4, 16, 256) if s <= 1 << bits]
NONUNIFORM = [(bits, None, k) for bits in (1, 2, 4, 8) for k in (1, 3, 16, 256) if k <= 1 << bits]
SMALL_SHAPES = [(500, 1600), (10, 1408), (1, 1), (3, 5)]
BUCKETS = [256, 64, 1000, None]


@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from quantized_distillation_b200 import _native as N
    from quantized_distillation_b200 import codec
    assert N.PACKED_LINEAR_MAX_ROWS == MAX
    return N, codec


def _weights(N, out_f, in_f, bits, s, k, bucket, seed):
    """(packed, alpha, beta, points, q): random codes packed with qd_pack_indices, random scales, and q decoded by
    qd_unpack_dequant_*."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    n = out_f * in_f
    b = bucket or 0
    codes = torch.randint(0, s or k, (n,), generator=g, device="cuda", dtype=torch.int32).to(torch.uint8)
    packed = torch.empty((n * bits + 7) // 8, dtype=torch.uint8, device="cuda")
    N.check(N.lib().qd_pack_indices(N.ptr(codes), N.ptr(packed), n, bits, N.stream_ptr()))
    rows = N.geometry(n, b)[0]
    alpha = torch.rand(rows, generator=g, device="cuda") * 0.1 + 0.01
    beta = torch.randn(rows, generator=g, device="cuda") * 0.05
    pts = None if k is None else torch.sort(torch.rand(k, generator=g, device="cuda")).values
    q = torch.empty(n, device="cuda")
    if pts is None:
        N.check(N.lib().qd_unpack_dequant_uniform(N.ptr(packed), bits, N.ptr(alpha), N.ptr(beta), N.ptr(q), n, b, s, N.stream_ptr()))
    else:
        N.check(N.lib().qd_unpack_dequant_nonuniform(N.ptr(packed), bits, N.ptr(pts), k, N.ptr(alpha), N.ptr(beta), N.ptr(q), n, b,
                                                     N.stream_ptr()))
    return packed, alpha, beta, pts, q


def _call(N, x, out_f, packed, bits, alpha, beta, pts, s, bucket, bias, y=None, stream=None):
    m, in_f = x.shape
    y = torch.empty(m, out_f, device="cuda") if y is None else y
    rc = N.lib().qd_packed_linear(N.ptr(x), m, in_f, out_f, N.ptr(packed), bits, N.ptr(alpha), N.ptr(beta), N.ptr(pts),
                                  0 if pts is None else pts.numel(), s or 0, bucket or 0, N.ptr(bias), N.ptr(y),
                                  stream if stream is not None else N.stream_ptr())
    return rc, y


def _reference(x, q, bias, out_f, in_f):
    """float64 reference x @ q.T + b (on the GPU, from the decoded weights) and the oracle's tolerance, per element."""
    xd, wd = x.double(), q.view(out_f, in_f).double()
    ref = xd @ wd.T + (0 if bias is None else bias.double())
    mag = xd.abs() @ wd.abs().T
    return ref, in_f * 2.0 ** -23 * mag + 2.0 ** -23 * ref.abs()


def _within(y, ref, tol):
    err = (y.double() - ref).abs()
    assert torch.all(err <= tol), float((err - tol).max())


def _check_against_oracle(y, x, q, bias, out_f, in_f):
    _within(y, *_reference(x, q, bias, out_f, in_f))


def _sweep(N, out_f, in_f, bits, s, k, bucket, seed, ms=MS):
    packed, alpha, beta, pts, q = _weights(N, out_f, in_f, bits, s, k, bucket, seed)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    x = torch.randn(MAX, in_f, generator=g, device="cuda")
    bias = torch.randn(out_f, generator=g, device="cuda")
    for b in (None, bias):
        ref, tol = _reference(x, q, b, out_f, in_f)      # rows are independent: the first m rows serve batch m
        full = None
        for m in sorted(ms, reverse=True):
            rc, y = _call(N, x[:m], out_f, packed, bits, alpha, beta, pts, s, bucket, b)
            N.check(rc)
            _within(y, ref[:m], tol[:m])
            if full is None:
                full = y
            else:                        # the order of a row's sum does not depend on the batch size
                assert torch.equal(y.view(torch.int32), full[:m].view(torch.int32)), (m, out_f, in_f, bits, s, k, bucket)


@pytest.mark.parametrize("bucket", BUCKETS, ids=lambda b: f"bucket{b}")
@pytest.mark.parametrize("bits,s,k", UNIFORM + NONUNIFORM)
def test_sweep_small_shapes(env, bits, s, k, bucket):
    N, _ = env
    for i, (out_f, in_f) in enumerate(SMALL_SHAPES):
        _sweep(N, out_f, in_f, bits, s, k, bucket, seed=bits * 1000 + (s or 0) * 7 + (k or 0) * 13 + i)


@pytest.mark.parametrize("bucket", BUCKETS, ids=lambda b: f"bucket{b}")
@pytest.mark.parametrize("bits,s,k", UNIFORM + NONUNIFORM)
def test_sweep_alexnet_head(env, bits, s, k, bucket):
    """(4096, 9216): the x tile is chunked (K = 9216 floats exceed the tile at 4 and 8 rows per tile)."""
    N, _ = env
    _sweep(N, 4096, 9216, bits, s, k, bucket, seed=bits * 1000 + (s or 0) * 7 + (k or 0) * 13)


def test_oracle_restatement_agrees_on_a_small_layer(env):
    """The NumPy oracle itself, codes to float64 product, on one layer with buckets straddling rows."""
    N, _ = env
    out_f, in_f, bits, s, bucket = 7, 37, 2, 3, 16
    packed, alpha, beta, _, q = _weights(N, out_f, in_f, bits, s, None, bucket, seed=5)
    x = torch.randn(5, in_f, device="cuda")
    bias = torch.randn(out_f, device="cuda")
    rc, y = _call(N, x, out_f, packed, bits, alpha, beta, None, s, bucket, bias)
    N.check(rc)
    want_q = P.dequantize(P.unpack_codes(packed.cpu().numpy(), out_f * in_f, bits), alpha.cpu().numpy(), beta.cpu().numpy(), bucket, levels=s)
    assert np.array_equal(want_q.view(np.int32), q.cpu().numpy().view(np.int32))
    ref, mag = P.packed_linear(x.cpu().numpy(), packed.cpu().numpy(), bits, alpha.cpu().numpy(), beta.cpu().numpy(), out_f, in_f, bucket,
                               levels=s, bias=bias.cpu().numpy())
    assert np.all(np.abs(y.cpu().numpy().astype(np.float64) - ref) <= P.tolerance(ref, mag, in_f))


@pytest.mark.parametrize("bits,s,k", [(1, 2, None), (2, 3, None), (4, 16, None), (8, 256, None), (4, None, 5), (8, None, 256)])
@pytest.mark.parametrize("in_f,bucket", [(64, 256), (60, 7), (33, None), (64, 1000)])
def test_kernel_weights_are_the_unpacked_weights(env, bits, s, k, in_f, bucket):
    """x = identity rows: y[i, o] = q[o, i] exactly, whatever the bucket or alignment."""
    N, _ = env
    out_f = 45
    packed, alpha, beta, pts, q = _weights(N, out_f, in_f, bits, s, k, bucket, seed=in_f + bits)
    eye = torch.eye(in_f, device="cuda")
    for m0 in range(0, in_f, MAX):
        rc, y = _call(N, eye[m0:m0 + MAX].contiguous(), out_f, packed, bits, alpha, beta, pts, s, bucket, None)
        N.check(rc)
        want = q.view(out_f, in_f)[:, m0:m0 + MAX].T
        assert torch.equal(y.view(torch.int32), want.contiguous().view(torch.int32))


def test_unaligned_views(env):
    """packed at an odd byte, x rows not 16-byte aligned: the general loads give the same bits as aligned copies."""
    N, _ = env
    out_f, in_f, bits, s, bucket = 300, 1600, 4, 16, 256
    packed, alpha, beta, _, q = _weights(N, out_f, in_f, bits, s, None, bucket, seed=11)
    x = torch.randn(9, in_f + 1, device="cuda")
    xa = x[:, 1:].contiguous()
    ref = _call(N, xa, out_f, packed, bits, alpha, beta, None, s, bucket, None)[1]
    arena = torch.empty(packed.numel() + 1, dtype=torch.uint8, device="cuda")
    arena[1:] = packed
    xu = torch.empty(9 * in_f + 1, device="cuda")[1:].view(9, in_f)
    xu.copy_(xa)
    rc, y = _call(N, xu, out_f, arena[1:], bits, alpha, beta, None, s, bucket, None)
    N.check(rc)
    assert torch.equal(y.view(torch.int32), ref.view(torch.int32))


def test_repeated_calls_and_four_streams_give_identical_bits(env):
    N, _ = env
    out_f, in_f, bits, s, bucket = 4096, 9216, 2, 4, 256
    packed, alpha, beta, _, _ = _weights(N, out_f, in_f, bits, s, None, bucket, seed=3)
    x = torch.randn(16, in_f, device="cuda")
    bias = torch.randn(out_f, device="cuda")
    ref = _call(N, x, out_f, packed, bits, alpha, beta, None, s, bucket, bias)[1]
    for _ in range(3):
        assert torch.equal(_call(N, x, out_f, packed, bits, alpha, beta, None, s, bucket, bias)[1].view(torch.int32), ref.view(torch.int32))
    torch.cuda.synchronize()
    outs, errs = [torch.empty_like(ref) for _ in range(4)], []

    def work(i):
        try:
            st = torch.cuda.Stream()
            with torch.cuda.stream(st):
                for _ in range(5):
                    N.check(_call(N, x, out_f, packed, bits, alpha, beta, None, s, bucket, bias, y=outs[i], stream=st.cuda_stream)[0])
            st.synchronize()
        except Exception as e:           # surfaced in the main thread
            errs.append(e)
    threads = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errs, errs
    for o in outs:
        assert torch.equal(o.view(torch.int32), ref.view(torch.int32))


def test_c_abi_refusals(env):
    N, _ = env
    out_f, in_f, bits, s, bucket = 10, 64, 2, 4, 256
    packed, alpha, beta, _, _ = _weights(N, out_f, in_f, bits, s, None, bucket, seed=1)
    pts = torch.rand(5, device="cuda")
    x = torch.randn(MAX + 1, in_f, device="cuda")
    y = torch.empty(MAX + 1, out_f, device="cuda")
    L = N.lib()

    def rc(**kw):
        a = dict(x=N.ptr(x), m=4, K=in_f, O=out_f, packed=N.ptr(packed), bits=bits, alpha=N.ptr(alpha), beta=N.ptr(beta), points=None,
                 k=0, levels=s, bucket=bucket, bias=None, y=N.ptr(y))
        a.update(kw)
        return L.qd_packed_linear(*a.values(), N.stream_ptr())
    assert rc() == N.QD_OK
    assert rc(m=MAX) == N.QD_OK
    assert rc(m=MAX + 1) == N.QD_ERR_UNSUPPORTED
    assert "at most 64" in L.qd_last_error().decode()
    for bad in (dict(x=None), dict(packed=None), dict(alpha=None), dict(beta=None), dict(y=None), dict(m=0), dict(K=0), dict(O=-1),
                dict(bits=3), dict(levels=5),                     # 5 levels do not fit in 2-bit codes
                dict(levels=1), dict(levels=0, points=N.ptr(pts), k=5),   # 5 points do not fit either
                dict(levels=0, points=None, k=3), dict(levels=0, points=N.ptr(pts), k=0),
                dict(points=N.ptr(pts), k=4),                     # points given to a uniform call
                dict(bucket=-1), dict(y=N.ptr(x))):               # y overlapping x
        assert rc(**bad) == N.QD_ERR_INVALID_ARG, bad
        assert L.qd_last_error().decode()


# ------------------------------------------------------------------------------------------------ the module
def _layer(codec, N, out_f, in_f, bits=4, s=16, bucket=256, bias=True, seed=0):
    packed, alpha, beta, _, q = _weights(N, out_f, in_f, bits, s, None, bucket, seed)
    b = torch.randn(out_f, device="cuda") if bias else None
    e = codec.PackedEntry("w", (out_f, in_f), bits=bits, packed=packed, alpha=alpha, beta=beta)
    return codec.PackedLinear(e, "uniform", s, bucket, b), q.view(out_f, in_f), b


def test_module_paths(env):
    N, codec = env
    layer, w, b = _layer(codec, N, 500, 1600)
    cross = codec.PackedLinear.CROSSOVER_ROWS
    assert 1 <= cross <= MAX
    assert torch.equal(layer.decoded_weight().view(torch.int32), w.view(torch.int32))
    with torch.no_grad():
        for m in (1, cross, cross + 1, MAX, MAX + 1, 300):
            x = torch.randn(m, 1600, device="cuda")
            y = layer(x)
            if m > cross:                # decode + F.linear: what an unpack_-loaded nn.Linear computes
                assert torch.equal(y, torch.nn.functional.linear(x, w, b)), m
            else:
                _check_against_oracle(y, x, w.reshape(-1), b, 500, 1600)
        assert layer(torch.randn(0, 1600, device="cuda")).shape == (0, 500)


@pytest.mark.parametrize("lead", [(1, 3), (2, 3)], ids=["kernel", "decode"])
def test_module_takes_3d_and_non_contiguous_inputs(env, lead):
    """Both sides of the crossover: (1, 3, K) and 3 transposed rows run the kernel, (2, 3, K) and 6 rows decode."""
    N, codec = env
    layer, w, b = _layer(codec, N, 500, 1600)
    rows = lead[0] * lead[1]
    assert (rows <= codec.PackedLinear.CROSSOVER_ROWS) == (lead == (1, 3))
    with torch.no_grad():
        x3 = torch.randn(*lead, 1600, device="cuda")
        y3 = layer(x3)
        assert y3.shape == (*lead, 500)
        assert torch.equal(y3, layer(x3.reshape(rows, 1600)).view(*lead, 500))
        _check_against_oracle(y3.reshape(rows, 500), x3.reshape(rows, 1600), w.reshape(-1), b, 500, 1600)
        xt = torch.randn(1600, rows, device="cuda").T          # non-contiguous
        assert not xt.is_contiguous()
        assert torch.equal(layer(xt), layer(xt.contiguous()))


def test_module_refusals(env):
    N, codec = env
    layer, _, _ = _layer(codec, N, 10, 64)
    with torch.no_grad():
        with pytest.raises(ValueError):
            layer(torch.randn(3, 63, device="cuda"))
        with pytest.raises(ValueError):
            layer(torch.randn(3, 64, device="cuda", dtype=torch.float64))
        with pytest.raises(ValueError):
            layer(torch.randn(3, 64))
    with pytest.raises(RuntimeError):
        layer(torch.randn(3, 64, device="cuda", requires_grad=True))
    with torch.no_grad():
        layer(torch.randn(3, 64, device="cuda", requires_grad=True))          # no gradient needed: fine
    layer(torch.randn(3, 64, device="cuda"))                                     # grad mode, input without grad: fine
    cast = _layer(codec, N, 10, 64)[0].double()           # scales, points and bias must stay float32 for the kernel
    with torch.no_grad(), pytest.raises(RuntimeError, match="float32"):
        cast(torch.randn(3, 64, device="cuda"))
    assert not isinstance(layer.decoded_weight, torch.nn.Parameter)


@pytest.mark.parametrize("rows", [2, 8], ids=["kernel", "decode"])
def test_cuda_graph_replay(env, rows):
    N, codec = env
    layer, _, _ = _layer(codec, N, 500, 1600)
    assert (rows <= codec.PackedLinear.CROSSOVER_ROWS) == (rows == 2)
    x = torch.randn(rows, 1600, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.no_grad(), torch.cuda.stream(side):
        ref = layer(x).clone()                                               # warm up on the capture stream
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.no_grad(), torch.cuda.graph(g):
        out = layer(x)
    for _ in range(3):
        out.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int32), ref.view(torch.int32))


# ------------------------------------------------------------------------------------------------ whole models
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
        for _ in range(3):
            model(torch.randn(16, 3, 32, 32, device="cuda"))
    return model


def _pack(codec, model, kind):
    if kind == "uniform":
        return codec.pack_model(model, 4, 256, quantize_first_and_last_layer=False, include_buffers=True)
    n_q = len(list(model.parameters())) - 2
    pts = [np.sort(np.random.default_rng(i).random(3 + i % 14)).astype(np.float32) for i in range(n_q)]
    return codec.pack_model(model, points=pts, bucket_size=256, quantize_first_and_last_layer=False, include_buffers=True)


@pytest.mark.parametrize("make,kind,linear", [(_student, "uniform", "linear_layers.0"), (_student, "nonuniform", "linear_layers.0"),
                                              (_wrn, "uniform", "linear")], ids=["student", "student_nonuniform", "wrn_16_22"])
def test_attach_whole_model(env, make, kind, linear):
    N, codec = env
    pm = _pack(codec, _trained(make), kind)
    torch.manual_seed(1)
    ref = make()
    codec.unpack_(pm, ref)
    torch.manual_seed(2)
    fresh = make()
    lin = fresh.get_submodule(linear)
    entry = pm.tensors[[n for n, _ in fresh.named_parameters()].index(linear + ".weight")]
    del lin
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    names = codec.attach_packed_linear_(pm, fresh)
    torch.cuda.synchronize()
    after = torch.cuda.memory_allocated()
    assert names == [linear]
    assert isinstance(fresh.get_submodule(linear), codec.PackedLinear)
    if make is _student:
        assert type(fresh.out_layer) is torch.nn.Linear
    w_bytes = entry.numel * 4
    kept = entry.packed.numel() + (entry.alpha.numel() + entry.beta.numel()) * 4
    assert before - after >= w_bytes - kept, (before, after, w_bytes, kept)
    got = dict(fresh.named_parameters())
    got.update(dict(fresh.named_buffers()))
    for name, t in list(ref.named_parameters()) + list(ref.named_buffers()):
        if name == linear + ".weight":
            assert name not in got
            continue
        assert torch.equal(got[name].view(-1).view(torch.int8), t.data.view(-1).view(torch.int8)), name
    assert torch.equal(fresh.get_submodule(linear).decoded_weight().view(torch.int32), ref.get_submodule(linear).weight.data.view(torch.int32))
    ref.eval(), fresh.eval()
    gen = torch.Generator(device="cuda").manual_seed(3)
    with torch.no_grad():
        # a batch of 2 runs the kernel: its rows agree within the kernel's tolerance, later layers amplify that by at
        # most a few ulps of the logits
        x = torch.randn(2, 3, 32, 32, device="cuda", generator=gen)
        want, out = ref(x), fresh(x)
        assert out.shape == want.shape
        assert torch.allclose(out, want, rtol=1e-4, atol=1e-4 * float(want.abs().max())), float((out - want).abs().max())
        # a batch of 8 decodes the weight and calls F.linear: the unpack_-loaded model's logits, bit for bit
        x = torch.randn(8, 3, 32, 32, device="cuda", generator=gen)
        assert torch.equal(fresh(x), ref(x))


class _Tied(torch.nn.Module):
    """An embedding whose matrix a generator Linear shares (NMT share_decoder_embeddings), one Linear registered under
    two parents, and two Linear layers of their own."""

    def __init__(self):
        super().__init__()
        self.emb = torch.nn.Embedding(50, 32)
        self.lin1 = torch.nn.Linear(32, 64)
        self.lin2 = torch.nn.Linear(64, 32)
        self.shared = torch.nn.Linear(32, 32)
        self.block = torch.nn.Sequential(self.shared)
        self.gen = torch.nn.Linear(32, 50)
        self.gen.weight = self.emb.weight

    def forward(self, tokens):
        h = self.lin2(torch.relu(self.lin1(self.emb(tokens))))
        return self.gen(self.block(self.shared(h)))


def test_attach_leaves_shared_weights_to_unpack(env):
    N, codec = env
    torch.manual_seed(0)
    pm = codec.pack_model(_Tied().cuda(), 4, 64, quantize_first_and_last_layer=True)
    torch.manual_seed(1)
    ref = _Tied().cuda()
    codec.unpack_(pm, ref)
    torch.manual_seed(2)
    fresh = _Tied().cuda()
    assert codec.attach_packed_linear_(pm, fresh) == ["lin1", "lin2"]
    assert type(fresh.gen) is torch.nn.Linear and fresh.gen.weight is fresh.emb.weight
    assert type(fresh.shared) is torch.nn.Linear and fresh.block[0] is fresh.shared
    got = dict(fresh.named_parameters())
    got.update(dict(fresh.named_buffers()))
    for name, t in ref.named_parameters():
        if name in ("lin1.weight", "lin2.weight"):
            continue
        assert torch.equal(got[name].view(torch.int32), t.data.view(torch.int32)), name
    tokens = torch.randint(0, 50, (2,), device="cuda")
    with torch.no_grad():
        want, out = ref(tokens), fresh(tokens)
    assert torch.allclose(out, want, rtol=1e-4, atol=1e-4 * float(want.abs().max())), float((out - want).abs().max())


def test_attach_refuses_a_mismatched_model_before_writing(env):
    N, codec = env
    pm = _pack(codec, _trained(_student), "uniform")
    net = _student()
    snap = {k: v.clone() for k, v in net.state_dict().items()}
    pm.tensors[3] = codec.PackedEntry(pm.tensors[3].name, (1, 2, 3), raw=torch.zeros(6, device="cuda"))
    with pytest.raises(ValueError, match="shape"):
        codec.attach_packed_linear_(pm, net)
    assert type(net.linear_layers[0]) is torch.nn.Linear
    for k, v in net.state_dict().items():
        assert torch.equal(v, snap[k]), k
