"""Convolution layers run from their packed codes: qd_packed_conv2d against the float64 oracle bound over every code
width, level / point count and bucket (straddling output channels, ragged, None), the student's and WRN's layer shapes,
edge shapes and batch sizes crossing every tile edge; its weights against qd_unpack_dequant_* bit for bit; determinism
across batches, calls and streams; refusals at the C ABI and in the module; PackedConv2d on both sides of its crossover
and in a CUDA graph; attach_packed_ on the student, a non-uniform student, a small WRN and WRN-16-22 against unpack_;
and the layers attach_packed_ must leave to unpack_."""
import gc
import threading

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import packed_conv_oracle as PC

pytestmark = pytest.mark.gpu

UNIFORM = [(bits, s, None) for bits in (1, 2, 4, 8) for s in (2, 3, 4, 16, 256) if s <= 1 << bits]
NONUNIFORM = [(bits, None, k) for bits in (1, 2, 4, 8) for k in (1, 3, 16, 256) if k <= 1 << bits]
BUCKETS = [256, 64, 1000, None]
# (C, O, H, W, kh, kw, stride, padding): edge shapes.  The tile is 64 positions x 64 channels x 16 taps.
EDGE_SHAPES = [
    (3, 5, 7, 7, 3, 3, (1, 1), (1, 1)),
    (1, 1, 1, 1, 1, 1, (1, 1), (0, 0)),            # C = O = 1 on a 1x1 input
    (2, 70, 9, 11, 3, 5, (2, 1), (0, 2)),          # kernel (3, 5), stride (2, 1), padding (0, 2); O crosses a tile
    (16, 65, 9, 9, 1, 1, (2, 2), (0, 0)),          # 1x1 at stride 2, K = 16: exactly one slab
    (1, 3, 2, 3, 5, 5, (1, 1), (2, 2)),            # kernel wider than the input: most taps are padding
]
EDGE_BATCHES = [1, 2, 5, 13]                       # 25, 45, 125, 325 ... positions: partial and several M tiles
# (name, C, O, H, W, k, stride, padding) of the layers the models run
MODEL_SHAPES = [
    ("student0", 3, 75, 32, 32, 5, 1, 2), ("student1", 75, 50, 32, 32, 5, 1, 2), ("student2", 50, 50, 16, 16, 5, 1, 2),
    ("student3", 50, 25, 16, 16, 5, 1, 2),
    ("wrn_stem", 3, 16, 32, 32, 3, 1, 1), ("wrn_16_352", 16, 352, 32, 32, 3, 1, 1), ("wrn_3x3_s1", 352, 352, 32, 32, 3, 1, 1),
    ("wrn_3x3_s2", 704, 704, 32, 32, 3, 2, 1), ("wrn_1x1_s1", 16, 352, 32, 32, 1, 1, 0), ("wrn_1x1_s2", 704, 1408, 16, 16, 1, 2, 0),
]


@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from quantized_distillation_b200 import _native as N
    from quantized_distillation_b200 import codec
    return N, codec


@pytest.fixture
def deterministic_cudnn():
    saved = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    yield
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = saved


@pytest.fixture
def no_tf32():
    saved = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = saved


def _weights(N, shape, bits, s, k, bucket, seed):
    """(packed, alpha, beta, points, q): random codes packed with qd_pack_indices, random scales, and q [O, C, kh, kw]
    decoded by qd_unpack_dequant_*."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    n = int(np.prod(shape))
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
    return packed, alpha, beta, pts, q.view(shape)


def _out_size(h, w, kh, kw, stride, padding):
    return (h + 2 * padding[0] - kh) // stride[0] + 1, (w + 2 * padding[1] - kw) // stride[1] + 1


def _call(N, x, shape, stride, padding, packed, bits, alpha, beta, pts, s, bucket, bias, y=None, stream=None):
    n, c, h, w = x.shape
    o, _, kh, kw = shape
    ho, wo = _out_size(h, w, kh, kw, stride, padding)
    y = torch.empty(n, o, ho, wo, device="cuda") if y is None else y
    rc = N.lib().qd_packed_conv2d(N.ptr(x), n, c, h, w, o, kh, kw, stride[0], stride[1], padding[0], padding[1], N.ptr(packed), bits,
                                  N.ptr(alpha), N.ptr(beta), N.ptr(pts), 0 if pts is None else pts.numel(), s or 0, bucket or 0,
                                  N.ptr(bias), N.ptr(y), stream if stream is not None else N.stream_ptr())
    return rc, y


def _reference(x, q, bias, stride, padding):
    """float64 convolution of the decoded weights (on the GPU) and the oracle's tolerance per output:
    K * 2^-23 * sum |x q| + 2^-23 * |y| (oracle/packed_linear_oracle.tolerance)."""
    xd, wd = x.double(), q.double()
    ref = F.conv2d(xd, wd, None if bias is None else bias.double(), stride, padding)
    mag = F.conv2d(xd.abs(), wd.abs(), None, stride, padding)
    K = q[0].numel()
    return ref, K * 2.0 ** -23 * mag + 2.0 ** -23 * ref.abs()


def _within(y, ref, tol):
    err = (y.double() - ref).abs()
    assert torch.all(err <= tol), float((err - tol).max())


def _sweep(N, geom, bits, s, k, bucket, seed, batches):
    c, o, h, w, kh, kw, stride, padding = geom
    shape = (o, c, kh, kw)
    packed, alpha, beta, pts, q = _weights(N, shape, bits, s, k, bucket, seed)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    x = torch.randn(max(batches), c, h, w, generator=g, device="cuda")
    bias = torch.randn(o, generator=g, device="cuda")
    for b in (None, bias):
        ref, tol = _reference(x, q, b, stride, padding)        # images are independent: the first n serve batch n
        full = None
        for n in sorted(batches, reverse=True):
            rc, y = _call(N, x[:n], shape, stride, padding, packed, bits, alpha, beta, pts, s, bucket, b)
            N.check(rc)
            _within(y, ref[:n], tol[:n])
            if full is None:
                full = y
            else:                        # the order of an output's sum does not depend on the batch size
                assert torch.equal(y.view(torch.int32), full[:n].view(torch.int32)), (n, geom, bits, s, k, bucket)


@pytest.mark.parametrize("bucket", BUCKETS, ids=lambda b: f"bucket{b}")
@pytest.mark.parametrize("bits,s,k", UNIFORM + NONUNIFORM)
def test_sweep_widths_on_edge_shapes(env, bits, s, k, bucket):
    N, _ = env
    for i, geom in enumerate(EDGE_SHAPES):
        _sweep(N, geom, bits, s, k, bucket, seed=bits * 1000 + (s or 0) * 7 + (k or 0) * 13 + i, batches=EDGE_BATCHES)


@pytest.mark.parametrize("bits,s,k", [(2, 4, None), (4, 16, None), (8, 256, None), (4, None, 11)])
@pytest.mark.parametrize("name,c,o,h,w,ks,st,pd", MODEL_SHAPES, ids=[m[0] for m in MODEL_SHAPES])
def test_model_layer_shapes(env, name, c, o, h, w, ks, st, pd, bits, s, k):
    """The student's four convolutions and WRN's: the 3->16 stem (left float32 by quantize_first_and_last_layer=False,
    tested as a layer), the 16->352 first conv of layer1, 3x3 at stride 1 and 2, the 1x1 shortcut at stride 1 and 2."""
    N, _ = env
    _sweep(N, (c, o, h, w, ks, ks, (st, st), (pd, pd)), bits, s, k, 256, seed=c + o + bits, batches=[1, 3])


def test_oracle_agrees_on_a_small_layer(env):
    """The NumPy oracle itself, codes to float64 convolution, on one layer with buckets straddling channels."""
    N, _ = env
    shape, stride, padding, bits, s, bucket = (7, 3, 3, 2), (2, 1), (1, 0), 2, 3, 16
    packed, alpha, beta, _, q = _weights(N, shape, bits, s, None, bucket, seed=5)
    x = torch.randn(2, 3, 6, 5, device="cuda")
    bias = torch.randn(7, device="cuda")
    rc, y = _call(N, x, shape, stride, padding, packed, bits, alpha, beta, None, s, bucket, bias)
    N.check(rc)
    ref, mag = PC.packed_conv2d(x.cpu().numpy(), packed.cpu().numpy(), bits, alpha.cpu().numpy(), beta.cpu().numpy(), shape, bucket,
                                stride, padding, levels=s, bias=bias.cpu().numpy())
    assert np.all(np.abs(y.cpu().numpy().astype(np.float64) - ref) <= PC.tolerance(ref, mag, 3 * 3 * 2))


@pytest.mark.parametrize("bits,s,k", [(1, 2, None), (2, 3, None), (4, 16, None), (8, 256, None), (4, None, 5), (8, None, 256)])
@pytest.mark.parametrize("padding,bucket", [((0, 0), 256), ((1, 2), 7), ((2, 1), None)])
def test_one_hot_inputs_reproduce_the_unpacked_weights(env, bits, s, k, padding, bucket):
    """An image with a single 1.0 gives, at every output whose window covers it, exactly the weight of that tap."""
    N, _ = env
    c, o, h, w, kh, kw = 4, 70, 5, 6, 3, 4
    shape = (o, c, kh, kw)
    packed, alpha, beta, pts, q = _weights(N, shape, bits, s, k, bucket, seed=bits + (s or 0) + (k or 0))
    x = torch.zeros(c * h * w, c, h, w, device="cuda")
    x.view(c * h * w, -1)[torch.arange(c * h * w), torch.arange(c * h * w)] = 1.0
    rc, y = _call(N, x, shape, (1, 1), padding, packed, bits, alpha, beta, pts, s, bucket, None)
    N.check(rc)
    ho, wo = y.shape[2:]
    want = torch.zeros(y.shape)
    qc = q.cpu()
    img = 0
    for ci in range(c):
        for hi in range(h):
            for wi in range(w):
                for i in range(ho):
                    for j in range(wo):
                        r, t = hi - i + padding[0], wi - j + padding[1]
                        if 0 <= r < kh and 0 <= t < kw:
                            want[img, :, i, j] = qc[:, ci, r, t]
                img += 1
    want = want.cuda()
    covered = want != 0
    assert torch.equal(y[covered].view(torch.int32), want[covered].view(torch.int32))
    assert torch.all(y[~covered] == 0)


def test_an_image_gives_the_same_bits_alone_and_in_any_batch(env):
    N, _ = env
    shape, stride, padding, bits, s, bucket = (50, 75, 5, 5), (1, 1), (2, 2), 4, 16, 256
    packed, alpha, beta, _, _ = _weights(N, shape, bits, s, None, bucket, seed=21)
    bias = torch.randn(50, device="cuda")
    img = torch.randn(1, 75, 32, 32, device="cuda")
    alone = _call(N, img, shape, stride, padding, packed, bits, alpha, beta, None, s, bucket, bias)[1]
    for n, at in ((2, 1), (5, 0), (5, 3), (17, 16), (33, 7)):
        batch = torch.randn(n, 75, 32, 32, device="cuda")
        batch[at] = img[0]
        y = _call(N, batch, shape, stride, padding, packed, bits, alpha, beta, None, s, bucket, bias)[1]
        assert torch.equal(y[at].view(torch.int32), alone[0].view(torch.int32)), (n, at)


def test_repeated_calls_and_four_streams_give_identical_bits(env):
    N, _ = env
    shape, stride, padding, bits, s, bucket = (352, 352, 3, 3), (1, 1), (1, 1), 2, 4, 256
    packed, alpha, beta, _, _ = _weights(N, shape, bits, s, None, bucket, seed=3)
    x = torch.randn(2, 352, 32, 32, device="cuda")
    bias = torch.randn(352, device="cuda")
    call = lambda **kw: _call(N, x, shape, stride, padding, packed, bits, alpha, beta, None, s, bucket, bias, **kw)  # noqa: E731
    ref = call()[1]
    for _ in range(3):
        assert torch.equal(call()[1].view(torch.int32), ref.view(torch.int32))
    torch.cuda.synchronize()
    outs, errs = [torch.empty_like(ref) for _ in range(4)], []

    def work(i):
        try:
            st = torch.cuda.Stream()
            with torch.cuda.stream(st):
                for _ in range(5):
                    N.check(call(y=outs[i], stream=st.cuda_stream)[0])
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
    shape, bits, s, bucket = (10, 4, 3, 3), 2, 4, 256
    packed, alpha, beta, _, _ = _weights(N, shape, bits, s, None, bucket, seed=1)
    pts = torch.rand(5, device="cuda")
    x = torch.randn(2, 4, 8, 8, device="cuda")
    y = torch.empty(2, 10, 8, 8, device="cuda")
    L = N.lib()

    def rc(**kw):
        a = dict(x=N.ptr(x), n=2, c=4, h=8, w=8, o=10, kh=3, kw=3, sh=1, sw=1, ph=1, pw=1, packed=N.ptr(packed), bits=bits,
                 alpha=N.ptr(alpha), beta=N.ptr(beta), points=None, k=0, levels=s, bucket=bucket, bias=None, y=N.ptr(y))
        a.update(kw)
        return L.qd_packed_conv2d(*a.values(), N.stream_ptr())
    assert rc() == N.QD_OK
    torch.cuda.synchronize()
    for bad in (dict(x=None), dict(packed=None), dict(alpha=None), dict(beta=None), dict(y=None),
                dict(n=0), dict(c=0), dict(h=0), dict(w=-1), dict(o=0), dict(kh=0), dict(kw=-2),
                dict(sh=0), dict(sw=-1), dict(ph=-1), dict(pw=-1),
                dict(kh=11, ph=1), dict(kw=9, pw=0),              # kernel larger than the padded input: empty output
                dict(bits=3), dict(levels=5),                     # 5 levels do not fit in 2-bit codes
                dict(levels=1), dict(levels=0, points=N.ptr(pts), k=5),   # 5 points do not fit either
                dict(levels=0, points=None, k=3), dict(levels=0, points=N.ptr(pts), k=0),
                dict(points=N.ptr(pts), k=4),                     # points given to a uniform call
                dict(bucket=-1), dict(y=N.ptr(x)),                # y overlapping x
                dict(y=N.ptr(x) + 4 * 100),
                dict(n=1 << 40, c=1 << 20, h=1 << 10, w=1 << 10)):   # sizes past 64-bit indexing
        assert rc(**bad) == N.QD_ERR_INVALID_ARG, bad
        assert L.qd_last_error().decode()
    # outside the supported set (refused before anything is read)
    for unsupported in (dict(h=1 << 29, ph=0), dict(c=1 << 31, kh=1, kw=1, ph=0, pw=0),
                        dict(n=1 << 40, c=1, h=1, w=1, kh=1, kw=1, ph=0, pw=0), dict(o=1 << 23)):
        assert rc(**unsupported) == N.QD_ERR_UNSUPPORTED, unsupported
        assert L.qd_last_error().decode()


# ------------------------------------------------------------------------------------------------ the module
def _layer(codec, N, o, c, k, stride=1, padding=2, bits=4, s=16, bucket=256, bias=True, seed=0):
    packed, alpha, beta, _, q = _weights(N, (o, c, k, k), bits, s, None, bucket, seed)
    b = torch.randn(o, device="cuda") if bias else None
    e = codec.PackedEntry("w", (o, c, k, k), bits=bits, packed=packed, alpha=alpha, beta=beta)
    return codec.PackedConv2d(e, "uniform", s, bucket, stride, padding, b), q, b


# the module tests' layer: 3 -> 25 channels, 3x3 (K = 27 taps) on 16x16 images, which runs the kernel at batch 1
def _module_layer(codec, N):
    return _layer(codec, N, 25, 3, 3, padding=1)


def _batches(layer):
    """(kernel batch, decode batch): the largest batch that runs the kernel and the next one."""
    assert layer.runs_kernel(1, 16, 16), "the module tests need a layer whose single image runs the kernel"
    n = 1
    while layer.runs_kernel(n + 1, 16, 16):
        n += 1
    return n, n + 1


def test_module_paths(env, deterministic_cudnn):
    N, codec = env
    layer, w, b = _module_layer(codec, N)
    nk, nd = _batches(layer)
    assert torch.equal(layer.decoded_weight().view(torch.int32), w.view(torch.int32))
    ref = torch.nn.Conv2d(3, 25, 3, padding=1).cuda()
    with torch.no_grad():
        ref.weight.copy_(w)
        ref.bias.copy_(b)
        for n in sorted({1, nk, nd, nd + 7}):
            x = torch.randn(n, 3, 16, 16, device="cuda")
            y = layer(x)
            if n > nk:                   # decode + F.conv2d: what an unpack_-loaded nn.Conv2d computes
                assert torch.equal(y, ref(x)), n
            else:
                _within(y, *_reference(x, w, b, (1, 1), (1, 1)))
        assert layer(torch.randn(0, 3, 16, 16, device="cuda")).shape == (0, 25, 16, 16)


@pytest.mark.parametrize("side", ["kernel", "decode"])
def test_module_takes_3d_and_non_contiguous_inputs(env, side, deterministic_cudnn):
    N, codec = env
    layer, w, b = _module_layer(codec, N)
    nk, nd = _batches(layer)
    n = nk if side == "kernel" else nd
    with torch.no_grad():
        if side == "kernel":             # one CHW image
            x3 = torch.randn(3, 16, 16, device="cuda")
            y3 = layer(x3)
            assert y3.shape == (25, 16, 16)
            assert torch.equal(y3, layer(x3[None])[0])
        xt = torch.randn(n, 16, 16, 3, device="cuda").permute(0, 3, 1, 2)        # channels-last strides
        assert not xt.is_contiguous()
        if side == "kernel":             # the kernel reads a contiguous copy
            assert torch.equal(layer(xt), layer(xt.contiguous()))
        else:                            # F.conv2d gets the input as nn.Conv2d would, strides included
            ref = torch.nn.Conv2d(3, 25, 3, padding=1).cuda()
            ref.weight.copy_(w)
            ref.bias.copy_(b)
            assert torch.equal(layer(xt), ref(xt))


def test_module_refusals(env):
    N, codec = env
    layer, _, _ = _layer(codec, N, 10, 4, 3, padding=1)
    with torch.no_grad():
        for bad in (torch.randn(2, 5, 8, 8, device="cuda"), torch.randn(2, 4, 8, 8, device="cuda", dtype=torch.float64),
                    torch.randn(2, 4, 8, 8), torch.randn(4, 8, device="cuda"), torch.randn(1, 2, 4, 8, 8, device="cuda")):
            with pytest.raises(ValueError):
                layer(bad)
        with pytest.raises(ValueError, match="smaller than"):          # a 3x3 kernel does not fit 2 rows unpadded
            _layer(codec, N, 10, 4, 3, padding=0)[0](torch.randn(2, 4, 2, 8, device="cuda"))
    with pytest.raises(RuntimeError):
        layer(torch.randn(2, 4, 8, 8, device="cuda", requires_grad=True))
    with torch.no_grad():
        layer(torch.randn(2, 4, 8, 8, device="cuda", requires_grad=True))      # no gradient needed: fine
    layer(torch.randn(2, 4, 8, 8, device="cuda"))                                 # grad mode, input without grad: fine
    cast = _layer(codec, N, 10, 4, 3)[0].double()
    with torch.no_grad(), pytest.raises(RuntimeError, match="float32"):
        cast(torch.randn(2, 4, 8, 8, device="cuda"))
    packed, alpha, beta, _, _ = _weights(N, (10, 4), 4, 16, None, 256, 0)
    with pytest.raises(ValueError, match="four-dimensional"):
        codec.PackedConv2d(codec.PackedEntry("w", (10, 4), bits=4, packed=packed, alpha=alpha, beta=beta), "uniform", 16, 256)
    with pytest.raises(ValueError):
        _layer(codec, N, 10, 4, 3, stride=0)


@pytest.mark.parametrize("side", ["kernel", "decode"])
def test_cuda_graph_replay(env, side):
    N, codec = env
    layer, _, _ = _module_layer(codec, N)
    nk, nd = _batches(layer)
    x = torch.randn(nk if side == "kernel" else nd, 3, 16, 16, device="cuda")
    side_stream = torch.cuda.Stream()
    side_stream.wait_stream(torch.cuda.current_stream())
    with torch.no_grad(), torch.cuda.stream(side_stream):
        ref = layer(x).clone()                                               # warm up on the capture stream
    torch.cuda.current_stream().wait_stream(side_stream)
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


def _wrn_small():
    from quantized_distillation_b200.cnn_models.wide_resnet import Wide_ResNet
    return Wide_ResNet(depth=10, widen_factor=2, dropout_rate=0.3, num_classes=10).cuda()


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


def _block_bytes(ptrs):
    """{address: size} of the caching allocator's allocated blocks that start at the given addresses."""
    sizes = {}
    for seg in torch.cuda.memory_snapshot():
        addr = seg["address"]
        for blk in seg["blocks"]:
            if blk["state"] == "active_allocated" and addr in ptrs:
                sizes[addr] = blk["size"]
            addr += blk["size"]
    return sizes


def _eligible(codec, pm, model):
    """Names of the modules attach_packed_ must replace: Linear and Conv2d layers with a weight stored quantized."""
    quantized = {name for (name, _), t in zip(model.named_parameters(), pm.tensors) if t.quantized}
    return [name for name, m in model.named_modules()
            if isinstance(m, (torch.nn.Linear, torch.nn.Conv2d)) and name + ".weight" in quantized]


@pytest.mark.parametrize("make,kind", [(_student, "uniform"), (_student, "nonuniform"), (_wrn_small, "uniform"), (_wrn, "uniform")],
                         ids=["student", "student_nonuniform", "wrn_10_2", "wrn_16_22"])
def test_attach_whole_model(env, make, kind, deterministic_cudnn):
    N, codec = env
    pm = _pack(codec, _trained(make), kind)
    torch.manual_seed(1)
    ref = make()
    codec.unpack_(pm, ref)
    torch.manual_seed(2)
    fresh = make()
    want_names = _eligible(codec, pm, fresh)
    index = {name: i for i, (name, _) in enumerate(fresh.named_parameters())}
    w_bytes = sum(pm.tensors[index[n + ".weight"]].numel * 4 for n in want_names)
    blocks = _block_bytes({fresh.get_submodule(n).weight.data_ptr() for n in want_names})
    gc.collect()                         # tensors earlier tests left in reference cycles must not be freed in between
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    names = codec.attach_packed_(pm, fresh)
    gc.collect()
    torch.cuda.synchronize()
    after = torch.cuda.memory_allocated()
    assert names == want_names
    assert any(isinstance(fresh.get_submodule(n), codec.PackedConv2d) for n in names)
    for n in names:
        assert isinstance(fresh.get_submodule(n), (codec.PackedLinear, codec.PackedConv2d)), n
    # exactly the allocator blocks that held the released float32 weights: each weight's bytes rounded up to 512, or a
    # reused cached block that the allocator did not split (up to 1 MB larger); the codes and scales the packed layers
    # hold belong to pm and were allocated before
    assert len(blocks) == len(names) and sum(blocks.values()) >= w_bytes
    assert before - after == sum(blocks.values()), (before, after, w_bytes, sum(blocks.values()))
    got = dict(fresh.named_parameters())
    got.update(dict(fresh.named_buffers()))
    for name, t in list(ref.named_parameters()) + list(ref.named_buffers()):
        if name.endswith(".weight") and name[:-7] in names:
            assert name not in got
            assert torch.equal(fresh.get_submodule(name[:-7]).decoded_weight().view(torch.int32), t.data.view(torch.int32)), name
            continue
        assert torch.equal(got[name].view(-1).view(torch.int8), t.data.view(-1).view(torch.int8)), name
    ref.eval(), fresh.eval()
    gen = torch.Generator(device="cuda").manual_seed(3)
    sides = {}                                   # packed convolution -> output side (Ho, Wo)
    convs = [m for m in fresh.modules() if isinstance(m, codec.PackedConv2d)]
    hooks = [m.register_forward_hook(lambda m, inp, out: sides.__setitem__(m, tuple(out.shape[-2:]))) for m in convs]
    with torch.no_grad():
        fresh(torch.randn(1, 3, 32, 32, device="cuda", generator=gen))
        for h in hooks:
            h.remove()
        if make is not _student:         # the student's convolutions have 75 to 1875 taps: they always decode
            assert any(m.runs_kernel(1, *sides[m]) for m in convs)      # batch 1 runs the kernel on some convolution
        decode_batch = 8
        while any(m.runs_kernel(decode_batch, *sides[m]) for m in convs):
            decode_batch *= 2
        # at decode_batch every packed convolution decodes and calls F.conv2d, and every PackedLinear calls F.linear:
        # the unpack_-loaded model's logits, bit for bit (TF32 as torch sets it by default)
        x = torch.randn(decode_batch, 3, 32, 32, device="cuda", generator=gen)
        want = ref(x)
        fresh(x)                                         # warm up: library workspaces are allocated once
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        got_logits = fresh(x)
        assert torch.equal(got_logits, want)
        del got_logits
        torch.cuda.synchronize()
        assert torch.cuda.memory_allocated() == base          # the decode path's scratch weights are freed
        # a batch of 1 runs the kernel on the layers under the crossover (and PackedLinear's kernel).  With TF32 off, both models sum in float32:
        # each layer's sums differ by reordering only, a few ulps, which the later layers carry to the logits; 1e-4 of
        # the largest logit is far above that and far below the gap between distinct logits of these networks
        saved = torch.backends.cudnn.allow_tf32
        torch.backends.cudnn.allow_tf32 = False
        try:
            x = torch.randn(1, 3, 32, 32, device="cuda", generator=gen)
            want, out = ref(x), fresh(x)
        finally:
            torch.backends.cudnn.allow_tf32 = saved
        assert out.shape == want.shape
        assert torch.allclose(out, want, rtol=1e-4, atol=1e-4 * float(want.abs().max())), float((out - want).abs().max())
        assert torch.equal(out.argmax(1), want.argmax(1))


class _Convs(torch.nn.Module):
    """One plain Conv2d that attach_packed_ replaces, and convolutions it must leave to unpack_: two sharing one
    weight, a grouped one, a dilated one, a Conv2d subclass, "same" padding of an even kernel (asymmetric) and
    reflect padding."""

    class Sub(torch.nn.Conv2d):
        def forward(self, x):
            return super().forward(x) * 2

    def __init__(self):
        super().__init__()
        self.plain = torch.nn.Conv2d(4, 8, 3, padding=1)
        self.tied_a = torch.nn.Conv2d(8, 8, 3, padding=1)
        self.tied_b = torch.nn.Conv2d(8, 8, 3, padding=1)
        self.tied_b.weight = self.tied_a.weight
        self.grouped = torch.nn.Conv2d(8, 8, 3, padding=1, groups=2)
        self.dilated = torch.nn.Conv2d(8, 8, 3, padding=2, dilation=2)
        self.sub = _Convs.Sub(8, 8, 3, padding=1)
        self.same_even = torch.nn.Conv2d(8, 8, 4, padding="same")
        self.reflect = torch.nn.Conv2d(8, 8, 3, padding=1, padding_mode="reflect")
        self.valid = torch.nn.Conv2d(8, 8, 1, padding="valid")
        self.same = torch.nn.Conv2d(8, 8, (3, 5), padding="same")

    def forward(self, x):
        x = self.tied_b(self.tied_a(self.plain(x)))
        x = self.reflect(self.same_even(self.sub(self.dilated(self.grouped(x)))))
        return self.same(self.valid(x))


def test_attach_leaves_ineligible_convolutions_to_unpack(env, no_tf32):
    N, codec = env
    torch.manual_seed(0)
    pm = codec.pack_model(_Convs().cuda(), 4, 64, quantize_first_and_last_layer=True)
    torch.manual_seed(1)
    ref = _Convs().cuda()
    codec.unpack_(pm, ref)
    torch.manual_seed(2)
    fresh = _Convs().cuda()
    assert codec.attach_packed_(pm, fresh) == ["plain", "valid", "same"]
    assert fresh.same.padding == (1, 2) and fresh.valid.padding == (0, 0)
    for name in ("tied_a", "tied_b", "grouped", "dilated", "same_even", "reflect"):
        assert type(fresh.get_submodule(name)) is torch.nn.Conv2d, name
    assert type(fresh.sub) is _Convs.Sub
    assert fresh.tied_b.weight is fresh.tied_a.weight
    got = dict(fresh.named_parameters())
    got.update(dict(fresh.named_buffers()))                  # a replaced layer holds its bias as a buffer
    for name, t in ref.named_parameters():
        if name in ("plain.weight", "valid.weight", "same.weight"):
            continue
        assert torch.equal(got[name].view(torch.int32), t.data.view(torch.int32)), name
    x = torch.randn(2, 4, 9, 9, device="cuda")
    with torch.no_grad():
        want, out = ref(x), fresh(x)
    assert torch.allclose(out, want, rtol=1e-4, atol=1e-4 * float(want.abs().max())), float((out - want).abs().max())


def test_attach_refuses_a_mismatched_model_before_writing(env):
    N, codec = env
    pm = _pack(codec, _trained(_student), "uniform")
    net = _student()
    snap = {k: v.clone() for k, v in net.state_dict().items()}
    pm.tensors[3] = codec.PackedEntry(pm.tensors[3].name, (1, 2, 3), raw=torch.zeros(6, device="cuda"))
    with pytest.raises(ValueError, match="shape"):
        codec.attach_packed_(pm, net)
    assert all(type(m) is torch.nn.Conv2d for m in net.conv_layers)
    assert type(net.linear_layers[0]) is torch.nn.Linear
    for k, v in net.state_dict().items():
        assert torch.equal(v, snap[k]), k
