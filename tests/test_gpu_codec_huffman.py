"""Huffman-coded model container on the GPU: encoder bytes against the NumPy restatement of the format
(oracle/huffman_oracle.py), decode -> q bit-identical to the fake-quantization ops, and whole models through
compress -> save -> load -> decompress_, with the sizes set against get_size_quantized_model."""
import numpy as np
import pytest
import torch

from oracle import huffman_oracle as HO

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import quantized_distillation_b200.quantization as Q
    from quantized_distillation_b200 import _native as N
    from quantized_distillation_b200 import codec
    return Q, N, codec


def gpu_encode(N, codec, idx, lengths):
    """(words, offsets) from qd_huffman_encode, as uint32 numpy arrays."""
    n = idx.numel()
    table = torch.from_numpy(codec.huffman_table(lengths)).cuda()
    counts = np.bincount(idx.cpu().numpy(), minlength=256)
    bits = int(sum(int(counts[s]) * l for s, l in lengths.items()))
    chunks = -(-n // codec.HUFFMAN_CHUNK)
    cap = -(-bits // 32) + chunks
    words = torch.full((cap + 1,), -1, dtype=torch.int32, device="cuda")
    offs = torch.empty(chunks, dtype=torch.int32, device="cuda")
    total = torch.zeros(1, dtype=torch.int64, device="cuda")
    N.check(N.lib().qd_huffman_encode(N.ptr(idx), n, N.ptr(table), N.ptr(words), cap, N.ptr(offs), N.ptr(total), N.stream_ptr()))
    t = int(total.item())
    assert t <= cap and int(words[cap].item()) == -1                 # nothing written past the capacity
    return words[:t].cpu().numpy().view(np.uint32), offs.cpu().numpy().view(np.uint32), table


def gpu_decode(N, codec, words, offs, table, alpha, beta, n, bucket, levels=None, points=None):
    w = torch.from_numpy(words.view(np.int32)).cuda()
    o = torch.from_numpy(offs.view(np.int32)).cuda()
    q = torch.empty(n, device="cuda")
    b = 0 if bucket is None else bucket
    wp = N.ptr(w) if w.numel() else None
    if points is None:
        N.check(N.lib().qd_huffman_decode_dequant_uniform(wp, w.numel(), N.ptr(o), N.ptr(table), N.ptr(alpha), N.ptr(beta), N.ptr(q),
                                                           n, b, levels, N.stream_ptr()))
    else:
        N.check(N.lib().qd_huffman_decode_dequant_nonuniform(wp, w.numel(), N.ptr(o), N.ptr(table), N.ptr(points), points.numel(),
                                                              N.ptr(alpha), N.ptr(beta), N.ptr(q), n, b, N.stream_ptr()))
    return q


def uniform_levels(N, x, s, bucket):
    n = x.numel()
    b = 0 if bucket is None else bucket
    rows = N.geometry(n, b)[0]
    alpha, beta = torch.empty(rows, device="cuda"), torch.empty(rows, device="cuda")
    idx = torch.empty(n, dtype=torch.uint8, device="cuda")
    ws = N.workspace(n, b, x.device)
    N.check(N.lib().qd_uniform_fwd(N.ptr(x), None, N.ptr(idx), N.ptr(alpha), N.ptr(beta), None, None, n, b, s, None, 0.0, 0, 0, 0,
                                   N.ptr(ws), ws.numel(), N.stream_ptr()))
    return idx, alpha, beta


SMALL_N = [1, 10, 255, 256, 257, 1023, 1024, 1025]


@pytest.mark.parametrize("n,s,bucket", [(n, s, b) for n in SMALL_N for s in (2, 4, 16, 256) for b in (256, 1024, None)] +
                         [(1_000_003, s, b) for s in (2, 4, 16, 256) for b in (256, None)] + [((1 << 24) + 5, 16, 256), ((1 << 24) + 5, 256, None)])
def test_uniform_stream_matches_oracle_and_decodes_to_q(env, n, s, bucket):
    Q, N, codec = env
    g = torch.Generator(device="cuda").manual_seed(n * 7 + s)
    x = torch.randn(n, generator=g, device="cuda") * 0.05
    idx, alpha, beta = uniform_levels(N, x, s, bucket)
    lengths = codec.huffman_code_lengths(np.bincount(idx.cpu().numpy(), minlength=256))
    words, offs, table = gpu_encode(N, codec, idx, lengths)
    ow, oo = HO.encode(idx.cpu().numpy(), lengths)
    assert np.array_equal(offs, oo) and np.array_equal(words, ow)
    q = gpu_decode(N, codec, words, offs, table, alpha, beta, n, bucket, levels=s)
    ref = Q.uniformQuantization(x.clone(), s, bucket_size=bucket)[0].view(-1)
    assert torch.equal(q.view(torch.int32), ref.view(torch.int32))


@pytest.mark.parametrize("K", [3, 4, 16])
@pytest.mark.parametrize("n,bucket", [(257, 256), (1025, None), (1_000_003, 256), (1_000_003, 1024)])
def test_nonuniform_stream_decodes_to_q(env, K, n, bucket):
    Q, N, codec = env
    g = torch.Generator(device="cuda").manual_seed(K * 1000 + n)
    x = torch.randn(n, generator=g, device="cuda") * 0.05
    pts = torch.sort(torch.rand(K, generator=g, device="cuda"))[0]
    q_ref, idx, _ = Q.nonUniformQuantization(x.clone(), pts, bucket_size=bucket, index_dtype=torch.uint8)
    b = 0 if bucket is None else bucket
    rows = N.geometry(n, b)[0]
    alpha, beta = torch.empty(rows, device="cuda"), torch.empty(rows, device="cuda")
    idx8 = torch.empty(n, dtype=torch.uint8, device="cuda")
    ws = N.workspace(n, b, x.device)
    N.check(N.lib().qd_nonuniform_fwd(N.ptr(x), N.ptr(pts), K, N.RULE_NEAREST, None, N.ptr(idx8), None, N.ptr(alpha), N.ptr(beta), n, b,
                                      None, 0.0, N.ptr(ws), ws.numel(), N.stream_ptr()))
    assert torch.equal(idx8, idx.view(-1).to(torch.uint8))
    lengths = codec.huffman_code_lengths(np.bincount(idx8.cpu().numpy(), minlength=256))
    words, offs, table = gpu_encode(N, codec, idx8, lengths)
    ow, oo = HO.encode(idx8.cpu().numpy(), lengths)
    assert np.array_equal(offs, oo) and np.array_equal(words, ow)
    q = gpu_decode(N, codec, words, offs, table, alpha, beta, n, bucket, points=pts)
    assert torch.equal(q.view(torch.int32), q_ref.view(-1).view(torch.int32))


@pytest.mark.parametrize("n", [1000, 1_000_003])
def test_skewed_histogram_long_codes_and_unaligned_views(env, n):
    """Codes of 20+ bits (geometric level histogram), symbols read from views at every byte offset, two runs."""
    Q, N, codec = env
    rng = np.random.default_rng(n)
    sym = np.minimum(rng.geometric(0.45, n + 3) - 1, 255).astype(np.uint8)
    base = torch.from_numpy(sym).cuda()
    lengths = None
    for shift in range(4):
        view = base[shift:shift + n]
        if lengths is None:
            lengths = codec.huffman_code_lengths(np.bincount(view.cpu().numpy(), minlength=256))
            if n > 100_000:
                assert max(lengths.values()) >= 20
        counts = np.bincount(view.cpu().numpy(), minlength=256)
        if any(counts[s] and s not in lengths for s in range(256)):
            lengths = codec.huffman_code_lengths(counts)
        words, offs, table = gpu_encode(N, codec, view, lengths)
        w2, o2, _ = gpu_encode(N, codec, view, lengths)
        assert np.array_equal(words, w2) and np.array_equal(offs, o2)          # deterministic bytes
        ow, oo = HO.encode(view.cpu().numpy(), lengths)
        assert np.array_equal(offs, oo) and np.array_equal(words, ow)
        # identity dequantization (points = symbol / 256, alpha 1, beta 0): q carries the decoded symbols
        pts = torch.arange(256, dtype=torch.float32, device="cuda") / 256
        one, zero = torch.ones(1, device="cuda"), torch.zeros(1, device="cuda")
        q = gpu_decode(N, codec, words, offs, table, one, zero, n, None, points=pts)
        assert torch.equal((q * 256).to(torch.uint8), view)
        # decode into an output that is not 16-byte aligned
        out = torch.empty(n + 1, device="cuda")[1:]
        w = torch.from_numpy(words.view(np.int32)).cuda()
        o = torch.from_numpy(offs.view(np.int32)).cuda()
        N.check(N.lib().qd_huffman_decode_dequant_nonuniform(N.ptr(w), w.numel(), N.ptr(o), N.ptr(table), N.ptr(pts), 256, N.ptr(one),
                                                              N.ptr(zero), N.ptr(out), n, 0, N.stream_ptr()))
        assert torch.equal(out, q)


def test_single_symbol_tensor(env):
    Q, N, codec = env
    x = torch.full((5000,), 0.25, device="cuda")
    idx, alpha, beta = uniform_levels(N, x, 16, 256)
    lengths = codec.huffman_code_lengths(np.bincount(idx.cpu().numpy(), minlength=256))
    assert list(lengths.values()) == [0]
    words, offs, table = gpu_encode(N, codec, idx, lengths)
    assert words.size == 0 and not offs.any()
    q = gpu_decode(N, codec, words, offs, table, alpha, beta, 5000, 256, levels=16)
    assert torch.equal(q, Q.uniformQuantization(x.clone(), 16, bucket_size=256)[0].view(-1))


# ---------------------------------------------------------------------------------------------------- models
def _student():
    from quantized_distillation_b200.cnn_models import conv_forward_model as cfm
    spec = dict(cfm.smallerModelSpec)
    spec["spec_dropout_rates"] = []
    return cfm.ConvolForwardNet(**spec, useBatchNorm=True, useAffineTransformInBatchNorm=True).cuda()


def _wrn():
    from quantized_distillation_b200.cnn_models.wide_resnet import Wide_ResNet
    return Wide_ResNet(depth=16, widen_factor=22, dropout_rate=0.3, num_classes=10).cuda()


def _check_model(env, tmp_path, make, numBits, bucket, qfl, overhead, points=None):
    Q, N, codec = env
    torch.manual_seed(0)
    model = make()
    params = list(model.parameters())
    with torch.no_grad():           # weight-like values: at its uniform initialisation every level is equally likely
        for p in params:
            p.normal_(0, 0.05)
    sel = range(len(params)) if qfl else range(1, len(params) - 1)
    if points is not None:
        gen = torch.Generator().manual_seed(3)
        points = [torch.sort(torch.rand(16, generator=gen))[0].cuda() for _ in sel]     # own 16 points per tensor: 4 bits
    cm = codec.compress_model(model, numBits if points is None else None, bucket_size=bucket, quantize_first_and_last_layer=qfl,
                              points=points)
    path = tmp_path / "model.qdh"
    size = codec.save_compressed(cm, path)
    back = codec.load_compressed(path)
    torch.manual_seed(1)
    fresh = make()
    fresh.load_state_dict({k: v for k, v in model.state_dict().items() if k not in dict(fresh.named_parameters())}, strict=False)
    handles = [p for p in fresh.parameters()]
    codec.decompress_(back, fresh)
    assert all(a is b for a, b in zip(handles, fresh.parameters()))
    expected = []
    for i, p in enumerate(params):
        if i in sel:
            k = list(sel).index(i)
            if points is None:
                expected.append(Q.uniformQuantization(p.data.clone(), 2 ** numBits, bucket_size=bucket)[0])
            else:
                expected.append(Q.nonUniformQuantization(p.data.clone(), points[k], bucket_size=bucket)[0])
        else:
            expected.append(p.data)
    for e, p in zip(expected, fresh.parameters()):
        assert torch.equal(p.data.view(-1).view(torch.int32), e.reshape(-1).view(torch.int32))
    # sizes against the reference's accounting (helpers/functions.py:226-262)
    count_q = sum(params[i].numel() for i in sel)
    if points is None:
        qf = lambda t: Q.uniformQuantization(t, 2 ** numBits, bucket_size=bucket)   # noqa: E731
        mean_bits = Q.help_functions.get_huffman_encoding_mean_bit_length(iter([params[i] for i in sel]), qf, "uniform", s=2 ** numBits)
        ref_mb = codec.get_size_quantized_model(model, numBits, qf, bucket_size=bucket, quantizeFirstLastLayer=qfl)
    else:
        qf = [lambda t, p_=p_: Q.nonUniformQuantization(t, p_, bucket_size=bucket) for p_ in points]
        mean_bits = Q.help_functions.get_huffman_encoding_mean_bit_length(iter([params[i] for i in sel]), qf, "nonUniform")
        ref_mb = codec.get_size_quantized_model(model, 4, qf, bucket_size=bucket, type_quantization="nonUniform", quantizeFirstLastLayer=qfl)
    sb = back.size_breakdown()
    assert sb == cm.size_breakdown() and sb["file_bytes"] == size
    assert sb["code_bits"] == pytest.approx(mean_bits * count_q, rel=1e-12)
    accounted = sb["code_bits"] / 8 + sb["scale_bytes"] + sb["unquantized_bytes"]
    assert abs(accounted - ref_mb * 1e6) <= 8 * len(sel) + 1e-6 * ref_mb * 1e6
    rest = sb["chunk_index_bytes"] + sb["padding_bits"] / 8 + sb["header_bytes"] + sb["alignment_bytes"]
    assert rest <= overhead * size, (rest / size, sb)
    fixed4 = sum((params[i].numel() * 4 + 7) // 8 + 8 * N.geometry(params[i].numel(), bucket or 0)[0] for i in sel) + sb["unquantized_bytes"]
    assert size < fixed4

    # the decoded model computes what the fake-quantized one does (sizes above use the original weights)
    with torch.no_grad():
        for e, p in zip(expected, model.parameters()):
            p.data.copy_(e.view_as(p))
    model.eval(), fresh.eval()
    x = torch.randn(8, 3, 32, 32, device="cuda")
    with torch.no_grad():
        assert torch.equal(model(x), fresh(x))


def test_student_uniform_4bit_round_trip_and_size(env, tmp_path):
    _check_model(env, tmp_path, _student, 4, 256, False, 0.04)


def test_student_differentiable_quantization_points_round_trip(env, tmp_path):
    _check_model(env, tmp_path, _student, None, 256, False, 0.04, points=True)


def test_wrn_16_22_uniform_2bit_round_trip_and_size(env, tmp_path):
    _check_model(env, tmp_path, _wrn, 2, 256, False, 0.03)
