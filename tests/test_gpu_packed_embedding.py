"""Embedding tables run from their packed codes: qd_packed_embedding against qd_unpack_dequant_*'s rows and the NumPy
restatement bit for bit over every code width, level / point count, bucket (straddling rows, None), odd and large row
widths, 1 to 50,000 rows, int32 / int64 indices in every order and unaligned outputs and codes; the NMT-sized table at
262,144 tokens; out-of-range indices (NaN rows, counted, never dereferenced); determinism across streams and under CUDA
graph replay; refusals at the C ABI and in the module; and attach_packed_(..., embeddings=True) on an NMT-shaped model
with a tied generator, on the Huffman route, and on the embeddings it must leave to unpack_."""
import gc
import threading

import numpy as np
import pytest
import torch

from oracle import packed_linear_oracle as P

pytestmark = pytest.mark.gpu

UNIFORM = [(bits, s, None) for bits in (1, 2, 4, 8) for s in (2, 3, 4, 16, 256) if s <= 1 << bits]
NONUNIFORM = [(bits, None, k) for bits in (1, 2, 4, 8) for k in (1, 3, 16, 256) if k <= 1 << bits]
# 3 and 2: buckets shorter than a lane's group of four, so (alpha, beta) change inside a group and a lane's cursor
# steps over several buckets at once
BUCKETS = [256, 100, 1024, 3, 2, None]
# (dim, num_embeddings): odd widths whose rows start inside a byte, widths around the 32-lane row, one row to 50,000.
# 9, 20 and 48 leave lanes of a row without a group (lanes per row are a power of two); 9 x 100 and 48 x 1200 fill
# whole buckets of 100 and 256 exactly, so such a lane's first element on the last row lies past the last bucket.
TABLES = [(1, 1), (3, 50_000), (7, 1), (9, 100), (20, 77), (31, 977), (48, 1200), (255, 3), (256, 4096), (257, 129),
          (500, 2000), (1023, 17), (4097, 5)]


@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from quantized_distillation_b200 import _native as N
    from quantized_distillation_b200 import codec
    return N, codec


def _table(N, V, D, bits, s, k, bucket, seed):
    """(packed, alpha, beta, points, q): random codes packed with qd_pack_indices, random scales, and q [V, D] decoded
    by qd_unpack_dequant_*."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    n = V * D
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
    return packed, alpha, beta, pts, q.view(V, D)


def _call(N, idx, V, D, packed, bits, alpha, beta, pts, s, bucket, out=None, invalid=None, stream=None):
    out = torch.empty(idx.numel(), D, device="cuda") if out is None else out
    rc = N.lib().qd_packed_embedding(N.ptr(idx), idx.element_size(), idx.numel(), V, D, N.ptr(packed), bits, N.ptr(alpha), N.ptr(beta),
                                     N.ptr(pts), 0 if pts is None else pts.numel(), s or 0, bucket or 0, N.ptr(out), N.ptr(invalid),
                                     stream if stream is not None else N.stream_ptr())
    return rc, out


def _oracle(idx, packed, bits, alpha, beta, V, D, bucket, s, pts):
    """oracle/packed_linear_oracle's decode reshaped to [V, D] and indexed."""
    q = P.dequantize(P.unpack_codes(packed.cpu().numpy(), V * D, bits), alpha.cpu().numpy(), beta.cpu().numpy(), bucket, s,
                     None if pts is None else pts.cpu().numpy())
    return q.reshape(V, D)[idx.cpu().numpy().astype(np.int64)]


def _same(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _orders(V, m, g):
    r = torch.randint(0, V, (m,), generator=g, device="cuda")
    r[-1] = V - 1                                    # the last row: the one that ends at the tensor's last element
    srt = torch.sort(r).values
    rep = r[:3].repeat_interleave(m // 3 + 1)[:m]
    return {"random": r, "sorted": srt, "reversed": srt.flip(0), "repeated": rep}


@pytest.mark.parametrize("bucket", BUCKETS, ids=lambda b: f"bucket{b}")
@pytest.mark.parametrize("bits,s,k", UNIFORM + NONUNIFORM)
def test_sweep_rows_bit_for_bit(env, bits, s, k, bucket):
    N, _ = env
    for t, (D, V) in enumerate(TABLES):
        seed = bits * 1000 + (s or 0) * 7 + (k or 0) * 13 + t
        packed, alpha, beta, pts, q = _table(N, V, D, bits, s, k, bucket, seed)
        g = torch.Generator(device="cuda").manual_seed(seed)
        for order, idx in _orders(V, 301, g).items():
            want = q[idx]
            for dt in (torch.int32, torch.int64):
                rc, out = _call(N, idx.to(dt), V, D, packed, bits, alpha, beta, pts, s, bucket)
                N.check(rc)
                assert _same(out, want), (D, V, order, dt)
            if order == "random":
                ref = _oracle(idx, packed, bits, alpha, beta, V, D, bucket, s, pts)
                assert np.array_equal(out.cpu().numpy().view(np.uint32), ref.view(np.uint32)), (D, V)


@pytest.mark.parametrize("bits,s,k", [(1, 2, None), (2, 3, None), (4, None, 11), (8, 256, None)])
@pytest.mark.parametrize("D", [3, 256, 257, 500])
def test_unaligned_outputs_and_codes(env, bits, s, k, D):
    """An output view 4 bytes past a 16-byte boundary (scalar stores on every row) and codes starting 1 byte past a
    word (byte loads) give the same bits."""
    N, _ = env
    V = 300
    packed, alpha, beta, pts, q = _table(N, V, D, bits, s, k, 256, seed=D + bits)
    idx = torch.randint(0, V, (77,), device="cuda")
    buf = torch.empty(77 * D + 4, device="cuda")
    out = buf[1:1 + 77 * D].view(77, D)
    N.check(_call(N, idx, V, D, packed, bits, alpha, beta, pts, s, 256, out=out)[0])
    assert _same(out, q[idx])
    shifted = torch.zeros(packed.numel() + 1, dtype=torch.uint8, device="cuda")
    shifted[1:] = packed
    rc, out2 = _call(N, idx, V, D, shifted[1:], bits, alpha, beta, pts, s, 256)
    N.check(rc)
    assert _same(out2, q[idx])


def test_nmt_table_at_262144_tokens(env):
    """The NMT default: a 50,000 x 500 table at 2 bits, bucket 256, gathered at 262,144 random tokens."""
    N, codec = env
    V, D, bits, s = 50_000, 500, 2, 4
    packed, alpha, beta, _, q = _table(N, V, D, bits, s, None, 256, seed=7)
    ref = P.dequantize(P.unpack_codes(packed.cpu().numpy(), V * D, bits), alpha.cpu().numpy(), beta.cpu().numpy(), 256, s)
    assert np.array_equal(q.cpu().numpy().reshape(-1).view(np.uint32), ref.view(np.uint32))
    emb = codec.PackedEmbedding(codec.PackedEntry("w", (V, D), bits=bits, packed=packed, alpha=alpha, beta=beta), "uniform", s, 256)
    idx = torch.randint(0, V, (262_144,), device="cuda")
    out = emb(idx)
    assert _same(out, q[idx])
    assert emb.invalid_index_count() == 0


# ------------------------------------------------------------------------------------------------ the module
def _module(codec, N, V=1000, D=37, bits=4, s=16, k=None, bucket=256, padding_idx=None, seed=0):
    packed, alpha, beta, pts, q = _table(N, V, D, bits, s, k, bucket, seed)
    e = codec.PackedEntry("w", (V, D), bits=bits, packed=packed, alpha=alpha, beta=beta, points=pts)
    return codec.PackedEmbedding(e, "uniform" if k is None else "nonuniform", s, bucket, padding_idx), q


def test_bad_indices_give_nan_rows_and_are_counted(env):
    N, codec = env
    emb, q = _module(codec, N)
    V = emb.num_embeddings
    for dt in (torch.int32, torch.int64):
        idx = torch.randint(0, V, (500,), device="cuda").to(dt)
        bad = torch.zeros(500, dtype=torch.bool, device="cuda")
        bad[torch.randperm(500, device="cuda")[:40]] = True
        idx[bad] = torch.where(torch.arange(500, device="cuda")[bad] % 2 == 0, -1, V).to(dt)
        idx[3], bad[3] = -(2 ** 31) if dt == torch.int32 else -(2 ** 62), True
        idx[4], bad[4] = 2 ** 31 - 1 if dt == torch.int32 else 2 ** 62, True
        out = emb(idx)
        assert _same(out[~bad], q[idx[~bad].long()])
        assert torch.isnan(out[bad]).all()
        assert emb.invalid_index_count() == int(bad.sum())
        assert emb.invalid_index_count() == 0                  # reset by the read
    emb(torch.tensor([0, V + 5, -3], device="cuda"))
    emb(torch.tensor([[V]], device="cuda"))
    assert emb.invalid_index_count() == 3
    packed, alpha, beta = emb.packed, emb.alpha, emb.beta      # the C ABI with no counter
    rc, out = _call(N, torch.tensor([1, -1, V], device="cuda"), V, emb.embedding_dim, packed, emb.bits, alpha, beta, None, 16, 256)
    N.check(rc)
    assert _same(out[0], q[1]) and torch.isnan(out[1:]).all()


def test_index_shapes(env):
    N, codec = env
    emb, q = _module(codec, N, padding_idx=-2)
    V, D = emb.num_embeddings, emb.embedding_dim
    assert emb.padding_idx == V - 2 and "padding_idx=998" in repr(emb)
    assert _same(emb.decoded_weight(), q)
    x0 = torch.tensor(5, device="cuda")
    assert _same(emb(x0), q[5])
    x2 = torch.randint(0, V, (4, 25), device="cuda", dtype=torch.int32)
    assert _same(emb(x2), q[x2.long()])
    xt = torch.randint(0, V, (25, 4), device="cuda").t()
    assert not xt.is_contiguous()
    assert _same(emb(xt), q[xt])
    assert _same(emb(torch.arange(V, device="cuda")[::3]), q[::3])
    assert _same(emb(torch.tensor([V - 2, V - 2], device="cuda")), q[[V - 2, V - 2]])   # padding_idx: the stored row
    for shape in ((0,), (3, 0), (0, 5)):
        e = emb(torch.empty(shape, dtype=torch.int64, device="cuda"))
        assert e.shape == shape + (D,) and e.dtype == torch.float32


def test_module_refusals(env):
    N, codec = env
    emb, _ = _module(codec, N)
    for bad in (torch.tensor([1, 2]), torch.tensor([1.0, 2.0], device="cuda"), torch.tensor([1, 2], dtype=torch.int16, device="cuda"),
                [1, 2]):
        with pytest.raises(ValueError):
            emb(bad)
    cast = _module(codec, N)[0].double()
    with pytest.raises(RuntimeError, match="float32"):
        cast(torch.tensor([1, 2], device="cuda"))
    packed, alpha, beta, _, _ = _table(N, 4, 5, 4, 16, None, 256, 0)
    with pytest.raises(ValueError, match="two-dimensional"):
        codec.PackedEmbedding(codec.PackedEntry("w", (4, 5, 1), bits=4, packed=packed, alpha=alpha, beta=beta), "uniform", 16, 256)
    with pytest.raises(ValueError, match="padding_idx"):
        codec.PackedEmbedding(codec.PackedEntry("w", (4, 5), bits=4, packed=packed, alpha=alpha, beta=beta), "uniform", 16, 256, 4)


def test_c_abi_refusals(env):
    N, _ = env
    V, D, bits, s = 10, 7, 2, 4
    packed, alpha, beta, _, _ = _table(N, V, D, bits, s, None, 256, seed=1)
    pts = torch.rand(5, device="cuda")
    idx = torch.arange(6, device="cuda")
    out = torch.empty(6, D, device="cuda")
    L = N.lib()

    def rc(**kw):
        a = dict(idx=N.ptr(idx), ib=8, count=6, V=V, D=D, packed=N.ptr(packed), bits=bits, alpha=N.ptr(alpha), beta=N.ptr(beta),
                 points=None, k=0, levels=s, bucket=256, out=N.ptr(out), invalid=None)
        a.update(kw)
        return L.qd_packed_embedding(*a.values(), N.stream_ptr())
    assert rc() == N.QD_OK
    torch.cuda.synchronize()
    for bad in (dict(idx=None), dict(packed=None), dict(alpha=None), dict(beta=None), dict(out=None),
                dict(ib=2), dict(ib=0), dict(count=0), dict(count=-1), dict(V=0), dict(D=0), dict(D=-3),
                dict(bits=3), dict(levels=5), dict(levels=1),                 # 5 levels do not fit in 2-bit codes
                dict(levels=0, points=N.ptr(pts), k=5),                       # nor 5 points
                dict(levels=0, points=None, k=3), dict(levels=0, points=N.ptr(pts), k=0),
                dict(points=N.ptr(pts), k=4),                                 # points given to a uniform call
                dict(bucket=-1), dict(out=N.ptr(idx)),                        # out overlapping the indices
                dict(V=1 << 40, D=1 << 30), dict(count=1 << 62, D=2)):        # sizes past 64-bit indexing
        assert rc(**bad) == N.QD_ERR_INVALID_ARG, bad
        assert L.qd_last_error().decode()
    assert rc(count=1 << 40) == N.QD_ERR_UNSUPPORTED                         # refused before anything is read
    assert L.qd_last_error().decode()


def test_four_streams_give_identical_bits(env):
    N, codec = env
    emb, q = _module(codec, N, V=50_000, D=500, bits=2, s=4)
    idx = torch.randint(0, 50_000, (1600,), device="cuda")
    ref = emb(idx)
    assert _same(ref, q[idx])
    torch.cuda.synchronize()
    outs, errs = [None] * 4, []

    def work(i):
        try:
            st = torch.cuda.Stream()
            with torch.cuda.stream(st):
                for _ in range(5):
                    outs[i] = emb(idx)
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
        assert _same(o, ref)


def test_cuda_graph_replay(env):
    N, codec = env
    emb, q = _module(codec, N, V=3000, D=257, bits=4, s=None, k=11)
    idx = torch.randint(0, 3000, (64, 25), device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ref = emb(idx).clone()                                             # warm up on the capture stream
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = emb(idx)
    for _ in range(3):
        out.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert _same(out, ref)
    assert _same(ref, q[idx])
    idx[0, 0] = -1                                                         # the counter is live under replay too
    g.replay()
    assert torch.isnan(out[0, 0]).all() and emb.invalid_index_count() == 1


# ------------------------------------------------------------------------------------------------ attaching
class _NMT(torch.nn.Module):
    """The reference's NMT shape in small: source and target embeddings with a padding index, an LSTM encoder and
    decoder, and a generator tied to the target embedding (or not)."""

    def __init__(self, vs=1500, vt=1200, d=48, tie=True):
        super().__init__()
        self.src_emb = torch.nn.Embedding(vs, d, padding_idx=1)
        self.tgt_emb = torch.nn.Embedding(vt, d, padding_idx=1)
        self.encoder = torch.nn.LSTM(d, d, num_layers=2)
        self.decoder = torch.nn.LSTM(d, d)
        self.generator = torch.nn.Linear(d, vt)
        if tie:
            self.generator.weight = self.tgt_emb.weight

    def forward(self, src, tgt):
        _, state = self.encoder(self.src_emb(src))
        out, _ = self.decoder(self.tgt_emb(tgt), (state[0][-1:], state[1][-1:]))
        return self.generator(out)


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


def _nmt(seed, **kw):
    torch.manual_seed(seed)
    return _NMT(**kw).cuda()


def _tokens(vs, vt, g):
    src = torch.randint(0, vs, (25, 64), device="cuda", generator=g)
    tgt = torch.randint(0, vt, (25, 64), device="cuda", generator=g)
    src[-3:, :5] = 1                                                       # padding
    return src, tgt


@pytest.mark.parametrize("kind", ["uniform", "nonuniform"])
def test_attach_nmt_model(env, kind):
    N, codec = env
    trained = _nmt(0)
    if kind == "uniform":
        pm = codec.pack_model(trained, 4, 256, quantize_first_and_last_layer=True)
    else:
        n_q = len(list(trained.parameters()))
        pts = [np.sort(np.random.default_rng(i).random(3 + i % 14)).astype(np.float32) for i in range(n_q)]
        pm = codec.pack_model(trained, points=pts, bucket_size=256, quantize_first_and_last_layer=True)
    ref = _nmt(1)
    codec.unpack_(pm, ref)
    fresh = _nmt(2)
    released = {fresh.src_emb.weight.data_ptr(), fresh.tgt_emb.weight.data_ptr()}
    w_bytes = 4 * (fresh.src_emb.weight.numel() + fresh.tgt_emb.weight.numel())
    blocks = _block_bytes(released)
    gc.collect()
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    names = codec.attach_packed_(pm, fresh, embeddings=True)
    gc.collect()
    torch.cuda.synchronize()
    after = torch.cuda.memory_allocated()
    assert names == ["src_emb", "tgt_emb", "generator"]
    assert type(fresh.src_emb) is codec.PackedEmbedding and type(fresh.tgt_emb) is codec.PackedEmbedding
    assert type(fresh.generator) is codec.PackedLinear
    assert fresh.src_emb.padding_idx == 1 and fresh.tgt_emb.padding_idx == 1
    for sec in ("packed", "alpha", "beta", "points"):                     # the tied pair holds one set of sections
        a, b = getattr(fresh.tgt_emb, sec), getattr(fresh.generator, sec)
        assert (a is None and b is None and kind == "uniform") or a.data_ptr() == b.data_ptr(), sec
    # the two float32 tables (the second is the generator's weight) are released; each embedding holds a 4-byte
    # invalid-index counter (one 512-byte allocator block); the codes and scales belong to pm and were allocated before
    assert len(blocks) == 2 and sum(blocks.values()) >= w_bytes
    assert before - after == sum(blocks.values()) - 2 * 512, (before, after, sum(blocks.values()))
    got = dict(fresh.named_parameters())
    got.update(dict(fresh.named_buffers()))                               # a replaced Linear holds its bias as a buffer
    for name, t in ref.named_parameters():                                # the LSTMs and the generator's bias as unpack_ wrote them
        if name in ("src_emb.weight", "tgt_emb.weight"):
            assert name not in got
            continue
        assert _same(got[name].data, t.data), name
    g = torch.Generator(device="cuda").manual_seed(3)
    src, tgt = _tokens(1500, 1200, g)
    with torch.no_grad():
        assert _same(fresh.src_emb(src), ref.src_emb(src))
        assert _same(fresh.tgt_emb(tgt), ref.tgt_emb(tgt))
        assert _same(fresh.tgt_emb.decoded_weight(), fresh.generator.decoded_weight())
        h = torch.randn(64, 48, device="cuda", generator=g)                 # above the crossover: decode + F.linear
        assert torch.equal(fresh.generator(h), ref.generator(h))
        h1 = h[:2]                                                          # the kernel: PackedLinear's float64 bound
        y, w = fresh.generator(h1).double(), ref.generator.weight.double()
        want = h1.double() @ w.T + ref.generator.bias.double()
        tol = 48 * 2.0 ** -23 * (h1.double().abs() @ w.abs().T) + 2.0 ** -23 * want.abs()
        assert torch.all((y - want).abs() <= tol)
        # the whole model: the same embeddings and weights, cuDNN's LSTM in both, 1600 generator rows (decode + F.linear)
        want, out = ref(src, tgt), fresh(src, tgt)
        assert torch.allclose(out, want, rtol=1e-4, atol=1e-4 * float(want.abs().max())), float((out - want).abs().max())
    assert fresh.src_emb.invalid_index_count() == 0


def test_default_keeps_todays_choices(env):
    N, codec = env
    for tie, want in ((True, []), (False, ["generator"])):
        pm = codec.pack_model(_nmt(0, tie=tie), 4, 256, quantize_first_and_last_layer=True)
        fresh = _nmt(2, tie=tie)
        assert codec.attach_packed_(pm, fresh) == want
        assert type(fresh.src_emb) is torch.nn.Embedding and type(fresh.tgt_emb) is torch.nn.Embedding
        ref = _nmt(1, tie=tie)
        codec.unpack_(pm, ref)
        assert _same(fresh.src_emb.weight.data, ref.src_emb.weight.data)
        if tie:
            assert type(fresh.generator) is torch.nn.Linear and fresh.generator.weight is fresh.tgt_emb.weight
    fresh = _nmt(2, tie=False)
    assert codec.attach_packed_(pm, fresh, embeddings=True) == ["src_emb", "tgt_emb", "generator"]
    assert fresh.tgt_emb.packed.data_ptr() != fresh.generator.packed.data_ptr()    # untied: two weights


class _Ineligible(torch.nn.Module):
    """Embeddings attach_packed_ must leave to unpack_ even with embeddings=True: one with max_norm, a subclass, two
    sharing one weight, and a generator whose tied weight has a third holder; one plain embedding it replaces."""

    class Sub(torch.nn.Embedding):
        def forward(self, x):
            return super().forward(x) * 2

    def __init__(self):
        super().__init__()
        self.plain = torch.nn.Embedding(50, 8)
        self.normed = torch.nn.Embedding(50, 8, max_norm=1.0)
        self.sub = _Ineligible.Sub(50, 8)
        self.shared_a = torch.nn.Embedding(50, 8)
        self.shared_b = torch.nn.Embedding(50, 8)
        self.shared_b.weight = self.shared_a.weight
        self.tri_emb = torch.nn.Embedding(50, 8)
        self.tri_gen = torch.nn.Linear(8, 50)
        self.tri_gen.weight = self.tri_emb.weight
        self.tri_other = torch.nn.Linear(8, 50, bias=False)
        self.tri_other.weight = self.tri_emb.weight
        self.normed_emb = torch.nn.Embedding(50, 8, max_norm=2.0)
        self.normed_gen = torch.nn.Linear(8, 50)
        self.normed_gen.weight = self.normed_emb.weight


def test_attach_leaves_ineligible_embeddings_to_unpack(env):
    N, codec = env
    torch.manual_seed(0)
    pm = codec.pack_model(_Ineligible().cuda(), 4, 64, quantize_first_and_last_layer=True)
    torch.manual_seed(1)
    ref = _Ineligible().cuda()
    codec.unpack_(pm, ref)
    torch.manual_seed(2)
    fresh = _Ineligible().cuda()
    assert codec.attach_packed_(pm, fresh, embeddings=True) == ["plain"]
    for name in ("normed", "shared_a", "shared_b", "tri_emb", "normed_emb"):
        assert type(fresh.get_submodule(name)) is torch.nn.Embedding, name
    for name in ("tri_gen", "tri_other", "normed_gen"):
        assert type(fresh.get_submodule(name)) is torch.nn.Linear, name
    assert type(fresh.sub) is _Ineligible.Sub
    assert fresh.shared_b.weight is fresh.shared_a.weight and fresh.normed_gen.weight is fresh.normed_emb.weight
    got = dict(fresh.named_parameters())
    for name, t in ref.named_parameters():
        if name != "plain.weight":
            assert _same(got[name].data, t.data), name
    idx = torch.arange(50, device="cuda")
    assert _same(fresh.plain(idx), ref.plain(idx))


def test_attach_huffman_route(env):
    """A Huffman-coded model transcoded to fixed-width codes and attached gives the rows decompress_ writes."""
    N, codec = env
    cm = codec.compress_model(_nmt(0), 4, bucket_size=256, quantize_first_and_last_layer=True)
    net = _nmt(2)
    assert codec.attach_packed_(codec.pack_compressed(cm), net, embeddings=True) == ["src_emb", "tgt_emb", "generator"]
    ref = _nmt(1)
    codec.decompress_(cm, ref)
    g = torch.Generator(device="cuda").manual_seed(4)
    src, tgt = _tokens(1500, 1200, g)
    assert _same(net.src_emb(src), ref.src_emb(src))
    assert _same(net.tgt_emb(tgt), ref.tgt_emb(tgt))
    assert _same(net.generator.decoded_weight(), ref.generator.weight.data)
