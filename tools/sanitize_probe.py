"""Small invocations of every kernel family for compute-sanitizer (memcheck / racecheck / synccheck)."""
import os
import sys

# every tensor in its own cudaMalloc, so that memcheck sees its exact bounds: the caching allocator would place small
# tensors inside larger segments, where a read past one tensor's end lands in memory the process owns
os.environ.setdefault("PYTORCH_NO_CUDA_MEMORY_CACHING", "1")

import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import quantized_distillation_b200.quantization as Q  # noqa: E402
from quantized_distillation_b200 import codec  # noqa: E402
from quantized_distillation_b200.plan import QuantizationPlan  # noqa: E402
from oracle import quant_oracle as O  # noqa: E402

rng = np.random.default_rng(0)
# row lengths: warp path (256, 100, 1024, 7), staged ring with 64 / 128 / 256 / 512 / 1024-thread CTAs, one and two rows in
# flight, aligned and alternating-unaligned rows (1026, 3002), grid path (None)
for n, bucket in ((1000, 256), (5000, 100), (70001, 1024), (20000, 2048), (150000, 49152), (300001, None), (257, 7),
                  (30000, 1026), (40000, 3002), (100000, 8192), (120000, 20000), (200000, 32768)):
    x = (rng.standard_normal(n) * 0.05).astype(np.float32)
    xd = torch.from_numpy(x).cuda()
    q, sf = Q.uniformQuantization(xd, 16, bucket_size=bucket)
    ref, _, st = O.uniform_fwd(x, 16, bucket)
    assert np.array_equal(q.cpu().numpy(), ref), (n, bucket)
    Q.uniformQuantization(xd, 16, bucket_size=bucket, stochastic_rounding=True)
    pts = torch.linspace(0, 1, 4).cuda()
    f = Q.nonUniformQuantization_variable(bucket_size=bucket, pre_process_tensors=True, tensor=xd)
    f.forward(None, pts)
    f.backward(torch.randn(n).cuda())
    Q.nonUniformQuantization(xd, torch.linspace(0, 1, 40).cuda(), bucket_size=bucket)
    if bucket is not None:
        g = Q.uniformQuantization_variable(16, bucket_size=bucket)
        g.forward(xd)
        g.backward(torch.randn(n).cuda())
    sfn = Q.ScalingFunction("linear", False, False, bucket, False)
    sfn.inv_scale_down(sfn.scale_down(xd))
    codec.decode(codec.encode_uniform(xd, 16, bucket))
params = [torch.randn(n).cuda() * 0.05 for n in (5000, 10, 93750, 75, 257, 1)]
plan = QuantizationPlan(params, 16, 256)
plan.save_and_quantize_()
plan.restore_master()
plan.backward_([torch.randn_like(p) for p in params], "complicated")
# round 2: fused optimizer step, long-row plan (bucket None), centroid plan, order statistics, multi-tensor norm, a10 extension
from quantized_distillation_b200.plan import CentroidPlan  # noqa: E402
from quantized_distillation_b200.quantization import help_functions as H  # noqa: E402
from quantized_distillation_b200.quantization import quant_functions as QF  # noqa: E402
plan.save_and_quantize_()
for style in ("none", "truncated", "complicated"):
    plan.fused_step_([torch.randn_like(p) for p in params], style, 1e-2, 0.9, 2e-4, True)
big = [torch.randn(n).cuda() * 0.05 for n in (432, 200000, 49153, 16385, 3)]
lplan = QuantizationPlan(big, 4, None)
lplan.save_and_quantize_()
lplan.restore_master()
lplan.backward_([torch.randn_like(p) for p in big], "truncated")
src = [torch.randn(n).cuda() * 0.05 for n in (5000, 10, 93750, 257)]
pts = [torch.sort(torch.rand(k).cuda())[0] for k in (4, 32, 7, 16)]
cplan = CentroidPlan(src, [torch.empty_like(t) for t in src], pts, 256)
cplan.forward_()
cplan.backward_([torch.randn_like(t) for t in src])
v = torch.rand(100003).cuda()
assert torch.equal(H.order_statistics(v, [0, 7, 50000, 100002]), torch.sort(v)[0][[0, 7, 50000, 100002]])
H.gradient_norms(src)
QF.ALLOW_UNPINNED_SCALING = True
for kind in ("absmax", "absnorm"):
    for bucket in (256, 4096, None):
        Q.uniformQuantization(src[2], 8, type_of_scaling=kind, bucket_size=bucket)
        sfa = Q.ScalingFunction(kind, False, False, bucket, False)
        sfa.inv_scale_down(sfa.scale_down(src[2]))
QF.ALLOW_UNPINNED_SCALING = False
# tiled helper kernels past one tile per thread-group (full-tile fast paths + general tails), 1 / 2 / 4 / 8-bit codes
from quantized_distillation_b200 import _native as N  # noqa: E402
xb = torch.randn(70_001).cuda() * 0.05
for s_levels, bucket in ((2, 256), (4, 100), (16, 256), (256, 1000), (16, None)):
    assert torch.equal(codec.decode(codec.encode_uniform(xb, s_levels, bucket)), Q.uniformQuantization(xb, s_levels, bucket_size=bucket)[0])
sfb = Q.ScalingFunction("linear", False, False, 256, False)
sfb.inv_scale_down(sfb.scale_down(xb))
# host entry points: one launch on pinned host pointers (small), chunked pipeline (pageable memory)
for pinned in (True, False):
    m = 300_001
    hx, hg = torch.randn(m) * 0.05, torch.randn(m)
    hq, hgo = torch.zeros(m), torch.zeros(m)
    if pinned:
        hx, hg, hq, hgo = hx.pin_memory(), hg.pin_memory(), hq.pin_memory(), hgo.pin_memory()
    N.check(N.lib().qd_uniform_fwd_bwd_host(N.ptr(hx), N.ptr(hg), N.ptr(hq), N.ptr(hgo), m, 256, 16, N.BWD_MINMAX, 0))
    assert torch.equal(hq, Q.uniformQuantization(hx.cuda(), 16, bucket_size=256)[0].cpu())
# packed embedding lookup: odd rows starting inside a byte at 1 / 2 / 4 bits, the tensor's last code byte, an output
# 4 bytes off a 16-byte boundary, codes 1 byte off a word, out-of-range indices; widths 9 and 48 leave lanes of a row
# without a group, on tables that end exactly at a bucket's end (9 x 100 at bucket 100, 25 x 48 at bucket 100, 11 x 9
# at bucket None); bucket 3 is shorter than a lane's group
for bits, V, D, bucket in ((1, 37, 7, 100), (2, 50, 3, 100), (4, 9, 31, 100), (8, 5, 257, 100), (2, 100, 9, 100),
                           (4, 25, 48, 100), (2, 11, 9, None), (4, 40, 5, 3)):
    s_levels = 1 << bits
    pe = codec.pack_model(torch.nn.Embedding(V, D).cuda(), bits, bucket).tensors[0]   # numBits = bits: 2^bits levels
    emb = codec.PackedEmbedding(pe, "uniform", s_levels, bucket)
    idx = torch.tensor([V - 1, 0, -1, V, V - 1, 3 % V], device="cuda")
    want = emb.decoded_weight()[idx.clamp(0, V - 1)]
    ok = (idx >= 0) & (idx < V)
    assert torch.equal(emb(idx)[ok], want[ok]) and emb.invalid_index_count() == 2
    buf = torch.empty(idx.numel() * D + 1, device="cuda")
    shifted = torch.zeros(emb.packed.numel() + 1, dtype=torch.uint8, device="cuda")
    shifted[1:] = emb.packed
    N.check(N.lib().qd_packed_embedding(N.ptr(idx), 8, idx.numel(), V, D, N.ptr(shifted) + 1, bits, N.ptr(emb.alpha), N.ptr(emb.beta),
                                        None, 0, s_levels, bucket or 0, N.ptr(buf) + 4, None, N.stream_ptr()))
    assert torch.equal(buf[1:].view(-1, D)[ok], want[ok])
# packed LSTM cell and layer: odd sizes whose rows start inside a byte, buckets straddling gate rows, 1 / 4 / 8 rows
# (row tiles of 1, 4 and 8), a bidirectional two-layer LSTM over an unsorted PackedSequence
for bits, I, Hd, bucket in ((1, 7, 5, 100), (2, 33, 17, 3), (4, 129, 250, 256), (8, 10, 9, None)):
    lstm_pm = codec.pack_model(torch.nn.LSTM(I, Hd, num_layers=2, bidirectional=True).cuda(), bits, bucket)
    net = torch.nn.Sequential(torch.nn.LSTM(I, Hd, num_layers=2, bidirectional=True)).cuda()
    assert codec.attach_packed_(lstm_pm, net, recurrent=True) == ["0"]
    xs = torch.nn.utils.rnn.pack_padded_sequence(torch.randn(6, 8, I).cuda(), torch.tensor([6, 1, 3, 6, 2, 5, 4, 1]), enforce_sorted=False)
    net[0].CROSSOVER_ROWS = N.PACKED_LSTM_MAX_ROWS                  # the kernel path, not decode + torch
    with torch.no_grad():
        net[0](xs)
        cell_pm = codec.pack_model(torch.nn.LSTMCell(I, Hd).cuda(), bits, bucket)
        cell = codec.PackedLSTMCell(cell_pm.tensors[0], cell_pm.tensors[1], "uniform", 1 << bits, bucket)
        cell.CROSSOVER_ROWS = N.PACKED_LSTM_MAX_ROWS
        for m_rows in (1, 4, 8):
            cell(torch.randn(m_rows, I).cuda())
# packed GRU cell and layer: the same sizes, buckets and row tiles, a bidirectional two-layer GRU over an unsorted
# PackedSequence
for bits, I, Hd, bucket in ((1, 7, 5, 100), (2, 33, 17, 3), (4, 129, 250, 256), (8, 10, 9, None)):
    gru_pm = codec.pack_model(torch.nn.GRU(I, Hd, num_layers=2, bidirectional=True).cuda(), bits, bucket)
    net = torch.nn.Sequential(torch.nn.GRU(I, Hd, num_layers=2, bidirectional=True)).cuda()
    assert codec.attach_packed_(gru_pm, net, gru=True) == ["0"]
    xs = torch.nn.utils.rnn.pack_padded_sequence(torch.randn(6, 8, I).cuda(), torch.tensor([6, 1, 3, 6, 2, 5, 4, 1]), enforce_sorted=False)
    net[0].CROSSOVER_ROWS = N.PACKED_GRU_MAX_ROWS                   # the kernel path, not decode + torch
    with torch.no_grad():
        net[0](xs)
        cell_pm = codec.pack_model(torch.nn.GRUCell(I, Hd).cuda(), bits, bucket)
        cell = codec.PackedGRUCell(cell_pm.tensors[0], cell_pm.tensors[1], "uniform", 1 << bits, bucket)
        cell.CROSSOVER_ROWS = N.PACKED_GRU_MAX_ROWS
        for m_rows in (1, 4, 8):
            cell(torch.randn(m_rows, I).cuda())
# fused NMT loss, forward and backward: rows shorter than a group of four, odd rows (every 16-byte phase), rows of
# several groups per thread, with and without a teacher, padding and out-of-range targets, and an offset view
from quantized_distillation_b200.nmt_loss import nmt_loss  # noqa: E402
for R, V in ((3, 1), (5, 3), (7, 1025), (4, 10_004)):
    for teacher in (False, True):
        buf = torch.randn(R * V + 1, device="cuda")
        zs = (buf[1:] if V > 4 else buf[:R * V]).view(R, V).detach().requires_grad_(True)
        zt = torch.randn(R, V, device="cuda") if teacher else None
        tg = torch.randint(0, V, (R,), device="cuda")
        tg[0] = 0
        tg[-1] = V + 2
        loss, stats = nmt_loss(zs, tg, 0, zt)
        loss.backward()
# beam search step: every row-list width, V = K (one group) to several groups per thread, an offset (unaligned) view,
# the first step and a later one with a row that ended on EOS, on logits and on log-probabilities
from quantized_distillation_b200.beam import BatchBeam  # noqa: E402
for K, B, V in ((1, 3, 1), (2, 1, 5), (5, 7, 1025), (16, 2, 10_004)):
    bb = BatchBeam(B, K, 2, 0, V - 1, 0, 3, "cuda")
    for t, normalized in enumerate((False, True, False)):
        buf = torch.randn(K * B * V + 1, device="cuda")
        bb.advance(buf[1:].view(K * B, V), torch.rand(K * B, 4, device="cuda"), normalized)
        bb.tokens[t + 1, 0, 0] = V - 1
    bb.done()
# SRU recurrence, forward and backward: k = 3 and 4 (the float4 path and, at an offset view, the scalar one), both
# directions, len 1 and longer than the load ring, one column and several CTAs
from quantized_distillation_b200.sru import sru_compute  # noqa: E402
for L, B, d, k, bi, off in ((1, 1, 1, 4, False, 0), (7, 3, 5, 3, True, 0), (9, 2, 70, 4, True, 1), (5, 4, 40, 3, False, 1)):
    D = d * (2 if bi else 1)
    xin = torch.randn(L, B, D if k == 3 else 3, device="cuda", requires_grad=True)
    ubuf = torch.randn(L * B * D * k + off, device="cuda")
    u = ubuf[off:].view(L * B, D * k).detach().requires_grad_(True)
    init = torch.randn(B, D, device="cuda", requires_grad=True)
    h, last = sru_compute(u, xin, torch.randn(2 * D, device="cuda"), d, bi, 1, init=init, mask_h=torch.rand(B, D, device="cuda"))
    (h.sum() + last.sum()).backward()
# "mlp" global attention, forward and backward: one row and partial and full row tiles, S = 1 and past one source
# chunk, H = 1 and past one CTA, the transposed bank and contiguous [N, S, H] slabs, at offset (unaligned) views
from quantized_distillation_b200.attention import mlp_attention_core  # noqa: E402
for Nb, T, S, H, off in ((1, 1, 1, 1, 0), (3, 5, 9, 40, 1), (2, 9, 17, 300, 0), (4, 1, 33, 550, 1)):
    wq, inp = (torch.randn(Nb * T * H + off, device="cuda")[off:].view(Nb, T, H).requires_grad_(True) for _ in range(2))
    uh = torch.randn(S * Nb * H + off, device="cuda")[off:].view(S, Nb, H).transpose(0, 1).requires_grad_(True)
    ctx = torch.randn(Nb, S, H, device="cuda", requires_grad=True)
    v = torch.randn(H, device="cuda", requires_grad=True)
    align, concat = mlp_attention_core(wq, uh, v, inp, ctx)
    (concat.sum() + (align * align).sum()).backward()
torch.cuda.synchronize()
print("sanitize probe ok")
