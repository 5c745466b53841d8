"""The SRU recurrence at the reference's NMT shapes, three arms on the same seeded inputs:
  fused  qd_sru_fwd / qd_sru_bwd (libqd_b200.so);
  ref    the reference's own kernels (oracle/_ref/libsru_ref.so, default contraction, as NVRTC built them) with the
         reference's launch shape, min(512, ncols) threads per block, and its torch sum of the bias partials;
  chain  the recurrence as a per-step chain of stock torch ops with autograd: the only way to run SRU without custom
         kernels.
"fwd" times the forward alone; "fwd+bwd" a forward and its backward.  Per shape: the median per-call time between
CUDA events over rounds through autograd (what a module pays, host work included), and the kernels alone: the fused
and the reference kernels' launches (the reference's bias sum included) captured `iters` times into a CUDA graph and
replayed, so that no host work is timed.  The fused kernels' bytes per call from the byte model below over their
graph-replay time give GB/s and the fraction of the H100 SXM data-sheet 3.35 TB/s.  Also one whole 2-layer
bidirectional encoder, SRU(500, 250) as onmt's RNNEncoder builds it for rnn_size 500, at len 50 and batch 64, forward
and backward, on each arm.
Prints one JSON line per row, with the card's name and power limit, and writes them to profiles/sru_bench.json.

    python tools/sru_bench.py [--rounds 7] [--iters 20]
"""
import argparse
import ctypes as C
import itertools
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from quantized_distillation_b200 import _native as N  # noqa: E402
from quantized_distillation_b200.sru import SRU, SRUCell  # noqa: E402

PEAK = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(), "unknown"
    return name, power


def ref_lib():
    path = os.path.join(ROOT, "oracle", "_ref", "libsru_ref.so")
    if not os.path.exists(path):
        raise SystemExit(f"{path} missing: run oracle/sru_ref_build.py (or __graft_entry__.build()) with a reference checkout")
    lib = C.CDLL(path)
    lib.sru_ref_fwd.argtypes = [C.c_int] + [C.c_void_p] * 5 + [C.c_int] * 4 + [C.c_void_p] * 2 + [C.c_int, C.c_void_p]
    lib.sru_ref_bwd.argtypes = [C.c_int] + [C.c_void_p] * 8 + [C.c_int] * 4 + [C.c_void_p] * 4 + [C.c_int, C.c_void_p]
    return lib


def fused_bytes(L, B, d, k, bi, backward):
    """Bytes the fused kernels must move at least: forward reads u (and x for k = 3), init, mask_h and writes h, c;
    backward reads u, x, c, grad_h, init, mask_h, grad_last and writes grad_u, grad_x, grad_init and the bias partials,
    which the second launch reads back.  The bias is negligible and left out."""
    n = B * d * (2 if bi else 1)
    seq = L * n * 4
    fwd = seq * k + (seq if k == 3 else 0) + 2 * n * 4 + 2 * seq
    if not backward:
        return fwd
    bwd = seq * k + (seq if k == 3 else 0) + 2 * seq + 3 * n * 4 + seq * k + (seq if k == 3 else 0) + n * 4 + 4 * n * 4
    return fwd + bwd


def time_call(fn, rounds, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b) * 1e3 / iters)
    return sorted(times)[len(times) // 2]


def graph_time(fn, rounds, iters):
    """Median device time per fn() of `iters` calls captured into one CUDA graph."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        for _ in range(iters):
            fn()
    return time_call(g.replay, rounds, 1) / iters


def kernel_calls(lib, u, x, bias, init, gh, d, bi, backward):
    """(fused, ref): the raw kernel launches of one forward (and backward) on preallocated outputs."""
    L, B = x.shape[0], x.shape[1]
    D = d * (2 if bi else 1)
    k = u.shape[-1] // D
    xk = x if k == 3 else None
    h, c, gu = torch.empty(L, B, D, device="cuda"), torch.empty(L, B, D, device="cuda"), torch.empty_like(u)
    gx = torch.empty_like(x) if k == 3 else None
    gl, gi, gb = torch.randn(B, D, device="cuda"), torch.empty(B, D, device="cuda"), torch.empty(2 * D, device="cuda")
    gbp = torch.empty(2, B, D, device="cuda")
    ws = torch.empty(int(N.lib().qd_sru_workspace_bytes(B, d, int(bi))), dtype=torch.uint8, device="cuda")
    P = N.ptr

    def fused():
        N.check(N.lib().qd_sru_fwd(P(u), P(xk), P(bias), P(init), None, L, B, d, k, int(bi), 1, P(h), P(c), N.stream_ptr()))
        if backward:
            N.check(N.lib().qd_sru_bwd(P(u), P(xk), P(bias), P(init), None, P(c), P(gh), P(gl), L, B, d, k, int(bi), 1, P(gu),
                                       P(gx), P(gb), P(gi), P(ws), ws.numel(), N.stream_ptr()))

    def ref():
        lib.sru_ref_fwd(int(bi), P(u), P(xk), P(bias), P(init), None, L, B, d, k, P(h), P(c), 1, N.stream_ptr())
        if backward:
            lib.sru_ref_bwd(int(bi), P(u), P(xk), P(bias), P(init), None, P(c), P(gh), P(gl), L, B, d, k, P(gu), P(gx),
                            P(gbp), P(gi), 1, N.stream_ptr())
            torch.sum(gbp, 1, out=gb.view(2, D))
    return fused, ref


def chain(u, x, bias, d, bi, act, init, mask_h):
    """The reference's recurrence in stock torch ops, one step at a time (x: [len, batch, n_in])."""
    L, B = x.shape[0], x.shape[1]
    dir_ = 2 if bi else 1
    D = dir_ * d
    k = u.shape[-1] // D
    u4 = u.view(L, B, D, k)
    xh = u4[..., 3] if k == 4 else x
    g1 = torch.sigmoid(u4[..., 1] + bias[:D])
    g2 = torch.sigmoid(u4[..., 2] + bias[D:])
    cur0 = init if init is not None else x.new_zeros(B, D)
    parts = []
    for r in range(dir_):
        sl = slice(r * d, (r + 1) * d)
        cur, cs = cur0[:, sl], [None] * L
        for t in (range(L) if r == 0 else range(L - 1, -1, -1)):
            cur = (cur - u4[t, :, sl, 0]) * g1[t, :, sl] + u4[t, :, sl, 0]
            cs[t] = cur
        parts.append(torch.stack(cs))
    c = torch.cat(parts, 2)
    a = torch.tanh(c) if act == 1 else (torch.relu(c) if act == 2 else c)
    h = (a * (mask_h if mask_h is not None else 1.0) - xh) * g2 + xh
    last = torch.stack((c[-1, :, :d], c[0, :, d:])) if bi else c[-1]
    return h, last


class RefCompute(torch.autograd.Function):
    """The reference's SRU_Compute on its own kernels: zero init when None, grad_bias partials summed by torch."""

    @staticmethod
    def forward(ctx, u, x, bias, init, lib, d, bi, act):
        L, B = x.shape[0], x.shape[1]
        D = d * (2 if bi else 1)
        k = u.shape[-1] // D
        init_ = init if init is not None else x.new_zeros(B, D)
        h, c = x.new_empty(L, B, D), x.new_empty(L, B, D)
        xk = x.contiguous() if k == 3 else None
        lib.sru_ref_fwd(int(bi), u.data_ptr(), N.ptr(xk), bias.data_ptr(), init_.data_ptr(), None, L, B, d, k,
                        h.data_ptr(), c.data_ptr(), act, N.stream_ptr())
        ctx.save_for_backward(u, xk, bias, init_, c)
        ctx.args = (lib, d, bi, act, L, B, D, k, init is not None)
        last = torch.stack((c[-1, :, :d], c[0, :, d:])) if bi else c[-1]
        return h, last

    @staticmethod
    def backward(ctx, gh, gl):
        u, xk, bias, init_, c = ctx.saved_tensors
        lib, d, bi, act, L, B, D, k, has_init = ctx.args
        if bi:
            gl = torch.cat((gl[0], gl[1]), 1)
        gh, gl = gh.contiguous(), gl.contiguous()
        gu = torch.empty_like(u)
        gx = torch.empty_like(xk) if k == 3 else None
        gb, gi = u.new_empty(2, B, D), u.new_empty(B, D)
        lib.sru_ref_bwd(int(bi), u.data_ptr(), N.ptr(xk), bias.data_ptr(), init_.data_ptr(), None, c.data_ptr(),
                        gh.data_ptr(), gl.data_ptr(), L, B, d, k, gu.data_ptr(), N.ptr(gx), gb.data_ptr(), gi.data_ptr(),
                        act, N.stream_ptr())
        return gu, gx, gb.sum(1).view(-1), gi if has_init else None, None, None, None, None


def recurrence_case(lib, L, B, d, k, bi, backward, rounds, iters):
    from quantized_distillation_b200.sru import sru_compute
    g = torch.Generator(device="cuda").manual_seed(L * 1000 + B + d)
    D = d * (2 if bi else 1)
    x = torch.randn(L, B, D if k == 3 else 500, generator=g, device="cuda").requires_grad_(backward)
    u = torch.randn(L * B, D * k, generator=g, device="cuda").requires_grad_(backward)
    bias = torch.randn(2 * D, generator=g, device="cuda").requires_grad_(backward)
    init = torch.randn(B, D, generator=g, device="cuda").requires_grad_(backward)
    gh = torch.randn(L, B, D, generator=g, device="cuda")
    arms = {"fused": lambda: sru_compute(u, x, bias, d, bi, 1, init=init),
            "ref": lambda: RefCompute.apply(u, x, bias, init, lib, d, bi, 1),
            "chain": lambda: chain(u, x, bias, d, bi, 1, init, None)}
    row = {"len": L, "batch": B, "d": d, "k": k, "bidirectional": bi, "pass": "fwd+bwd" if backward else "fwd"}
    for name, f in arms.items():
        def call(f=f):
            if backward:
                h, last = f()
                torch.autograd.backward([h, last], [gh, torch.ones_like(last)])
            else:
                with torch.no_grad():
                    f()
        row[f"{name}_us"] = round(time_call(call, rounds, iters), 2)
    row["vs_ref"] = round(row["ref_us"] / row["fused_us"], 3)
    row["vs_chain"] = round(row["chain_us"] / row["fused_us"], 3)
    with torch.no_grad():
        fk, rk = kernel_calls(lib, u.detach(), x.detach(), bias.detach(), init.detach(), gh, d, bi, backward)
        row["fused_kernel_us"] = round(graph_time(fk, rounds, iters), 2)
        row["ref_kernel_us"] = round(graph_time(rk, rounds, iters), 2)
    row["kernel_vs_ref"] = round(row["ref_kernel_us"] / row["fused_kernel_us"], 3)
    row["fused_bytes"] = fused_bytes(L, B, d, k, bi, backward)
    row["fused_GBps"] = round(row["fused_bytes"] / row["fused_kernel_us"] / 1e3, 1)
    row["fused_of_peak"] = round(row["fused_bytes"] / (row["fused_kernel_us"] * 1e-6) / PEAK, 4)
    return row


def encoder_case(lib, rounds, L=50, B=64, n_in=500, hidden=250):
    torch.manual_seed(0)
    fused = SRU(n_in, hidden, num_layers=2, bidirectional=True).cuda()
    x = torch.randn(L, B, n_in, device="cuda", requires_grad=True)
    row = {"encoder": "SRU(500, 250, 2 layers, bidirectional), len 50, batch 64, fwd+bwd"}

    def cell_forward(self, input, c0=None, mode="chain"):
        u = input.contiguous().view(-1, self.n_in).mm(self.weight)
        if mode == "chain":
            return chain(u, input, self.bias, self.n_out, self.bidirectional, self.activation_type, c0, None)
        return RefCompute.apply(u, input, self.bias, c0, lib, self.n_out, self.bidirectional, self.activation_type)

    for name in ("fused", "ref", "chain"):
        for m in fused.modules():
            if isinstance(m, SRUCell):
                if name == "fused":
                    m.__dict__.pop("forward", None)
                else:
                    m.forward = (lambda self, mode: lambda input, c0=None: cell_forward(self, input, c0, mode))(m, name)

        def call():
            h, fh = fused(x)
            (h.sum() + fh.sum()).backward()
        row[f"{name}_ms"] = round(time_call(call, rounds, 3) / 1e3, 3)
    row["vs_ref"] = round(row["ref_ms"] / row["fused_ms"], 3)
    row["vs_chain"] = round(row["chain_ms"] / row["fused_ms"], 3)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "sru_bench.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sru_bench needs a CUDA device")
    lib = ref_lib()
    name, power = card()
    rows = []
    for L, B, d, k, bi, bwd in itertools.product((1, 20, 50), (1, 64, 320), (250, 500, 550), (3, 4), (False, True),
                                                (False, True)):
        rows.append(recurrence_case(lib, L, B, d, k, bi, bwd, args.rounds, args.iters))
    rows.append(encoder_case(lib, args.rounds))
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        for r in rows:
            r.update(card=name, power_limit=power)
            print(json.dumps(r))
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
