"""Times the loss of the NMT training step over the target vocabulary, forward + backward, three ways:
  (a) fused: nmt_loss (qd_nmt_loss_fwd + qd_nmt_loss_bwd), the whole batch in one call;
  (b) torch: the reference's chain (onmt/Loss.py:97-120) on current torch, unsharded -- log_softmax, nll_loss with weight
      0 at the padding index, and with a teacher log_softmax -> exp -> kl_div masked to the non-padding rows;
  (c) torch sharded: the same chain over shards of 32 time steps (64 sentences per batch, so 2,048 rows per shard), one
      loss and one backward per shard, as onmt's shards() does.
The unsharded paths get the logits leaf itself, so its gradient is the one tensor the backward writes (a view of it
would make autograd allocate a second R x V gradient and copy into it); each shard gets its own leaf, the way a shard's
logits are their own tensor in onmt.  With the generator, the paths slice its input (rows x 500) instead.
Shapes: V in {10,004; 24,004; 50,004}, R in {2,048; 3,264} rows (batch 64 at 32 and 51 target steps), with and without
the teacher (weight 0.7).  The teacher's logits are given, so its generator, the same in every path, is not timed.  Three
more rows (R = 3,264, teacher on) also run the student's generator Linear(500 -> V) forward and backward inside every
timed call, to show the loss's share of the generator step (TF32 off, the torch default; the setting is recorded).
Each timed unit is one forward + backward between CUDA events; rounds alternate the paths, and the table gives the
median per call, GB/s at 20 (teacher) or 12 (no teacher) bytes per logit -- the traffic of the fused pass -- and the peak
allocated device memory above the inputs.  The card name and power limit are read in the same run.

    python -m tools.nmt_loss_bench [--out profiles/nmt_loss_bench.json] [--rounds 7] [--quick]"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

VOCABS = [10_004, 24_004, 50_004]
ROWS = [2_048, 3_264]
BATCH = 64
SHARD_STEPS = 32
HIDDEN = 500
PAD = 1
W = 0.7


def _card():
    import torch
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        out["nvidia_smi"] = q
    except Exception as e:  # pragma: no cover - depends on the host
        out["nvidia_smi"] = f"unavailable ({type(e).__name__})"
    return out


def _torch_loss(logits, target, teacher_logits):
    import torch.nn.functional as F
    import torch
    weight = torch.ones(logits.shape[1], device=logits.device)
    weight[PAD] = 0
    scores = F.log_softmax(logits, dim=1)
    loss = F.nll_loss(scores, target, weight=weight, reduction="sum")
    if teacher_logits is not None:
        pt = F.log_softmax(teacher_logits, dim=1).exp().detach()
        kl = F.kl_div(scores, pt, reduction="none") * target.ne(PAD).float()[:, None]
        loss = (1 - W) * loss + W * kl.sum()
    return loss


def _paths(R, V, teacher, generator, seed):
    """name -> callable running one forward + backward; the inputs they share; the loss of each for a cross-check."""
    import torch
    from quantized_distillation_b200.nmt_loss import nmt_loss
    g = torch.Generator(device="cuda").manual_seed(seed)
    target = torch.randint(0, V, (R,), generator=g, device="cuda")
    target[::7] = PAD
    zt = torch.randn(R, V, generator=g, device="cuda") * 2 if teacher else None
    if generator:
        lin = torch.nn.Linear(HIDDEN, V).cuda()
        hidden = torch.randn(R, HIDDEN, generator=g, device="cuda", requires_grad=True)

        def inputs(rows):
            return lin(hidden if rows is None else hidden[rows])
    else:
        leaf = (torch.randn(R, V, generator=g, device="cuda") * 2).requires_grad_(True)

        def inputs(rows):
            return leaf if rows is None else leaf.detach()[rows].requires_grad_(True)
    shard = SHARD_STEPS * BATCH
    losses = {}

    def zero():
        for p in ([lin.weight, lin.bias, hidden] if generator else [leaf]):
            p.grad = None

    def fused():
        zero()
        loss, _ = nmt_loss(inputs(None), target, PAD, zt, W)
        loss.backward()
        losses["fused"] = loss.detach()

    def torch_full():
        zero()
        loss = _torch_loss(inputs(None), target, zt)
        loss.backward()
        losses["torch"] = loss.detach()

    def torch_sharded():
        zero()
        total = 0.0
        for r0 in range(0, R, shard):
            rows = slice(r0, min(R, r0 + shard))
            loss = _torch_loss(inputs(rows), target[rows], None if zt is None else zt[rows])
            loss.backward()
            total = total + loss.detach()
        losses["torch_sharded"] = total

    return {"fused": fused, "torch": torch_full, "torch_sharded": torch_sharded}, losses


def _run(R, V, teacher, generator, rounds):
    import torch
    fns, losses = _paths(R, V, teacher, generator, seed=V + R)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    peak = {}
    for name, fn in fns.items():                 # warm-up, and the peak of one call above the inputs
        fn()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        fn()
        torch.cuda.synchronize()
        peak[name] = torch.cuda.max_memory_allocated() - base
    times = {k: [] for k in fns}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for _ in range(rounds):
        for name, fn in fns.items():
            ev[0].record()
            fn()
            ev[1].record()
            torch.cuda.synchronize()
            times[name].append(ev[0].elapsed_time(ev[1]) * 1e3)          # microseconds
    ref = losses["torch"].item()
    bytes_per_logit = 20 if teacher else 12
    row = {"R": R, "V": V, "teacher": teacher, "generator": generator,
           "loss_rel_diff_fused_vs_torch": abs(losses["fused"].item() - ref) / abs(ref)}
    for name in fns:
        med = statistics.median(times[name])
        row[name] = {"us_median": med, "us_min": min(times[name]), "us_max": max(times[name]),
                     "GBps_at_fused_bytes": bytes_per_logit * R * V / (med * 1e-6) / 1e9, "peak_alloc_MB": peak[name] / 2 ** 20}
    return row


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "nmt_loss_bench.json"))
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--quick", action="store_true", help="one small shape, for a rehearsal")
    args = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("nmt_loss_bench needs a CUDA device: there is nothing to time without one")
    card = _card()
    print(json.dumps(card))
    shapes = [(R, V, t, False) for V in VOCABS for R in ROWS for t in (False, True)]
    shapes += [(3_264, V, True, True) for V in VOCABS]
    if args.quick:
        shapes = [(256, 1_004, True, False), (256, 1_004, True, True)]
    rows = []
    hdr = f"{'R':>5} {'V':>6} {'teach':>5} {'gen':>3} | " + " | ".join(f"{n:>26}" for n in ("fused us GB/s MB", "torch", "torch sharded"))
    print(hdr)
    for R, V, t, gen in shapes:
        r = _run(R, V, t, gen, args.rounds)
        rows.append(r)
        cells = [f"{r[n]['us_median']:9.1f} {r[n]['GBps_at_fused_bytes']:7.0f} {r[n]['peak_alloc_MB']:8.0f}"
                 for n in ("fused", "torch", "torch_sharded")]
        print(f"{R:5d} {V:6d} {str(t):>5} {'y' if gen else 'n':>3} | " + " | ".join(cells)
              + f"   speed-up {r['torch']['us_median'] / r['fused']['us_median']:.2f}x / "
              f"{r['torch_sharded']['us_median'] / r['fused']['us_median']:.2f}x  d_loss {r['loss_rel_diff_fused_vs_torch']:.1e}")
        torch.cuda.empty_cache()
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump({"card": card, "tf32_matmul": torch.backends.cuda.matmul.allow_tf32, "rounds": args.rounds, "rows": rows}, f, indent=1)
    print(f"wrote {args.out}")


if __name__ == "__main__":
    main()
