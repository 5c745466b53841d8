"""Steps/s of data-parallel differentiable quantization (``optimize_quantization_points`` on a
``FlatDataParallel``-wrapped network): every step reduces only the float64 centroid-gradient table,
one NCCL all-reduce of (tensors x 32) doubles.

Workloads, each with eager steps and with the whole step captured in a CUDA graph (all-reduce included):
* the student of BASELINE config 4: 4 points per tensor, bucket 256, batch 25 per rank;
* Wide_ResNet-16-22: 4 points per tensor, bucket 256, global batch 100 (13 per rank on 8 GPUs).

    python tools/diffquant_dp_bench.py [--gpus 1,2,4,8] [--steps 40] [--warmup 8] [--out profiles/diffquant_dp.md]

The launcher runs ``torchrun --nproc-per-node N`` of this file once per N that fits on the visible GPUs, and reports
the others as not measured.  N = 1 runs the same data-parallel path over a one-rank NCCL group.  The card's name,
power limit and the GPU count are read in the same run.  Synthetic data and random weights: steps/s does not depend
on either.  Reported time per step is the slowest rank's, from CUDA events around the timed steps.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

MODELS = ("student", "wrn16-22")


def _build(kind, dev):
    import torch
    from quantized_distillation_b200.cnn_models import conv_forward_model as cfm
    from quantized_distillation_b200.cnn_models.wide_resnet import Wide_ResNet
    torch.manual_seed(1234)
    with torch.device(dev):
        if kind == "student":
            spec = dict(cfm.smallerModelSpec)
            spec["spec_dropout_rates"] = []
            return cfm.ConvolForwardNet(**spec, useBatchNorm=True, useAffineTransformInBatchNorm=True)
        return Wide_ResNet(depth=16, widen_factor=22, dropout_rate=0.3, num_classes=10)


def _per_rank_batch(kind, world):
    if kind == "student":
        return 25
    return 100 // world if 100 % world == 0 else 13


def worker(args):
    import torch
    import torch.distributed as dist
    from quantized_distillation_b200 import distributed as D
    from quantized_distillation_b200.cnn_models import conv_forward_model as cfm
    from quantized_distillation_b200.cnn_models import help_fun as hf

    world, rank, local = D.env_world()
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    rows = []
    try:
        for kind in MODELS:
            for graph in (False, True):
                model = D.FlatDataParallel(_build(kind, dev))
                batch = _per_rank_batch(kind, world)
                total = args.warmup + args.steps
                data = hf.synthetic_cifar_loader(total, batch, seed=100 + rank)
                ev = {}

                def hook(i, loss):
                    if i in (args.warmup, total):
                        ev[i] = torch.cuda.Event(enable_timing=True)
                        ev[i].record()

                _, pts, info = cfm.optimize_quantization_points(
                    model, data, data, initial_learning_rate=1e-5, epochs_to_train=1, print_every=total,
                    numPointsPerTensor=4, bucket_size=256, use_distillation_loss=True, initialize_method="quantiles",
                    verbose=False, evaluate=False, max_steps=total, step_hook=hook, cuda_graph_step=graph)
                torch.cuda.synchronize(dev)
                ms = D.max_over_ranks(ev[args.warmup].elapsed_time(ev[total]) / args.steps, dev)
                tensors = len(pts)
                table = tensors * 32 * 8
                rows.append({"model": kind, "gpus": world, "per_rank_batch": batch, "global_batch": batch * world,
                             "captured": bool(info["cuda_graph_step"]), "requested_graph": graph,
                             "multi_tensor_plan": bool(info["multi_tensor_plan"]), "tensors": tensors,
                             "ms_per_step": round(ms, 4), "steps_per_s": round(1000.0 / ms, 2),
                             "table_bytes": table,
                             "ring_bytes_sent_per_rank": int(round(2 * (world - 1) / world * table))})
                del model, data
                torch.cuda.empty_cache()
    finally:
        dist.destroy_process_group()
    if rank == 0:
        with open(args.json, "w") as f:
            json.dump(rows, f)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()
        return out
    except Exception as e:
        return [f"nvidia-smi unavailable: {e}"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", default="1,2,4,8")
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--out", default=None, help="markdown table (default: print only)")
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--json", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("diffquant_dp_bench needs CUDA GPUs")
    visible = torch.cuda.device_count()
    cards = card()
    print(json.dumps({"visible_gpus": visible, "cards": cards}))
    rows, skipped = [], []
    for n in [int(v) for v in args.gpus.split(",")]:
        if n > visible:
            skipped.append(n)
            continue
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "rows.json")
            cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", f"--nproc-per-node={n}", os.path.abspath(__file__),
                   "--worker", "--steps", str(args.steps), "--warmup", str(args.warmup), "--json", path]
            subprocess.run(cmd, check=True, cwd=ROOT)
            with open(path) as f:
                got = json.load(f)
        for r in got:
            print(json.dumps(r))
        rows += got
    lines = [f"Card: {'; '.join(cards)} ({visible} visible). {args.steps} timed steps after {args.warmup} warm-up steps.", "",
             "| model | GPUs | batch per rank | step | steps/s | ms/step | table bytes | bytes sent per rank (ring) |",
             "|---|---:|---:|---|---:|---:|---:|---:|"]
    for r in rows:
        step = "captured" if r["captured"] else ("eager (capture fell back)" if r["requested_graph"] else "eager")
        lines.append(f"| {r['model']} | {r['gpus']} | {r['per_rank_batch']} | {step} | {r['steps_per_s']} | {r['ms_per_step']} | "
                     f"{r['table_bytes']} | {r['ring_bytes_sent_per_rank']} |")
    for n in skipped:
        lines.append(f"| both | {n} | | | not measured ({visible} GPU(s) visible) | | | |")
    text = "\n".join(lines)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
