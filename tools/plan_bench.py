"""Per-step quantization cost on the real parameter lists (BASELINE configs 2/3):

  * ours: QuantizationPlan save / quantize_ / restore / backward_ (one launch each)
  * ours, per-tensor API loop (launch-latency bound for the 10-500 element tensors)
  * the reference's choreography with stock torch ops ON THE SAME GPU
    (oracle/torch_chain.py run on CUDA tensors: ~12 launches per tensor, rebinding + copy back)

    python -m tools.plan_bench [--out gpurun_out/plan_bench.json]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import quantized_distillation_b200.quantization as Q  # noqa: E402
from oracle import torch_chain as T  # noqa: E402
from quantized_distillation_b200.cnn_models import conv_forward_model as cfm  # noqa: E402
from quantized_distillation_b200.cnn_models.wide_resnet import Wide_ResNet  # noqa: E402
from quantized_distillation_b200.plan import QuantizationPlan  # noqa: E402


def timed(fn, iters=50, warm=5):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3      # us


def run(out_path=None):
    dev = torch.device("cuda", 0)
    spec = dict(cfm.smallerModelSpec)
    spec["spec_dropout_rates"] = []
    models = {
        "student_22_tensors_1.0M": (cfm.ConvolForwardNet(**spec, useBatchNorm=True, useAffineTransformInBatchNorm=True).to(dev), 16, True),
        "wrn16-22_60_tensors_82.7M": (Wide_ResNet(depth=16, widen_factor=22, dropout_rate=0.3, num_classes=10).to(dev), 4, False),
    }
    res = {}
    for name, (model, s, first_last) in models.items():
        params = [p.data for p in cfm._selected_parameters(model, first_last)]
        numel = sum(p.numel() for p in params)
        plan = QuantizationPlan(params, s, 256)
        grads = [torch.randn_like(p) for p in params]
        iters = 100 if numel < 5e6 else 20
        r = {"tensors": len(params), "numel": numel, "levels": s, "bucket": 256}
        r["plan_save_us"] = timed(plan.save_master, iters)
        plan.save_master()
        r["plan_quantize_us"] = timed(plan.quantize_, iters)
        r["plan_restore_us"] = timed(plan.restore_master, iters)
        r["plan_backward_minmax_us"] = timed(lambda: plan.backward_(grads, "complicated"), iters)
        plan.restore_master()
        plan.restore_master()
        r["plan_save_and_quantize_us"] = timed(lambda: (plan.restore_master(), plan.save_and_quantize_()), iters) - r["plan_restore_us"]
        plan.restore_master()
        r["plan_step_total_us"] = r["plan_save_and_quantize_us"] + r["plan_restore_us"]
        r["hbm_floor_us_20B_per_elt"] = numel * 20 / 3350e9 * 1e6

        def per_tensor():
            for p in params:
                Q.uniformQuantization(p, s, bucket_size=256, modify_in_place=True)
        r["per_tensor_api_quantize_us"] = timed(per_tensor, max(iters // 4, 5))
        plan.restore_master()

        saved = [p.clone() for p in params]

        def reference_chain():                      # conv_forward_model.py:286-302 with stock torch ops
            new = T.quantize_model_step(params, s, 256)
            for p, q_, m in zip(params, new, saved):
                p.copy_(m)                          # load_state_dict copy-back
            return new
        r["reference_torch_ops_on_gpu_us"] = timed(reference_chain, max(iters // 10, 3), warm=2)
        r["speedup_vs_reference_torch_ops_on_gpu"] = r["reference_torch_ops_on_gpu_us"] / r["plan_step_total_us"]
        # ---- round 2: the tail of a step (restore + fix-up + SGD) and the head of the next one (save + quantize)
        # unfused (four launches + torch's multi-tensor SGD) against the fused optimizer step (one launch, 24 B/elt)
        ref_params = [torch.nn.Parameter(p.clone()) for p in params]
        opt = torch.optim.SGD(ref_params, lr=1e-3, momentum=0.9, nesterov=True, weight_decay=2.2e-4)
        ref_plan = QuantizationPlan([p.data for p in ref_params], s, 256)
        for p, g_ in zip(ref_params, grads):
            p.grad = g_.clone()
        ref_plan.save_and_quantize_()

        def unfused_tail():
            ref_plan.restore_master()
            ref_plan.backward_([p.grad for p in ref_params], "complicated")
            opt.step()
            ref_plan.save_and_quantize_()
        r["unfused_restore_fixup_sgd_requantize_us"] = timed(unfused_tail, iters)
        plan.save_and_quantize_()
        if 256 <= 512:
            r["fused_sgd_step_us"] = timed(lambda: plan.fused_step_(grads, "complicated", 1e-3, 0.9, 2.2e-4, True), iters)
            r["fused_sgd_hbm_floor_us_24B_per_elt"] = numel * 24 / 3350e9 * 1e6
        # ---- differentiable-quantization step: CentroidPlan (3 launches for the model) vs the per-tensor ops
        from quantized_distillation_b200.plan import CentroidPlan
        src = [p.clone() for p in params]
        pts = [torch.linspace(0, 1, 4, device=dev) for _ in params]
        cplan = CentroidPlan(src, [torch.empty_like(t) for t in src], pts, 256)
        funs = [Q.nonUniformQuantization_variable(bucket_size=256, pre_process_tensors=True, tensor=t) for t in src]

        def per_tensor_centroids():
            for f_, pt, g_ in zip(funs, pts, grads):
                f_.forward(None, pt)
                f_.backward(g_)

        def plan_centroids():
            cplan.forward_()
            cplan.backward_(grads)
        r["centroid_step_per_tensor_ops_us"] = timed(per_tensor_centroids, max(iters // 4, 5))
        r["centroid_step_plan_us"] = timed(plan_centroids, iters)
        res[name] = {k: (round(v, 2) if isinstance(v, float) else v) for k, v in r.items()}
        del plan, ref_plan, cplan
    # single big tensor: stock torch chain vs fused kernel (BASELINE config 5 flavour)
    n = 1 << 26
    x = torch.randn(n, device=dev) * 0.05
    res["single_64Mi_tensor"] = {
        "reference_torch_ops_on_gpu_uniform_fwd_us": round(timed(lambda: T.uniform_fwd(x, 16, 256), 5, 2), 1),
        "ours_uniform_fwd_us": round(timed(lambda: Q.uniformQuantization(x, 16, bucket_size=256), 20, 3), 1),
    }
    out_path = out_path or os.path.join(ROOT, "gpurun_out", "plan_bench.json")
    os.makedirs(os.path.dirname(out_path), exist_ok=True)
    json.dump(res, open(out_path, "w"), indent=1)
    print(json.dumps(res, indent=1))
    return out_path


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    run(ap.parse_args().out)
