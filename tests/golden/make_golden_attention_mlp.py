"""Generates tests/golden/reference_attention_mlp.npz: the reference's own onmt/modules/GlobalAttention.py with
attn_type "mlp" (Bahdanau), loaded unmodified by make_golden_attention.py's loader (a stub onmt.Utils.aeq), run in
float64 on the CPU as the decoders call it: the context is the transpose of a contiguous [S, N, H] memory bank; a
one-step input is [N, H], a multi-step input the contiguous [N, T, H].

Per case: the inputs (float32 values, stored as float64), all six weights (linear_context.weight, linear_query.weight
and .bias, v.weight, linear_out.weight and .bias), both outputs and, for random upstream gradients of both outputs,
the gradients of the input, the memory bank and every weight.  The file is written with fixed zip timestamps, so a
rerun gives the same bytes.

Run in the build container only:  python tests/golden/make_golden_attention_mlp.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden_attention import _f32, _load_global_attention, _write_npz  # noqa: E402

OUT = os.path.join(HERE, "reference_attention_mlp.npz")

# (N, T (0: one step), S, H)
CASES = [(3, 0, 5, 4), (2, 0, 1, 3), (2, 0, 4, 1), (2, 0, 9, 33), (4, 0, 40, 6),
         (2, 3, 4, 5), (3, 4, 6, 7), (2, 2, 1, 2), (2, 3, 3, 1), (2, 3, 35, 9), (2, 2, 7, 33)]

# weight key in the state_dict -> (short name, shape of H)
WEIGHTS = [("linear_context.weight", "w_ctx"), ("linear_query.weight", "w_q"), ("linear_query.bias", "b_q"),
           ("v.weight", "v"), ("linear_out.weight", "w_out"), ("linear_out.bias", "b_out")]


def _weights(rng, H):
    return {"w_ctx": _f32(rng, H, H, scale=H ** -0.5), "w_q": _f32(rng, H, H, scale=H ** -0.5),
            "b_q": _f32(rng, H, scale=0.5), "v": _f32(rng, 1, H, scale=2 * H ** -0.5),
            "w_out": _f32(rng, H, 2 * H, scale=(2 * H) ** -0.5), "b_out": _f32(rng, H, scale=0.5)}


def run_case(torch, GA, i, N, T, S, H):
    rng = np.random.default_rng([11, i])
    m = GA(H, attn_type="mlp").double()
    w = _weights(rng, H)
    sd = m.state_dict()
    assert sorted(sd) == sorted(k for k, _ in WEIGHTS), sorted(sd)
    m.load_state_dict({k: torch.from_numpy(w[s]) for k, s in WEIGHTS}, strict=True)
    inp = _f32(rng, *((N, H) if T == 0 else (N, T, H)))
    bank = _f32(rng, S, N, H)
    x = torch.tensor(inp, requires_grad=True)
    mb = torch.tensor(bank, requires_grad=True)
    attn_h, align = m(x, mb.transpose(0, 1))
    g_h = _f32(rng, *attn_h.shape)
    g_a = _f32(rng, *align.shape)
    ((attn_h * torch.from_numpy(g_h)).sum() + (align * torch.from_numpy(g_a)).sum()).backward()
    params = dict(m.named_parameters())
    out = {"input": inp, "bank": bank, "attn_h": attn_h.detach().numpy(), "align": align.detach().numpy(),
           "grad_h": g_h, "grad_align": g_a, "grad_input": x.grad.numpy(), "grad_bank": mb.grad.numpy()}
    for k, s in WEIGHTS:
        out[s] = w[s]
        out["grad_" + s] = params[k].grad.numpy()
    return {f"c{i}_{k}": v for k, v in out.items()}


def main():
    import warnings

    import torch
    GA = _load_global_attention()
    out = {"cases": np.array([[N, T, S, H] for N, T, S, H in CASES], np.int64)}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")        # nn.Softmax() without a dim
        for i, c in enumerate(CASES):
            out.update(run_case(torch, GA, i, *c))
    _write_npz(OUT, out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
