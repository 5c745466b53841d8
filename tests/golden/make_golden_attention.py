"""Generates tests/golden/reference_attention.npz: the reference's own onmt/modules/GlobalAttention.py (with its
UtilClass.py), loaded unmodified by file path with a stub onmt.Utils.aeq, run in float64 on the CPU as the decoders
call it (onmt/Models.py:254-257, 338-339): the context is the transpose of a contiguous [S, N, H] memory bank; a
one-step input is [N, H], a multi-step input the contiguous [N, T, H].  Its nn.Softmax() without a dim takes dim 1 of
the [N*T, S] scores: the source axis.

Per case: the inputs (float32 values, stored as float64), the weights, both outputs and, for random upstream gradients
of both outputs, the gradients of the input, the memory bank and every weight.  The file is written with fixed zip
timestamps, so a rerun gives the same bytes.

Run in the build container only:  python tests/golden/make_golden_attention.py
"""
import importlib.util
import io
import os
import sys
import types
import zipfile

import numpy as np

REF = "/root/reference/onmt/modules"
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_attention.npz")

# (attn_type, N, T (0: one step), S, H)
CASES = [
    ("general", 3, 0, 5, 4), ("dot", 3, 0, 5, 4), ("general", 2, 0, 1, 1), ("dot", 1, 0, 1, 3),
    ("general", 4, 0, 7, 3), ("general", 2, 0, 9, 33), ("dot", 5, 0, 3, 7),
    ("general", 3, 4, 6, 7), ("dot", 2, 3, 4, 5), ("general", 2, 3, 1, 2), ("general", 2, 2, 3, 1), ("dot", 3, 5, 33, 9),
]


def _load_global_attention():
    import torch.nn  # noqa: F401  (the reference modules import torch themselves)
    onmt = types.ModuleType("onmt")
    utils = types.ModuleType("onmt.Utils")

    def aeq(*args):
        assert all(a == args[0] for a in args[1:]), f"size mismatch {args}"
    utils.aeq = aeq
    modules = types.ModuleType("onmt.modules")
    onmt.Utils, onmt.modules = utils, modules
    sys.modules.update({"onmt": onmt, "onmt.Utils": utils, "onmt.modules": modules})
    for name in ("UtilClass", "GlobalAttention"):
        spec = importlib.util.spec_from_file_location(f"onmt.modules.{name}", os.path.join(REF, f"{name}.py"))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[f"onmt.modules.{name}"] = mod
        spec.loader.exec_module(mod)
        setattr(modules, name, mod)
    return sys.modules["onmt.modules.GlobalAttention"].GlobalAttention


def _f32(rng, *shape, scale=1.0):
    return (rng.standard_normal(shape) * scale).astype(np.float32).astype(np.float64)


def run_case(torch, GA, i, attn_type, N, T, S, H):
    rng = np.random.default_rng([7, i])
    m = GA(H, attn_type=attn_type).double()
    with torch.no_grad():
        if attn_type == "general":
            m.linear_in.weight.copy_(torch.from_numpy(_f32(rng, H, H, scale=H ** -0.5)))
        m.linear_out.weight.copy_(torch.from_numpy(_f32(rng, H, 2 * H, scale=(2 * H) ** -0.5)))
    inp = _f32(rng, *((N, H) if T == 0 else (N, T, H)))
    bank = _f32(rng, S, N, H)
    x = torch.tensor(inp, requires_grad=True)
    mb = torch.tensor(bank, requires_grad=True)
    attn_h, align = m(x, mb.transpose(0, 1))
    g_h = _f32(rng, *attn_h.shape)
    g_a = _f32(rng, *align.shape)
    ((attn_h * torch.from_numpy(g_h)).sum() + (align * torch.from_numpy(g_a)).sum()).backward()
    out = {"input": inp, "bank": bank, "w_out": m.linear_out.weight.detach().numpy().copy(),
           "attn_h": attn_h.detach().numpy(), "align": align.detach().numpy(), "grad_h": g_h, "grad_align": g_a,
           "grad_input": x.grad.numpy(), "grad_bank": mb.grad.numpy(), "grad_w_out": m.linear_out.weight.grad.numpy()}
    if attn_type == "general":
        out["w_in"] = m.linear_in.weight.detach().numpy().copy()
        out["grad_w_in"] = m.linear_in.weight.grad.numpy()
    return {f"c{i}_{k}": v for k, v in out.items()}


def _write_npz(path, arrays):
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asarray(arrays[k]), allow_pickle=False)
            z.writestr(zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0)), buf.getvalue(), zipfile.ZIP_DEFLATED)


def main():
    import warnings

    import torch
    GA = _load_global_attention()
    out = {"cases": np.array([[["dot", "general"].index(a), N, T, S, H] for a, N, T, S, H in CASES], np.int64)}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")        # nn.Softmax() without a dim
        for i, c in enumerate(CASES):
            out.update(run_case(torch, GA, i, *c))
    _write_npz(OUT, out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
