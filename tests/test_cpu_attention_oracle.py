"""The float64 oracle of global attention (oracle/attention_oracle.py) against the reference's own GlobalAttention run by
tests/golden/make_golden_attention.py (tests/golden/reference_attention.npz): outputs and the gradients of the input,
the memory bank and every weight, "dot" and "general", one-step and multi-step, S = 1, H = 1 and odd H."""
import importlib.util
import os

import numpy as np
import pytest

from oracle import attention_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "golden", "reference_attention.npz")
DATA = np.load(FIXTURE)
CASES = DATA["cases"]


def _close(got, want):
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12 * max(1.0, np.abs(want).max()))


@pytest.mark.parametrize("i", range(len(CASES)))
def test_oracle_reproduces_reference(i):
    kind, N, T, S, H = CASES[i].tolist()
    attn_type = ["dot", "general"][kind]
    d = {k[len(f"c{i}_"):]: DATA[k] for k in DATA.files if k.startswith(f"c{i}_")}
    context = d["bank"].transpose(1, 0, 2)
    o = O.global_attention(d["input"], context, attn_type, d.get("w_in"), d["w_out"], d["grad_h"], d["grad_align"])
    _close(o["attn_h"], d["attn_h"])
    _close(o["align"], d["align"])
    _close(o["grad_input"], d["grad_input"])
    _close(o["grad_context"].transpose(1, 0, 2), d["grad_bank"])
    _close(o["grad_w_out"], d["grad_w_out"])
    if attn_type == "general":
        _close(o["grad_w_in"], d["grad_w_in"])
    assert d["attn_h"].shape == ((N, H) if T == 0 else (T, N, H))
    assert d["align"].shape == ((N, S) if T == 0 else (T, N, S))


def test_core_composes_to_the_module():
    """core() is the middle of global_attention(): the same align, and concat feeds linear_out + tanh."""
    rng = np.random.default_rng(3)
    x, ctx, w = rng.standard_normal((3, 4, 5)), rng.standard_normal((3, 6, 5)), rng.standard_normal((5, 10))
    c = O.core(x, x, ctx)
    m = O.global_attention(x, ctx, "dot", None, w)
    _close(c["align"], m["align"])
    _close(np.tanh(c["concat"] @ w.T), m["attn_h"])


def test_bounds_cover_float32_rounding_of_the_inputs():
    """The stated bounds are positive and grow with the magnitudes; a float32 evaluation of the same chain lies within."""
    rng = np.random.default_rng(4)
    q, inp, ctx = rng.standard_normal((2, 3, 40)), rng.standard_normal((2, 3, 40)), rng.standard_normal((2, 70, 40))
    gc, ga = rng.standard_normal((3, 2, 80)), rng.standard_normal((3, 2, 70))
    b = O.core_bounds(q, inp, ctx, ga, gc)
    o = O.core(q, inp, ctx, ga, gc)
    s = np.einsum("nth,nsh->nts", q.astype(np.float32), ctx.astype(np.float32)).astype(np.float32)
    p = np.exp(s - s.max(2, keepdims=True))
    p = (p / p.sum(2, keepdims=True)).astype(np.float32).transpose(1, 0, 2)
    assert np.all(np.abs(p - o["align"]) <= b["align"])
    assert all(np.all(v > 0) for v in b.values())


def test_fixture_is_small_and_regenerates():
    assert os.path.getsize(FIXTURE) < 1 << 20
    spec = importlib.util.spec_from_file_location("make_golden_attention", os.path.join(HERE, "golden", "make_golden_attention.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    assert [list(c) for c in CASES] == [[["dot", "general"].index(a), N, T, S, H] for a, N, T, S, H in gen.CASES]
