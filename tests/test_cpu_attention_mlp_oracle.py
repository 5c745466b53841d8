"""The float64 oracle of "mlp" (Bahdanau) global attention (oracle/attention_mlp_oracle.py) against the reference's own
GlobalAttention(attn_type="mlp") run by tests/golden/make_golden_attention_mlp.py
(tests/golden/reference_attention_mlp.npz): outputs and the gradients of the input, the memory bank and all six
weights, one-step and multi-step, S = 1, H = 1, H = 33 and S up to 40; the fused core composes to the module; the
stated bounds cover a float32 evaluation of the chain."""
import importlib.util
import os

import numpy as np
import pytest

from oracle import attention_mlp_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "golden", "reference_attention_mlp.npz")
DATA = np.load(FIXTURE)
CASES = DATA["cases"]
WEIGHTS = ("w_ctx", "w_q", "b_q", "v", "w_out", "b_out")


def _close(got, want):
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12 * max(1.0, np.abs(want).max()))


def _case(i):
    return {k[len(f"c{i}_"):]: DATA[k] for k in DATA.files if k.startswith(f"c{i}_")}


@pytest.mark.parametrize("i", range(len(CASES)))
def test_oracle_reproduces_reference(i):
    N, T, S, H = CASES[i].tolist()
    d = _case(i)
    context = d["bank"].transpose(1, 0, 2)
    o = O.mlp_global_attention(d["input"], context, *(d[w] for w in WEIGHTS), d["grad_h"], d["grad_align"])
    _close(o["attn_h"], d["attn_h"])
    _close(o["align"], d["align"])
    _close(o["grad_input"], d["grad_input"])
    _close(o["grad_context"].transpose(1, 0, 2), d["grad_bank"])
    for w in WEIGHTS:
        _close(o["grad_" + w], d["grad_" + w])
    assert d["attn_h"].shape == ((N, H) if T == 0 else (T, N, H))
    assert d["align"].shape == ((N, S) if T == 0 else (T, N, S))


@pytest.mark.parametrize("i", [0, 6, 9])
def test_core_composes_to_the_module(i):
    """mlp_core() is the middle of mlp_global_attention(): on the fixture's projections it gives the reference's align,
    linear_out of its concat gives attn_h, and its gradients carried through the projections give the reference's."""
    d = _case(i)
    x = d["input"] if d["input"].ndim == 3 else d["input"][:, None, :]
    ctx = d["bank"].transpose(1, 0, 2)
    wq, uh = x @ d["w_q"].T + d["b_q"], ctx @ d["w_ctx"].T
    T = x.shape[1]
    g_h = d["grad_h"].reshape(T, *d["grad_h"].shape[-2:])
    g_a = d["grad_align"].reshape(T, *d["grad_align"].shape[-2:])
    gc = g_h @ d["w_out"]                                                   # the gradient of concat
    c = O.mlp_core(wq, uh, d["v"], x, ctx, g_a, gc)
    _close(c["align"].reshape(d["align"].shape), d["align"])
    _close((c["concat"] @ d["w_out"].T + d["b_out"]).reshape(d["attn_h"].shape), d["attn_h"])
    _close(c["grad_v"], d["grad_v"][0])
    _close(np.einsum("nth,nti->hi", c["grad_wq"], x), d["grad_w_q"])
    _close(c["grad_wq"].sum((0, 1)), d["grad_b_q"])
    _close(np.einsum("nsh,nsi->hi", c["grad_uh"], ctx), d["grad_w_ctx"])
    grad_bank = (c["grad_context"] + c["grad_uh"] @ d["w_ctx"]).transpose(1, 0, 2)
    _close(grad_bank, d["grad_bank"])
    grad_x = c["grad_input"] + c["grad_wq"] @ d["w_q"]
    _close(grad_x.reshape(d["grad_input"].shape), d["grad_input"])


def test_bounds_cover_float32_rounding_of_the_inputs():
    """The stated bounds are positive; a float32 evaluation of the same chain (numpy's tanh) lies within them."""
    rng = np.random.default_rng(4)
    Nb, T, S, H = 2, 3, 70, 40
    wq, uh, v = rng.standard_normal((Nb, T, H)), rng.standard_normal((Nb, S, H)), rng.standard_normal(H) * H ** -0.5
    inp, ctx = rng.standard_normal((Nb, T, H)), rng.standard_normal((Nb, S, H))
    gc, ga = rng.standard_normal((T, Nb, 2 * H)), rng.standard_normal((T, Nb, S))
    b = O.mlp_core_bounds(wq, uh, v, inp, ctx, ga, gc)
    o = O.mlp_core(wq, uh, v, inp, ctx, ga, gc)
    f = np.float32
    e = np.tanh(wq.astype(f)[:, :, None, :] + uh.astype(f)[:, None, :, :])
    s = (e * v.astype(f)).sum(-1, dtype=f)
    p = np.exp(s - s.max(2, keepdims=True))
    p = (p / p.sum(2, keepdims=True)).astype(f).transpose(1, 0, 2)
    assert np.all(np.abs(p - o["align"]) <= b["align"])
    assert all(np.all(v > 0) for v in b.values())
    assert set(b) == {"align", "c", "grad_wq", "grad_uh", "grad_v", "grad_context"}


def test_fixture_is_small_and_regenerates():
    assert os.path.getsize(FIXTURE) < 1 << 20
    spec = importlib.util.spec_from_file_location("make_golden_attention_mlp",
                                                  os.path.join(HERE, "golden", "make_golden_attention_mlp.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    assert [list(c) for c in CASES] == [list(c) for c in gen.CASES]
    T0 = [c for c in gen.CASES if c[1] == 0]
    assert T0 and len(T0) < len(gen.CASES)                        # one step and several steps
    assert any(c[2] == 1 for c in gen.CASES) and any(c[3] == 1 for c in gen.CASES)
    assert any(c[3] == 33 for c in gen.CASES) and any(c[2] >= 33 for c in gen.CASES)
