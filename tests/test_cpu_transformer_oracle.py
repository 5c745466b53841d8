"""The float64 oracle of onmt's Transformer sublayers (oracle/mha_oracle.py) against the reference's own modules run by
tests/golden/make_golden_transformer.py (tests/golden/reference_transformer.npz): MultiHeadedAttention (self and
context attention, Lq != Lk, no mask, padding, padding plus subsequent, an all-masked row, dh = 1, one key),
BottleLayerNorm (2-D, 3-D, width 1), PositionwiseFeedForward, TransformerEncoderLayer and TransformerDecoderLayer:
outputs and the gradients of the inputs and of every parameter."""
import importlib.util
import os

import numpy as np
import pytest

from oracle import mha_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "golden", "reference_transformer.npz")
DATA = np.load(FIXTURE)


def _gen():
    spec = importlib.util.spec_from_file_location("make_golden_transformer",
                                                  os.path.join(HERE, "golden", "make_golden_transformer.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    return gen


CASES = _gen().CASES


def _case(name):
    pre = name + "/"
    return {k[len(pre):]: DATA[k] for k in DATA.files if k.startswith(pre)}


def _params(d):
    return {k[2:]: v for k, v in d.items() if k.startswith("p_")}


def _close(got, want):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape
    assert np.array_equal(np.isnan(got), np.isnan(want))
    fin = ~np.isnan(want)
    scale = max(1.0, np.abs(want[fin]).max()) if fin.any() else 1.0
    np.testing.assert_allclose(got[fin], want[fin], rtol=1e-12, atol=1e-12 * scale)


def _oracle(kind, sz, d):
    P = _params(d)
    if kind == "mha":
        B, Lq, Lk, dm, h, mk = sz
        ctx = d.get("context", d["query"])
        return O.multi_headed_attention(P, ctx, ctx, d["query"], h, d.get("mask"), [d["g0"], d["g1"]])
    if kind == "ln":
        o = O.bottle_layer_norm(d["x"], P["a_2"], P["b_2"], 1e-3, d["g0"])
        return {"out0": o["y"], "grad_in0": o["grad_x"], "grad_a_2": o["grad_a_2"], "grad_b_2": o["grad_b_2"]}
    if kind == "ffn":
        return O.feed_forward(P, d["x"], [d["g0"]])
    if kind == "enc":
        return O.encoder_layer(P, d["x"], d["mask"], sz[3], [d["g0"]])
    return O.decoder_layer(P, d["x"], d["context"], d["src_pad_mask"], d["tgt_pad_mask"], sz[4], [d["g0"], d["g1"]])


@pytest.mark.parametrize("name,kind,sz", CASES, ids=[c[0] for c in CASES])
def test_oracle_reproduces_reference(name, kind, sz):
    d = _case(name)
    o = _oracle(kind, sz, d)
    outs = [k for k in d if k.startswith("out")]
    grads = [k for k in d if k.startswith("grad_")]
    assert outs and grads
    for k in outs + grads:
        if k == "grad_in0" and kind == "mha" and "context" not in d:
            _close(o["grad_in0"] + o["grad_in1"] + o["grad_in2"], d["grad_in2"])     # key, value and query are one
            continue
        if k == "grad_in2" and kind == "mha" and "context" not in d:
            continue
        if k == "grad_in0" and kind == "mha":
            _close(o["grad_in0"] + o["grad_in1"], d["grad_in0"])                      # key and value are one tensor
            continue
        _close(o[k], d[k])


def test_fixture_covers_the_issue_cases():
    mha = {n: _case(n) for n, k, _ in CASES if k == "mha"}
    assert any(np.isnan(d["out0"]).any() for d in mha.values()), "one case has an all-masked row"
    assert any("mask" not in d for d in mha.values()) and any("mask" in d for d in mha.values())
    assert any(d["out1"].shape[1] != d["out1"].shape[2] for d in mha.values()), "Lq != Lk"
    assert any(_case(n)["x"].shape[-1] == 1 for n, k, _ in CASES if k == "ln"), "width 1"


def test_state_dict_keys_of_the_layers():
    enc = [str(k) for k in DATA["keys/encoder_layer"]]
    dec = [str(k) for k in DATA["keys/decoder_layer"]]
    assert "self_attn.linear_keys.weight" in enc and "feed_forward.layer_norm.a_2" in enc
    assert "context_attn.layer_norm.b_2" in dec and "mask" in dec


def test_core_composes_to_the_module():
    """core() and layer_norm() compose to multi_headed_attention()."""
    rng = np.random.default_rng(3)
    B, L, d, h = 2, 5, 16, 4
    x = rng.standard_normal((B, L, d))
    P = {f"linear_{n}.weight": rng.standard_normal((d, d)) / 4 for n in ("keys", "values", "query")}
    P.update({"layer_norm.a_2": 1 + rng.standard_normal(d) / 5, "layer_norm.b_2": rng.standard_normal(d) / 5})
    m = O.multi_headed_attention(P, x, x, x, h)
    c = O.core(x @ P["linear_query.weight"].T, x @ P["linear_keys.weight"].T, x @ P["linear_values.weight"].T, h)
    y = O.layer_norm(c["out"].reshape(B * L, d), P["layer_norm.a_2"], P["layer_norm.b_2"], 1e-3, x.reshape(B * L, d))
    _close(y["y"].reshape(B, L, d), m["out0"])
    _close(c["top"], m["out1"])


def test_bounds_cover_float32_rounding():
    """The stated bounds are positive where finite, and a float32 evaluation of the same chain lies within them."""
    rng = np.random.default_rng(4)
    B, Lq, Lk, h, dh = 2, 5, 37, 2, 40
    q, k, v = (rng.standard_normal((B, L, h * dh)) for L in (Lq, Lk, Lk))
    mask = rng.random((B, Lq, Lk)) < 0.3
    mask[:, :, 0] = False
    go, gt = rng.standard_normal((B, Lq, h * dh)), rng.standard_normal((B, Lq, Lk))
    b = O.core_bounds(q, k, v, h, mask, None, 0.0, go, gt)
    o = O.core(q, k, v, h, mask, None, 0.0, go, gt)
    f = O.core(q.astype(np.float32), k.astype(np.float32), v.astype(np.float32), h, mask)
    # a float64 chain on float32-rounded inputs stays within the bounds of rounding the inputs' products
    assert np.all(np.abs(f["top"] - o["top"]) <= b["top"] + 1e-6 * np.abs(o["top"]))
    assert all(np.all(v[np.isfinite(v)] >= 0) for v in b.values())
    x, a, bb = rng.standard_normal((7, 300)), 1 + rng.standard_normal(300) / 5, rng.standard_normal(300)
    r, gy = rng.standard_normal((7, 300)), rng.standard_normal((7, 300))
    lb = O.layer_norm_bounds(x, a, bb, 1e-3, r, gy)
    z = (x + r).astype(np.float32)
    mu = z.mean(1, keepdims=True, dtype=np.float32)
    sd = np.sqrt(((z - mu) ** 2).sum(1, keepdims=True, dtype=np.float32) / np.float32(299))
    y32 = (z - mu) / (sd + np.float32(1e-3)) * a.astype(np.float32) + bb.astype(np.float32)
    assert np.all(np.abs(y32 - O.layer_norm(x, a, bb, 1e-3, r)["y"]) <= lb["y"])
    assert all(np.all(v > 0) for v in lb.values())


def test_fixture_is_small():
    assert os.path.getsize(FIXTURE) < 1 << 20
