"""The NumPy beam oracle (oracle/beam_oracle.py) against the reference's own onmt/Beam.py, executed by
tests/golden/make_golden_beam.py into tests/golden/reference_beam.npz: every step's scores, back pointers and tokens,
done(), the order of sortFinished (with the `minimum` quirk) and getHyp's hypotheses and attention, bit for bit, at
K in {1, 2, 5, 8, 16}, n_best in {1, 2, 3} and V from K to 1,000."""
import importlib.util
import os

import numpy as np
import pytest

from oracle import beam_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))


def _gen():
    spec = importlib.util.spec_from_file_location("make_golden_beam", os.path.join(HERE, "golden", "make_golden_beam.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


G = _gen()
DATA = np.load(os.path.join(HERE, "golden", "reference_beam.npz"))
N_CASES = int(DATA["n_cases"])


def case(c):
    return {k[len(f"c{c}_"):]: DATA[k] for k in DATA.files if k.startswith(f"c{c}_")}


def replay(c):
    """The oracle's batch of Beams on the case's inputs, as translateBatch drives them."""
    r = case(c)
    seed, K, n_best, V, B, max_len, T = (int(v) for v in r["meta"])
    eos = G.eos_of(V)
    steps = iter(range(T))

    def step(inp):
        i = next(steps)
        return G.draw(seed, i, int(r["attempts"][i]), K * B, V, float(r["eos_scale"]))

    hyps, scores, attn, beams = O.translate_batch(step, B, K, n_best, max_len, G.BOS, eos, G.PAD)
    return r, (K, n_best, V, B, T), (hyps, scores, attn, beams)


@pytest.mark.parametrize("c", range(N_CASES))
def test_oracle_replays_reference_beam(c):
    r, (K, n_best, V, B, T), (hyps, scores, attn, beams) = replay(c)
    assert all(len(b.prevKs) == T for b in beams)
    for t in range(T):
        for j, b in enumerate(beams):
            assert np.array_equal(b.prevKs[t], r["prev"][t, j]), (t, j)
            assert np.array_equal(b.nextYs[t + 1], r["next"][t + 1, j]), (t, j)
    # the scores after each step, bit for bit (the oracle keeps only the last; re-run step by step to see each)
    r2 = case(c)
    seed = int(r2["meta"][0])
    bs = [O.Beam(K, n_best, G.BOS, G.eos_of(V), G.PAD) for _ in range(B)]
    for t in range(T):
        lp, at = G.draw(seed, t, int(r["attempts"][t]), K * B, V, float(r["eos_scale"]))
        lp, at = lp.reshape(K, B, V), at.reshape(K, B, -1)
        for j, b in enumerate(bs):
            b.advance(lp[:, j], at[:, j])
            assert np.array_equal(b.scores.view(np.uint32), r["scores"][t, j].view(np.uint32)), (t, j)
            assert b.done() == bool(r["done"][t, j]), (t, j)
    # sortFinished(minimum=n_best) and getHyp
    fs, ftk = np.split(r["fin_scores"], np.cumsum(r["n_finished"])[:-1]), np.split(r["fin_tk"], np.cumsum(r["n_finished"])[:-1])
    lens = iter(r["hyp_len"].tolist())
    tok_off = att_off = 0
    for j, b in enumerate(beams):
        assert np.array_equal(np.array(scores[j], np.float32).view(np.uint32), fs[j].view(np.uint32)), j
        assert [(t, int(k)) for _, t, k in b.finished] == [tuple(x) for x in ftk[j].tolist()], j
        for n in range(n_best):
            L = next(lens)
            assert hyps[j][n] == r["hyp_tok"][tok_off:tok_off + L].tolist(), (j, n)
            assert np.array_equal(attn[j][n].view(np.uint32), r["hyp_attn"][att_off:att_off + L].view(np.uint32)), (j, n)
            tok_off += L
            att_off += L


def test_fixture_covers_the_documented_ground():
    Ks, nbs, Vs, on_done, on_limit, quirk, eos_rows = set(), set(), [], 0, 0, 0, 0
    for c in range(N_CASES):
        r = case(c)
        seed, K, n_best, V, B, max_len, T = (int(v) for v in r["meta"])
        Ks.add(K), nbs.add(n_best), Vs.append(V)
        if T < max_len:
            on_done += 1
        else:
            on_limit += 1
        # short of n_best finished, sortFinished appended the top beam of the last step again and again
        for j, tk in enumerate(np.split(r["fin_tk"], np.cumsum(r["n_finished"])[:-1])):
            quirk += sum(1 for t, k in tk.tolist() if t == T and k == 0) > 1
        eos = G.eos_of(V)
        eos_rows += int(np.sum(r["next"][1:T] == eos))       # beams that ended on EOS and had -1e20 rows next step
    assert Ks == {1, 2, 5, 8, 16} and nbs == {1, 2, 3}
    assert min(Vs) <= 2 and max(Vs) >= 1000 and any(V == K for K, V in ((int(case(c)["meta"][1]), int(case(c)["meta"][3])) for c in range(N_CASES)))
    assert on_done >= 3 and on_limit >= 3 and quirk >= 1 and eos_rows >= 20
    assert os.path.getsize(os.path.join(HERE, "golden", "reference_beam.npz")) < 1 << 20


def test_top_k_order_and_ties():
    k = np.array([1.0, np.nan, 3.0, 3.0, -np.inf, np.inf, -0.0, 0.0, np.nan], np.float32)
    assert O.top_k(k, 9).tolist() == [1, 8, 5, 2, 3, 0, 6, 7, 4]
    assert O.top_k(np.full(7, -1e20, np.float32), 3).tolist() == [0, 1, 2]
