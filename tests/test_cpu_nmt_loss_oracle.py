"""The float64 oracle of the fused NMT loss (oracle/nmt_loss_oracle.py) against the reference's formula
(onmt/Loss.py:97-120, 68-77) restated in float64 torch: log_softmax, nll_loss with weight 0 at the padding index,
kl_div to exp(teacher log-probs) with the padding rows masked, the stats' argmax, and autograd for the gradient."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import nmt_loss_oracle as O


def reference(zs, y, padding_idx, zt=None, w=0.7):
    """(loss, grad, [n_words, n_correct]) of the reference chain in float64 torch."""
    zs = torch.tensor(zs, dtype=torch.float64, requires_grad=True)
    y = torch.tensor(y, dtype=torch.int64)
    V = zs.shape[1]
    weight = torch.ones(V, dtype=torch.float64)
    if padding_idx >= 0:
        weight[padding_idx] = 0
    scores = F.log_softmax(zs, dim=1)
    loss = F.nll_loss(scores, y, weight=weight, reduction="sum")
    if zt is not None:
        w = float(np.float32(w))             # the ABI takes the weight as float32
        pt = F.log_softmax(torch.tensor(zt, dtype=torch.float64), dim=1).exp()
        kl = F.kl_div(scores, pt, reduction="none")
        # the reference's torch summed target * (log target - input) only where target > 0 (current torch's xlogy form
        # gives 0 * inf = NaN where the target is 0 and the input -inf); the padding rows are what its weight= meant
        kl = torch.where(pt > 0, kl, torch.zeros_like(kl))
        keep = (y != padding_idx).to(torch.float64)[:, None]
        loss = (1 - w) * loss + w * (kl * keep).sum()
    loss.backward()
    non_padding = y.ne(padding_idx)
    pred = scores.max(1)[1]
    n_correct = int(pred.eq(y).masked_select(non_padding).sum())
    return loss.item(), zs.grad.numpy(), [int(non_padding.sum()), n_correct]


def check(zs, y, padding_idx, zt=None, w=0.7):
    o = O.nmt_loss(zs, y, padding_idx, zt, w)
    loss, grad, counts = reference(zs, y, padding_idx, zt, w)
    if not np.isfinite(loss):
        np.testing.assert_equal(o["loss"], loss)
    else:
        assert o["loss"] == pytest.approx(loss, rel=1e-12, abs=1e-12)
    np.testing.assert_allclose(o["grad"], grad, rtol=0, atol=1e-12)
    assert list(o["counts"]) == counts + [0]
    return o


@pytest.mark.parametrize("teacher", [False, True])
@pytest.mark.parametrize("w", [0.0, 0.7, 1.0])
@pytest.mark.parametrize("padding_idx", [-1, 0, 1])
def test_oracle_matches_reference_formula(teacher, w, padding_idx):
    rng = np.random.default_rng(17)
    R, V = 37, 53
    zs = rng.standard_normal((R, V)) * 3
    zt = rng.standard_normal((R, V)) * 3 if teacher else None
    y = rng.integers(0, V, R)
    if padding_idx >= 0:
        y[::4] = padding_idx
    check(zs, y, padding_idx, zt, w)


@pytest.mark.parametrize("w", [0.0, 0.7, 1.0])
def test_minus_inf_logits(w):
    rng = np.random.default_rng(3)
    R, V = 16, 40
    zs = rng.standard_normal((R, V))
    zt = rng.standard_normal((R, V))
    y = rng.integers(0, V, R)
    # student and teacher -inf together: the teacher term is 0, not 0 * inf
    both = rng.random((R, V)) < 0.3
    zs[both] = -np.inf
    zt[both] = -np.inf
    # teacher alone -inf: its term is 0 as well
    zt[rng.random((R, V)) < 0.2] = -np.inf
    y = np.where(np.isinf(zs[np.arange(R), y]), np.argmax(zs, axis=1), y)
    o = check(zs, y, 1, zt, w)
    assert np.isfinite(o["loss"]) and np.isfinite(o["grad"]).all()
    # a student -inf where the teacher is positive: the KL is +inf, the gradient stays finite
    zs2 = zs.copy()
    zs2[0, np.flatnonzero(np.isfinite(zt[0]) & (np.arange(V) != y[0]))[0]] = -np.inf
    o2 = check(zs2, y, -1, zt, w)
    assert np.isfinite(o2["grad"]).all()
    if w > 0:
        assert o2["loss"] == np.inf        # (at w = 0 the term is 0 * inf: NaN, in the reference as here)
    # student -inf at the target: the NLL is +inf
    zs3 = zs.copy()
    zs3[2, y[2]] = -np.inf
    assert check(zs3, y, -1, None, w)["loss"] == np.inf


@pytest.mark.parametrize("teacher", [False, True])
def test_all_padding_rows(teacher):
    rng = np.random.default_rng(5)
    R, V = 9, 11
    zs = rng.standard_normal((R, V))
    zt = rng.standard_normal((R, V)) if teacher else None
    y = np.zeros(R, np.int64)
    o = check(zs, y, 0, zt)
    assert o["loss"] == 0.0 and not o["grad"].any() and list(o["counts"]) == [0, 0, 0]
    # padding rows among others contribute nothing
    y2 = rng.integers(1, V, R)
    y2[[1, 4, 7]] = 0
    full = O.nmt_loss(zs, y2, 0, zt)
    keep = y2 != 0
    part = O.nmt_loss(zs[keep], y2[keep], 0, None if zt is None else zt[keep])
    assert full["loss"] == pytest.approx(part["loss"], rel=1e-14)
    assert not full["grad"][~keep].any()


def test_argmax_ties_take_first_occurrence():
    rng = np.random.default_rng(9)
    R, V = 20, 30
    zs = rng.standard_normal((R, V))
    first = rng.integers(0, V // 2, R)
    second = first + rng.integers(1, V // 2, R)
    top = zs.max(axis=1) + 1.0
    zs[np.arange(R), first] = top
    zs[np.arange(R), second] = top
    y = np.where(np.arange(R) % 2 == 0, first, second)       # even rows hit the first tie, odd rows the second
    o = check(zs, y, -1, None)
    assert list(o["argmax"]) == list(first)
    assert o["counts"][1] == (R + 1) // 2


def test_invalid_targets_are_nan_and_counted():
    rng = np.random.default_rng(1)
    zs = rng.standard_normal((6, 10))
    y = np.array([3, -1, 10, 0, 12, 2])
    o = O.nmt_loss(zs, y, 0, zs[::-1].copy())
    assert np.isnan(o["loss"]) and list(o["counts"]) == [2, int(o["argmax"][0] == 3) + int(o["argmax"][5] == 2), 3]
    assert np.isnan(o["grad"][[1, 2, 4]]).all() and not o["grad"][3].any() and np.isfinite(o["grad"][[0, 5]]).all()


def test_teacher_term_against_student_minus_inf_is_inf_even_when_p_t_underflows():
    # p_t = exp(-1000 - lse_t) is 0 in float64, yet a positive teacher probability against a zero student one is +inf
    zs = np.array([[0.0, 1.0, -np.inf, 0.5]])
    zt = np.array([[0.0, 1.0, -1000.0, 0.5]])
    assert O.nmt_loss(zs, np.array([1]), -1, zt, 0.7)["loss"] == np.inf
    zt[0, 2] = -np.inf                       # teacher -inf there: the column adds 0
    o = check(zs, np.array([1]), -1, zt, 0.7)
    assert np.isfinite(o["loss"])
