"""The float64 oracle of the SRU recurrence (oracle/sru_oracle.py) against the reference's own SRU kernels compiled for
the CPU by tests/golden/make_golden_sru.py (tests/golden/reference_sru.npz): h, c, grad_u, grad_x, the batch-summed
grad_bias and grad_init within the oracle's float32 bounds, both directions, k = 3 and 4, the three activations, with
and without mask_h, len 1 and len > 1, zero and non-zero init and grad_last."""
import os

import numpy as np
import pytest

from oracle import sru_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
DATA = np.load(os.path.join(HERE, "golden", "reference_sru.npz"))
CASES = DATA["cases"]


def case(i):
    return {k[len(f"c{i}_"):]: DATA[k] for k in DATA.files if k.startswith(f"c{i}_")}


def oracle(i, d_):
    bi, k, act, _, L, B, d, _, _ = CASES[i].tolist()
    return O.sru(d_["u"], d_.get("x"), d_["bias"], d, bool(bi), act, init=d_["init"], mask_h=d_.get("mask_h"),
                 grad_h=d_["grad_h"], grad_last=d_["grad_last"])


@pytest.mark.parametrize("i", range(len(CASES)))
def test_oracle_bounds_the_reference_kernels(i):
    d_ = case(i)
    vals, errs = oracle(i, d_)
    bnd = O.bounds(errs, CASES[i][4])
    got = dict(d_, grad_bias=d_["grad_bias_partial"].astype(np.float64).sum(1).reshape(-1))
    names = ["h", "c", "grad_u", "grad_bias", "grad_init"] + (["grad_x"] if "x" in d_ else [])
    for name in names:
        err = np.abs(got[name].astype(np.float64) - vals[name])
        assert np.all(err <= bnd[name]), f"{name}: worst err/bound {(err / bnd[name]).max():.3f}"
    assert vals["h"].shape == d_["h"].shape and vals["grad_u"].shape == d_["u"].shape


def test_fixture_covers_the_matrix():
    bi, k, act, mask, L, init, gl = (set(CASES[:, j].tolist()) for j in (0, 1, 2, 3, 4, 7, 8))
    assert bi == {0, 1} and k == {3, 4} and act == {0, 1, 2} and mask == {0, 1} and init == {0, 1} and gl == {0, 1}
    assert 1 in L and max(L) > 1


def test_bounds_are_tight_enough_to_mean_something():
    # the bound of a well-conditioned case stays within a few hundred ulps of the values it bounds
    d_ = case(0)
    vals, errs = oracle(0, d_)
    bnd = O.bounds(errs, CASES[0][4])
    assert np.all(bnd["h"] <= 1e-4 * (1 + np.abs(vals["h"])))
    assert np.all(bnd["grad_u"] <= 1e-4 * (1 + np.abs(vals["grad_u"])))
