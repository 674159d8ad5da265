"""CPU tests of the automatically scaled split's model (tests/train_range_ref.py): the host weight scale
b2second.tc.pow2_scale follows the same exponent rule, and the model itself keeps its stated properties."""
import numpy as np
import pytest
import torch

import train_range_ref as trr
from b2second import tc

CASES = trr.crafted_cases()


@pytest.mark.parametrize("name", sorted(CASES))
def test_pow2_scale_follows_the_rule(name):
    x = CASES[name]
    assert tc.pow2_scale(torch.from_numpy(x)) == 2.0 ** trr.exponent(x)


def test_exponent_edges():
    assert trr.exponent(CASES["all_zero"]) == 0 and trr.exponent(CASES["neg_zero"]) == 0
    assert trr.exponent(CASES["no_finite"]) == 0
    assert trr.exponent(CASES["max_2^12"]) == 1 and trr.exponent(CASES["max_2^13"]) == 0
    assert trr.exponent(CASES["max_above_2^13"]) == -1
    assert trr.exponent(CASES["flt_max"]) == 13 - 128
    assert trr.exponent(CASES["min_normal"]) == 126 and trr.exponent(CASES["below_clamp"]) == 126
    assert trr.exponent(CASES["min_subnormal"]) == 126
    # a non-finite element does not take the scale: the rest keeps the exponent it has alone
    for v in ("+inf", "-inf", "nan"):
        x = CASES[v + "_middle"]
        assert trr.exponent(x) == trr.exponent(np.where(np.isfinite(x), x, 0))


@pytest.mark.parametrize("name", sorted(CASES))
def test_split_model(name):
    x = CASES[name]
    e = trr.exponent(x)
    hi, lo = trr.split(x, e)
    fin = np.isfinite(x)
    assert trr.same_bits(hi[~fin], x[~fin].astype(np.float16))
    assert (lo[~fin].view(np.uint16) == 0).all()                 # +0
    assert np.isfinite(hi[fin]).all() and (np.abs(hi[fin].astype(np.float64)) <= 2.0 ** 13).all()
    v = x[fin].astype(np.float64) * 2.0 ** e
    err = np.abs(hi[fin].astype(np.float64) + lo[fin].astype(np.float64) - v)
    # 22 significant bits while lo is a normal fp16, 2^-25 absolute below
    assert (err <= np.maximum(np.abs(v) * 2.0 ** -22, 2.0 ** -25)).all()
