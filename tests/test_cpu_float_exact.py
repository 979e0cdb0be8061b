"""CPU rehearsal of the designed float data of test_float_exact_gpu.py: every generator runs against the CPU oracle and
checks its own exactness bound and coverage. Also checks that the checks bite: data that breaks the bound, a grid
without ties, and split-term data whose expected value equals the full product are all refused."""
import numpy as np
import pytest

import float_exact as F
from anakin_b200 import saber_abi as A


@pytest.mark.parametrize("variant", list(F.DENSE_VARIANTS))
@pytest.mark.parametrize("case", F.DENSE_F_CASES)
def test_dense_case(case, variant, oracle):
    x, w, bias, res, want = F.dense_case(case, variant)
    assert want.dtype == (np.float16 if F.DENSE_VARIANTS[variant][1] == A.HALF else np.float32)


@pytest.mark.parametrize("variant", list(F.GRID_VARIANTS))
def test_grid_case(variant, oracle):
    F.grid_case(variant)


@pytest.mark.parametrize("math", ["tf32x3"])
@pytest.mark.parametrize("case", [(1, 14, 14, 128, 200, 3, 3, 1, 1), (2, 9, 9, 256, 72, 1, 1, 1, 0),
                                  (1, 12, 30, 64, 200, 3, 3, 1, 1)])
def test_split_term_case(case, math, oracle):
    F.x3_case(case)


def test_split_term_truncation_case(oracle):
    F.x3_trunc_case()


@pytest.mark.parametrize("math", ["f16", "tf32x3"])
def test_stem_case(math, oracle):
    F.stem_case((2, 3, 40, 44, 64, 7, 7, 2, 3, (3, 2, 0)), math)


@pytest.mark.parametrize("k", [1024, 25088])
@pytest.mark.parametrize("out", [A.HALF, A.FLOAT])
def test_fc_case(k, out, oracle):
    F.fc_case(k, "f16", out, True)


def test_dw_case(oracle):
    F.dw_case(2, 28, 28, 32, 3, 1, 1)


def test_pool_tie_planes(oracle):
    x = F.pool_tie_planes(1, 4, 4, 64)
    mean = x.astype(np.float64).reshape(1, 2, 2, 2, 2, 64).mean((2, 4))
    tie, up = F.f16_ties(mean.astype(np.float32))
    assert tie.all() and up.any() and (~up).any()


def test_quantum_and_bound():
    assert F.quantum_of(np.array([3 * 2.0 ** -7, 0.5], np.float32)) == 2.0 ** -7
    assert F.quantum_of(np.zeros(3)) == 1.0
    x = np.full((1, 4, 4, 512), 15 * 2.0 ** -4, np.float32)
    w = np.full((8, 512, 3, 3), 15 * 2.0 ** -3, np.float32)
    assert F.check_conv_exact(x, w, pad=(1, 1)) == 4608 * 225          # within 2^22 quanta of 2^-7
    with pytest.raises(AssertionError, match="not exact"):
        F.check_conv_exact(np.concatenate([x] * 8, -1), np.concatenate([w] * 8, 1), pad=(1, 1))


def test_checks_refuse_vacuous_data(oracle):
    # a grid without the f16 tie classes (every value an f16 number)
    with pytest.raises(AssertionError):
        F.assert_f16_classes(np.arange(-2048, 2048, dtype=np.float32))


X3_REFUSAL_CASE = (1, 14, 14, 128, 200, 3, 3, 1, 1)


@pytest.mark.parametrize("drop", ["weights", "activations"])
def test_split_terms_refuse_data_without_low_parts(drop, oracle):
    """Without weight low parts Ahi*Wlo vanishes and the three-term sum is the full product; without activation low
    parts Alo*Whi vanishes. The separation shares then fall to zero, and the generator refuses the data."""
    x, w, bias = F.x3_data(X3_REFUSAL_CASE)
    if drop == "weights":
        w = F.tf32_hi(w)
        gone = ["Ahi*Wlo", "full product"]
    else:
        x = F.tf32_hi(x)
        gone = ["Alo*Whi", "full product"]
    kw = dict(stride=(1, 1), pad=(1, 1))
    three, wrong = F.x3_outputs(x, w, bias, kw)
    for name in gone:
        assert np.array_equal(wrong[name], three), name
    with pytest.raises(AssertionError, match="only 0.00 of the outputs separate the three-term sum from the " +
                       gone[0].replace("*", r"\*")):
        F.x3_expected(x, w, bias, 1, 1)
