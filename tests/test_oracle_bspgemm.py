"""The block SpGEMM checker (oracle/kk_oracle_bspgemm.c) against the reference's own bspgemm_debug_numeric compiled in place
(oracle/kkref_bspgemm.cpp, sparse/impl/KokkosSparse_bspgemm_impl_seq.hpp:39-130 with SerialGemmInternal<Unblocked>): bit
for bit, on the reference's sweep (Test_Sparse_bspgemm.hpp:232-242) and on unsorted rows, repeated columns, signed zeros,
NaN and Inf.  Also: the restatement lies within a rounding-error bound of a dense wide-precision product."""
import os

import numpy as np
import pytest

import bspgemm_cases as BC


@pytest.fixture(scope="module")
def orc():
    return BC.BlockOracle()


def _need_ref(orc):
    if orc.ref is None:
        pytest.skip("oracle/_ref/libkkref_bspgemm.so was not built (the reference tree is needed to build it)")


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("bs", BC.BLOCK_SIZES)
def test_restatement_equals_reference_sweep(orc, bs, dtype):
    _need_ref(orc)
    for name, bs_, A, B, m, n, k in BC.ref_sweep_cases(bs, dtype):
        got = orc.bspgemm(bs_, A, B, m, n, k)
        exp = orc.bspgemm_ref(bs_, A, B, m, n, k)
        assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1]), name
        assert BC.same_bits(got[2], exp[2]), name


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("bs", [1, 2, 3, 5])
def test_restatement_equals_reference_special(orc, bs, dtype):
    _need_ref(orc)
    for name, bs_, A, B, m, n, k in BC.special_cases(bs, dtype) + [BC.long_row_case(bs, dtype, products=1500)]:
        got = orc.bspgemm(bs_, A, B, m, n, k)
        exp = orc.bspgemm_ref(bs_, A, B, m, n, k)
        assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1]), name
        assert BC.same_bits(got[2], exp[2]), name
        if name == "zeros_signed":  # chains start at +0.0, so no product row of -0.0 blocks can make a -0.0 entry
            assert not np.any(np.signbit(got[2]) & (got[2] == 0)), name


def test_sorted_rows(orc):
    for name, bs, A, B, m, n, k in BC.special_cases(3):
        rpC, ciC, _ = orc.bspgemm(bs, A, B, m, n, k)
        for i in range(m):
            row = ciC[rpC[i]:rpC[i + 1]]
            assert np.all(np.diff(row) > 0), name


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("bs", [1, 2, 3, 4, 5])
def test_restatement_within_dense_bound(orc, bs, dtype):
    cases = [c for c in BC.ref_sweep_cases(bs, dtype) if c[4] <= 50] + BC.special_cases(bs, dtype)[:3]
    for name, bs_, A, B, m, n, k in cases:
        rpC, ciC, vC = orc.bspgemm(bs_, A, B, m, n, k)
        assert BC.dense_bound_ok(bs_, A, B, m, n, k, rpC, ciC, vC), name
