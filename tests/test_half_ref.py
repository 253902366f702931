"""The fp16 reference and bound of tests/half_ref.py checked on the CPU: the bound holds for the emulated fp16 kernels
(tools/emu), it is not vacuous (it fails a kernel that accumulates in fp16, and a dropped term), and the reference agrees
with rational arithmetic."""
from fractions import Fraction

import numpy as np

import half_ref as H
import spmm_cases as cases
from test_emulated_spmm_f16 import case16, emu, operands16, run16  # noqa: F401  (emu is a fixture)


def _bound_fails(got, A, X, Y0, alpha, beta):
    rp, ci, v, _ = A
    try:
        H.assert_within16(got, H.spmm_exact16(rp, ci, v, X, Y0, alpha, beta), H.spmm_bound16(rp, ci, v, X, Y0, alpha, beta), "x")
    except AssertionError:
        return True
    return False


def test_bound_holds_for_the_emulated_kernel(emu):
    for name in ("thresholds", "small_mod2", "duplicates", "cancelling"):
        A = case16(name, seed=11)
        for k in (4, 16):
            X, Y0 = operands16(A, k, "C", seed=3)
            got, _ = run16(A, X, Y0, 1.25, -0.75)
            assert not _bound_fails(got, A, X, Y0, 1.25, -0.75), (name, k)


def test_bound_rejects_fp16_accumulation():
    """Rows of 300..1200 positive terms: every fp16 partial sum is rounded to 11 bits, and the errors add up to far more
    than one fp16 rounding of the result."""
    rng = np.random.default_rng(0)
    ncols = 50
    rp, ci, v = cases.from_lengths([600, 900, 1200, 300], ncols, rng, np.float32)
    v = np.abs(v).astype(np.float16)
    X = (np.abs(cases.dense_operands(rng, ncols, 4, np.float32)) + 1).astype(np.float16)
    Y0 = np.zeros((4, 4), dtype=np.float16)
    A = (rp, ci, v, ncols)
    assert _bound_fails(H.fp16_accumulation(rp, ci, v, X, Y0, 1.0, 0.0), A, X, Y0, 1.0, 0.0)
    # the same inputs through fp32 accumulation and one rounding pass
    exact = H.spmm_exact16(rp, ci, v, X, Y0, 1.0, 0.0)
    assert not _bound_fails(exact.astype(np.float32).astype(np.float16), A, X, Y0, 1.0, 0.0)


def test_bound_rejects_a_dropped_term(emu):
    A = case16("small_mod1", seed=2)
    X, Y0 = operands16(A, 8, "C", seed=4)
    rp, ci, v, nc = A
    v2 = v.copy()
    row = int(np.argmax(np.diff(rp)))
    v2[rp[row + 1] - 1] = 0  # the last entry of the longest row
    got, _ = run16((rp, ci, v2, nc), X, Y0, 1.0, 0.0)
    assert _bound_fails(got, A, X, Y0, 1.0, 0.0)


def test_reference_is_exact():
    rng = np.random.default_rng(1)
    ncols = 20
    rp, ci, v = cases.from_lengths([7, 0, 33, 5], ncols, rng, np.float32)
    v = v.astype(np.float16)
    X = cases.dense_operands(rng, ncols, 3, np.float16)
    Y0 = cases.dense_operands(rng, 4, 3, np.float16)
    alpha, beta = np.float32(0.3), np.float32(-1.7)
    got = H.spmm_exact16(rp, ci, v, X, Y0, alpha, beta)
    for i in range(4):
        for j in range(3):
            s = sum(Fraction(float(v[e])) * Fraction(float(X[ci[e], j])) for e in range(rp[i], rp[i + 1]))
            want = Fraction(float(beta)) * Fraction(float(Y0[i, j])) + Fraction(float(alpha)) * s
            assert abs(Fraction(float(got[i, j])) - want) <= abs(want) * Fraction(1, 2**50) + Fraction(1, 2**80)
