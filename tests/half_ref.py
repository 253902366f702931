"""Exact reference and per-entry error bound of half-precision rank-2 SpMV (b200sp_spmm_f16_i32): A's values, X and Y in
IEEE binary16, products and sums in fp32, one rounding to binary16 at the end.

spmm_exact16 is the exact product of the fp16 inputs, computed in float64 by exact_ref.spmm_exact on the widened inputs (a
product of two fp16 numbers is exact in fp32 already).  alpha and beta are taken as the float32 values the C ABI receives.

spmm_bound16 is, per entry,

    |y_hat - y| <= 2^-11 |y| + (1 + 2^-11) gamma_fp32(len_i + 3) (|alpha| sum |a||x| + |beta||y0|) + 2^-25

The fp32 part is exact_ref.spmm_bound's derivation with len_i + 3 roundings of unit 2^-24: the kernel's fp32 result s carries
|s - y| <= gamma_fp32(len_i + 3) * scale.  Rounding s to binary16 adds at most 2^-11 |s| <= 2^-11 |y| + 2^-11 |s - y| for a
normal result, and at most half the subnormal spacing, 2^-25, below 2^-14.  A kernel that accumulates in fp16 makes errors of
about 2^-11 times its partial sums at every addition and fails the bound on rows whose partial sums exceed the result."""
import numpy as np

import exact_ref as R

HALF_MAX_ROUNDED = 65520.0  # 65504 + half an ulp: from here on, round-to-nearest gives +-inf


def widen(a):
    return None if a is None else np.asarray(a, dtype=np.float16).astype(np.float32)


def spmm_exact16(rp, ci, v16, X16, Y16, alpha, beta, trans=False):
    """beta*Y0 + alpha*op(A)*X in float64 for fp16 v, X, Y0 and float32 alpha, beta."""
    return R.spmm_exact(rp, ci, widen(v16), widen(X16), widen(Y16), np.float32(alpha), np.float32(beta), trans)


def spmm_bound16(rp, ci, v16, X16, Y16, alpha, beta, trans=False):
    """The per-entry bound of the module docstring, against spmm_exact16 (whose own error, < 2^-50 relative, is far
    inside the spare terms)."""
    v32, X32, Y32 = widen(v16), widen(X16), widen(Y16)
    scale = R.spmm_scale(rp, ci, v32, X32, Y32, np.float32(alpha), np.float32(beta), trans)
    lens = R.op_row_lengths(rp, ci, scale.shape[0], trans).astype(np.float64)
    exact = np.abs(spmm_exact16(rp, ci, v16, X16, Y16, alpha, beta, trans).astype(np.float64))
    g = R.gamma(lens + 3, 2.0**-24)[:, None]
    return 2.0**-11 * exact + (1 + 2.0**-11) * g * scale + 2.0**-25


def assert_within16(got16, exact, bound, what):
    """exact_ref.assert_within for an fp16 result: an fp16 +-inf is also accepted where the exact value is within the bound
    of the overflow threshold (|y| + bound >= 65520) and has the same sign."""
    got = np.asarray(got16, dtype=np.float16).astype(np.float64)
    exact = np.asarray(exact, dtype=np.float64)
    bound = np.asarray(bound, dtype=np.float64)
    with np.errstate(invalid="ignore"):
        ovf = np.isinf(got) & np.isfinite(exact) & (np.sign(got) == np.sign(exact)) & (np.abs(exact) + bound >= HALF_MAX_ROUNDED)
    R.assert_within(np.where(ovf, exact, got), exact, bound, what)


def round16(y32):
    """round_fp16 of an fp32 result: the identity of the item paths is Y16 == round16(Y32)."""
    return np.asarray(y32, dtype=np.float32).astype(np.float16)


def fp16_accumulation(rp, ci, v16, X16, Y16, alpha, beta):
    """What a kernel accumulating in fp16 would compute (mode N, storage order): every product and partial sum rounded to
    binary16.  Only used to show that spmm_bound16 rejects it."""
    v, X, Y0 = (np.asarray(a, dtype=np.float16) for a in (v16, X16, Y16))
    a16, b16 = np.float16(alpha), np.float16(beta)
    out = np.zeros(Y0.shape, dtype=np.float16)
    with np.errstate(over="ignore", invalid="ignore"):
        for i in range(len(rp) - 1):
            s = np.zeros(Y0.shape[1], dtype=np.float16)
            for e in range(rp[i], rp[i + 1]):
                s = (s + v[e] * X[ci[e]]).astype(np.float16)
            out[i] = (a16 * s + (b16 * Y0[i] if b16 != 0 else np.float16(0))).astype(np.float16)
    return out
