"""The rank-2 SpMV kernel paths EXECUTED on the CPU (tools/emu) on the shared cases of spmm_cases.py, each result checked
entry by entry against the exact product within the per-entry rounding bound (tests/exact_ref.py) -- the same inputs
and the same check as tests/test_gpu_spmm_paths.py, at the sizes the emulation can afford (small m, k <= 64)."""
import numpy as np
import pytest

import emu_lib as E
import exact_ref as R
import spmm_cases as cases
from test_emulated_kernels import env

PATHS = {
    "items": {},
    "items16": {"B200SP_SPMM_ITEM_LMAX": "16"},
    "items64": {"B200SP_SPMM_ITEM_LMAX": "64"},
    "items256": {"B200SP_SPMM_ITEM_LMAX": "256"},
}
KS = [1, 4, 5, 16, 33, 64]


@pytest.fixture(scope="module")
def emu():
    return E.lib()


def run(A_np, X, Y0, alpha, beta, trans=False, y_nan=False):
    rp, ci, v, ncols = A_np
    Y = Y0.copy(order="K")
    if y_nan:
        Y[...] = np.nan
    plan = E.SpmvPlan()
    try:
        E.spmm(plan, "T" if trans else "N", len(rp) - 1, ncols, rp, ci, v, X, Y, alpha, beta)
        return Y, plan.kernel()
    finally:
        plan.close()


def operands(A_np, k, dtype, order, trans=False):
    rp, ci, v, ncols = A_np
    rng = np.random.default_rng(k)
    xr, yr = (len(rp) - 1, ncols) if trans else (ncols, len(rp) - 1)
    return (np.asarray(cases.dense_operands(rng, xr, k, dtype), order=order),
            np.asarray(cases.dense_operands(rng, yr, k, dtype), order=order))


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("case", ["thresholds", "small_mod1", "small_mod3", "duplicates", "cancelling"])
def test_paths_on_shared_cases(emu, case, path, dtype):
    A_np = cases.SMALL_CASES[case](5, dtype)
    with env(**PATHS[path]):
        for k in KS:
            for order in "CF":
                X, Y0 = operands(A_np, k, dtype, order)
                for alpha, beta in ((2.5, -0.5), (1.0, 0.0)):
                    got, kern = run(A_np, X, Y0, alpha, beta, y_nan=beta == 0)
                    what = f"{kern} {case} {path} k={k} order={order} a={alpha} b={beta}"
                    assert kern.startswith("spmm_"), what
                    R.assert_within(got, R.spmm_exact(*A_np[:3], X, Y0, alpha, beta), R.spmm_bound(*A_np[:3], X, Y0, alpha, beta), what)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("case", ["thresholds", "duplicates", "wide_short", "small_mod2"])
def test_transpose_and_degenerate(emu, case, dtype):
    A_np = cases.SMALL_CASES[case](5, dtype)
    for k in (1, 5, 16):
        for order in "CF" if A_np[3] else "C":  # an array without rows has no layout to speak of
            for trans in (False, True):
                X, Y0 = operands(A_np, k, dtype, order, trans)
                for alpha, beta in ((-1.5, 0.5), (0.0, 2.5), (1.0, 0.0)):
                    got, kern = run(A_np, X, Y0, alpha, beta, trans, y_nan=beta == 0)
                    what = f"{kern} {case} trans={trans} k={k} order={order} a={alpha} b={beta}"
                    R.assert_within(got, R.spmm_exact(*A_np[:3], X, Y0, alpha, beta, trans),
                                    R.spmm_bound(*A_np[:3], X, Y0, alpha, beta, trans), what)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_item_path_identities(emu, dtype):
    """Same bits on a second call, for LayoutLeft as for LayoutRight, and for misaligned (scalar) as for aligned (vector)
    operands."""
    A_np = cases.thresholds(5, dtype)
    for k in (4, 16, 64):
        X, Y0 = operands(A_np, k, dtype, "C")
        ref, kern = run(A_np, X, Y0, 1.5, -0.5)
        assert kern == "spmm_items_vec", kern
        again, _ = run(A_np, X, Y0, 1.5, -0.5)
        left, kern_l = run(A_np, np.asfortranarray(X), np.asfortranarray(Y0), 1.5, -0.5)
        assert kern_l == "spmm_relayout+items", kern_l
        bx = np.empty(X.size + 1, dtype)
        by = np.empty(Y0.size + 1, dtype)
        Xo = bx[1:].reshape(X.shape)
        Yo = by[1:].reshape(Y0.shape)
        Xo[...] = X
        Yo[...] = Y0
        plan = E.SpmvPlan()
        E.spmm(plan, "N", len(A_np[0]) - 1, A_np[3], *A_np[:3], Xo, Yo, 1.5, -0.5)
        kern_o = plan.kernel()
        plan.close()
        if (Xo.ctypes.data | Yo.ctypes.data) % 16:
            assert kern_o == "spmm_items", kern_o
        for other in (again, left, Yo):
            assert np.array_equal(np.ascontiguousarray(other).view(np.uint8), ref.view(np.uint8)), (k, kern, kern_l, kern_o)


# variables that once selected kernels of spmm.cu; nothing reads them any more
RETIRED = [dict(B200SP_SPMM_KERNEL=kern, B200SP_SPMM_SEG="vec", B200SP_SPMM_VEC="1", B200SP_SPMM_CFG="2", B200SP_SPMM_LMAX="16")
           for kern in ("row", "split", "tilev")]


@pytest.mark.parametrize("dtype", [np.float64, np.float32, np.float16])
def test_retired_variables_are_inert(emu, dtype):
    """With every retired selection variable set, fp64, fp32 and fp16 calls report the default kernel and give the same bits
    as without them, for LayoutRight and LayoutLeft operands."""
    from test_emulated_spmm_f16 import case16, run16

    A_np = case16("thresholds") if dtype == np.float16 else cases.thresholds(5, dtype)
    call = run16 if dtype == np.float16 else run
    for k in (5, 16):
        for order in "CF":
            X, Y0 = operands(A_np, k, dtype, order)
            ref, kern = call(A_np, X, Y0, 1.5, -0.5)
            assert kern in ("spmm_items", "spmm_items_vec", "spmm_relayout+items"), kern
            for retired in RETIRED:
                with env(**retired):
                    got, kern_r = call(A_np, X, Y0, 1.5, -0.5)
                what = f"{np.dtype(dtype).name} k={k} order={order} {retired}"
                assert kern_r == kern, (what, kern_r, kern)
                assert np.array_equal(np.ascontiguousarray(got).view(np.uint8), np.ascontiguousarray(ref).view(np.uint8)), what
