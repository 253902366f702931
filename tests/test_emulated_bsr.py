"""BsrMatrix SpMV / SpMM kernels executed on the CPU (tools/emu, see tests/test_emulated_kernels.py) against the
oracle: the sweep of the reference's unit test (sparse/unit_test/Test_Sparse_spmv_bsr.hpp:351-456,595-700: shapes x
block sizes {1,2,5,9} + the 7 / 11 x 499 case, modes N T C H, alpha x beta, 1 and 7 vectors, both layouts) with its
tolerance law, plus cases sized to wrap the TMA ring, with block rows longer than a stage, unaligned arrays and
every block size 2..17."""
import numpy as np
import pytest

import emu_lib as E
import exact_ref as R
import spmm_cases
from bsr_cases import BLOCK_SIZES, COEFS_ALPHA, COEFS_BETA, PRIME_CASE, SHAPES, bsr_random, op_max_nnz_per_row, tolerance


@pytest.fixture(scope="module")
def emu():
    return E.lib()


def expected(oracle, mode, bs, nb, rp, ci, v, X, Y0, alpha, beta):
    """Mode N: the reference's GPU-space functor order (B1, pinned on the reference's own code); T/H: its host
    functor (B3)."""
    Yc = np.nan_to_num(Y0.copy(order="K")) if beta == 0.0 else Y0.copy(order="K")
    if mode in "NC":
        return oracle.bsr_spmv_v42(bs, rp, ci, v, X, Yc, alpha, beta)
    return oracle.bsr_spmv_v41(mode, bs, nb, rp, ci, v, X, Yc, alpha, beta)


def run_rank1(oracle, plan, mode, bs, mb, nb, rp, ci, v, rng, alpha, beta, dtype, signed=False):
    """signed: mixed-sign values (spmm_cases._values), x and y0, checked against the exact product only (the reference's
    law assumes entries in [0, 10)); every call is checked against it."""
    trans = mode in "TH"
    nx, ny = (mb * bs, nb * bs) if trans else (nb * bs, mb * bs)
    x = rng.uniform(0, 10, nx).astype(dtype)
    y0 = rng.uniform(0, 10, ny).astype(dtype)
    if signed:
        v = spmm_cases._values(rng, len(v), dtype)
        x = spmm_cases.dense_operands(rng, nx, 1, dtype)[:, 0]
        y0 = spmm_cases.dense_operands(rng, ny, 1, dtype)[:, 0]
    if beta == 0.0:
        y0[::7] = np.nan
    y = y0.copy()
    E.bsr_spmv(plan, mode, mb, nb, bs, rp, ci, v, x, y, alpha, beta)
    prp, pci, pv = R.bsr_to_point_crs(bs, rp, ci, v)
    R.assert_within(y, R.spmm_exact(prp, pci, pv, x, y0, alpha, beta, trans), R.spmm_bound(prp, pci, pv, x, y0, alpha, beta, trans),
                    f"{plan.kernel()} mode {mode} bs {bs} alpha {alpha} beta {beta} signed {signed}")
    if signed:
        return
    exp = expected(oracle, mode, bs, nb, rp, ci, v, x, y0, alpha, beta)
    assert not np.isnan(y).any(), "NaN survived beta == 0"
    tol = tolerance(dtype, alpha, beta, op_max_nnz_per_row(bs, rp, ci, nb, trans))
    err = np.max(np.abs(y - exp), initial=0.0)
    assert err <= tol, f"{plan.kernel()} mode {mode} bs {bs} alpha {alpha} beta {beta}: err {err:.3e} > {tol:.3e}"


CASES = [(bs, mb, nb) for (mb, nb) in SHAPES for bs in BLOCK_SIZES] + [PRIME_CASE]


@pytest.mark.parametrize("bs,mb,nb", CASES)
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_reference_sweep_rank1(emu, oracle, bs, mb, nb, dtype):
    rp, ci, v = bsr_random(bs, mb, nb, seed=3 + bs + mb, dtype=dtype, sort=False)
    rng = np.random.default_rng(17)
    for signed in (False, True):
        plan = E.BsrPlan()
        for mode in "NTCH":
            for alpha in COEFS_ALPHA:
                for beta in COEFS_BETA:
                    run_rank1(oracle, plan, mode, bs, mb, nb, rp, ci, v, rng, alpha, beta, dtype, signed)
        plan.close()


@pytest.mark.parametrize("bs,mb,nb", CASES)
@pytest.mark.parametrize("order", ["F", "C"])
def test_reference_sweep_multivector(emu, oracle, bs, mb, nb, order):
    dtype = np.float64
    rp, ci, v = bsr_random(bs, mb, nb, seed=5 + bs + nb, dtype=dtype, sort=False)
    rng = np.random.default_rng(19)
    plan = E.BsrPlan()
    for mode in "NTCH":
        trans = mode in "TH"
        nx, ny = (mb * bs, nb * bs) if trans else (nb * bs, mb * bs)
        max_row = op_max_nnz_per_row(bs, rp, ci, nb, trans)
        for k in (1, 7):
            X = np.asarray(rng.uniform(0, 10, (nx, k)), order=order)
            Y0 = np.asarray(rng.uniform(0, 10, (ny, k)), order=order)
            for alpha in COEFS_ALPHA:
                for beta in COEFS_BETA:
                    Yin = Y0.copy(order=order)
                    if beta == 0.0 and ny:
                        Yin[::5] = np.nan
                    Y = Yin.copy(order=order)
                    E.bsr_spmm(plan, mode, mb, nb, bs, rp, ci, v, X, Y, alpha, beta)
                    exp = expected(oracle, mode, bs, nb, rp, ci, v, X, Yin, alpha, beta)
                    assert not np.isnan(Y).any()
                    assert np.max(np.abs(Y - exp), initial=0.0) <= tolerance(dtype, alpha, beta, max_row), (plan.kernel(), mode, k, alpha, beta)
    plan.close()


@pytest.mark.parametrize("bs", list(range(2, 18)))
def test_tile_kernel_every_block_size(emu, oracle, bs):
    """Enough blocks per CTA (emulated device: 8 SMs) to wrap the ring; bs = 17 exceeds the tile path (vector kernel)."""
    mb = max(300, 24000 // (bs * bs))
    nb = mb + 13
    rp, ci, v = bsr_random(bs, mb, nb, seed=bs, min_blocks=0, max_blocks=12, sort=False)
    plan = E.BsrPlan()
    rng = np.random.default_rng(bs)
    import os
    for knob in (None, "walk"):  # default: element-per-lane kernel for bs 2..5; "walk": the run-time-bs kernel for every bs
        if knob:
            os.environ["B200SP_BSR_KERNEL"] = knob
        try:
            for alpha, beta in ((1.0, 0.0), (3.7, -1.5)):
                for dtype in (np.float64, np.float32):
                    vv = v.astype(dtype)
                    run_rank1(oracle, plan, "N", bs, mb, nb, rp, ci, vv, rng, alpha, beta, dtype)
                    run_rank1(oracle, plan, "N", bs, mb, nb, rp, ci, vv, rng, alpha, beta, dtype, signed=True)
                    # default: element-per-lane tile kernel for bs 2..5, row-vector kernel above (the measured choice)
                    if bs > 5 and not knob:  # default: tensor-core kernel for double up to bs = 16, row-vector kernel otherwise
                        want = "bsr_mm_tc<f64" if (dtype == np.float64 and bs <= 16) else "bsr_vector"
                    else:
                        want = "bsr_vector" if bs > 16 else ("bsr_tile_e<" if (bs <= 5 and not knob) else "bsr_tile<")
                    assert plan.kernel().startswith(want), plan.kernel()
        finally:
            os.environ.pop("B200SP_BSR_KERNEL", None)
    run_rank1(oracle, plan, "T", bs, mb, nb, rp, ci, v, rng, -1.0, 1.0, np.float64)
    plan.close()


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_long_block_rows_and_tail(emu, oracle, dtype):
    """Block rows beyond the stage (left to the per-row kernel), empty block rows, and nnzb % 4 != 0 (the last
    blocks of the matrix are staged by plain loads)."""
    bs, mb, nb = 3, 900, 1500
    rng = np.random.default_rng(23)
    lens = rng.integers(0, 6, mb)
    lens[[5, 400, 899]] = [700, 227, 1300]
    if int(lens.sum()) % 4 == 0:
        lens[10] += 1
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    ci = np.concatenate([rng.choice(nb, int(l), replace=False) for l in lens]).astype(np.int32)
    v = rng.uniform(0, 10, len(ci) * bs * bs).astype(dtype)
    plan = E.BsrPlan()
    for alpha, beta in ((1.0, 0.0), (-1.0, 1.0), (3.7, -1.5)):
        for signed in (False, True):
            run_rank1(oracle, plan, "N", bs, mb, nb, rp, ci, v, rng, alpha, beta, dtype, signed)
            assert plan.kernel().startswith("bsr_tile"), plan.kernel()
    plan.close()


def test_unaligned_arrays_take_the_vector_kernel(emu, oracle):
    bs, mb, nb = 4, 500, 500
    rp, ci, v = bsr_random(bs, mb, nb, seed=2, sort=False)
    cib = np.empty(len(ci) + 1, np.int32)
    cib[1:] = ci
    plan = E.BsrPlan()
    rng = np.random.default_rng(3)
    run_rank1(oracle, plan, "N", bs, mb, nb, rp, cib[1:], v, rng, 3.7, -1.5, np.float64)
    assert plan.kernel().startswith("bsr_vector"), plan.kernel()
    plan.close()


def test_corner_cases_and_arguments(emu):
    """bsr_corner_case_0_by_0 / 0_by_1 / 1_by_0 (Test_Sparse_spmv_bsr.hpp:101-116,221-278) and argument errors."""
    L = emu
    plan = E.BsrPlan()
    z = np.zeros(1, np.int32)
    e = np.zeros(0, np.int32)
    for bs in BLOCK_SIZES:
        for mode in "NTCH":
            E.bsr_spmv(plan, mode, 0, 0, bs, z, e, np.zeros(0), np.zeros(0), np.zeros(0), 1.0, 1.0)  # 0 x 0
            y = np.full(bs, 2.0)
            if mode in "TH":  # 0 x 1 blocks: y has bs entries for T
                E.bsr_spmv(plan, mode, 0, 1, bs, z, e, np.zeros(0), np.zeros(0), y, 3.7, -1.5)
                assert np.array_equal(y, np.full(bs, -3.0))
            else:  # 1 x 0 blocks: one empty block row
                E.bsr_spmv(plan, mode, 1, 0, bs, np.zeros(2, np.int32), e, np.zeros(0), np.zeros(0), y, 3.7, 0.0)
                assert np.array_equal(y, np.zeros(bs))
    y = np.zeros(4)
    rc = L.b200sp_bsr_spmv_f64_i32(plan.h, None, b"N", 1, 1, 0, 0, 1.0, E.ptr(np.zeros(2, np.int32)), None, None, E.ptr(y), 0.0, E.ptr(y))
    assert rc != 0 and b"block size" in L.b200sp_last_error_string()
    rc = L.b200sp_bsr_spmv_f64_i32(plan.h, None, b"X", 1, 1, 0, 2, 1.0, E.ptr(np.zeros(2, np.int32)), None, None, E.ptr(y), 0.0, E.ptr(y))
    assert rc != 0 and b"mode" in L.b200sp_last_error_string()
    plan.close()
