"""Block SpGEMM on the H100 (kokkos-kernels_b200/csrc/bspgemm.cu through sparse.block_spgemm_* and the view-level
spgemm_numeric_views(..., block_dim)): structure exact and sorted, values bit-identical to the restatement of the reference's
bspgemm_debug_numeric (oracle/kk_oracle_bspgemm.c, pinned on the reference in tests/test_oracle_bspgemm.py), and the
reference's own relative law (5e-7 fp64 / 3e-2 fp32, Test_Sparse_bspgemm.hpp:120-125) as a second check."""
import numpy as np
import pytest
import torch

import bspgemm_cases as BC

pytestmark = pytest.mark.gpu

DTYPES = [np.float64, np.float32]


@pytest.fixture(scope="module")
def kk():
    import __graft_entry__ as g

    return g.build(verbose=False)


@pytest.fixture(scope="module")
def orc():
    return BC.BlockOracle()


def _bsr(kk, bs, A, ncols):
    dev = torch.device("cuda:0")
    rp, ci, v = (torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in A)
    return kk.sparse.BsrMatrix(rp, ci, v, ncols, bs)


def _check(orc, bs, A, B, m, n, k, C, name):
    exp = BC.BlockOracle.bspgemm(orc, bs, A, B, m, n, k)
    rpC, ciC, vC = (t.cpu().numpy() for t in (C.row_map, C.entries, C.values))
    assert np.array_equal(rpC, exp[0]), name
    assert np.array_equal(ciC, exp[1]), name
    for i in range(m):
        assert np.all(np.diff(ciC[rpC[i]:rpC[i + 1]]) > 0), name
    # bs = 1 is the point numeric: bit-identical to the oracle on rows of up to 8192 products (its expand / sort / compress
    # kernels); its hash kernels for longer rows add with atomics, so there the law below is the check
    prods = [sum(B[0][c + 1] - B[0][c] for c in A[1][A[0][i]:A[0][i + 1]]) for i in range(m)] if bs == 1 else [0]
    if max(prods, default=0) <= 8192:
        assert BC.same_bits(vC, exp[2]), name
    # the reference's law: |a - b| / max(|a|, |b|) <= eps entry by entry (finite entries)
    eps = 5e-7 if vC.dtype == np.float64 else 3e-2
    fin = np.isfinite(exp[2]) & np.isfinite(vC)
    a, b = vC[fin].astype(np.float64), exp[2][fin].astype(np.float64)
    den = np.maximum(np.maximum(np.abs(a), np.abs(b)), np.finfo(np.float64).tiny)
    assert np.all(np.abs(a - b) / den <= eps), name
    return vC


def _product(kk, bs, A, B, m, n, k):
    kh = kk.sparse.KokkosKernelsHandle()
    kh.create_spgemm_handle()
    Am, Bm = _bsr(kk, bs, A, n), _bsr(kk, bs, B, k)
    C = kk.sparse.block_spgemm_symbolic(kh, Am, False, Bm, False)
    kk.sparse.block_spgemm_numeric(kh, Am, False, Bm, False, C)
    torch.cuda.synchronize()
    assert kh.get_spgemm_handle().is_numeric_called()
    return kh, Am, Bm, C


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("bs", BC.BLOCK_SIZES)
def test_reference_sweep(kk, orc, bs, dtype):
    for name, bs_, A, B, m, n, k in BC.ref_sweep_cases(bs, dtype):
        _, _, _, C = _product(kk, bs_, A, B, m, n, k)
        assert C.blockDim() == bs_ and C.values.numel() == C.nnz() * bs_ * bs_
        _check(orc, bs_, A, B, m, n, k, C, name)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("bs", [2, 3, 4, 17])
def test_special_inputs(kk, orc, bs, dtype):
    """unsorted rows, repeated columns, explicit and signed zero blocks, NaN and Inf in A"""
    for name, bs_, A, B, m, n, k in BC.special_cases(bs, dtype):
        _, _, _, C = _product(kk, bs_, A, B, m, n, k)
        _check(orc, bs_, A, B, m, n, k, C, name)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("bs,products", [(2, 2000), (2, 6000), (3, 20000), (8, 5000)])
def test_long_rows(kk, orc, bs, products, dtype):
    """a block row in the 4096-product bin, and rows past it (per-CTA global scratch; A's blocks unstaged at bs = 8)"""
    name, bs_, A, B, m, n, k = BC.long_row_case(bs, dtype, products=products)
    _, _, _, C = _product(kk, bs_, A, B, m, n, k)
    _check(orc, bs_, A, B, m, n, k, C, name)


@pytest.mark.parametrize("dtype", DTYPES)
def test_numeric_rerun_and_determinism(kk, orc, dtype):
    """numeric again on the same structure with new values (Test_Sparse_spgemm.hpp:112-122), and two runs give the same bits"""
    name, bs, A, B, m, n, k = BC.ref_sweep_cases(3, dtype)[0]
    kh, Am, Bm, C = _product(kk, bs, A, B, m, n, k)
    first = _check(orc, bs, A, B, m, n, k, C, name)
    kk.sparse.block_spgemm_numeric(kh, Am, False, Bm, False, C)
    torch.cuda.synchronize()
    assert BC.same_bits(C.values.cpu().numpy(), first)
    A2 = (A[0], A[1], (A[2] * -2.5).astype(dtype))
    Am.values.copy_(torch.from_numpy(A2[2]))
    kk.sparse.block_spgemm_numeric(kh, Am, False, Bm, False, C)
    torch.cuda.synchronize()
    _check(orc, bs, A2, B, m, n, k, C, name + "_rerun")


@pytest.mark.parametrize("dtype", DTYPES)
def test_view_level(kk, orc, dtype):
    """spgemm_symbolic_views on the block graphs + spgemm_numeric_views(..., block_dim=bs); block_dim=1 stays the point product"""
    sp = kk.sparse
    dev = torch.device("cuda:0")
    name, bs, A, B, m, n, k = BC.ref_sweep_cases(4, dtype)[1]
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    kh = sp.KokkosKernelsHandle()
    kh.create_spgemm_handle()
    rpC = torch.empty(m + 1, dtype=torch.int32, device=dev)
    sp.spgemm_symbolic_views(kh, m, n, k, t(A[0]), t(A[1]), False, t(B[0]), t(B[1]), False, rpC)
    nnz = kh.get_spgemm_handle().get_c_nnz()
    ciC = torch.empty(nnz, dtype=torch.int32, device=dev)
    vC = torch.empty(nnz * bs * bs, dtype=t(A[2]).dtype, device=dev)
    sp.spgemm_numeric_views(kh, m, n, k, t(A[0]), t(A[1]), t(A[2]), False, t(B[0]), t(B[1]), t(B[2]), False, rpC, ciC, vC, block_dim=bs)
    torch.cuda.synchronize()
    _check(orc, bs, A, B, m, n, k, sp.BsrMatrix(rpC, ciC, vC, k, bs), name)
    # block_dim = 1 (the default): the point product on the same graphs, unchanged behaviour
    Ap = (A[0], A[1], A[2][:: bs * bs].copy())
    Bp = (B[0], B[1], B[2][:: bs * bs].copy())
    kh1 = sp.KokkosKernelsHandle()
    kh1.create_spgemm_handle()
    rp1 = torch.empty(m + 1, dtype=torch.int32, device=dev)
    sp.spgemm_symbolic_views(kh1, m, n, k, t(Ap[0]), t(Ap[1]), False, t(Bp[0]), t(Bp[1]), False, rp1)
    nz1 = kh1.get_spgemm_handle().get_c_nnz()
    ci1 = torch.empty(nz1, dtype=torch.int32, device=dev)
    v1 = torch.empty(nz1, dtype=t(Ap[2]).dtype, device=dev)
    sp.spgemm_numeric_views(kh1, m, n, k, t(Ap[0]), t(Ap[1]), t(Ap[2]), False, t(Bp[0]), t(Bp[1]), t(Bp[2]), False, rp1, ci1, v1)
    torch.cuda.synchronize()
    exp = orc.bspgemm(1, Ap, Bp, m, n, k)
    assert np.array_equal(ci1.cpu().numpy(), exp[1])
    assert BC.same_bits(v1.cpu().numpy(), exp[2])


def test_bs1_equals_point_entry(kk):
    """bs = 1 forwards to the point numeric: the same bits as spgemm on the same CrsMatrix"""
    sp = kk.sparse
    name, bs, A, B, m, n, k = BC.ref_sweep_cases(1, np.float64)[0]
    _, _, _, C = _product(kk, 1, A, B, m, n, k)
    dev = torch.device("cuda:0")
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    P = sp.spgemm(sp.CrsMatrix(t(A[0]), t(A[1]), t(A[2]), n), False, sp.CrsMatrix(t(B[0]), t(B[1]), t(B[2]), k), False)
    torch.cuda.synchronize()
    assert torch.equal(P.entries, C.entries) and BC.same_bits(P.values.cpu().numpy(), C.values.cpu().numpy())


def test_errors(kk):
    sp = kk.sparse
    name, bs, A, B, m, n, k = BC.ref_sweep_cases(2, np.float64)[0]
    Am, Bm = _bsr(kk, 2, A, n), _bsr(kk, 2, B, k)
    B3 = BC.random_bsr(n, k, 100, 50, 5, 3, 1)
    kh = sp.KokkosKernelsHandle()
    kh.create_spgemm_handle()
    with pytest.raises(sp.B200SparseInvalidArgument, match="Block SpGEMM must be called for matrices with the same block size"):
        sp.block_spgemm_symbolic(kh, Am, False, _bsr(kk, 3, B3, k), False)
    with pytest.raises(sp.B200SparseError, match="transpos"):
        sp.block_spgemm_symbolic(kh, Am, True, Bm, False)
    # numeric before symbolic
    C0 = sp.BsrMatrix(torch.zeros(m + 1, dtype=torch.int32, device="cuda"), torch.zeros(0, dtype=torch.int32, device="cuda"),
                      torch.zeros(0, dtype=torch.float64, device="cuda"), k, 2)
    with pytest.raises(sp.B200SparseError, match="symbolic"):
        sp.block_spgemm_numeric(kh, Am, False, Bm, False, C0)
    C = sp.block_spgemm_symbolic(kh, Am, False, Bm, False)
    with pytest.raises(sp.B200SparseError, match="transpos"):
        sp.block_spgemm_numeric(kh, Am, False, Bm, True, C)
    # mixed scalar types
    Bf = sp.BsrMatrix(Bm.row_map, Bm.entries, Bm.values.float(), k, 2)
    with pytest.raises(sp.B200SparseError, match="same scalar type"):
        sp.block_spgemm_symbolic(kh, Am, False, Bf, False)
    with pytest.raises(sp.B200SparseError, match="same scalar type"):
        sp.block_spgemm_numeric(kh, Am, False, Bf, False, C)
    # 64-bit offsets are not provided
    with pytest.raises(sp.B200SparseError, match="64-bit"):
        sp.spgemm_numeric_views(kh, m, n, k, Am.row_map.long(), Am.entries, Am.values, False, Bm.row_map, Bm.entries, Bm.values,
                                False, C.row_map, C.entries, C.values, block_dim=2)
    # C ABI: bs < 1 and negative sizes
    import ctypes as Cc

    L = kk._lib.sparse()
    null = Cc.c_void_p(0)
    for bad in ((m, n, k, 0), (-1, n, k, 2)):
        rc = L.b200sp_bspgemm_numeric_f64_i32(kh.get_spgemm_handle()._plan, null, *bad, *([null] * 9))
        assert rc == 1  # B200SP_ERR_INVALID_ARGUMENT


def test_plan_without_symbolic_is_state_error(kk):
    import ctypes as Cc

    L = kk._lib.sparse()
    h = Cc.c_void_p()
    assert L.b200sp_spgemm_plan_create(Cc.byref(h)) == 0
    null = Cc.c_void_p(0)
    rc = L.b200sp_bspgemm_numeric_f64_i32(h, null, 4, 4, 4, 2, *([null] * 9))
    assert rc == 3 and "spgemm_symbolic" in L.b200sp_last_error_string().decode()  # B200SP_ERR_STATE
    assert L.b200sp_spgemm_plan_destroy(h, null) == 0
