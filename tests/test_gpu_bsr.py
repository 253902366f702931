"""GPU parity of BsrMatrix SpMV / SpMM through the C ABI (kokkos_kernels_b200.sparse.spmv on a BsrMatrix) against the
oracle -- the reference's own sweep (sparse/unit_test/Test_Sparse_spmv_bsr.hpp:351-456,595-700) with its tolerance
law, plus sizes that wrap the TMA ring, block rows longer than a stage and every block size 2..17.  Same cases as
tests/test_emulated_bsr.py, which runs these kernels on the CPU."""
import numpy as np
import pytest
import torch

from bsr_cases import BLOCK_SIZES, COEFS_ALPHA, COEFS_BETA, PRIME_CASE, SHAPES, bsr_random, op_max_nnz_per_row, tolerance

pytestmark = pytest.mark.gpu

CASES = [(bs, mb, nb) for (mb, nb) in SHAPES for bs in BLOCK_SIZES] + [PRIME_CASE]


def to_dev(sp, dev, bs, nb, rp, ci, v):
    return sp.BsrMatrix(torch.from_numpy(rp).to(dev), torch.from_numpy(ci).to(dev), torch.from_numpy(v).to(dev), nb, bs)


def expected(oracle, mode, bs, nb, rp, ci, v, X, Y0, alpha, beta):
    Yc = np.nan_to_num(Y0.copy(order="K")) if beta == 0.0 else Y0.copy(order="K")
    if mode in "NC":
        return oracle.bsr_spmv_v42(bs, rp, ci, v, X, Yc, alpha, beta)
    return oracle.bsr_spmv_v41(mode, bs, nb, rp, ci, v, X, Yc, alpha, beta)


def run_rank1(sp, oracle, dev, handle, A, host, mode, rng, alpha, beta, dtype):
    bs, mb, nb, rp, ci, v = host
    trans = mode in "TH"
    nx, ny = (mb * bs, nb * bs) if trans else (nb * bs, mb * bs)
    x = rng.uniform(0, 10, nx).astype(dtype)
    y0 = rng.uniform(0, 10, ny).astype(dtype)
    if beta == 0.0:
        y0[::7] = np.nan
    yd = torch.from_numpy(y0).to(dev)
    sp.spmv(handle, mode, alpha, A, torch.from_numpy(x).to(dev), beta, yd)
    torch.cuda.synchronize()
    got = yd.cpu().numpy()
    exp = expected(oracle, mode, bs, nb, rp, ci, v, x, y0, alpha, beta)
    assert not np.isnan(got).any(), "NaN survived beta == 0"
    tol = tolerance(dtype, alpha, beta, op_max_nnz_per_row(bs, rp, ci, nb, trans))
    err = np.max(np.abs(got - exp), initial=0.0)
    assert err <= tol, f"{handle.last_kernel()} mode {mode} bs {bs} alpha {alpha} beta {beta}: err {err:.3e} > {tol:.3e}"


@pytest.mark.parametrize("bs,mb,nb", CASES)
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_reference_sweep_rank1(cuda, oracle, bs, mb, nb, dtype):
    from kokkos_kernels_b200 import sparse as sp

    rp, ci, v = bsr_random(bs, mb, nb, seed=3 + bs + mb, dtype=dtype, sort=False)
    A = to_dev(sp, cuda, bs, nb, rp, ci, v)
    rng = np.random.default_rng(17)
    for algo in (sp.SPMV_DEFAULT, sp.SPMV_NATIVE, sp.SPMV_BSR_V41):  # test_spmv_combos (:364)
        h = sp.SPMVHandle(algo)
        for mode in "NTCH":
            for alpha in COEFS_ALPHA:
                for beta in COEFS_BETA:
                    run_rank1(sp, oracle, cuda, h, A, (bs, mb, nb, rp, ci, v), mode, rng, alpha, beta, dtype)


@pytest.mark.parametrize("bs,mb,nb", CASES)
@pytest.mark.parametrize("layout", ["left", "right"])
def test_reference_sweep_multivector(cuda, oracle, bs, mb, nb, layout):
    from kokkos_kernels_b200 import sparse as sp

    dtype = np.float64
    rp, ci, v = bsr_random(bs, mb, nb, seed=5 + bs + nb, dtype=dtype, sort=False)
    A = to_dev(sp, cuda, bs, nb, rp, ci, v)
    rng = np.random.default_rng(19)
    h = sp.SPMVHandle()

    def dev2d(a):
        t = torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
        return t if layout == "right" else t.t().contiguous().t()

    for mode in "NTCH":
        trans = mode in "TH"
        nx, ny = (mb * bs, nb * bs) if trans else (nb * bs, mb * bs)
        max_row = op_max_nnz_per_row(bs, rp, ci, nb, trans)
        for k in (1, 7):
            X = rng.uniform(0, 10, (nx, k))
            Y0 = rng.uniform(0, 10, (ny, k))
            for alpha in COEFS_ALPHA:
                for beta in COEFS_BETA:
                    Yin = Y0.copy()
                    if beta == 0.0 and ny:
                        Yin[::5] = np.nan
                    Yd = dev2d(Yin)
                    sp.spmv(h, mode, alpha, A, dev2d(X), beta, Yd)
                    torch.cuda.synchronize()
                    got = Yd.cpu().numpy()
                    exp = expected(oracle, mode, bs, nb, rp, ci, v, X, Yin, alpha, beta)
                    assert not np.isnan(got).any()
                    assert np.max(np.abs(got - exp), initial=0.0) <= tolerance(dtype, alpha, beta, max_row), (h.last_kernel(), mode, k, alpha, beta)


@pytest.mark.parametrize("bs", [1, 2, 3, 4, 5, 7, 8, 11, 16, 17])
@pytest.mark.parametrize("layout", ["left", "right"])
def test_tensor_core_multivector(cuda, oracle, bs, layout):
    """SPMV_BSR_TC (the reference's tensor-core functor, spmv_bsrmatrix_impl.hpp:74-459, selected by the handle's algorithm,
    spmv_bsrmatrix_spec.hpp:176-245): mma.sync m8n8k4 kernel for double / mode N / bs <= 16, the default kernels otherwise."""
    from kokkos_kernels_b200 import sparse as sp

    dtype = np.float64
    mb, nb = 300, 280
    rp, ci, v = bsr_random(bs, mb, nb, seed=40 + bs, dtype=dtype, sort=False)
    A = to_dev(sp, cuda, bs, nb, rp, ci, v)
    rng = np.random.default_rng(29)
    h = sp.SPMVHandle(sp.SPMV_BSR_TC)

    def dev2d(a):
        t = torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
        return t if layout == "right" else t.t().contiguous().t()

    for mode in "NT":
        trans = mode == "T"
        nx, ny = (mb * bs, nb * bs) if trans else (nb * bs, mb * bs)
        max_row = op_max_nnz_per_row(bs, rp, ci, nb, trans)
        for k in (2, 8, 13, 16, 33):
            X = rng.uniform(0, 10, (nx, k))
            Y0 = rng.uniform(0, 10, (ny, k))
            for alpha, beta in ((1.0, 0.0), (-2.5, 1.0), (3.7, -1.5)):
                Yin = Y0.copy()
                if beta == 0.0:
                    Yin[::5] = np.nan
                Yd = dev2d(Yin)
                sp.spmv(h, mode, alpha, A, dev2d(X), beta, Yd)
                torch.cuda.synchronize()
                got = Yd.cpu().numpy()
                exp = expected(oracle, mode, bs, nb, rp, ci, v, X, Yin, alpha, beta)
                assert not np.isnan(got).any()
                assert np.max(np.abs(got - exp), initial=0.0) <= tolerance(dtype, alpha, beta, max_row), (h.last_kernel(), mode, k, alpha, beta)
                if mode == "N" and 2 <= bs <= 16:
                    assert h.last_kernel().startswith("bsr_mm_tc<f64"), h.last_kernel()
                else:
                    assert not h.last_kernel().startswith("bsr_mm_tc"), h.last_kernel()
    # the scalar functors on request (SPMV_BSR_V42), the default's choice by the number of columns
    for algo, k, tc in ((sp.SPMV_BSR_V42, 8, False), (sp.SPMV_DEFAULT, 8, True), (sp.SPMV_DEFAULT, 3, False)):
        h2 = sp.SPMVHandle(algo)
        X = rng.uniform(0, 10, (nb * bs, k))
        Yin = rng.uniform(0, 10, (mb * bs, k))
        Yd = dev2d(Yin)
        sp.spmv(h2, "N", 1.5, A, dev2d(X), -0.5, Yd)
        torch.cuda.synchronize()
        exp = expected(oracle, "N", bs, nb, rp, ci, v, X, Yin, 1.5, -0.5)
        assert np.max(np.abs(Yd.cpu().numpy() - exp), initial=0.0) <= tolerance(dtype, 1.5, -0.5, op_max_nnz_per_row(bs, rp, ci, nb, False))
        assert h2.last_kernel().startswith("bsr_mm_tc") == (tc and 2 <= bs <= 16), (h2.last_kernel(), algo, k)


@pytest.mark.parametrize("force", [None, "walk"])
@pytest.mark.parametrize("bs", list(range(2, 18)))
def test_tile_kernel_every_block_size(cuda, oracle, bs, force, monkeypatch):
    """Default selection (element-per-lane tile kernel for bs <= 5, row-vector kernel above: the measured choice) and the
    run-time block size tile kernel forced for every bs it supports."""
    from kokkos_kernels_b200 import sparse as sp

    if force:
        monkeypatch.setenv("B200SP_BSR_KERNEL", force)
    else:
        monkeypatch.delenv("B200SP_BSR_KERNEL", raising=False)

    mb = max(20000, 4000000 // (bs * bs))  # enough tiles per CTA to wrap the ring on 132 SMs
    nb = mb + 13
    rp, ci, v = bsr_random(bs, mb, nb, seed=bs, min_blocks=0, max_blocks=12, sort=False)
    A = to_dev(sp, cuda, bs, nb, rp, ci, v)
    h = sp.SPMVHandle()
    rng = np.random.default_rng(bs)
    for alpha, beta in ((1.0, 0.0), (3.7, -1.5)):
        run_rank1(sp, oracle, cuda, h, A, (bs, mb, nb, rp, ci, v), "N", rng, alpha, beta, np.float64)
        if force:
            assert h.last_kernel().startswith("bsr_tile<" if bs <= 16 else "bsr_vector"), h.last_kernel()
        else:
            want = "bsr_tile_e" if bs <= 5 else ("bsr_mm_tc<f64" if bs <= 16 else "bsr_vector")  # double: tensor cores for bs 6..16
            assert h.last_kernel().startswith(want), h.last_kernel()
    run_rank1(sp, oracle, cuda, h, A, (bs, mb, nb, rp, ci, v), "T", rng, -1.0, 1.0, np.float64)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_long_block_rows_and_tail(cuda, oracle, dtype):
    from kokkos_kernels_b200 import sparse as sp

    bs, mb, nb = 3, 900, 1500
    rng = np.random.default_rng(23)
    lens = rng.integers(0, 6, mb)
    lens[[5, 400, 899]] = [700, 227, 1300]
    if int(lens.sum()) % 4 == 0:
        lens[10] += 1
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    ci = np.concatenate([rng.choice(nb, int(l), replace=False) for l in lens]).astype(np.int32)
    v = rng.uniform(0, 10, len(ci) * bs * bs).astype(dtype)
    A = to_dev(sp, cuda, bs, nb, rp, ci, v)
    h = sp.SPMVHandle()
    for alpha, beta in ((1.0, 0.0), (-1.0, 1.0), (3.7, -1.5)):
        run_rank1(sp, oracle, cuda, h, A, (bs, mb, nb, rp, ci, v), "N", rng, alpha, beta, dtype)
        assert h.last_kernel().startswith("bsr_tile"), h.last_kernel()


def test_errors(cuda):
    from kokkos_kernels_b200 import sparse as sp

    z = torch.zeros(2, dtype=torch.int32, device=cuda)
    e = torch.zeros(0, dtype=torch.int32, device=cuda)
    with pytest.raises(sp.B200SparseError):
        sp.BsrMatrix(z, e, torch.zeros(0, dtype=torch.float64, device=cuda), 1, 0)  # block size 0 (BsrMatrix.hpp:429-433)
    A = sp.BsrMatrix(z, e, torch.zeros(0, dtype=torch.float64, device=cuda), 1, 3)
    with pytest.raises(sp.B200SparseError):  # dimensions (KokkosSparse_spmv.hpp:126-142) are checked in POINT units
        sp.spmv(sp.SPMVHandle(), "N", 1.0, A, torch.zeros(1, dtype=torch.float64, device=cuda), 0.0,
                torch.zeros(3, dtype=torch.float64, device=cuda))
