"""GPU parity of SpMV / SpMM on 64-bit offsets (spmv64.cu: the (int64_t, size_t) instantiation of the reference's cuSPARSE slot,
sparse/tpls/KokkosSparse_spmv_tpl_spec_decl.hpp:246-257) through the C ABI (kokkos_kernels_b200.sparse.spmv on a CrsMatrix whose
row_map is int64): equal bits to the 32-bit entry points in the non-transposed modes, the oracle within the reference's tolerance
law (sparse/unit_test/Test_Sparse_spmv.hpp:120-150).  The window limit is lowered so that the matrices are cut into many 32-bit
windows; a matrix past 2^31 entries (26 GB) is left to tools/gpu_check --big.  Same cases as tests/test_emulated_spmv64.py, which
runs these kernels on the CPU."""
import numpy as np
import pytest
import torch

from test_emulated_spmv64 import random_crs

pytestmark = pytest.mark.gpu


def dev_matrix(sp, dev, rp, ci, v, n):
    return sp.CrsMatrix(torch.from_numpy(rp).to(dev), torch.from_numpy(ci).to(dev), torch.from_numpy(v).to(dev), n)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("col_bits", [32, 64])
@pytest.mark.parametrize("window", [None, 50000, 3000])
def test_rank1_equals_the_32_bit_path(cuda, oracle, dtype, col_bits, window):
    from kokkos_kernels_b200 import sparse as sp

    m, n = 20000, 15000
    rp64, ci32, v = random_crs(m, n, 11.0, seed=31, long_rows=4)
    v = v.astype(dtype)
    A32 = dev_matrix(sp, cuda, rp64.astype(np.int32), ci32, v, n)
    A64 = dev_matrix(sp, cuda, rp64, ci32.astype(np.int64) if col_bits == 64 else ci32, v, n)
    rng = np.random.default_rng(3)
    tol = 1e-13 if dtype == np.float64 else 1e-5
    short = np.diff(rp64) <= 512
    for mode, alpha, beta in (("N", 1.0, 0.0), ("N", -0.7, 1.3), ("C", 2.0, 1.0), ("T", 1.0, 0.0), ("H", 0.5, -2.0)):
        trans = mode in "TH"
        x = rng.uniform(-1, 1, m if trans else n).astype(dtype)
        y0 = rng.uniform(-1, 1, n if trans else m).astype(dtype)
        if beta == 0.0:
            y0[::7] = np.nan
        h32, h64 = sp.SPMVHandle(), sp.SPMVHandle()
        if window is not None:
            h64.set_window(window)
        xd = torch.from_numpy(x).to(cuda)
        for _ in range(5):  # through the self-tuning phases of every window's plan
            y32, y64 = torch.from_numpy(y0).to(cuda), torch.from_numpy(y0).to(cuda)
            sp.spmv(h32, mode, alpha, A32, xd, beta, y32)
            sp.spmv(h64, mode, alpha, A64, xd, beta, y64)
            torch.cuda.synchronize()
            g32, g64 = y32.cpu().numpy(), y64.cpu().numpy()
            assert not np.isnan(g64).any()
            if trans:
                assert np.allclose(g32, g64, rtol=0, atol=tol * 50)
            else:
                assert np.array_equal(g32[short], g64[short]), (h32.last_kernel(), h64.last_kernel())
                assert np.allclose(g32, g64, rtol=0, atol=tol * 50)
                if window is None:
                    assert np.array_equal(g32, g64)
        assert h64.windows() == (1 if window is None else h64.windows()) and (window is None or h64.windows() >= len(ci32) // window)
        if not trans:
            yo = np.where(np.isnan(y0), 0, y0).astype(dtype)
            oracle.spmv_serial(rp64.astype(np.int32), ci32, v, x, yo, alpha, beta)
            assert np.max(np.abs(g64.astype(np.float64) - yo.astype(np.float64))) <= tol * 100 * max(1.0, np.max(np.abs(yo)))


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_rank2_equals_the_32_bit_path(cuda, dtype):
    from kokkos_kernels_b200 import sparse as sp

    m, n, k = 12000, 9000, 6
    rp64, ci32, v = random_crs(m, n, 10.0, seed=41)
    v = v.astype(dtype)
    A32 = dev_matrix(sp, cuda, rp64.astype(np.int32), ci32, v, n)
    A64 = dev_matrix(sp, cuda, rp64, ci32.astype(np.int64), v, n)
    rng = np.random.default_rng(4)
    tol = 1e-12 if dtype == np.float64 else 2e-5
    for layout_left in (False, True):
        for mode, alpha, beta in (("N", 1.0, 0.0), ("N", 0.5, -1.5), ("T", 2.0, 0.0), ("T", -1.0, 1.0)):
            trans = mode == "T"
            xr, yr = (m, n) if trans else (n, m)
            X = torch.from_numpy(rng.uniform(-1, 1, (xr, k)).astype(dtype)).to(cuda)
            Y0 = torch.from_numpy(rng.uniform(-1, 1, (yr, k)).astype(dtype)).to(cuda)
            if layout_left:
                X, Y0 = X.t().contiguous().t(), Y0.t().contiguous().t()
            h32, h64 = sp.SPMVHandle(), sp.SPMVHandle()
            h64.set_window(8000)
            Y32, Y64 = Y0.clone(memory_format=torch.preserve_format), Y0.clone(memory_format=torch.preserve_format)
            sp.spmv(h32, mode, alpha, A32, X, beta, Y32)
            sp.spmv(h64, mode, alpha, A64, X, beta, Y64)
            torch.cuda.synchronize()
            assert h64.windows() >= 10
            if trans:
                assert torch.allclose(Y32, Y64, rtol=0, atol=tol * 20)
            else:
                assert torch.equal(Y32, Y64)


def test_errors_and_int32_only_operations(cuda):
    from kokkos_kernels_b200 import sparse as sp

    m, n = 500, 400
    rp64, ci32, v = random_crs(m, n, 6.0, seed=2)
    A64 = dev_matrix(sp, cuda, rp64, ci32.astype(np.int64), v, n)
    x = torch.zeros(n, dtype=torch.float64, device=cuda)
    y = torch.zeros(m, dtype=torch.float64, device=cuda)
    h = sp.SPMVHandle()
    h.set_window(8)  # no row fits
    with pytest.raises(sp.B200SparseError, match="window"):
        sp.spmv(h, "N", 1.0, A64, x, 0.0, y)
    bad = ci32.astype(np.int64)
    bad[7] = 2**31 + 1
    with pytest.raises(sp.B200SparseError, match="31 bits"):
        sp.spmv(sp.SPMVHandle(), "N", 1.0, dev_matrix(sp, cuda, rp64, bad, v, n), x, 0.0, y)
    sp.spmv(None, "N", 1.0, A64, x, 0.0, y)  # the convenience overload builds its own handle
    with pytest.raises(sp.B200SparseError, match="int32"):  # everything else is (int32, int32)
        sp.transpose_matrix(A64)
