"""GPU run of the reference's GMRES unit test (sparse/unit_test/Test_Sparse_gmres.hpp:86-170) through
kokkos_kernels_b200.sparse.gmres -> b200sp_gmres_*: n = 5000, m = 15, B = 1, X = 0; CGS2, MGS and MatrixPrec(A); double
(tol 1e-8) and float (1e-5); acceptance = the test's (true relative residual < tol, flag Conv) plus the oracle's iteration
count."""
import numpy as np
import pytest
import torch

from gmres_cases import crs_to_bsr, gmres_matrix, true_rel_res

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("use_blocks", [False, True])  # run_test_gmres<false> / <true> (:202-203): CrsMatrix, BsrMatrix of 10 x 10 blocks
@pytest.mark.parametrize("dtype,tol", [(np.float64, 1e-8), (np.float32, 1e-5)])
def test_gmres_reference_test(cuda, oracle, dtype, tol, use_blocks):
    from kokkos_kernels_b200 import sparse as sp

    n, m = 5000, 15
    A = gmres_matrix(n, 1.0, dtype=dtype)
    if use_blocks:
        brp, bci, bv = crs_to_bsr(*A, 10)
        Ad = sp.BsrMatrix(torch.from_numpy(brp).to(cuda), torch.from_numpy(bci).to(cuda), torch.from_numpy(bv).to(cuda), n // 10, 10)
    else:
        Ad = sp.CrsMatrix(torch.from_numpy(A[0]).to(cuda), torch.from_numpy(A[1]).to(cuda), torch.from_numpy(A[2]).to(cuda), n)
    b = np.ones(n, dtype=dtype)
    Bd = torch.from_numpy(b).to(cuda)
    kh = sp.KokkosKernelsHandle()
    kh.create_gmres_handle(m, tol)
    gh = kh.get_gmres_handle()
    assert gh.get_conv_flag_val() == sp.GMRESHandle.NotRun
    for variant in ("cgs2", "mgs", "matrixprec"):
        gh.reset_handle(m, tol)
        if variant == "mgs":
            gh.set_ortho(sp.GMRESHandle.MGS)
        prec = sp.MatrixPrec(Ad) if variant == "matrixprec" else None
        Xd = torch.zeros(n, dtype=Bd.dtype, device=cuda)
        sp.gmres(kh, Ad, Bd, Xd, prec)
        x = Xd.cpu().numpy()
        assert true_rel_res(oracle, A, b, x) < gh.get_tol()  # EXPECT_LT(endRes, tol)
        assert gh.get_conv_flag_val() == sp.GMRESHandle.Conv  # EXPECT_EQ(conv_flag, Conv)
        xo = np.zeros(n, dtype=dtype)
        st, it_o, _, _ = oracle.gmres(A, b, xo, m=m, tol=tol, ortho=1 if variant == "mgs" else 0, prec=A if prec else None)
        assert st == 0 and abs(gh.get_num_iters() - it_o) <= 1
    with pytest.raises(sp.B200SparseError):
        sp.gmres(kh, Ad, Bd[:-1], torch.zeros(n, dtype=Bd.dtype, device=cuda))
