"""GPU parity of spgemm_jacobi (C = (I - omega D^-1 A) B) through the C ABI against the oracle's restatement of
spgemm_jacobi_seq: structure bit-identical, values by the reference's is_same_matrix law -- the shape of
test_spgemm_jacobi (sparse/unit_test/Test_Sparse_spgemm_jacobi.hpp:176-228)."""
import numpy as np
import pytest
import torch

from test_oracle_jacobi import diag_dominant

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n,per", [(1000, 10), (20000, 6)])
@pytest.mark.parametrize("dtype,eps", [(np.float64, 1e-7), (np.float32, 3.7e-3)])
def test_spgemm_jacobi(cuda, oracle, n, per, dtype, eps):
    from kokkos_kernels_b200 import sparse as sp

    rp, ci, v = diag_dominant(n, per, n)
    v = v.astype(dtype)
    omega, dinv = 3.0, np.full(n, 2.0, dtype=dtype)
    exp = oracle.spgemm_jacobi(rp, ci, v, rp, ci, v, n, dtype(omega), dinv)
    A = sp.CrsMatrix(torch.from_numpy(rp).to(cuda), torch.from_numpy(ci).to(cuda), torch.from_numpy(v).to(cuda), n)
    kh = sp.KokkosKernelsHandle()
    kh.create_spgemm_handle()
    with pytest.raises(Exception):
        sp.spgemm_jacobi(kh, A, False, A, False, A, omega, torch.from_numpy(dinv).to(cuda))  # symbolic first
    Cm = sp.spgemm_symbolic(kh, A, False, A, False)
    sp.spgemm_jacobi(kh, A, False, A, False, Cm, omega, torch.from_numpy(dinv).to(cuda).reshape(n, 1))
    torch.cuda.synchronize()
    assert np.array_equal(Cm.row_map.cpu().numpy(), exp[0]) and np.array_equal(Cm.entries.cpu().numpy(), exp[1])
    assert oracle.rel_mismatch(Cm.values.cpu().numpy().astype(np.float64), exp[2].astype(np.float64), eps) == 0
