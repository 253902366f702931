"""GPU parity of the CG driver (kokkos_kernels_b200.sparse.pcgsolve -> b200sp_cg_solve_f64_i32) against the oracle's
restatement of the reference's pcgsolve without preconditioner (perf_test/sparse/KokkosSparse_pcg.hpp:248-466; tolerance
1e-7 as its driver uses, perf_test/sparse/KokkosSparse_pcg.cpp:70)."""
import numpy as np
import pytest
import torch

from test_oracle_cg import spd_lap27

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("g", [14, 40])
def test_pcgsolve(cuda, oracle, g):
    from kokkos_kernels_b200 import sparse as sp

    rp, ci, v = spd_lap27(g, shift=0.5)
    n = len(rp) - 1
    rng = np.random.default_rng(0)
    xs = rng.uniform(-1, 1, n)
    b = np.zeros(n)
    oracle.spmv_serial(rp, ci, v, xs, b, 1.0, 0.0)
    xo = np.zeros(n)
    it_o, nr_o = oracle.cg(rp, ci, v, b, xo, 100000, 1e-7)
    A = sp.CrsMatrix(torch.from_numpy(rp).to(cuda), torch.from_numpy(ci).to(cuda), torch.from_numpy(v).to(cuda), n)
    h = sp.SPMVHandle()
    bd = torch.from_numpy(b).to(cuda)
    for check_every in (1, 8):
        xd = torch.zeros(n, dtype=torch.float64, device=cuda)
        res = sp.pcgsolve(h, A, bd, xd, 100000, 1e-7, check_every)
        assert abs(res.iteration - it_o) <= 2 and res.norm_res <= 1e-7, (res.iteration, it_o, res.norm_res)
        x = xd.cpu().numpy()
        assert np.linalg.norm(x - xo) / np.linalg.norm(xo) < 1e-8
    xd = torch.zeros(n, dtype=torch.float64, device=cuda)
    res = sp.pcgsolve(h, A, bd, xd, 7, 1e-7, 3)
    xo7 = np.zeros(n)
    it7, nr7 = oracle.cg(rp, ci, v, b, xo7, 7, 1e-7)
    assert res.iteration == 7 == it7 and abs(res.norm_res - nr7) <= 1e-9 * nr7
    assert np.allclose(xd.cpu().numpy(), xo7, rtol=1e-10, atol=1e-12)
    with pytest.raises(sp.B200SparseError):
        sp.pcgsolve(h, A, bd.float(), xd.float())
