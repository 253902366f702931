"""GPU run of the point Gauss-Seidel kernels and the SGS-preconditioned CG through the Python mirror: proper colouring, sweeps equal to
the oracle's restatement of the reference functor over the same colour sets, the reference unit test's acceptance
(sparse/unit_test/Test_Sparse_gauss_seidel.hpp:180-216), and pcgsolve(use_sgs=True) against the oracle."""
import numpy as np
import pytest
import torch

from gmres_cases import gmres_matrix
from test_emulated_gs import check_coloring, symmetrize
from test_oracle_cg import spd_lap27

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("symmetric", [True, False])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_gauss_seidel(cuda, oracle, symmetric, dtype):
    from kokkos_kernels_b200 import sparse as sp

    n = 20000
    rp, ci, v = gmres_matrix(n, 1.0, seed=245)
    if symmetric:
        rp, ci, v = symmetrize(rp, ci, v, n)
    v = v.astype(dtype)
    rng = np.random.default_rng(3)
    xs = rng.uniform(-1, 1, n).astype(dtype)
    y = np.zeros(n, dtype=dtype)
    oracle.spmv_serial(rp, ci, v, xs, y, 1.0, 0.0)
    t = lambda a: torch.from_numpy(a).to(cuda)
    rpd, cid, vd, yd = t(rp), t(ci), t(v), t(y)
    kh = sp.KokkosKernelsHandle()
    kh.create_gs_handle()
    sp.gauss_seidel_symbolic(kh, n, n, rpd, cid, symmetric)
    sp.gauss_seidel_numeric(kh, n, n, rpd, cid, vd, symmetric)
    colors, cptr, crows = kh.get_gs_handle().get_coloring(n)
    check_coloring(n, rp, ci, len(cptr) - 1, colors, cptr, crows)
    rows = np.repeat(np.arange(n), np.diff(rp))
    dinv = (1.0 / np.bincount(rows[rows == ci], weights=v[rows == ci].astype(np.float64), minlength=n)).astype(dtype)
    init = np.linalg.norm(xs.astype(np.float64))
    applies = (sp.symmetric_gauss_seidel_apply, sp.forward_sweep_gauss_seidel_apply, sp.backward_sweep_gauss_seidel_apply)
    for direction, fn in enumerate(applies):
        xd = torch.ones(n, dtype=vd.dtype, device=cuda)
        fn(kh, n, n, rpd, cid, vd, xd, yd, True, True, 0.9, 2)
        torch.cuda.synchronize()
        x = xd.cpu().numpy()
        xo = oracle.gs_apply(rp, ci, v, cptr, crows, dinv, y, np.ones(n, dtype), True, dtype(0.9), 2, direction)
        tol = 1e-12 if dtype == np.float64 else 2e-5
        assert np.max(np.abs(x.astype(np.float64) - xo.astype(np.float64))) <= tol * max(1.0, np.max(np.abs(xo)))
        assert np.linalg.norm(x.astype(np.float64) - xs.astype(np.float64)) < init
    kh.destroy_gs_handle()


def test_pcgsolve_sgs(cuda, oracle):
    from kokkos_kernels_b200 import sparse as sp

    rp, ci, v = spd_lap27(24, shift=0.5)
    n = len(rp) - 1
    xs = np.random.default_rng(0).uniform(-1, 1, n)
    b = np.zeros(n)
    oracle.spmv_serial(rp, ci, v, xs, b, 1.0, 0.0)
    t = lambda a: torch.from_numpy(a).to(cuda)
    A = sp.CrsMatrix(t(rp), t(ci), t(v), n)
    gh = sp.GaussSeidelHandle()
    sp.gauss_seidel_symbolic(gh, n, n, A.row_map, A.entries, True)
    sp.gauss_seidel_numeric(gh, n, n, A.row_map, A.entries, A.values, True)
    colors, cptr, crows = gh.get_coloring(n)
    rows = np.repeat(np.arange(n), np.diff(rp))
    xo = np.zeros(n)
    it_o, _ = oracle.pcg(rp, ci, v, b, xo, 100000, 1e-7, cptr, crows, 1.0 / v[rows == ci])
    xd = torch.zeros(n, dtype=torch.float64, device=cuda)
    res = sp.pcgsolve(sp.SPMVHandle(), A, t(b), xd, 100000, 1e-7, 8, use_sgs=True, gs_handle=gh)
    assert abs(res.iteration - it_o) <= 1 and res.norm_res <= 1e-7
    assert np.linalg.norm(xd.cpu().numpy() - xo) / np.linalg.norm(xo) < 1e-8
    xd2 = torch.zeros(n, dtype=torch.float64, device=cuda)
    res2 = sp.pcgsolve(None, A, t(b), xd2, 100000, 1e-7, 8, use_sgs=True)  # handles created inside, as the reference's driver does
    assert res2.iteration == res.iteration


def test_gauss_seidel_ghost_columns(cuda, oracle):
    """num_cols > num_rows (the local matrix of a distributed one): ghost entries of x are read, never written."""
    from kokkos_kernels_b200 import sparse as sp
    from test_oracle_gs2 import dd_matrix

    n, ghosts = 20000, 300
    rp, ci, v = dd_matrix(n, 31, extra_cols=ghosts)
    ncols = n + ghosts
    t = lambda a: torch.from_numpy(a).to(cuda)
    rpd, cid, vd = t(rp), t(ci), t(v)
    kh = sp.KokkosKernelsHandle()
    kh.create_gs_handle()
    sp.gauss_seidel_symbolic(kh, n, ncols, rpd, cid, False)
    sp.gauss_seidel_numeric(kh, n, ncols, rpd, cid, vd, False)
    colors, cptr, crows = kh.get_gs_handle().get_coloring(n)
    rows = np.repeat(np.arange(n), np.diff(rp))
    dinv = 1.0 / np.bincount(rows[rows == ci], weights=v[rows == ci], minlength=n)
    rng = np.random.default_rng(5)
    b, x0 = rng.uniform(-1, 1, n), rng.uniform(-1, 1, ncols)
    for direction, fn in enumerate((sp.symmetric_gauss_seidel_apply, sp.forward_sweep_gauss_seidel_apply, sp.backward_sweep_gauss_seidel_apply)):
        xd = t(x0)
        fn(kh, n, ncols, rpd, cid, vd, xd, t(b), False, True, 0.9, 2)
        torch.cuda.synchronize()
        x = xd.cpu().numpy()
        xo = oracle.gs_apply(rp, ci, v, cptr, crows, dinv, b, x0.copy(), False, 0.9, 2, direction)
        assert np.array_equal(x[n:], x0[n:]) and np.max(np.abs(x - xo)) <= 1e-12
