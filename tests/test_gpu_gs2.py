"""GPU run of the two-stage Gauss-Seidel (gs2.cu: GS_TWOSTAGE with inner Jacobi-Richardson sweeps, every product the library's
SpMV) through the Python mirror -- KokkosKernelsHandle::create_gs_handle(GS_TWOSTAGE), set_gs_set_num_inner_sweeps / ..., then
gauss_seidel_symbolic / numeric / apply: the oracle's restatement of the reference's TwostageGaussSeidel::apply, classic and
compact recurrences, and the reference unit test's acceptance (sparse/unit_test/Test_Sparse_gauss_seidel.hpp:236-241).  Same
cases as tests/test_emulated_gs2.py, which runs these kernels on the CPU."""
import numpy as np
import pytest
import torch

import exact_ref as R
from test_oracle_gs2 import dd_matrix

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("compact", [False, True])
def test_oracle_parity(cuda, oracle, dtype, compact):
    from kokkos_kernels_b200 import sparse as sp

    n, ghosts = 30000, 200
    rp, ci, v = dd_matrix(n, 11, extra_cols=ghosts)
    v = v.astype(dtype)
    ncols = n + ghosts
    rng = np.random.default_rng(4)
    b = rng.uniform(-1, 1, n).astype(dtype)
    x0 = rng.uniform(-1, 1, ncols).astype(dtype)
    t = lambda a: torch.from_numpy(a).to(cuda)
    rpd, cid, vd, bd = t(rp), t(ci), t(v), t(b)
    tol = 1e-13 if dtype == np.float64 else 1e-5
    applies = (sp.symmetric_gauss_seidel_apply, sp.forward_sweep_gauss_seidel_apply, sp.backward_sweep_gauss_seidel_apply)
    for inner, gamma, outer in ((1, 1.0, 1), (0, 0.7, 1), (3, 1.0, 1), (2, 0.9, 3)):
        kh = sp.KokkosKernelsHandle()
        kh.create_gs_handle(sp.GS_TWOSTAGE)
        kh.set_gs_twostage(True, n)
        kh.set_gs_twostage_compact_form(compact)
        kh.set_gs_set_num_inner_sweeps(inner)
        kh.set_gs_set_num_outer_sweeps(outer)
        kh.set_gs_set_inner_damp_factor(gamma)
        sp.gauss_seidel_symbolic(kh, n, ncols, rpd, cid, False)
        sp.gauss_seidel_numeric(kh, n, ncols, rpd, cid, vd, False)
        for direction, fn in enumerate(applies):
            for omega, init_zero, num_iter in ((1.0, False, 1), (0.9, True, 2)):
                xd = t(x0)
                fn(kh, n, ncols, rpd, cid, vd, xd, bd, init_zero, True, omega, num_iter)
                torch.cuda.synchronize()
                x = xd.cpu().numpy()
                xo = x0.copy()
                oracle.gs2_apply(rp, ci, v, ncols, xo, b, init_zero, dtype(omega), num_iter, direction, compact=compact, inner_sweeps=inner,
                                 outer_sweeps=outer, gamma=dtype(gamma))
                err = np.max(np.abs(x.astype(np.float64) - xo.astype(np.float64)))
                assert err <= tol * 20 * max(1.0, np.max(np.abs(xo))), (inner, gamma, outer, direction, omega, init_zero, err)
                ex, bnd = R.gs2_ref(rp, ci, v, ncols, x0, b, init_zero, omega, num_iter, direction, compact, inner, outer, gamma)
                R.assert_within(x, ex, bnd, str((inner, gamma, outer, direction, omega, init_zero)))
        kh.destroy_gs_handle()


def test_reference_unit_test_and_multivectors(cuda, oracle):
    from kokkos_kernels_b200 import sparse as sp

    n, k = 40000, 3
    rp, ci, v = dd_matrix(n, 245)
    rng = np.random.default_rng(3)
    xs = rng.uniform(-1, 1, (n, k))
    Y = np.zeros((n, k))
    for j in range(k):
        yj = np.zeros(n)
        oracle.spmv_serial(rp, ci, v, np.ascontiguousarray(xs[:, j]), yj, 1.0, 0.0)
        Y[:, j] = yj
    t = lambda a: torch.from_numpy(a).to(cuda)
    rpd, cid, vd = t(rp), t(ci), t(v)
    Yd = t(np.ascontiguousarray(Y.T)).t()  # LayoutLeft: columns contiguous
    kh = sp.KokkosKernelsHandle()
    kh.create_gs_handle(sp.GS_TWOSTAGE)
    sp.gauss_seidel_symbolic(kh, n, n, rpd, cid, False)
    sp.gauss_seidel_numeric(kh, n, n, rpd, cid, vd, False)
    init = np.linalg.norm(xs, axis=0)
    for direction, fn in enumerate((sp.symmetric_gauss_seidel_apply, sp.forward_sweep_gauss_seidel_apply, sp.backward_sweep_gauss_seidel_apply)):
        Xd = t(np.ascontiguousarray(rng.uniform(-1, 1, (k, n)))).t()
        fn(kh, n, n, rpd, cid, vd, Xd, Yd, True, True, 0.9, 2)
        torch.cuda.synchronize()
        X = Xd.cpu().numpy()
        assert np.all(np.linalg.norm(X - xs, axis=0) < init)  # EXPECT_LT(result_norm_res, initial_norm_res)
        for j in range(k):
            xo = np.zeros(n)
            oracle.gs2_apply(rp, ci, v, n, xo, np.ascontiguousarray(Y[:, j]), True, 0.9, 2, direction)
            assert np.allclose(X[:, j], xo, rtol=0, atol=1e-13)
            ex, bnd = R.gs2_ref(rp, ci, v, n, np.zeros(n), np.ascontiguousarray(Y[:, j]), True, 0.9, 2, direction)
            R.assert_within(X[:, j], ex, bnd, f"direction {direction} column {j}")
    kh.set_gs_twostage(False, n)  # the classic (sptrsv) form: tests/test_gpu_sptrsv.py; switching resets the phases
    assert not kh.get_twostage_gs_handle().isTwoStage() and not kh.get_twostage_gs_handle().is_symbolic_called()
    kh2 = sp.KokkosKernelsHandle()
    kh2.create_gs_handle()
    with pytest.raises(sp.B200SparseError):
        kh2.set_gs_set_num_inner_sweeps(2)  # not a two-stage handle (KokkosKernels_Handle.hpp:631-637)


def test_pcgsolve_with_two_stage_handle(cuda, oracle):
    from kokkos_kernels_b200 import sparse as sp
    from test_oracle_cg import spd_lap27

    rp, ci, v = spd_lap27(24, shift=0.5)
    n = len(rp) - 1
    xs = np.random.default_rng(0).uniform(-1, 1, n)
    b = np.zeros(n)
    oracle.spmv_serial(rp, ci, v, xs, b, 1.0, 0.0)
    xo = np.zeros(n)
    it_o, _ = oracle.pcg_gs2(rp, ci, v, b, xo, 500, 1e-9, inner_sweeps=2)
    it_c, _ = oracle.cg(rp, ci, v, b, np.zeros(n), 500, 1e-9)
    t = lambda a: torch.from_numpy(a).to(cuda)
    A = sp.CrsMatrix(t(rp), t(ci), t(v), n)
    kh = sp.KokkosKernelsHandle()
    kh.create_gs_handle(sp.GS_TWOSTAGE)
    kh.set_gs_set_num_inner_sweeps(2)
    xd = torch.zeros(n, dtype=torch.float64, device=cuda)
    res = sp.pcgsolve(None, A, t(b), xd, 500, 1e-9, use_sgs=True, gs_handle=kh)
    torch.cuda.synchronize()
    x = xd.cpu().numpy()
    assert abs(res.iteration - it_o) <= 1 and res.iteration < it_c
    assert res.norm_res <= 1e-9 and np.linalg.norm(x - xs) / np.linalg.norm(xs) < 1e-8
