"""GPU parity of rank-1 SpMV through the C ABI against the oracle -- mirrors the reference's
own sweep (sparse/unit_test/Test_Sparse_spmv.hpp:345-463,1060-1068)."""
import numpy as np
import pytest
import torch

import exact_ref as R
from helpers import kk_matrix, rowwise_scale, spmv_tolerance

pytestmark = pytest.mark.gpu

TOL64 = 1e-10  # north_star: within 1e-10 rel of the Serial path (row-wise scaled, SURVEY 8d)
TOL32 = 1e-4


def dev_matrix(sp, dev, rp, ci, v, ncols):
    return sp.CrsMatrix(torch.from_numpy(rp).to(dev), torch.from_numpy(ci).to(dev), torch.from_numpy(v).to(dev), ncols)


def run_case(sp, oracle, dev, handle, A, host, mode, alpha, beta, x, y0, ref_tol):
    rp, ci, v, ncols = host
    nrows = len(rp) - 1
    trans = mode in "TH"
    yd = torch.from_numpy(y0).to(dev)
    sp.spmv(handle, mode, alpha, A, torch.from_numpy(x).to(dev), beta, yd)
    torch.cuda.synchronize()
    got = yd.cpu().numpy()
    # Serial path of the reference (O1 for N/C, O5 for T/H) and the unit test's own oracle (O3)
    if not trans:
        exp = oracle.spmv_serial(rp, ci, v, x, y0.copy(), alpha, beta)
    else:
        exp = oracle.spmv_transpose(rp, ci, v, ncols, x, y0.copy(), alpha, beta)
    exp3 = oracle.spmv_test(mode, rp, ci, v, x, y0.copy(), alpha, beta)
    assert not np.isnan(got).any(), f"NaN survived (mode {mode} alpha {alpha} beta {beta})"
    scale = rowwise_scale(rp, ci, v, x, y0, alpha, beta, ncols_out=ncols, trans=trans)
    tol = TOL64 if v.dtype == np.float64 else TOL32
    err = np.abs(got.astype(np.float64) - exp.astype(np.float64))
    bad = err > tol * scale + 1e-300
    assert not bad.any(), f"mode {mode} a={alpha} b={beta}: {bad.sum()} rows beyond {tol} (max {np.max(err / np.maximum(scale, 1e-300)):.3e})"
    # the reference's own acceptance law against its own test oracle
    assert np.max(np.abs(got - exp3)) <= ref_tol + 1e-300
    # entry by entry within the rounding bound of the exact product (tests/exact_ref.py)
    R.assert_within(got, R.spmm_exact(rp, ci, v, x, y0, alpha, beta, trans), R.spmm_bound(rp, ci, v, x, y0, alpha, beta, trans),
                    f"{handle.last_kernel() if handle is not None else 'no plan'} mode {mode} a={alpha} b={beta}")
    return got


SWEEP = [  # Test_Sparse_spmv.hpp:1060-1068
    (1000, 3, 200, 10, True), (1000, 3, 100, 10, True), (1000, 20, 100, 5, True),
    (50000, 3, 20, 10, False), (50000, 3, 100, 10, False), (10000, 2, 100, 5, False),
]


@pytest.mark.parametrize("rows,per,bw,var,heavy", SWEEP)
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_spmv_sweep(cuda, oracle, rows, per, bw, var, heavy, dtype):
    from kokkos_kernels_b200 import sparse as sp

    rp, ci, v = kk_matrix(rows, rows, rows * per, var, bw, dtype=dtype)
    A = dev_matrix(sp, cuda, rp, ci, v, rows)
    rng = np.random.default_rng(13718)
    x = rng.random(rows).astype(dtype)
    y = rng.random(rows).astype(dtype)
    y_nan = y.copy()
    y_nan[::19] = np.nan
    yt_nan = y.copy()
    yt_nan[::23] = np.nan
    eps = np.finfo(dtype).eps
    coefs = [0.0, 1.0, -1.0, 2.5] if heavy else [0.0, 1.0]
    modes = ["N", "C", "T", "H"] if heavy else ["N", "T"]
    for algo in (sp.SPMV_DEFAULT, sp.SPMV_NATIVE, sp.SPMV_MERGE_PATH, sp.SPMV_NATIVE_MERGE_PATH):
        h = sp.SPMVHandle(algo)  # one handle reused for every call on this matrix (:425-427)
        for mode in modes:
            for alpha in coefs:
                for beta in coefs:
                    ref_tol = spmv_tolerance(eps, alpha, beta, per + var)
                    run_case(sp, oracle, cuda, h, A, (rp, ci, v, rows), mode, alpha, beta, x, y, ref_tol)
                    if beta == 0.0:
                        run_case(sp, oracle, cuda, h, A, (rp, ci, v, rows), mode, alpha, beta, x,
                                 yt_nan if mode in "TH" else y_nan, ref_tol)


@pytest.mark.parametrize("cfg", [0, 1, 2, 3, 4])
@pytest.mark.parametrize("lpr", [2, 4, 8, 16, 32])
def test_tile_kernel_all_configs(cuda, oracle, cfg, lpr):
    """Force the TMA-tiled kernel (every ring configuration x lanes-per-row) on matrices with ragged
    rows, empty rows, nnz % 4 != 0 tails and rows longer than the tile's row limit."""
    from kokkos_kernels_b200 import sparse as sp

    rng = np.random.default_rng(cfg * 10 + lpr)
    n = 6000 + cfg * 7 + lpr
    lens = rng.integers(0, 40, size=n)
    lens[rng.integers(0, n, size=n // 5)] = 0            # empty rows
    lens[100:400] = 0                                    # a long run of empty rows
    lens[rng.integers(0, n, size=6)] = rng.integers(1500, 9000, size=6)  # long rows (> LMAX)
    lens[n - 1] = 3
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    nnz = int(rp[-1])
    ci = rng.integers(0, n, size=nnz).astype(np.int32)   # duplicates allowed for spmv
    v = (rng.random(nnz) - 0.5)
    x = rng.random(n) - 0.5
    y0 = rng.random(n)
    A = dev_matrix(sp, cuda, rp, ci, v, n)
    h = sp.SPMVHandle(sp.SPMV_DEFAULT)
    h.tune(cfg, lpr, -1)
    for alpha, beta in ((1.0, 0.0), (2.5, -1.0), (-1.0, 1.0)):
        yin = y0.copy()
        if beta == 0.0:
            yin[::19] = np.nan
        got = run_case(sp, oracle, cuda, h, A, (rp, ci, v, n), "N", alpha, beta, x, yin,
                       spmv_tolerance(np.finfo(np.float64).eps, alpha, beta, 9000))
        assert h.last_kernel().startswith("tile"), h.last_kernel()
        # second call reuses the cached plan and must give identical bits (deterministic kernel)
        yd = torch.from_numpy(yin).to(cuda)
        sp.spmv(h, "N", alpha, A, torch.from_numpy(x).to(cuda), beta, yd)
        assert np.array_equal(yd.cpu().numpy(), got, equal_nan=True)


def test_tile_kernel_stencil_bitwise_vs_vector(cuda, oracle):
    """27-pt 2-dof Laplacian (the bench family): tiled kernel == row-vector kernel bit for bit when
    both use the same lanes-per-row (same per-row summation order)."""
    from kokkos_kernels_b200 import matgen, sparse as sp

    rp, ci, v = matgen.lap27(40, 37, 29, ndof=2, noise=0.5)
    n = len(rp) - 1
    x = matgen.fill(n, -1, 1, 1)
    A = dev_matrix(sp, cuda, rp, ci, v, n)
    xd = torch.from_numpy(x).to(cuda)
    outs = []
    for algo in (sp.SPMV_DEFAULT, sp.SPMV_FAST_SETUP):
        h = sp.SPMVHandle(algo)
        h.tune(-1, 8, -1)
        yd = torch.empty(n, dtype=torch.float64, device=cuda)
        sp.spmv(h, "N", 1.0, A, xd, 0.0, yd)
        outs.append((h.last_kernel(), yd.cpu().numpy()))
    assert outs[0][0].startswith("tile") and outs[1][0].startswith("vector")
    assert np.array_equal(outs[0][1], outs[1][1])
    exp = oracle.spmv_serial(rp, ci, v, x, np.zeros(n), 1.0, 0.0)
    scale = rowwise_scale(rp, ci, v, x, None, 1.0, 0.0)
    assert np.max(np.abs(outs[0][1] - exp) / scale) <= TOL64


def test_issue101_exact(cuda):
    """Known-answer test: y == 1 + eps_f/2 exactly in double (Test_Sparse_spmv.hpp:822-961)."""
    from kokkos_kernels_b200 import sparse as sp

    eps_f = float(np.finfo(np.float32).eps)
    A = sp.CrsMatrix(torch.tensor([0, 2], dtype=torch.int32, device=cuda), torch.tensor([0, 1], dtype=torch.int32, device=cuda),
                     torch.tensor([1.0, eps_f / 2], dtype=torch.float64, device=cuda), 2)
    x = torch.ones(2, dtype=torch.float64, device=cuda)
    y = torch.zeros(1, dtype=torch.float64, device=cuda)
    sp.spmv(None, "N", 1.0, A, x, 0.0, y)
    assert y.item() == 1.0 + eps_f / 2 and y.item() != 1.0
    for nv in range(1, 23):
        for rowmajor in (False, True):
            X = torch.ones((2, nv), dtype=torch.float64, device=cuda)
            Y = torch.zeros((1, nv), dtype=torch.float64, device=cuda)
            if not rowmajor:
                X = X.t().contiguous().t()
                Y = Y.t().contiguous().t()
            sp.spmv(None, "N", 1.0, A, X, 0.0, Y)
            assert torch.all(Y == 1.0 + eps_f / 2)


def test_interfaces_and_errors(cuda, oracle):
    """All overload shapes on a 111 x 99 matrix (Test_Sparse_spmv.hpp:963-1055) on a side stream;
    dimension / mode errors raise like the reference throws (KokkosSparse_spmv.hpp:126-142)."""
    from kokkos_kernels_b200 import sparse as sp
    from kokkos_kernels_b200 import B200SparseError

    rp, ci, v = kk_matrix(111, 99, 111 * 8, 4, 60)
    A = dev_matrix(sp, cuda, rp, ci, v, 99)
    rng = np.random.default_rng(1)
    x, y0 = rng.random(99), rng.random(111)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        for h in (None, sp.SPMVHandle(), sp.SPMVHandle(sp.SPMV_FAST_SETUP)):
            yd = torch.from_numpy(y0).to(cuda)
            sp.spmv(h, "N", 2.0, A, torch.from_numpy(x).to(cuda), 0.5, yd)
            side.synchronize()
            exp = oracle.spmv_serial(rp, ci, v, x, y0.copy(), 2.0, 0.5)
            assert np.allclose(yd.cpu().numpy(), exp, rtol=1e-13, atol=1e-13)
    bad = torch.zeros(98, dtype=torch.float64, device=cuda)
    yd = torch.zeros(111, dtype=torch.float64, device=cuda)
    with pytest.raises(B200SparseError, match="Dimensions do not match"):
        sp.spmv(None, "N", 1.0, A, bad, 0.0, yd)
    with pytest.raises(B200SparseError, match="Dimensions do not match"):
        sp.spmv(None, "T", 1.0, A, torch.zeros(99, dtype=torch.float64, device=cuda), 0.0, yd)
    with pytest.raises(B200SparseError, match="Invalid transpose mode"):
        sp.spmv(None, "X", 1.0, A, torch.zeros(99, dtype=torch.float64, device=cuda), 0.0, yd)


def test_empty_and_alpha_zero(cuda):
    """alpha == 0 or an empty matrix: y = beta*y, exact zeros for beta == 0 even over NaN
    (KokkosSparse_spmv.hpp:145-154)."""
    from kokkos_kernels_b200 import sparse as sp

    n = 500
    A0 = sp.CrsMatrix(torch.zeros(n + 1, dtype=torch.int32, device=cuda), torch.zeros(0, dtype=torch.int32, device=cuda),
                      torch.zeros(0, dtype=torch.float64, device=cuda), n)
    x = torch.ones(n, dtype=torch.float64, device=cuda)
    for h in (None, sp.SPMVHandle()):
        y = torch.full((n,), float("nan"), dtype=torch.float64, device=cuda)
        sp.spmv(h, "N", 1.0, A0, x, 0.0, y)
        assert torch.all(y == 0)
        y = torch.full((n,), 3.0, dtype=torch.float64, device=cuda)
        sp.spmv(h, "T", 1.0, A0, x, -2.0, y)
        assert torch.all(y == -6.0)
    Ae = sp.CrsMatrix(torch.zeros(1, dtype=torch.int32, device=cuda), torch.zeros(0, dtype=torch.int32, device=cuda),
                      torch.zeros(0, dtype=torch.float64, device=cuda), 0)
    sp.spmv(None, "N", 1.0, Ae, torch.zeros(0, dtype=torch.float64, device=cuda), 0.0, torch.zeros(0, dtype=torch.float64, device=cuda))


def test_hostvec_entry(cuda, oracle):
    from kokkos_kernels_b200 import matgen, sparse as sp

    rp, ci, v = matgen.lap27(30, 30, 30, ndof=2, noise=0.5)
    n = len(rp) - 1
    A = dev_matrix(sp, cuda, rp, ci, v, n)
    xh = torch.from_numpy(matgen.fill(n, -1, 1, 3)).pin_memory()
    yh = torch.full((n,), float("nan"), dtype=torch.float64).pin_memory()
    h = sp.SPMVHandle()
    sp.spmv_hostvec(h, "N", 1.0, A, xh, 0.0, yh)
    torch.cuda.synchronize()
    exp = oracle.spmv_serial(rp, ci, v, xh.numpy(), np.zeros(n), 1.0, 0.0)
    scale = rowwise_scale(rp, ci, v, xh.numpy(), None, 1.0, 0.0)
    assert np.max(np.abs(yh.numpy() - exp) / scale) <= TOL64


def test_hostvec_pipeline(cuda, oracle):
    """Large product -> pipelined host-vector path (double-buffered upload, piecewise download): three
    back-to-back calls with different x / beta on one handle, each checked against the Serial oracle."""
    from kokkos_kernels_b200 import matgen, sparse as sp

    rp, ci, v = matgen.lap27(56, 56, 56, ndof=2, noise=0.5)
    n = len(rp) - 1
    assert len(ci) >= (1 << 22)
    A = dev_matrix(sp, cuda, rp, ci, v, n)
    h = sp.SPMVHandle()
    xs = [torch.from_numpy(matgen.fill(n, -1, 1, s)).pin_memory() for s in (3, 4, 5)]
    y0 = matgen.fill(n, -1, 1, 9)
    ys = [torch.from_numpy(y0.copy()).pin_memory() for _ in range(3)]
    betas = [0.0, 0.5, 0.0]
    ys[0][::19] = float("nan")
    ys[2][::19] = float("nan")
    for k in range(3):  # enqueue all three before synchronising: exercises both device buffers
        sp.spmv_hostvec(h, "N", 2.0, A, xs[k], betas[k], ys[k])
    torch.cuda.synchronize()
    for k in range(3):
        exp = oracle.spmv_serial(rp, ci, v, xs[k].numpy(), y0.copy(), 2.0, betas[k])
        scale = rowwise_scale(rp, ci, v, xs[k].numpy(), y0, 2.0, betas[k])
        got = ys[k].numpy()
        assert not np.isnan(got).any()
        assert np.max(np.abs(got - exp) / scale) <= TOL64, k


@pytest.mark.parametrize("bandwidth", [100000, 1000])
def test_baseline_config1_shape(cuda, oracle, bandwidth):
    """BASELINE.json configs[0]: fp64 CrsMatrix 100k x 100k, ~20 nnz/row random (kk_generate with
    nnz = 2e6, row-size variance 10, bandwidth n or 0.01 n -- SURVEY.md 8d), single vector: the GPU result
    against the oracle's Serial path (the reference's own CPU-runnable case) within 1e-10 row-scaled,
    for the analysed (tile / self-tuned) and the no-analysis kernels."""
    from kokkos_kernels_b200 import sparse as sp

    n = 100000
    rp, ci, v = kk_matrix(n, n, 2_000_000, 10, bandwidth, lo=-1.0, hi=1.0)
    rng = np.random.default_rng(13718)
    x = rng.uniform(-1, 1, n)
    y0 = rng.uniform(-1, 1, n)
    A = dev_matrix(sp, cuda, rp, ci, v, n)
    for algo in (sp.SPMV_DEFAULT, sp.SPMV_FAST_SETUP):
        h = sp.SPMVHandle(algo)
        for alpha, beta in ((1.0, 0.0), (2.5, -0.5)):
            for _ in range(4):  # passes through the plan's self-tuning phases (tile, tile timed, vector timed, choice)
                run_case(sp, oracle, cuda, h, A, (rp, ci, v, n), "N", alpha, beta, x, y0,
                         spmv_tolerance(np.finfo(np.float64).eps, alpha, beta, 30))
