"""GPU parity of rank-2 (multivector) SpMV (Test_Sparse_spmv.hpp:465-606,1075-1092)."""
import numpy as np
import pytest
import torch

import exact_ref as R
from helpers import kk_matrix, spmv_tolerance

pytestmark = pytest.mark.gpu


def _mk(dev, a, rowmajor):
    t = torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    if not rowmajor:
        t = t.t().contiguous().t()  # LayoutLeft: stride (1, rows)
    return t


@pytest.mark.parametrize("rows,per,bw,var", [(1000, 3, 200, 10), (1000, 20, 100, 5), (10000, 2, 100, 5), (5000, 30, 400, 20)])
@pytest.mark.parametrize("nv", [1, 5, 10, 16, 30])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_spmm_sweep(cuda, oracle, rows, per, bw, var, nv, dtype):
    from kokkos_kernels_b200 import sparse as sp

    ncols = rows - 37
    rp, ci, v = kk_matrix(rows, ncols, rows * per, var, bw, dtype=dtype)
    A = sp.CrsMatrix(torch.from_numpy(rp).to(cuda), torch.from_numpy(ci).to(cuda), torch.from_numpy(v).to(cuda), ncols)
    rng = np.random.default_rng(13718)
    X = rng.random((ncols, nv)).astype(dtype)
    Y0 = rng.random((rows, nv)).astype(dtype)
    Xt = rng.random((rows, nv)).astype(dtype)
    Yt0 = rng.random((ncols, nv)).astype(dtype)
    eps = np.finfo(dtype).eps
    h = sp.SPMVHandle()
    for xrm, yrm in ((True, True), (False, False), (True, False), (False, True)):
        for alpha, beta in ((1.0, 0.0), (2.5, -1.0), (-1.0, 1.0), (0.0, 2.5), (1.0, 2.5)):
            tol = 16 * spmv_tolerance(eps, alpha, beta, per + var) + 1e-300
            Y0n = Y0.copy()
            if beta == 0.0:
                Y0n[::19, :] = np.nan
            Yd = _mk(cuda, Y0n, yrm)
            sp.spmv(h if (xrm, yrm) != (True, False) else None, "N", alpha, A, _mk(cuda, X, xrm), beta, Yd)
            exp = oracle.spmv_mv(rp, ci, v, ncols, X, np.where(np.isnan(Y0n), 0, Y0n) if beta == 0 else Y0n.copy(), alpha, beta)
            got = Yd.cpu().numpy()
            assert not np.isnan(got).any()
            assert np.max(np.abs(got - exp)) <= tol, (xrm, yrm, alpha, beta, np.max(np.abs(got - exp)), tol)
            what = f"{h.last_kernel() if (xrm, yrm) != (True, False) else 'no plan'} {(xrm, yrm)} a={alpha} b={beta}"
            R.assert_within(got, R.spmm_exact(rp, ci, v, X, Y0, alpha, beta), R.spmm_bound(rp, ci, v, X, Y0, alpha, beta), what)
            # transpose
            Ytd = _mk(cuda, Yt0, yrm)
            sp.spmv(h, "T", alpha, A, _mk(cuda, Xt, xrm), beta, Ytd)
            expt = oracle.spmv_mv_transpose(rp, ci, v, ncols, Xt, Yt0.copy(), alpha, beta)
            gott = Ytd.cpu().numpy()
            assert np.max(np.abs(gott - expt)) <= 4 * tol + 1e-300
            R.assert_within(gott, R.spmm_exact(rp, ci, v, Xt, Yt0, alpha, beta, trans=True),
                            R.spmm_bound(rp, ci, v, Xt, Yt0, alpha, beta, trans=True), f"{h.last_kernel()} T {(xrm, yrm)} a={alpha} b={beta}")


@pytest.mark.parametrize("dtype,k", [(np.float32, 16), (np.float64, 5), (np.float32, 40)])
def test_spmm_hub_rows(cuda, oracle, dtype, k):
    """Rows of thousands of entries (more than 64 pieces of 64: the CTA-per-row reduce of the item kernel) next to short
    and empty rows; beta != 0; twice through one handle (run-to-run identical)."""
    from kokkos_kernels_b200 import sparse as sp

    rng = np.random.default_rng(77)
    m, n = 3000, 9000
    lens = rng.integers(0, 12, m)
    lens[[7, 1500, 2999]] = [9000, 4097, 6500]
    lens[100:110] = rng.integers(65, 700, 10)  # a few rows of several pieces (the warp-per-row reduce)
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    ci = np.concatenate([rng.choice(n, int(l), replace=False) for l in lens]).astype(np.int32)
    v = rng.uniform(-1, 1, len(ci)).astype(dtype)
    X = rng.uniform(-1, 1, (n, k)).astype(dtype)
    Y0 = rng.uniform(-1, 1, (m, k)).astype(dtype)
    A = sp.CrsMatrix(torch.from_numpy(rp).to(cuda), torch.from_numpy(ci).to(cuda), torch.from_numpy(v).to(cuda), n)
    exp = oracle.spmv_mv(rp, ci, v, n, X, Y0.copy(), 1.5, -0.5)
    tol = 10 * np.finfo(dtype).eps * 9000 * 1.5
    exact, bound = R.spmm_exact(rp, ci, v, X, Y0, 1.5, -0.5), R.spmm_bound(rp, ci, v, X, Y0, 1.5, -0.5)
    h = sp.SPMVHandle()
    outs = []
    for _ in range(2):
        Y = _mk(cuda, Y0.copy(), True)
        sp.spmv(h, "N", 1.5, A, _mk(cuda, X, True), -0.5, Y)
        outs.append(Y.cpu().numpy())
        assert np.max(np.abs(outs[-1] - exp)) <= tol
        R.assert_within(outs[-1], exact, bound, h.last_kernel())
    assert np.array_equal(outs[0], outs[1])
    assert h.last_kernel().startswith("spmm_items"), h.last_kernel()


def test_spmm_powerlaw_rows(cuda, oracle):
    """R-MAT structure (skewed rows), fp32, 16 columns: the config-3 shape at a small scale."""
    from kokkos_kernels_b200 import matgen, sparse as sp

    rp, ci = matgen.rmat(14, 16)
    n = len(rp) - 1
    v = matgen.fill(len(ci), 0, 1, 23, dtype=np.float32)
    X = matgen.fill(n * 16, -1, 1, 5, dtype=np.float32).reshape(n, 16)
    A = sp.CrsMatrix(torch.from_numpy(rp).to(cuda), torch.from_numpy(ci).to(cuda), torch.from_numpy(v).to(cuda), n)
    exp = oracle.spmv_mv(rp, ci, v, n, X, np.zeros((n, 16), dtype=np.float32), 1.0, 0.0)
    maxrow = int(np.diff(rp).max())
    Y0 = np.zeros((n, 16), dtype=np.float32)
    exact, bound = R.spmm_exact(rp, ci, v, X, Y0, 1.0, 0.0), R.spmm_bound(rp, ci, v, X, Y0, 1.0, 0.0)
    for rowmajor in (True, False):
        Y = _mk(cuda, np.full((n, 16), np.nan, dtype=np.float32), rowmajor)
        h = sp.SPMVHandle()
        sp.spmv(h, "N", 1.0, A, _mk(cuda, X, rowmajor), 0.0, Y)
        got = Y.cpu().numpy()
        err = np.max(np.abs(got - exp))
        assert err <= 10 * np.finfo(np.float32).eps * maxrow
        R.assert_within(got, exact, bound, f"{h.last_kernel()} rowmajor={rowmajor}")


def test_config3_full_size(cuda, oracle):
    """BASELINE.json configs[2] at full size: R-MAT scale 23 (8,388,608 rows, 1.3e8 entries, longest row 152,801), fp32,
    16-column multivector, both layouts -- EVERY row against the oracle's CPU multivector loop (O4, spmv_impl.hpp:745-926;
    OpenMP over rows changes no bit of a row).  Criterion (SURVEY.md section 8d): component-wise error scaled by
    |alpha| sum_j |a_ij||x_jc| + |beta||y0_ic| at most 1e-4 (fp32); alpha = 1.5, beta = 0.5 and the beta == 0 / NaN case.
    In addition, 200,000 rows chosen by a fixed seed plus every row of more than 4,096 entries are held to the exact
    product's per-entry bound (tests/exact_ref.py)."""
    import os

    from kokkos_kernels_b200 import matgen, sparse as sp

    rp, ci = matgen.rmat(23, 16)
    n, k = len(rp) - 1, 16
    assert n == 1 << 23
    v = matgen.fill(len(ci), 0.0, 1.0, 23, dtype=np.float32)
    X = matgen.fill(n * k, -1.0, 1.0, 5, dtype=np.float32).reshape(n, k)
    Y0 = matgen.fill(n * k, -1.0, 1.0, 6, dtype=np.float32).reshape(n, k)
    threads = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    A = sp.CrsMatrix(torch.from_numpy(rp).to(cuda), torch.from_numpy(ci).to(cuda), torch.from_numpy(v).to(cuda), n)
    h = sp.SPMVHandle()
    scale_a = oracle.spmv_mv(rp, ci, np.abs(v), n, np.abs(X), np.zeros((n, k), dtype=np.float32), 1.0, 0.0, threads=threads)
    lens = np.diff(rp)
    sample = np.union1d(np.random.default_rng(8).choice(n, 200000, replace=False), np.flatnonzero(lens > 4096))
    rp_s = np.concatenate([[0], np.cumsum(lens[sample])]).astype(np.int32)
    take = np.concatenate([np.arange(rp[r], rp[r + 1]) for r in sample])
    ci_s, v_s = ci[take], v[take]
    for alpha, beta, rowmajor in ((1.0, 0.0, True), (1.5, 0.5, True), (1.5, 0.5, False)):
        y_in = Y0.copy()
        if beta == 0.0:
            y_in[::23] = np.nan  # beta == 0 must overwrite, not scale (Test_Sparse_spmv.hpp:394-408)
        Yd = _mk(cuda, y_in, rowmajor)
        sp.spmv(h, "N", alpha, A, _mk(cuda, X, rowmajor), beta, Yd)
        got = Yd.cpu().numpy()
        exp = oracle.spmv_mv(rp, ci, v, n, X, np.zeros((n, k), dtype=np.float32) if beta == 0.0 else Y0.copy(), alpha, beta, threads=threads)
        assert not np.isnan(got).any()
        scale = abs(alpha) * scale_a.astype(np.float64) + abs(beta) * np.abs(Y0).astype(np.float64)
        err = np.abs(got.astype(np.float64) - exp.astype(np.float64)) / np.maximum(scale, 1e-30)
        assert float(err.max()) <= 1e-4, (alpha, beta, rowmajor, float(err.max()), int(err.argmax()) // k)
        R.assert_within(got[sample], R.spmm_exact(rp_s, ci_s, v_s, X, Y0[sample], alpha, beta),
                        R.spmm_bound(rp_s, ci_s, v_s, X, Y0[sample], alpha, beta), f"{h.last_kernel()} rowmajor={rowmajor} (row = index in the sample)")
