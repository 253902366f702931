"""GPU parity of the CrsMatrix utilities (sort_crs_matrix, sort_and_merge_matrix, transpose_matrix,
spadd) through the C ABI against the oracle's restatement of the reference's host path: every
output array bit-identical (int32 structure AND floating-point values -- the kernels keep the
reference's per-row operation order), plus the reference's own acceptance laws
(Test_Sparse_SortCrs.hpp, Test_Sparse_spadd.hpp)."""
import numpy as np
import pytest
import torch

from crs_cases import MERGE_CASES, random_matrix, spadd_dense_check
from helpers import kk_matrix

pytestmark = pytest.mark.gpu


def dev_mat(sp, dev, rp, ci, v, ncols):
    return sp.CrsMatrix(torch.from_numpy(rp.copy()).to(dev), torch.from_numpy(ci.copy()).to(dev),
                        torch.from_numpy(v.copy()).to(dev), ncols)


def host(t):
    return t.cpu().numpy()


def long_row_matrix(rng, m, n, long_lens, dtype=np.float64):
    """Short random rows plus a few rows in the CTA (257..4096) and global (>4096) sort classes, with
    duplicate columns so that stability matters."""
    lens = rng.integers(0, 40, m)
    lens[: len(long_lens)] = long_lens
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    ci = rng.integers(0, n, rp[-1]).astype(np.int32)
    v = rng.uniform(-1, 1, rp[-1]).astype(dtype)
    return rp, ci, v


@pytest.mark.parametrize("m,n,nnz", [(10, 10, 20), (100, 100, 2000), (1000, 1000, 30000), (50, 200, 3000), (20000, 20000, 600000)])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_sort_crs_matrix_sweep(cuda, oracle, m, n, nnz, dtype):
    """testSortCRS (Test_Sparse_SortCrs.hpp:44-139): kk_generate_sparse_matrix rows are unsorted."""
    from kokkos_kernels_b200 import sparse as sp

    rp, ci, v = kk_matrix(m, n, nnz, 2, n // 2, dtype=dtype)
    A = dev_mat(sp, cuda, rp, ci, v, n)
    sp.sort_crs_matrix(A)
    G = torch.from_numpy(ci.copy()).to(cuda)
    sp.sort_crs_graph(A.row_map, G)
    oracle.sort_crs_stable(rp, ci, v)
    assert np.array_equal(host(A.entries), ci) and np.array_equal(host(A.values), v)
    assert np.array_equal(host(G), ci)
    # idempotent, and already-sorted input is left untouched
    sp.sort_crs_matrix(A)
    assert np.array_equal(host(A.entries), ci) and np.array_equal(host(A.values), v)


def test_sort_long_rows_and_stability(cuda, oracle):
    from kokkos_kernels_b200 import sparse as sp

    rng = np.random.default_rng(11)
    rp, ci, v = long_row_matrix(rng, 3000, 500, [9000, 5000, 4097, 4096, 300, 257, 256, 255, 33, 32, 31, 2, 1, 0])
    A = dev_mat(sp, cuda, rp, ci, v, 500)
    sp.sort_crs_matrix(A)
    oracle.sort_crs_stable(rp, ci, v)
    assert np.array_equal(host(A.entries), ci)
    assert np.array_equal(host(A.values), v), "ties must keep their original order (stable sort)"


@pytest.mark.parametrize("case", sorted(MERGE_CASES))
def test_sort_and_merge_golden(cuda, case):
    from kokkos_kernels_b200 import sparse as sp

    c = MERGE_CASES[case]
    A = dev_mat(sp, cuda, c["rowmap"], c["entries"], c["values"], c["ncols"])
    M = sp.sort_and_merge_matrix(A)
    assert np.array_equal(host(M.row_map), c["gold_rowmap"])
    assert np.array_equal(host(M.entries), c["gold_entries"])
    assert np.array_equal(host(M.values), c["gold_values"])
    rm, en = sp.sort_and_merge_graph(torch.from_numpy(c["rowmap"].copy()).to(cuda), torch.from_numpy(c["entries"].copy()).to(cuda))
    assert np.array_equal(host(rm), c["gold_rowmap"]) and np.array_equal(host(en), c["gold_entries"])


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_sort_and_merge_random(cuda, oracle, dtype):
    from kokkos_kernels_b200 import sparse as sp

    rng = np.random.default_rng(3)
    rp, ci, v = long_row_matrix(rng, 5000, 60, [5000, 700, 100], dtype=dtype)   # 60 columns: many duplicates
    A = dev_mat(sp, cuda, rp, ci, v, 60)
    M = sp.sort_and_merge_matrix(A)
    rpo, cio, vo = oracle.sort_and_merge(rp, ci, v)
    assert np.array_equal(host(M.row_map), rpo) and np.array_equal(host(M.entries), cio)
    assert np.array_equal(host(M.values), vo), "duplicates are summed in the sorted row's order: bit-identical"
    assert np.array_equal(host(A.entries), ci), "the input is sorted in place on the way"


@pytest.mark.parametrize("m,n,nnz", [(100, 300, 2000), (3000, 1000, 90000), (1, 5, 3), (7, 1, 4)])
def test_transpose_matrix(cuda, oracle, m, n, nnz):
    from kokkos_kernels_b200 import sparse as sp

    rng = np.random.default_rng(m)
    lens = rng.multinomial(nnz, np.ones(m) / m)
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    ci = rng.integers(0, n, nnz).astype(np.int32)          # duplicates within a row are allowed
    v = rng.uniform(-1, 1, nnz)
    T = sp.transpose_matrix(dev_mat(sp, cuda, rp, ci, v, n))
    trp, tci, tv = oracle.transpose(rp, ci, v, n)
    assert T.numRows() == n and T.numCols() == m
    assert np.array_equal(host(T.row_map), trp) and np.array_equal(host(T.entries), tci) and np.array_equal(host(T.values), tv)


def test_transpose_empty(cuda):
    from kokkos_kernels_b200 import sparse as sp

    A = sp.CrsMatrix(torch.zeros(6, dtype=torch.int32, device=cuda), torch.zeros(0, dtype=torch.int32, device=cuda),
                     torch.zeros(0, dtype=torch.float64, device=cuda), 9)
    T = sp.transpose_matrix(A)
    assert T.row_map.numel() == 10 and not host(T.row_map).any() and T.nnz() == 0


@pytest.mark.parametrize("sort_rows", [True, False])
@pytest.mark.parametrize("m,n,lo,hi", [(10, 10, 0, 0), (10, 10, 0, 2), (100, 100, 50, 100), (50, 50, 75, 100), (20000, 3000, 0, 60)])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_spadd(cuda, oracle, sort_rows, m, n, lo, hi, dtype):
    """test_spadd (Test_Sparse_spadd.hpp:96-187), incl. duplicated entries when maxNNZ > ncols; C's row
    map is pre-filled with 5 and C's entries / values with 5 like the reference test does."""
    from kokkos_kernels_b200 import sparse as sp

    A = random_matrix(m, n, lo, hi, sort_rows, seed=(m << 1) ^ n, dtype=dtype)
    B = random_matrix(m, n, lo, hi, sort_rows, seed=((m << 1) ^ n) + 1, dtype=dtype)
    Ad, Bd = dev_mat(sp, cuda, *A, n), dev_mat(sp, cuda, *B, n)
    kh = sp.KokkosKernelsHandle()
    kh.create_spadd_handle(sort_rows, hi <= n)
    ah = kh.get_spadd_handle()
    c_rowmap = torch.full((m + 1,), 5, dtype=torch.int32, device=cuda)
    sp.spadd_symbolic_views(kh, m, n, Ad.row_map, Ad.entries, Bd.row_map, Bd.entries, c_rowmap)
    assert ah.is_symbolic_called() and not ah.is_numeric_called()
    c_entries = torch.full((ah.get_c_nnz(),), 5, dtype=torch.int32, device=cuda)
    c_values = torch.full((ah.get_c_nnz(),), 5, dtype=Ad.values.dtype, device=cuda)
    one = dtype(1)
    sp.spadd_numeric_views(kh, m, n, Ad.row_map, Ad.entries, Ad.values, one, Bd.row_map, Bd.entries, Bd.values, one, c_rowmap,
                           c_entries, c_values)
    assert ah.is_numeric_called()
    got = (host(c_rowmap), host(c_entries), host(c_values))
    spadd_dense_check(A, B, got, n, 1.0, 1.0)
    exp = oracle.spadd(*A, one, *B, one, sort_rows)
    for g, e in zip(got, exp):
        assert np.array_equal(g, e)
    # numeric again with other coefficients on the same symbolic
    a2, b2 = dtype(0.3), dtype(-1.7)  # not powers of two: the products round (no FMA contraction in the kernels)
    sp.spadd_numeric_views(kh, m, n, Ad.row_map, Ad.entries, Ad.values, a2, Bd.row_map, Bd.entries, Bd.values, b2, c_rowmap,
                           c_entries, c_values)
    exp2 = oracle.spadd(*A, a2, *B, b2, sort_rows)
    assert np.array_equal(host(c_values), exp2[2])
    kh.destroy_spadd_handle()


@pytest.mark.parametrize("group", ["0", "8", "32"])
def test_spadd_sorted_kernel_variants(cuda, oracle, monkeypatch, group):
    """the sorted spadd kernels -- one thread per row (0) and a group of 8 / 32 lanes per row placing every entry by its rank in the
    union (crs_utils.cu) -- give the oracle's bits: rows with common and disjoint columns, an empty A_i or B_i, a long row, signed
    zeros (0 + (-0) = +0 as in `acc = 0; acc += ...`), and rows with a repeated column (the serial fallback inside the group kernels)"""
    from kokkos_kernels_b200 import sparse as sp

    monkeypatch.setenv("B200SP_SPADD_GROUP", group)
    rng = np.random.default_rng(3)
    m, n = 400, 5000
    def mat(seed, repeats):
        r = np.random.default_rng(seed)
        rp, ci, v = [0], [], []
        for i in range(m):
            ln = 0 if i % 17 == seed % 17 else (3000 if i == 7 else int(r.integers(1, 70)))
            cols = np.sort(r.choice(n, ln, replace=False))
            if repeats and i % 29 == 3 and ln >= 2:
                cols[1] = cols[0]  # a repeated column inside a sorted row
            vals = r.uniform(-1, 1, ln)
            vals[r.random(ln) < 0.1] = -0.0
            ci += list(cols)
            v += list(vals)
            rp.append(len(ci))
        return np.array(rp, np.int32), np.array(ci, np.int32), np.array(v)
    A, B = mat(1, True), mat(2, False)
    B[1][B[0][5]:B[0][5] + 3] = A[1][A[0][5]:A[0][5] + 3] if A[0][6] - A[0][5] >= 3 and B[0][6] - B[0][5] >= 3 else B[1][B[0][5]:B[0][5] + 3]
    # re-sort row 5 of B after planting common columns (and drop accidental repeats by leaving them: repeats are legal)
    s5, e5 = B[0][5], B[0][6]
    order = np.argsort(B[1][s5:e5], kind="stable")
    B[1][s5:e5], B[2][s5:e5] = B[1][s5:e5][order], B[2][s5:e5][order]
    Ad, Bd = dev_mat(sp, cuda, *A, n), dev_mat(sp, cuda, *B, n)
    for alpha, beta in ((1.0, 1.0), (0.3, -1.7), (-1.0, 0.0)):
        kh = sp.KokkosKernelsHandle()
        kh.create_spadd_handle(True, False)
        c_rowmap = torch.zeros(m + 1, dtype=torch.int32, device=cuda)
        sp.spadd_symbolic_views(kh, m, n, Ad.row_map, Ad.entries, Bd.row_map, Bd.entries, c_rowmap)
        nnz = kh.get_spadd_handle().get_c_nnz()
        c_entries = torch.full((nnz,), -1, dtype=torch.int32, device=cuda)
        c_values = torch.full((nnz,), np.nan, dtype=torch.float64, device=cuda)
        sp.spadd_numeric_views(kh, m, n, Ad.row_map, Ad.entries, Ad.values, alpha, Bd.row_map, Bd.entries, Bd.values, beta, c_rowmap,
                               c_entries, c_values)
        exp = oracle.spadd(*A, alpha, *B, beta, True)
        got = (host(c_rowmap), host(c_entries), host(c_values))
        assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1])
        assert np.array_equal(got[2].view(np.int64), exp[2].view(np.int64))  # bits: the sign of a zero counts
        kh.destroy_spadd_handle()


def test_spadd_unsorted_rows_bits(cuda, oracle):
    """the unsorted path (8 lanes per row: places by a ballot prefix, the three passes of the serial loop side by side on rows without a
    repeated column, lane 0 alone on the others): shuffled rows with a long row, empty rows, repeated columns and signed zeros"""
    from kokkos_kernels_b200 import sparse as sp

    m, n = 300, 4000
    def mat(seed, repeats):
        r = np.random.default_rng(seed)
        rp, ci, v = [0], [], []
        for i in range(m):
            ln = 0 if i % 13 == seed % 13 else (2500 if i == 11 else int(r.integers(1, 90)))
            cols = r.choice(n, ln, replace=False)
            if repeats and i % 7 == 2 and ln >= 3:
                cols[2] = cols[0]  # a repeated column somewhere in the unsorted row
            vals = r.uniform(-1, 1, ln)
            vals[r.random(ln) < 0.1] = -0.0
            ci += list(cols)
            v += list(vals)
            rp.append(len(ci))
        return np.array(rp, np.int32), np.array(ci, np.int32), np.array(v)
    A, B = mat(5, True), mat(6, True)
    Ad, Bd = dev_mat(sp, cuda, *A, n), dev_mat(sp, cuda, *B, n)
    for alpha, beta in ((1.0, 1.0), (0.3, -1.7)):
        kh = sp.KokkosKernelsHandle()
        kh.create_spadd_handle(False, False)
        c_rowmap = torch.zeros(m + 1, dtype=torch.int32, device=cuda)
        sp.spadd_symbolic_views(kh, m, n, Ad.row_map, Ad.entries, Bd.row_map, Bd.entries, c_rowmap)
        nnz = kh.get_spadd_handle().get_c_nnz()
        c_entries = torch.full((nnz,), -1, dtype=torch.int32, device=cuda)
        c_values = torch.full((nnz,), np.nan, dtype=torch.float64, device=cuda)
        sp.spadd_numeric_views(kh, m, n, Ad.row_map, Ad.entries, Ad.values, alpha, Bd.row_map, Bd.entries, Bd.values, beta, c_rowmap,
                               c_entries, c_values)
        exp = oracle.spadd(*A, alpha, *B, beta, False)
        got = (host(c_rowmap), host(c_entries), host(c_values))
        assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1])
        assert np.array_equal(got[2].view(np.int64), exp[2].view(np.int64))
        kh.destroy_spadd_handle()


def test_spadd_known_columns_and_misuse(cuda):
    from kokkos_kernels_b200 import sparse as sp
    from kokkos_kernels_b200 import B200SparseError

    rp = torch.tensor([0, 1, 2, 3, 4, 4, 4], dtype=torch.int32, device=cuda)
    A = sp.CrsMatrix(rp, torch.arange(4, dtype=torch.int32, device=cuda), torch.ones(4, dtype=torch.float64, device=cuda), 7)
    kh = sp.KokkosKernelsHandle()
    kh.create_spadd_handle(True)
    with pytest.raises(B200SparseError):
        sp.spadd_numeric(kh, 1.0, A, 1.0, A, A)
    Cm = sp.spadd_symbolic(kh, A, A)
    sp.spadd_numeric(kh, 1.0, A, 1.0, A, Cm)
    assert Cm.numRows() == 6 and Cm.numCols() == 7 and Cm.nnz() == A.nnz()
    assert torch.all(Cm.values == 2.0)
    # zero rows
    E = sp.CrsMatrix(torch.zeros(1, dtype=torch.int32, device=cuda), torch.zeros(0, dtype=torch.int32, device=cuda),
                     torch.zeros(0, dtype=torch.float64, device=cuda), 3)
    kh2 = sp.KokkosKernelsHandle()
    kh2.create_spadd_handle(False)
    C0 = sp.spadd_symbolic(kh2, E, E)
    sp.spadd_numeric(kh2, 1.0, E, 1.0, E, C0)
    assert C0.nnz() == 0 and host(C0.row_map).tolist() == [0]


@pytest.mark.parametrize("dtype,tol", [(np.float64, 1e-10), (np.float32, 1e-4)])
def test_spmv_cached_transpose(cuda, oracle, dtype, tol):
    """Modes T / H through the plan's explicit transpose (SPMVHandle.cache_transpose): same result law as
    the atomics path, and bit-reproducible from call to call."""
    from helpers import rowwise_scale
    from kokkos_kernels_b200 import sparse as sp

    m, n = 30000, 12000
    rp, ci, v = kk_matrix(m, n, 600000, 20, 4000, dtype=dtype, lo=-1.0, hi=1.0)
    rng = np.random.default_rng(2)
    x = rng.uniform(-1, 1, m).astype(dtype)
    y0 = rng.uniform(-1, 1, n).astype(dtype)
    alpha, beta = 1.25, -0.5
    yref = y0.astype(dtype).copy()
    oracle.spmv_transpose(rp, ci, v, n, x, yref, dtype(alpha), dtype(beta))
    scale = rowwise_scale(rp, ci, v, x, y0, alpha, beta, ncols_out=n, trans=True)
    A = dev_mat(sp, cuda, rp, ci, v, n)
    h = sp.SPMVHandle(sp.SPMV_DEFAULT)
    h.cache_transpose(True)
    xd = torch.from_numpy(x).to(cuda)
    outs = []
    for mode in ("T", "H", "T"):
        yd = torch.from_numpy(y0.copy()).to(cuda)
        sp.spmv(h, mode, alpha, A, xd, beta, yd)
        outs.append(host(yd))
    assert h.last_kernel().startswith("cached_transpose")
    err = np.max(np.abs(outs[0].astype(np.float64) - yref.astype(np.float64)) / np.maximum(scale, 1e-300))
    assert err <= tol, err
    assert np.array_equal(outs[0], outs[1]) and np.array_equal(outs[0], outs[2]), "deterministic: no atomics"
    # the values may change in place between calls: they are re-gathered
    A.values.mul_(2.0)
    yd = torch.from_numpy(y0.copy()).to(cuda)
    sp.spmv(h, "T", alpha / 2.0, A, xd, beta, yd)
    assert np.max(np.abs(host(yd).astype(np.float64) - yref.astype(np.float64)) / np.maximum(scale, 1e-300)) <= tol
