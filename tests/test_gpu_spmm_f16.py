"""Half-precision rank-2 SpMV on the GPU through the Python mirror (sparse.spmv on torch.float16 CrsMatrix values and
multivectors): every path with its last_kernel(), the bit identity with the fp32 call on the widened inputs on the item
paths (Y16 == round_fp16(Y32)), config 3 at full size, k from 1 to 64, fp32 accumulation, special values, strided and
misaligned views, determinism, and the mirror's errors for what half precision does not cover."""
import os

import numpy as np
import pytest
import torch

import half_ref as H
import spmm_cases as cases

pytestmark = pytest.mark.gpu

F16 = np.float16
EMULATED = os.environ.get("B200SP_TEST_EMULATED") == "1"
SPMM_VARS = ["B200SP_SPMM_ITEM_LMAX"]
LAYOUTS = ["RR", "LL", "RL", "LR"]  # X layout, Y layout: R = LayoutRight (row-major), L = LayoutLeft


@pytest.fixture(autouse=True)
def _clean_env(monkeypatch):
    for k in SPMM_VARS:
        monkeypatch.delenv(k, raising=False)


_MATS = {}


def matrix16(name, seed=5):
    """A shared case of spmm_cases.py with fp16 values (the cancelling case scaled by 2^-10 into the fp16 range)."""
    key = (name, seed)
    if key not in _MATS:
        builder = cases.SMALL_CASES.get(name) or getattr(cases, name)
        rp, ci, v, ncols = builder(seed, np.float32)
        if name == "cancelling":
            v = v * np.float32(2.0**-10)
        _MATS[key] = (rp, ci, v.astype(F16), ncols)
    return _MATS[key]


def dev_matrix(cuda, A, dtype=None):
    from kokkos_kernels_b200 import sparse as sp

    rp, ci, v, ncols = A
    v = v if dtype is None else v.astype(dtype)
    return sp.CrsMatrix(torch.from_numpy(rp).to(cuda), torch.from_numpy(ci).to(cuda), torch.from_numpy(v).to(cuda), ncols)


def dev(cuda, a, rowmajor):
    t = torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    return t if rowmajor else t.t().contiguous().t()


def host(t):
    return t.cpu().numpy()


def operands(A, k, seed, trans=False):
    rp, ci, v, ncols = A
    rng = np.random.default_rng(seed)
    xr, yr = (len(rp) - 1, ncols) if trans else (ncols, len(rp) - 1)
    return cases.dense_operands(rng, xr, k, F16), cases.dense_operands(rng, yr, k, F16)


def call(cuda, A16, X, Y0, alpha, beta, lay="RR", mode="N", handle=True, dtype=torch.float16, y_nan=False):
    """One sp.spmv call; returns (Y on the host, last_kernel() or None)."""
    from kokkos_kernels_b200 import sparse as sp

    npd = F16 if dtype == torch.float16 else np.float32
    A = dev_matrix(cuda, A16, npd)
    Xd = dev(cuda, X.astype(npd), lay[0] == "R")
    Yd = dev(cuda, Y0.astype(npd), lay[1] == "R")
    if y_nan:
        Yd.fill_(float("nan"))
    h = sp.SPMVHandle() if handle else None
    sp.spmv(h, mode, alpha, A, Xd, beta, Yd)
    torch.cuda.synchronize()
    return host(Yd), (h.last_kernel() if h else None)


def check_bound(A, X, Y0, got, alpha, beta, mode, what):
    rp, ci, v, _ = A
    t = mode in "TtHh"
    H.assert_within16(got, H.spmm_exact16(rp, ci, v, X, Y0, alpha, beta, t), H.spmm_bound16(rp, ci, v, X, Y0, alpha, beta, t), what)


def same_bits(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint16), np.ascontiguousarray(b).view(np.uint16))


def label(lay, k):
    if lay == "RR" or k == 1:  # one column: the mirror passes any view as row-major
        return "spmm_items_vec" if k % 8 == 0 else "spmm_items"
    return "spmm_relayout+items" if k >= 4 else "spmm_general"


@pytest.mark.parametrize("lay", LAYOUTS)
@pytest.mark.parametrize("case", ["thresholds", "small_mod3", "duplicates", "cancelling"])
def test_paths_within_bound(cuda, case, lay):
    A = matrix16(case)
    for k in (3, 5, 16):
        X, Y0 = operands(A, k, k)
        for alpha, beta in ((1.5, -0.5), (1.0, 0.0)):
            got, kern = call(cuda, A, X, Y0, alpha, beta, lay, y_nan=beta == 0)
            assert kern == label(lay, k), (kern, lay, k)
            check_bound(A, X, Y0, got, alpha, beta, "N", f"{kern} {case} {lay} k={k} a={alpha} b={beta}")


@pytest.mark.parametrize("mode", ["N", "C", "T", "H"])
def test_transpose_and_no_handle(cuda, mode):
    A = matrix16("thresholds")
    trans = mode in "TH"
    for lay in LAYOUTS:
        for k in (1, 8, 13):
            X, Y0 = operands(A, k, k, trans)
            for alpha, beta in ((-1.5, 0.5), (1.0, 0.0), (0.0, 2.0)):
                got, _ = call(cuda, A, X, Y0, alpha, beta, lay, mode, handle=False, y_nan=beta == 0)
                check_bound(A, X, Y0, got, alpha, beta, mode, f"no handle {mode} {lay} k={k} a={alpha} b={beta}")
                if trans:
                    got, kern = call(cuda, A, X, Y0, alpha, beta, lay, mode, y_nan=beta == 0)
                    assert alpha == 0 or kern == "spmm_transpose", kern
                    check_bound(A, X, Y0, got, alpha, beta, mode, f"{kern} {mode} {lay} k={k} a={alpha} b={beta}")


def identity(cuda, A, X, Y0, alpha, beta, lay, what):
    got, kern = call(cuda, A, X, Y0, alpha, beta, lay)
    y32, kern32 = call(cuda, A, X, Y0, alpha, beta, lay, dtype=torch.float32)
    assert kern in ("spmm_items", "spmm_items_vec", "spmm_relayout+items"), kern
    assert kern32.split("_vec")[0] == kern.split("_vec")[0], (kern, kern32)
    assert same_bits(got, H.round16(y32)), f"{kern} {what}"
    return got


IDENTITY_CASES = ["thresholds", "duplicates"] + ([] if EMULATED else ["many_multi_piece_rows", "many_long_rows"])


@pytest.mark.parametrize("lmax", [None, "16", "256"])
@pytest.mark.parametrize("case", IDENTITY_CASES)
def test_bit_identity_with_fp32(cuda, case, lmax, monkeypatch):
    """Single items, multi-piece rows (warp reduce) and rows of more than 64 pieces (CTA reduce), at every LMAX extreme."""
    if lmax:
        monkeypatch.setenv("B200SP_SPMM_ITEM_LMAX", lmax)
    A = matrix16(case)
    for lay in LAYOUTS:
        for k in (5, 16):
            X, Y0 = operands(A, k, 7)
            for alpha, beta in ((1.5, -0.5), (1.0, 0.0)):
                identity(cuda, A, X, Y0, alpha, beta, lay, f"{case} lmax={lmax} {lay} k={k} a={alpha} b={beta}")


def test_k_sweep(cuda):
    A = matrix16("small_mod1")
    for k in range(1, 65):
        X, Y0 = operands(A, k, k)
        for lay in ("RR", "LL"):
            got, kern = call(cuda, A, X, Y0, 1.5, -0.5, lay)
            assert kern == label(lay, k), (kern, lay, k)
            check_bound(A, X, Y0, got, 1.5, -0.5, "N", f"{kern} {lay} k={k}")
            if kern != "spmm_general":
                y32, _ = call(cuda, A, X, Y0, 1.5, -0.5, lay, dtype=torch.float32)
                assert same_bits(got, H.round16(y32)), (kern, lay, k)


def test_config3_full_size(cuda):
    """bench.py's config 3 (R-MAT scale 23, 16 columns, alpha = 1, beta = 0) with fp16 values and X: bit-identical to the
    fp32 call on the widened inputs, for LayoutRight and LayoutLeft."""
    from kokkos_kernels_b200 import matgen, sparse as sp

    k = 16
    rp, ci = matgen.rmat(23, 16)
    n, nnz = len(rp) - 1, len(ci)
    va = matgen.fill(nnz, 0.0, 1.0, 23, dtype=np.float32).astype(F16)
    X = matgen.fill(n * k, -1.0, 1.0, 5, dtype=np.float32).reshape(n, k).astype(F16)
    A16 = sp.CrsMatrix(torch.from_numpy(rp).to(cuda), torch.from_numpy(ci).to(cuda), torch.from_numpy(va).to(cuda), n)
    X16 = torch.from_numpy(X).to(cuda)
    for lay in ("RR", "LL"):
        h16, h32 = sp.SPMVHandle(), sp.SPMVHandle()
        Xa = X16 if lay == "RR" else X16.t().contiguous().t()
        Y16 = torch.full((n, k), float("nan"), dtype=torch.float16, device=cuda)
        Y16 = Y16 if lay == "RR" else Y16.t().contiguous().t()
        sp.spmv(h16, "N", 1.0, A16, Xa, 0.0, Y16)
        again = torch.empty_like(Y16)
        again.fill_(float("nan"))
        sp.spmv(h16, "N", 1.0, A16, Xa, 0.0, again)
        A32 = sp.CrsMatrix(A16.row_map, A16.entries, A16.values.float(), n)
        Y32 = torch.full_like(Y16, float("nan"), dtype=torch.float32)
        sp.spmv(h32, "N", 1.0, A32, Xa.float(), 0.0, Y32)
        torch.cuda.synchronize()
        assert h16.last_kernel() == ("spmm_items_vec" if lay == "RR" else "spmm_relayout+items"), h16.last_kernel()
        assert torch.equal(Y16.view(torch.int16), Y32.half().view(torch.int16)), lay
        assert torch.equal(Y16.view(torch.int16), again.view(torch.int16)), lay
        del Y16, Y32, again, A32, h16, h32


ACCUMULATION = [([2048, 1, -2048], 1.0, 1.0), ([60000, 60000, -60000], 1.0, 60000.0), ([60000, 60000], 0.5, 60000.0),
                ([60000, 60000], 1.0, np.inf), ([-60000, -60000], 1.0, -np.inf)]


@pytest.mark.parametrize("vals,alpha,want", ACCUMULATION)
def test_fp32_accumulation(cuda, vals, alpha, want):
    n = len(vals)
    row = (np.array([0, n], dtype=np.int32), np.arange(n, dtype=np.int32), np.asarray(vals, dtype=F16), n)
    col = (np.arange(n + 1, dtype=np.int32), np.zeros(n, dtype=np.int32), np.asarray(vals, dtype=F16), 1)
    for lay in LAYOUTS:
        for k in (3, 8):
            for handle in (True, False):
                got, kern = call(cuda, row, np.ones((n, k), F16), np.zeros((1, k), F16), alpha, 0.0, lay, handle=handle)
                assert np.all(got.astype(np.float64) == want), (got, want, kern)
                got, kern = call(cuda, col, np.ones((n, k), F16), np.zeros((1, k), F16), alpha, 0.0, lay, "T", handle=handle)
                assert np.all(got.astype(np.float64) == want), (got, want, kern)


def test_special_values(cuda):
    for vals, x, want in (([2.0**-14], 2.0**-10, 2.0**-24), ([2.0**-13] * 3, 2.0**-12, 2.0**-23), ([2.0**-14, -2.0**-15], 2.0**-10, 0.0)):
        n = len(vals)
        A = (np.array([0, n], dtype=np.int32), np.arange(n, dtype=np.int32), np.asarray(vals, dtype=F16), n)
        for lay in ("RR", "LL"):
            got, kern = call(cuda, A, np.full((n, 8), x, F16), np.zeros((1, 8), F16), 1.0, 0.0, lay)
            assert np.all(got.astype(np.float64) == want), (vals, got, want, kern)
    A = matrix16("small_mod1")
    X, Y0 = operands(A, 8, 1)
    X[3, :] = np.inf
    X[7, 2] = np.nan
    for lay in LAYOUTS:
        for alpha, beta in ((1.0, 0.0), (2.0, -1.0)):
            got, kern = call(cuda, A, X, Y0, alpha, beta, lay, y_nan=beta == 0)
            check_bound(A, X, Y0, got, alpha, beta, "N", f"{kern} inf/nan {lay}")
    got, _ = call(cuda, A, np.ones_like(X), Y0, 1.0, 0.0, "RR", y_nan=True)
    assert not np.isnan(got).any()


def test_strided_and_misaligned(cuda):
    from kokkos_kernels_b200 import sparse as sp

    A16 = matrix16("thresholds")
    k = 16
    X, Y0 = operands(A16, k, 2)
    ref, kern = call(cuda, A16, X, Y0, 1.5, -0.5)
    assert kern == "spmm_items_vec", kern
    A = dev_matrix(cuda, A16)
    for how in ("odd_ld", "offset"):
        if how == "odd_ld":
            Xd = torch.zeros((X.shape[0], k + 1), dtype=torch.float16, device=cuda)[:, :k]
            Yd = torch.zeros((Y0.shape[0], k + 1), dtype=torch.float16, device=cuda)[:, :k]
        else:
            Xd = torch.zeros(X.size + 1, dtype=torch.float16, device=cuda)[1:].view(X.shape)
            Yd = torch.zeros(Y0.size + 1, dtype=torch.float16, device=cuda)[1:].view(Y0.shape)
        Xd.copy_(torch.from_numpy(X).to(cuda))
        Yd.copy_(torch.from_numpy(Y0).to(cuda))
        h = sp.SPMVHandle()
        sp.spmv(h, "N", 1.5, A, Xd, -0.5, Yd)
        torch.cuda.synchronize()
        assert h.last_kernel() == "spmm_items", (how, h.last_kernel())
        assert same_bits(host(Yd), ref), how


def test_determinism(cuda):
    A = matrix16("thresholds" if EMULATED else "many_long_rows")
    X, Y0 = operands(A, 16, 3)
    for lay in ("RR", "LL"):
        a, ka = call(cuda, A, X, Y0, 1.5, -0.5, lay)
        b, kb = call(cuda, A, X, Y0, 1.5, -0.5, lay)
        assert ka == kb and same_bits(a, b), (lay, ka)


def test_coefficients_are_rounded_to_half(cuda):
    """alpha and beta reach the library as the half_t Kokkos would hold: 0.1 becomes 0.0999755859375."""
    A = matrix16("small_mod1")
    X, Y0 = operands(A, 8, 4)
    got, _ = call(cuda, A, X, Y0, 0.1, 0.3)
    ref, _ = call(cuda, A, X, Y0, float(F16(0.1)), float(F16(0.3)))
    assert same_bits(got, ref)


def test_mirror_errors(cuda):
    from kokkos_kernels_b200 import sparse as sp
    from kokkos_kernels_b200._lib import B200SparseError

    rp, ci, v, n = matrix16("small_mod1")
    m = len(rp) - 1
    A = dev_matrix(cuda, (rp, ci, v, n))
    X = torch.ones((n, 4), dtype=torch.float16, device=cuda)
    Y = torch.zeros((m, 4), dtype=torch.float16, device=cuda)
    h = sp.SPMVHandle()
    with pytest.raises(B200SparseError, match="rank 1"):
        sp.spmv(h, "N", 1.0, A, X[:, 0].contiguous(), 0.0, Y[:, 0].contiguous())
    with pytest.raises(B200SparseError, match="mixed precision"):
        sp.spmv(h, "N", 1.0, A, X.float(), 0.0, Y)
    with pytest.raises(B200SparseError, match="mixed precision"):
        sp.spmv(h, "N", 1.0, dev_matrix(cuda, (rp, ci, v, n), np.float32), X, 0.0, Y)
    A64 = sp.CrsMatrix(A.row_map.long(), A.entries, A.values, n)
    with pytest.raises(B200SparseError, match="64-bit offsets"):
        sp.spmv(h, "N", 1.0, A64, X, 0.0, Y)
    B = sp.BsrMatrix(A.row_map, A.entries, A.values, n, 1)
    with pytest.raises(B200SparseError, match="BsrMatrix"):
        sp.spmv(h, "N", 1.0, B, X, 0.0, Y)
    with pytest.raises(B200SparseError, match="Dimensions do not match"):
        sp.spmv(h, "N", 1.0, A, Y, 0.0, Y)
