"""Every rank-2 SpMV kernel path (csrc/spmm.cu) on the GPU, each call checked entry by entry against the exact product
(tests/exact_ref.py) within a rigorous per-entry rounding bound, in fp32 and fp64.  The operands' layouts, strides and alignment and the
presence of a plan select the path, B200SP_SPMM_ITEM_LMAX (read by getenv on every call) the item length, and every test
that runs with a plan asserts the handle's last_kernel(), so a dispatcher that quietly falls back cannot make a test
vacuous."""
import os

import numpy as np
import pytest
import torch

import exact_ref as R
import spmm_cases as cases

pytestmark = pytest.mark.gpu

DTYPES = [np.float32, np.float64]
TDT = {np.dtype(np.float32): torch.float32, np.dtype(np.float64): torch.float64}
LAYOUTS = ["RR", "LL", "RL", "LR"]  # X layout, Y layout: R = LayoutRight (row-major), L = LayoutLeft
SPMM_VARS = ["B200SP_SPMM_ITEM_LMAX"]
EMULATED = os.environ.get("B200SP_TEST_EMULATED") == "1"


@pytest.fixture(autouse=True)
def _clean_env(monkeypatch):
    for k in SPMM_VARS:
        monkeypatch.delenv(k, raising=False)


_MATS = {}


def matrix(name, dtype, seed=5):
    key = (name, np.dtype(dtype).name, seed)
    if key not in _MATS:
        builder = cases.SMALL_CASES.get(name) or getattr(cases, name)
        _MATS[key] = builder(seed, dtype)
    return _MATS[key]


def dev_matrix(cuda, rp, ci, v, ncols):
    from kokkos_kernels_b200 import sparse as sp

    return sp.CrsMatrix(torch.from_numpy(rp).to(cuda), torch.from_numpy(ci).to(cuda), torch.from_numpy(v).to(cuda), ncols)


def dev(cuda, a, rowmajor):
    if a.size == 0:
        return torch.empty(a.shape, dtype=TDT[a.dtype], device=cuda)
    t = torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    return t if rowmajor else t.t().contiguous().t()


def spmv(h, mode, alpha, A, X, beta, Y):
    from kokkos_kernels_b200 import sparse as sp

    sp.spmv(h, mode, alpha, A, X, beta, Y)
    torch.cuda.synchronize()
    return Y.cpu().numpy()


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def kernel(h):
    return h.last_kernel() if h is not None else "no plan"


def expected_kernel(k, dtype, layout, ld_vec=True):
    """The label spmm_impl reports for these operands (16-byte aligned, a plan).  ld_vec=False: a LayoutRight operand has a
    leading dimension that is not a multiple of the vector width, which rules out the 16-byte kernels."""
    if k == 1:
        layout = "RR"  # a single column is passed as LayoutRight whatever its strides
    if layout != "RR":
        return "spmm_relayout+items" if k >= 4 else "spmm_general"
    vec = k % (4 if np.dtype(dtype) == np.float32 else 2) == 0 and ld_vec
    return "spmm_items_vec" if vec else "spmm_items"


def check(got, A_np, X, Y0, alpha, beta, trans, what):
    rp, ci, v, _ = A_np
    R.assert_within(got, R.spmm_exact(rp, ci, v, X, Y0, alpha, beta, trans), R.spmm_bound(rp, ci, v, X, Y0, alpha, beta, trans), what)


def operands(A_np, k, dtype, trans=False, seed=0):
    rp, ci, v, ncols = A_np
    m = len(rp) - 1
    rng = np.random.default_rng(seed + 1000 * k)
    xr, yr = (m, ncols) if trans else (ncols, m)
    return cases.dense_operands(rng, xr, k, dtype), cases.dense_operands(rng, yr, k, dtype)


# ---- (a) each path ---------------------------------------------------------------------------------------------------
PATHS = [
    {},
    {"B200SP_SPMM_ITEM_LMAX": "16"},
    {"B200SP_SPMM_ITEM_LMAX": "64"},
    {"B200SP_SPMM_ITEM_LMAX": "256"},
]
PATH_IDS = ["-".join(f"{k.replace('B200SP_SPMM_', '').lower()}={v}" for k, v in p.items()) or "default" for p in PATHS]
PATH_KS = [1, 5, 16, 36, 132]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("env", PATHS, ids=PATH_IDS)
def test_each_path(cuda, monkeypatch, env, dtype):
    """The threshold matrix (row lengths around every batch and item limit) through the item path at one item length, with a
    fresh handle, for k crossing the vector width and the 32-lane strips, LayoutRight and LayoutLeft (relayout)."""
    from kokkos_kernels_b200 import sparse as sp

    for k_, v_ in env.items():
        monkeypatch.setenv(k_, v_)
    A_np = matrix("thresholds", dtype)
    A = dev_matrix(cuda, *A_np)
    h = sp.SPMVHandle()
    for k in PATH_KS:
        X, Y0 = operands(A_np, k, dtype)
        exact = R.spmm_exact(*A_np[:3], X, Y0, 2.5, -0.5)
        bound = R.spmm_bound(*A_np[:3], X, Y0, 2.5, -0.5)
        for layout in ("RR", "LL"):
            got = spmv(h, "N", 2.5, A, dev(cuda, X, layout[0] == "R"), -0.5, dev(cuda, Y0, layout[1] == "R"))
            assert h.last_kernel() == expected_kernel(k, dtype, layout), (env, k, layout, h.last_kernel())
            R.assert_within(got, exact, bound, f"{h.last_kernel()} {env} k={k} {layout} {np.dtype(dtype).name}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mode", ["T", "H"])
def test_transpose_every_layout(cuda, mode, dtype):
    """T / H (atomics) for every layout mix, with and without a plan; rectangular, duplicates, cancelling rows."""
    from kokkos_kernels_b200 import sparse as sp

    for name in ("thresholds", "duplicates", "cancelling", "wide_short"):
        A_np = matrix(name, dtype)
        A = dev_matrix(cuda, *A_np)
        for k in (1, 4, 17):
            X, Y0 = operands(A_np, k, dtype, trans=True)
            for alpha, beta in ((1.0, 0.0), (-1.5, 0.5)):
                exact = R.spmm_exact(*A_np[:3], X, Y0, alpha, beta, trans=True)
                bound = R.spmm_bound(*A_np[:3], X, Y0, alpha, beta, trans=True)
                for layout in LAYOUTS:
                    for h in (sp.SPMVHandle(), None):
                        Yd = dev(cuda, np.full_like(Y0, np.nan) if beta == 0 else Y0, layout[1] == "R")
                        got = spmv(h, mode, alpha, A, dev(cuda, X, layout[0] == "R"), beta, Yd)
                        if h is not None:
                            assert h.last_kernel() == "spmm_transpose", h.last_kernel()
                        R.assert_within(got, exact, bound, f"{kernel(h)} {name} {mode} k={k} {layout} a={alpha} b={beta}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_no_plan_paths(cuda, dtype):
    """handle=None: spmm_rowmajor_kernel for LayoutRight X and Y (k from 1 to 33: every group width KT from 1 to 32),
    spmm_general_kernel for any other mix."""
    for name in ("thresholds", "small_mod1", "duplicates", "cancelling"):
        A_np = matrix(name, dtype)
        A = dev_matrix(cuda, *A_np)
        for k in (1, 2, 3, 5, 8, 16, 17, 33):
            X, Y0 = operands(A_np, k, dtype)
            exact = R.spmm_exact(*A_np[:3], X, Y0, -1.0, 1.0)
            bound = R.spmm_bound(*A_np[:3], X, Y0, -1.0, 1.0)
            for layout in LAYOUTS:
                got = spmv(None, "N", -1.0, A, dev(cuda, X, layout[0] == "R"), 1.0, dev(cuda, Y0, layout[1] == "R"))
                R.assert_within(got, exact, bound, f"no plan {name} k={k} {layout}")


# ---- (b) k sweep -----------------------------------------------------------------------------------------------------
K_SWEEP = [1, 2, 3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 132, 256]


@pytest.mark.parametrize("dtype", DTYPES)
def test_k_sweep(cuda, dtype):
    """The default path for k across the vector width, KTL = 32, the multi-strip loop beyond KTL*W, the relayout's
    32-column tiles and the reduce kernels' column loop beyond 32; all four layout mixes."""
    from kokkos_kernels_b200 import sparse as sp

    A_np = matrix("thresholds", dtype)
    A = dev_matrix(cuda, *A_np)
    for k in K_SWEEP:
        X, Y0 = operands(A_np, k, dtype)
        exact = R.spmm_exact(*A_np[:3], X, Y0, 1.5, 0.5)
        bound = R.spmm_bound(*A_np[:3], X, Y0, 1.5, 0.5)
        for layout in LAYOUTS:
            h = sp.SPMVHandle()
            got = spmv(h, "N", 1.5, A, dev(cuda, X, layout[0] == "R"), 0.5, dev(cuda, Y0, layout[1] == "R"))
            assert h.last_kernel() == expected_kernel(k, dtype, layout), (k, layout, h.last_kernel())
            R.assert_within(got, exact, bound, f"{h.last_kernel()} k={k} {layout} {np.dtype(dtype).name}")


# ---- (c) strides and alignment ---------------------------------------------------------------------------------------
SENTINEL = -7.25e5


def padded(cuda, a, rowmajor, extra_cols, extra_rows=5):
    """a as a view into a wider tensor (ld = k + extra_cols for LayoutRight, ld > rows for LayoutLeft, columns beyond k
    either way); everything outside the view holds SENTINEL.  Returns (view, base)."""
    rows, k = a.shape
    t = torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    if rowmajor:
        base = torch.full((rows, k + extra_cols), SENTINEL, dtype=t.dtype, device=cuda)
        base[:, :k] = t
        return base[:, :k], base
    base = torch.full((k + extra_cols, rows + extra_rows), SENTINEL, dtype=t.dtype, device=cuda).t()
    base[:rows, :k] = t
    return base[:rows, :k], base


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("pad", [4, 3], ids=["ld_vector", "ld_odd"])
def test_strided_views(cuda, pad, dtype):
    """X and Y as slices of wider tensors in both layouts: correct, and nothing outside Y's view is written.  Padding
    LayoutRight rows by 4 keeps ld a multiple of the vector width, so the 16-byte kernels run with ld > k (a vector store
    past k would land in the padding); padding by 3 makes ld odd and selects the scalar kernels."""
    from kokkos_kernels_b200 import sparse as sp

    A_np = matrix("thresholds", dtype)
    A = dev_matrix(cuda, *A_np)
    for k in (4, 6, 16, 36, 132):
        X, Y0 = operands(A_np, k, dtype)
        exact = R.spmm_exact(*A_np[:3], X, Y0, 2.5, -0.5)
        bound = R.spmm_bound(*A_np[:3], X, Y0, 2.5, -0.5)
        for layout in LAYOUTS:
            h = sp.SPMVHandle()
            Xv, _ = padded(cuda, X, layout[0] == "R", pad)
            Yv, Yb = padded(cuda, Y0, layout[1] == "R", pad)
            before = Yb.cpu().numpy().copy()
            got = spmv(h, "N", 2.5, A, Xv, -0.5, Yv)
            what = f"{h.last_kernel()} k={k} {layout} strided pad={pad}"
            ld_vec = pad % (4 if np.dtype(dtype) == np.float32 else 2) == 0 or layout == "LL"  # LL: row-major scratch, ld = k
            assert h.last_kernel() == expected_kernel(k, dtype, layout, ld_vec), what
            R.assert_within(got, exact, bound, what)
            after = Yb.cpu().numpy()
            outside = np.ones(after.shape, bool)
            outside[:Y0.shape[0], :k] = False
            assert np.array_equal(bits(after[outside]), bits(before[outside])), what + ": wrote outside the view"


def offset_by_one(cuda, a):
    """a row-major at a storage offset of one element (not 16-byte aligned)."""
    t = torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=cuda)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    return v


@pytest.mark.parametrize("dtype", DTYPES)
def test_misaligned_operands(cuda, dtype):
    """X / Y one element off 16-byte alignment: the scalar item kernel, with the same bits as the aligned vector kernel (per
    column the additions come in the same order)."""
    from kokkos_kernels_b200 import sparse as sp

    A_np = matrix("thresholds", dtype)
    A = dev_matrix(cuda, *A_np)
    for k in (4, 16, 132):
        X, Y0 = operands(A_np, k, dtype)
        exact = R.spmm_exact(*A_np[:3], X, Y0, 2.5, -0.5)
        bound = R.spmm_bound(*A_np[:3], X, Y0, 2.5, -0.5)
        h = sp.SPMVHandle()
        ref = spmv(h, "N", 2.5, A, dev(cuda, X, True), -0.5, dev(cuda, Y0, True))
        vec_kernel = h.last_kernel()
        assert vec_kernel == expected_kernel(k, dtype, "RR")
        for xoff, yoff in ((True, False), (False, True), (True, True)):
            Xd = offset_by_one(cuda, X) if xoff else dev(cuda, X, True)
            Yd = offset_by_one(cuda, Y0) if yoff else dev(cuda, Y0, True)
            got = spmv(h, "N", 2.5, A, Xd, -0.5, Yd)
            what = f"{h.last_kernel()} k={k} offsets x={xoff} y={yoff}"
            assert h.last_kernel() == "spmm_items", what
            R.assert_within(got, exact, bound, what)
            assert np.array_equal(bits(got), bits(ref)), what + ": differs from the aligned vector kernel"


@pytest.mark.parametrize("dtype", DTYPES)
def test_misaligned_matrix_arrays(cuda, dtype):
    """vals / col_idx one element off 16-byte alignment: the item path reads them entry by entry, so it takes them and must
    be right, in both layouts."""
    from kokkos_kernels_b200 import sparse as sp

    rp, ci, v, ncols = A_np = matrix("thresholds", dtype)
    A = sp.CrsMatrix(torch.from_numpy(rp).to(cuda), offset_by_one(cuda, ci[:, None])[:, 0], offset_by_one(cuda, v[:, None])[:, 0], ncols)
    assert A.entries.data_ptr() % 16 != 0 and A.values.data_ptr() % 16 != 0
    for k in (3, 16):
        X, Y0 = operands(A_np, k, dtype)
        exact = R.spmm_exact(rp, ci, v, X, Y0, 2.5, -0.5)
        bound = R.spmm_bound(rp, ci, v, X, Y0, 2.5, -0.5)
        for layout in ("RR", "LL"):
            h = sp.SPMVHandle()
            got = spmv(h, "N", 2.5, A, dev(cuda, X, layout[0] == "R"), -0.5, dev(cuda, Y0, layout[1] == "R"))
            assert h.last_kernel() == expected_kernel(k, dtype, layout), h.last_kernel()
            R.assert_within(got, exact, bound, f"{h.last_kernel()} k={k} {layout} misaligned vals/col_idx")


# ---- (d) scalars and special values ----------------------------------------------------------------------------------
SCALARS = [(1.0, 0.0), (-1.0, 1.0), (2.5, -0.5), (0.0, 2.5), (0.0, 0.0), (1.0, 1.0)]


@pytest.mark.parametrize("dtype", DTYPES)
def test_scalars(cuda, dtype):
    """Every (alpha, beta) pair; beta == 0 over a Y of NaN; alpha == 0 over an X of NaN gives exactly beta*Y0."""
    from kokkos_kernels_b200 import sparse as sp

    for name in ("thresholds", "cancelling", "small_mod2", "no_columns"):
        A_np = matrix(name, dtype)
        A = dev_matrix(cuda, *A_np)
        for k in (5, 16):
            X, Y0 = operands(A_np, k, dtype)
            for alpha, beta in SCALARS:
                for layout in ("RR", "LL", "RL") if A_np[3] else ("RR", "RL"):
                    h = sp.SPMVHandle()
                    Yin = np.full_like(Y0, np.nan) if beta == 0 else Y0
                    Xin = np.full_like(X, np.nan) if alpha == 0 else X
                    Xd, Yd = dev(cuda, Xin, layout[0] == "R"), dev(cuda, Yin, layout[1] == "R")
                    expect0 = Yd * beta if beta != 0 else torch.zeros_like(Yd)
                    got = spmv(h, "N", alpha, A, Xd, beta, Yd)
                    what = f"{h.last_kernel()} {name} k={k} {layout} a={alpha} b={beta}"
                    if alpha == 0 or A_np[3] == 0:  # only Y is scaled: no product kernel runs
                        assert h.last_kernel() == "none", what
                        assert torch.equal(torch.from_numpy(got).to(cuda), expect0), what
                    else:
                        assert h.last_kernel() == expected_kernel(k, dtype, layout), what
                        R.assert_within(got, R.spmm_exact(*A_np[:3], X, Y0, alpha, beta), R.spmm_bound(*A_np[:3], X, Y0, alpha, beta), what)


@pytest.mark.parametrize("dtype", DTYPES)
def test_single_inf_reaches_exactly_its_rows(cuda, dtype):
    """One Inf in X(c, j): exactly the rows of A that reference column c turn non-finite in column j (the reference
    says which: +-Inf, or NaN where terms of both signs meet); every other entry stays finite and within its bound."""
    from kokkos_kernels_b200 import sparse as sp

    rp, ci, v, ncols = A_np = matrix("thresholds", dtype)
    A = dev_matrix(cuda, *A_np)
    counts = np.bincount(ci, minlength=ncols)
    for k in (4, 16):
        X, Y0 = operands(A_np, k, dtype)
        for c in (int(ci[rp[1] - 1]), int(np.argmax(counts))):  # a column of the long first row; the most used column
            j = c % k
            Xi = X.copy()
            Xi[c, j] = np.inf
            exact = R.spmm_exact(rp, ci, v, Xi, Y0, 1.5, 0.5)
            hit = np.unique(np.repeat(np.arange(len(rp) - 1), np.diff(rp))[ci == c])
            assert set(np.flatnonzero(~np.isfinite(exact[:, j]))) == set(hit) and np.isfinite(np.delete(exact, j, 1)).all()
            for layout in ("RR", "LL"):
                h = sp.SPMVHandle()
                got = spmv(h, "N", 1.5, A, dev(cuda, Xi, layout[0] == "R"), 0.5, dev(cuda, Y0, layout[1] == "R"))
                assert h.last_kernel() == expected_kernel(k, dtype, layout), h.last_kernel()
                R.assert_within(got, exact, R.spmm_bound(rp, ci, v, Xi, Y0, 1.5, 0.5), f"{h.last_kernel()} Inf at X({c},{j}) k={k} {layout}")


# ---- (e) determinism and the stated identities -----------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_items_are_deterministic(cuda, dtype):
    """The item path uses no atomics: a second call through the same handle gives the same bits; and it gives the same bits
    for LayoutLeft as for LayoutRight (the relayout only moves data)."""
    from kokkos_kernels_b200 import sparse as sp

    A_np = matrix("thresholds", dtype)
    A = dev_matrix(cuda, *A_np)
    for k in (3, 16, 132):
        X, Y0 = operands(A_np, k, dtype)
        h = sp.SPMVHandle()
        outs = {}
        for layout in ("RR", "RR", "LL", "RL", "LR"):
            got = spmv(h, "N", 1.5, A, dev(cuda, X, layout[0] == "R"), -0.5, dev(cuda, Y0, layout[1] == "R"))
            check(got, A_np, X, Y0, 1.5, -0.5, False, f"{h.last_kernel()} k={k} {layout}")
            if layout in outs:
                assert np.array_equal(bits(got), bits(outs[layout])), (k, "second call differs")
            outs[layout] = got
        if k >= 4:  # below 4 columns LayoutLeft operands take spmm_general_kernel
            for layout in ("LL", "RL", "LR"):
                assert np.array_equal(bits(outs[layout]), bits(outs["RR"])), (k, layout, "differs from RR")


# ---- (f) one handle, changing shapes ---------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_one_handle_growing_and_shrinking_k(cuda, dtype):
    """k = 16, 129, 4, 64 through one handle and one matrix, layouts RR, LL, RL, LR in turn, beta alternating between 0
    and not: the plan's partial sums and relayout scratch are re-grown and reused."""
    from kokkos_kernels_b200 import sparse as sp

    A_np = matrix("thresholds", dtype)
    A = dev_matrix(cuda, *A_np)
    h = sp.SPMVHandle()
    step = 0
    for k in (16, 129, 4, 64):
        X, Y0 = operands(A_np, k, dtype)
        for layout in LAYOUTS:
            beta = 0.0 if step % 2 == 0 else 0.75
            step += 1
            Yin = np.full_like(Y0, np.nan) if beta == 0 else Y0
            got = spmv(h, "N", -2.0, A, dev(cuda, X, layout[0] == "R"), beta, dev(cuda, Yin, layout[1] == "R"))
            assert h.last_kernel() == expected_kernel(k, dtype, layout), (k, layout, h.last_kernel())
            check(got, A_np, X, Y0, -2.0, beta, False, f"{h.last_kernel()} k={k} {layout} b={beta}")


# ---- wrap cases: more work than one pass of the grid-stride loops on 132 SMs -------------------------------------------
@pytest.mark.skipif(EMULATED, reason="millions of entries: hours under the emulation")
@pytest.mark.parametrize("dtype,k", [(np.float32, 16), (np.float64, 4)])
def test_reduce_kernels_wrap(cuda, dtype, k):
    """More multi-piece rows than spmm_item_reduce_kernel's warps, and more rows of over 64 pieces than
    spmm_item_reduce_long_kernel's CTAs."""
    from kokkos_kernels_b200 import sparse as sp

    for name, layout in (("many_multi_piece_rows", "RR"), ("many_long_rows", "RR"), ("many_multi_piece_rows", "LL")):
        A_np = matrix(name, dtype)
        A = dev_matrix(cuda, *A_np)
        X, Y0 = operands(A_np, k, dtype)
        h = sp.SPMVHandle()
        got = spmv(h, "N", 1.5, A, dev(cuda, X, layout[0] == "R"), -0.5, dev(cuda, Y0, layout[1] == "R"))
        assert h.last_kernel() == expected_kernel(k, dtype, layout), h.last_kernel()
        check(got, A_np, X, Y0, 1.5, -0.5, False, f"{h.last_kernel()} {name} k={k} {layout}")


@pytest.mark.skipif(EMULATED, reason="300,000 rows: slow under the emulation")
@pytest.mark.parametrize("dtype", DTYPES)
def test_relayout_and_scale_wrap(cuda, dtype):
    """300,000 rows with LayoutLeft operands (relayout_kernel's grid wraps) and alpha == 0 / transposes over rows * k
    beyond scale2d_kernel's grid."""
    from kokkos_kernels_b200 import sparse as sp

    A_np = matrix("tall", dtype)
    A = dev_matrix(cuda, *A_np)
    for k in (4, 8):
        X, Y0 = operands(A_np, k, dtype)
        for layout in ("LL", "RL", "LR"):
            h = sp.SPMVHandle()
            got = spmv(h, "N", 2.5, A, dev(cuda, X, layout[0] == "R"), -0.5, dev(cuda, Y0, layout[1] == "R"))
            assert h.last_kernel() == expected_kernel(k, dtype, layout), h.last_kernel()
            check(got, A_np, X, Y0, 2.5, -0.5, False, f"{h.last_kernel()} tall k={k} {layout}")
            Yd = dev(cuda, Y0, layout[1] == "R")
            expect = Yd * 0.5
            spmv(h, "N", 0.0, A, dev(cuda, X, layout[0] == "R"), 0.5, Yd)
            assert torch.equal(Yd, expect), ("scale2d", k, layout)
        Xt, Yt0 = operands(A_np, k, dtype, trans=True)
        for layout in ("RR", "LL"):
            h = sp.SPMVHandle()
            got = spmv(h, "T", 2.5, A, dev(cuda, Xt, layout[0] == "R"), -0.5, dev(cuda, Yt0, layout[1] == "R"))
            assert h.last_kernel() == "spmm_transpose"
            check(got, A_np, Xt, Yt0, 2.5, -0.5, True, f"transpose tall k={k} {layout}")


# ---- (g) one large case: scale2d_kernel's 64-bit index branch --------------------------------------------------------
@pytest.mark.skipif(EMULATED, reason="8.6 GB on the device")
def test_scale_over_2_to_the_31_elements(cuda):
    """alpha == 0, beta = 0.5 on an fp32 Y of 2^31 + 16 elements: every entry is exactly 0.5 * Y0 (one rounding)."""
    from kokkos_kernels_b200 import sparse as sp

    free, _ = torch.cuda.mem_get_info()
    if free < 24 * 2**30:
        pytest.skip(f"needs 24 GB free on the device, {free / 2**30:.1f} GB free")
    k = 16
    rows = (1 << 31) // k + 1
    A = sp.CrsMatrix(torch.zeros(rows + 1, dtype=torch.int32, device=cuda), torch.zeros(1, dtype=torch.int32, device=cuda)[:0],
                     torch.zeros(1, dtype=torch.float32, device=cuda)[:0], 3)
    X = torch.ones((3, k), dtype=torch.float32, device=cuda)
    g = torch.Generator(device=cuda)
    g.manual_seed(17)
    Y0 = torch.randn((rows, k), dtype=torch.float32, device=cuda, generator=g)
    Y = Y0.clone()
    h = sp.SPMVHandle()
    sp.spmv(h, "N", 0.0, A, X, 0.5, Y)
    torch.cuda.synchronize()
    step = 1 << 24
    for r in range(0, rows, step):
        assert torch.equal(Y[r:r + step], Y0[r:r + step] * 0.5), r
    del Y, Y0
    torch.cuda.empty_cache()
