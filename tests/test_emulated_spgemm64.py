"""SpGEMM on 64-bit offsets (kokkos-kernels_b200/csrc/spgemm64.cu) executed on the CPU (tools/emu): with the window limit
lowered so that small products are cut into many windows, row_ptr_C must equal the 32-bit entry point's, and col_idx_C and
vals_C must equal them bit for bit (fp64 and fp32), on the SpGEMM case lists that drive every ESC bin, the hash kernels and
the bitmap / fallback rows.  The limits go down to the longest row's products, so window boundaries fall inside every bin.
The production limit (2^31 - 65537) cannot be reached in a test; tests/test_gpu_spgemm64.py runs a product past it."""
import ctypes as C
import os

import numpy as np
import pytest

import emu_lib as E
from spgemm_cases import cases

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "issue402.npz")
OK, ERR_INVALID, ERR_STATE, ERR_OVERFLOW = 0, 1, 3, 4


@pytest.fixture(scope="module")
def emu():
    return E.lib()


class Plan:
    def __init__(self, window=None):
        self.h = C.c_void_p()
        E.ok(E.lib().b200sp_spgemm_plan_create(C.byref(self.h)))
        if window is not None:
            E.ok(E.lib().b200sp_spgemm_plan_set_window(self.h, C.c_int64(window)))

    def windows(self):
        return E.lib().b200sp_spgemm_plan_windows(self.h)

    def close(self):
        E.ok(E.lib().b200sp_spgemm_plan_destroy(self.h, None))


def symbolic64_rc(plan, A, B, m, n, k, rpC):
    nnz, mx = C.c_int64(-1), C.c_int(-1)
    rc = E.lib().b200sp_spgemm_symbolic_i64(plan.h, None, m, n, k, E.ptr(A[0]), E.ptr(A[1]), E.ptr(B[0]), E.ptr(B[1]),
                                            E.ptr(rpC), C.byref(nnz), C.byref(mx))
    return rc, nnz.value, mx.value


def numeric_rc(plan, A, B, m, n, k, rpC, ciC, vC, bits):
    fn = getattr(E.lib(), "b200sp_spgemm_numeric_%s_i%d" % (E.sfx(vC.dtype), bits))
    return fn(plan.h, None, m, n, k, E.ptr(A[0]), E.ptr(A[1]), E.ptr(A[2]), E.ptr(B[0]), E.ptr(B[1]), E.ptr(B[2]), E.ptr(rpC),
              E.ptr(ciC), E.ptr(vC))


def wide(M):
    return (M[0].astype(np.int64), M[1], M[2])


def spgemm64(A, B, m, n, k, dtype, window=None):
    """C = A*B through the _i64 entries; returns (rpC, ciC, vC, c_max, windows)."""
    A64, B64 = wide(A), wide(B)
    p = Plan(window)
    try:
        rpC = np.full(m + 1, -7, dtype=np.int64)
        rc, nnz, mx = symbolic64_rc(p, A64, B64, m, n, k, rpC)
        E.ok(rc)
        ciC = np.full(nnz, -1, dtype=np.int32)
        vC = np.full(nnz, np.nan, dtype=dtype)
        E.ok(numeric_rc(p, A64, B64, m, n, k, rpC, ciC, vC, 64))
        return rpC, ciC, vC, mx, p.windows()
    finally:
        p.close()


def row_products(A, B):
    lenB = np.diff(B[0].astype(np.int64))
    rows = np.repeat(np.arange(len(A[0]) - 1), np.diff(A[0]))
    return np.bincount(rows, weights=lenB[A[1]], minlength=len(A[0]) - 1).astype(np.int64)


def expected_windows(A, B, limit):
    """The greedy cut the library documents: consecutive rows, at most `limit` products and `limit` entries of A."""
    P = np.concatenate([[0], np.cumsum(row_products(A, B))])
    Q = A[0].astype(np.int64)
    m, R, count = len(Q) - 1, 0, 0
    while R < m:
        end = min(np.searchsorted(P, P[R] + limit, "right"), np.searchsorted(Q, Q[R] + limit, "right")) - 1
        assert end > R
        count += 1
        R = end
    return count


def longest_row_limit(A, B):
    """The least limit that takes every row: the longest row's products (or entries of A)."""
    return max(int(row_products(A, B).max()), int(np.diff(A[0]).max()), 8)


def limits_for(A, B):
    """About 40 windows (boundary and boundary + 1), about 9, and the default (one window)."""
    lo, total = longest_row_limit(A, B), int(row_products(A, B).sum())
    base = max(lo, -(-total // 40))
    return sorted({base, base + 1, max(lo, total // 9)}) + [None]


def rows_around_longest(A, B, count=24):
    """A's rows [r0, r0 + count) around its longest product row, with a row map of its own."""
    m = len(A[0]) - 1
    r0 = max(0, min(m - count, int(np.argmax(row_products(A, B))) - count // 2))
    r1 = min(m, r0 + count)
    a0, a1 = int(A[0][r0]), int(A[0][r1])
    return (A[0][r0:r1 + 1] - a0, A[1][a0:a1].copy(), A[2][a0:a1].copy()), r1 - r0


def all_cases(dtype):
    out = list(cases(dtype))
    z = np.load(GOLD)
    import oracle_lib

    orc = oracle_lib.Oracle()
    rp, ci, v = z["rowmap"].copy(), z["entries"].copy(), z["values"].astype(dtype)
    n = len(rp) - 1
    trp, tci, tv = orc.transpose(rp, ci, v.astype(np.float64), n)
    out.append(("issue402", (rp, ci, v), (trp, tci, tv.astype(dtype)), n, n, n))
    return out


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_windows_equal_the_32_bit_path(emu, dtype):
    for name, A, B, m, n, k in all_cases(dtype):
        ref = E.spgemm(A, B, m, n, k, dtype)
        for limit in limits_for(A, B):
            rpC, ciC, vC, mx, nw = spgemm64(A, B, m, n, k, dtype, limit)
            what = (name, limit)
            assert np.array_equal(rpC, ref[0].astype(np.int64)), what
            assert np.array_equal(ciC, ref[1]), what
            assert np.array_equal(vC.view(np.uint8), ref[2].view(np.uint8)), what
            assert mx == ref[3], what
            assert nw == (1 if limit is None else expected_windows(A, B, limit)), what


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_limit_at_the_longest_row(emu, dtype):
    """At and just above the longest row's products nearly every row is a window of its own: on the rows around it."""
    for name, A, B, m, n, k in all_cases(dtype):
        As, ms = rows_around_longest(A, B)
        ref = E.spgemm(As, B, ms, n, k, dtype)
        lo = longest_row_limit(As, B)
        assert lo == longest_row_limit(A, B) or name == "issue402", name
        for limit in (lo, lo + 1):
            rpC, ciC, vC, mx, nw = spgemm64(As, B, ms, n, k, dtype, limit)
            what = (name, limit)
            assert np.array_equal(rpC, ref[0].astype(np.int64)) and np.array_equal(ciC, ref[1]), what
            assert np.array_equal(vC.view(np.uint8), ref[2].view(np.uint8)), what
            assert nw == expected_windows(As, B, limit) and nw > 1, what


def test_numeric_rerun_with_new_values(emu):
    name, A, B, m, n, k = cases(np.float64)[3]
    A64, B64 = wide(A), wide(B)
    limit = limits_for(A, B)[1]
    p = Plan(limit)
    rpC = np.zeros(m + 1, dtype=np.int64)
    rc, nnz, _ = symbolic64_rc(p, A64, B64, m, n, k, rpC)
    E.ok(rc)
    assert p.windows() > 3
    for scale in (1.0, -2.5):
        A2, B2 = (A[0], A[1], A[2] * scale), (B[0], B[1], B[2] + scale)
        ref = E.spgemm(A2, B2, m, n, k, np.float64)
        ciC, vC = np.full(nnz, -1, dtype=np.int32), np.full(nnz, np.nan)
        E.ok(numeric_rc(p, wide(A2), wide(B2), m, n, k, rpC, ciC, vC, 64))
        assert np.array_equal(ciC, ref[1]) and np.array_equal(vC.view(np.uint64), ref[2].view(np.uint64))
    # the same product again is idempotent, and keeps the cut
    rpC2 = np.full(m + 1, -7, dtype=np.int64)
    rc, nnz2, _ = symbolic64_rc(p, A64, B64, m, n, k, rpC2)
    assert rc == OK and nnz2 == nnz and np.array_equal(rpC2, rpC) and p.windows() == expected_windows(A, B, limit)
    p.close()


def test_degenerate_shapes(emu):
    rng = np.random.default_rng(1)
    A = (np.array([0, 2, 2, 3], np.int64), np.array([0, 1, 1], np.int32), rng.uniform(1, 2, 3))
    B = (np.array([0, 1, 3], np.int64), np.array([2, 0, 3], np.int32), rng.uniform(1, 2, 3))
    Bempty = (np.zeros(3, np.int64), np.zeros(0, np.int32), np.zeros(0))
    Aempty = (np.zeros(4, np.int64), np.zeros(0, np.int32), np.zeros(0))
    for Am, Bm, m, n, k in ((A, B, 0, 2, 4), (A, B, 3, 0, 4), (A, B, 3, 2, 0), (Aempty, B, 3, 2, 4), (A, Bempty, 3, 2, 4)):
        p = Plan(8)
        rpC = np.full(m + 1, -7, dtype=np.int64)
        rc, nnz, mx = symbolic64_rc(p, Am, Bm, m, n, k, rpC)
        assert (rc, nnz, mx) == (OK, 0, 0) and np.all(rpC == 0) and p.windows() == 0, (m, n, k)
        assert numeric_rc(p, Am, Bm, m, n, k, rpC, np.zeros(0, np.int32), np.zeros(0), 64) == OK
        p.close()


def test_overflow(emu):
    name, A, B, m, n, k = cases(np.float64)[0]  # 32 per row: 1024 products per row
    A64, B64 = wide(A), wide(B)
    # a row alone above the limit by its products
    for limit in (1023,):
        p = Plan(limit)
        rc, _, _ = symbolic64_rc(p, A64, B64, m, n, k, np.zeros(m + 1, np.int64))
        assert rc == ERR_OVERFLOW and "window limit" in E.lib().b200sp_last_error_string().decode()
        assert p.windows() == 0
        # numeric after a failed symbolic is a state error
        assert numeric_rc(p, A64, B64, m, n, k, np.zeros(m + 1, np.int64), np.zeros(1, np.int32), np.zeros(1), 64) == ERR_STATE
        p.close()
    # a row alone above the limit by its entries of A only: they point at empty rows of B (no products at all)
    Bz = (np.array([0, 0, 0, 2, 2], np.int64), np.array([0, 1], np.int32), np.ones(2))
    Az = (np.array([0, 40, 41], np.int64), np.concatenate([np.full(40, 1), [2]]).astype(np.int32), np.ones(41))
    p = Plan(39)
    rpC = np.zeros(3, np.int64)
    assert symbolic64_rc(p, Az, Bz, 2, 4, 2, rpC)[0] == ERR_OVERFLOW
    assert "row 0 holds more than 39 entries or products" in E.lib().b200sp_last_error_string().decode()
    p.close()
    p = Plan(40)
    assert symbolic64_rc(p, Az, Bz, 2, 4, 2, rpC) == (OK, 2, 2) and list(rpC) == [0, 0, 2] and p.windows() == 2
    p.close()
    # more than 4096 windows
    p = Plan(1024)
    big = (np.concatenate([A64[0], A64[0][1:] + A64[0][-1]]), np.concatenate([A[1], A[1]]), np.concatenate([A[2], A[2]]))
    assert symbolic64_rc(p, big, B64, 2 * m, n, k, np.zeros(2 * m + 1, np.int64))[0] == ERR_OVERFLOW
    assert "windows" in E.lib().b200sp_last_error_string().decode()
    p.close()
    # nnz(B) past the 32-bit limit: read from row_ptr_B[n] before anything else of B
    p = Plan()
    Bhuge = (np.array([0, 2 ** 31], np.int64), np.zeros(1, np.int32), np.zeros(1))
    Aone = (np.array([0, 1], np.int64), np.zeros(1, np.int32), np.ones(1))
    assert symbolic64_rc(p, Aone, Bhuge, 1, 1, 1, np.zeros(2, np.int64))[0] == ERR_OVERFLOW
    assert "nnz(B)" in E.lib().b200sp_last_error_string().decode()
    p.close()


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_windows_cut_by_entries_of_a(emu, dtype):
    """Rows whose entries of A mostly point at empty rows of B: few products, many entries, so the entries bound alone
    decides where the windows end (a cut by products alone would make one window)."""
    rng = np.random.default_rng(9)
    m, n, k = 400, 300, 500
    lensB = np.where(np.arange(n) % 100 == 0, rng.integers(1, 6, n), 0)
    ciB = np.concatenate([rng.choice(k, l, replace=False) for l in lensB]).astype(np.int32)
    Bm = (np.concatenate([[0], np.cumsum(lensB)]).astype(np.int32), ciB, rng.uniform(1, 2, len(ciB)).astype(dtype))
    lensA = rng.integers(20, 60, m)
    rpA = np.concatenate([[0], np.cumsum(lensA)]).astype(np.int32)
    ciA = np.concatenate([rng.choice(n, l, replace=False) for l in lensA]).astype(np.int32)
    Am = (rpA, ciA, rng.uniform(1, 2, len(ciA)).astype(dtype))
    total = int(row_products(Am, Bm).sum())
    limit = max(total + 1, int(lensA.max()))
    assert int(lensA.sum()) > 20 * limit  # the entries bound cuts
    ref = E.spgemm(Am, Bm, m, n, k, dtype)
    rpC, ciC, vC, mx, nw = spgemm64(Am, Bm, m, n, k, dtype, limit)
    assert nw == expected_windows(Am, Bm, limit) and nw > 20
    assert np.array_equal(rpC, ref[0].astype(np.int64)) and np.array_equal(ciC, ref[1])
    assert np.array_equal(vC.view(np.uint8), ref[2].view(np.uint8))


def test_plan_kind_state_errors(emu):
    import ctypes as Cc

    L = E.lib()
    name, A, B, m, n, k = cases(np.float64)[2]
    A64, B64 = wide(A), wide(B)
    ref = E.spgemm(A, B, m, n, k, np.float64)
    nnz = len(ref[1])
    ciC, vC = np.zeros(nnz, np.int32), np.zeros(nnz)
    # 64-bit numeric without a symbolic, and after a 32-bit symbolic
    p = Plan()
    assert numeric_rc(p, A64, B64, m, n, k, np.zeros(m + 1, np.int64), ciC, vC, 64) == ERR_STATE
    rp32 = np.zeros(m + 1, np.int32)
    E.ok(L.b200sp_spgemm_symbolic_i32(p.h, None, m, n, k, E.ptr(A[0]), E.ptr(A[1]), E.ptr(B[0]), E.ptr(B[1]), E.ptr(rp32),
                                      Cc.byref(Cc.c_int64()), Cc.byref(Cc.c_int())))
    assert numeric_rc(p, A64, B64, m, n, k, rp32.astype(np.int64), ciC, vC, 64) == ERR_STATE
    assert "32-bit" in L.b200sp_last_error_string().decode()
    assert symbolic64_rc(p, A64, B64, m, n, k, np.zeros(m + 1, np.int64))[0] == ERR_STATE
    assert numeric_rc(p, A, B, m, n, k, rp32, ciC, vC, 32) == OK  # the 32-bit product is untouched
    p.close()
    # the other direction: every 32-bit entry refuses a plan whose symbolic had 64-bit offsets
    p = Plan(300)
    rp64 = np.zeros(m + 1, np.int64)
    assert symbolic64_rc(p, A64, B64, m, n, k, rp64)[0] == OK
    rp32 = rp64.astype(np.int32)
    assert numeric_rc(p, A, B, m, n, k, rp32, ciC, vC, 32) == ERR_STATE
    assert numeric_rc(p, A, B, m, n, k, rp32, ciC, vC.astype(np.float32), 32) == ERR_STATE
    dinv = np.ones(m)
    assert L.b200sp_spgemm_jacobi_f64_i32(p.h, None, m, n, k, E.ptr(A[0]), E.ptr(A[1]), E.ptr(A[2]), E.ptr(B[0]), E.ptr(B[1]),
                                          E.ptr(B[2]), E.ptr(rp32), E.ptr(ciC), E.ptr(vC), 1.0, E.ptr(dinv)) == ERR_STATE
    assert "64-bit" in L.b200sp_last_error_string().decode()
    assert L.b200sp_bspgemm_numeric_f64_i32(p.h, None, m, n, k, 1, E.ptr(A[0]), E.ptr(A[1]), E.ptr(A[2]), E.ptr(B[0]),
                                            E.ptr(B[1]), E.ptr(B[2]), E.ptr(rp32), E.ptr(ciC), E.ptr(vC)) == ERR_STATE
    assert L.b200sp_bspgemm_numeric_f64_i32(p.h, None, m, n, k, 2, E.ptr(A[0]), E.ptr(A[1]), E.ptr(A[2]), E.ptr(B[0]),
                                            E.ptr(B[1]), E.ptr(B[2]), E.ptr(rp32), E.ptr(ciC), E.ptr(vC)) == ERR_STATE
    assert "64-bit" in L.b200sp_last_error_string().decode()
    assert L.b200sp_spgemm_symbolic_i32(p.h, None, m, n, k, E.ptr(A[0]), E.ptr(A[1]), E.ptr(B[0]), E.ptr(B[1]), E.ptr(rp32),
                                        Cc.byref(Cc.c_int64()), Cc.byref(Cc.c_int())) == ERR_STATE
    # one handle, one product
    assert symbolic64_rc(p, A64, B64, m, n, k - 1, rp64)[0] == ERR_STATE
    assert numeric_rc(p, A64, B64, m, n, k, rp64, ciC, vC, 64) == OK
    assert np.array_equal(ciC, ref[1]) and np.array_equal(vC, ref[2])
    p.close()


def test_argument_checks(emu):
    L = E.lib()
    null = C.c_void_p(0)
    p = Plan()
    assert L.b200sp_spgemm_symbolic_i64(null, None, 1, 1, 1, null, null, null, null, null, None, None) == ERR_INVALID
    assert L.b200sp_spgemm_symbolic_i64(p.h, None, -1, 1, 1, null, null, null, null, E.ptr(np.zeros(1, np.int64)), None,
                                        None) == ERR_INVALID
    assert L.b200sp_spgemm_symbolic_i64(p.h, None, 1, 1, 1, null, null, null, null, null, None, None) == ERR_INVALID
    for bad in (7, 2 ** 31):
        assert L.b200sp_spgemm_plan_set_window(p.h, C.c_int64(bad)) == ERR_INVALID
    assert L.b200sp_spgemm_plan_windows(null) == 0
    p.close()
