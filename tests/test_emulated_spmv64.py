"""SpMV on 64-bit offsets (spmv64.cu) executed on the CPU (tools/emu): the row windows, their relative 32-bit row maps and the
narrowed columns must reproduce, bit for bit in the non-transposed modes, what the 32-bit entry points give on the same
matrix (which the other emulated tests hold against the oracle), and the oracle's own answer within the unit test's
tolerance law (sparse/unit_test/Test_Sparse_spmv.hpp:120-150).  The window limit is lowered so that small matrices need many
windows; the production limit (2^31 - 65537 entries) cannot be reached in a test."""
import numpy as np
import pytest

import emu_lib as E


@pytest.fixture(scope="module")
def emu():
    return E.lib()


def random_crs(m, n, mean, seed, long_rows=0, empty_frac=0.1):
    rng = np.random.default_rng(seed)
    lens = rng.poisson(mean, m).astype(np.int64)
    lens[rng.random(m) < empty_frac] = 0
    for r in rng.integers(0, m, long_rows):
        lens[r] = rng.integers(600, 1500)
    lens = np.minimum(lens, n)
    rp = np.zeros(m + 1, np.int64)
    np.cumsum(lens, out=rp[1:])
    ci = np.concatenate([np.sort(rng.choice(n, k, replace=False)) for k in lens] + [np.zeros(0, np.int64)]).astype(np.int32)
    v = rng.uniform(-1, 1, len(ci))
    return rp, ci, v


def expected_windows(rp, limit):
    """The greedy cut the library documents: consecutive rows, each window ending at the last row whose offset lies within
    `limit` entries of the window's base, its first offset rounded down to a multiple of 4."""
    m, R, count = len(rp) - 1, 0, 0
    while R < m:
        end = np.searchsorted(rp, (int(rp[R]) & ~3) + limit, "right") - 1
        assert end > R
        count += 1
        R = end
    return count


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("long_rows", [0, 4])
def test_window_count_of_the_aligned_cut(emu, seed, long_rows):
    """Limits from the longest row plus the base's rounding upwards, on row maps with empty rows (and rows of 600 to 1500
    entries): the window count is the greedy cut's."""
    m, n = 3000, 2000
    rp, ci, v = random_crs(m, n, 6.0, seed=seed, long_rows=long_rows, empty_frac=0.3)
    x, y = np.ones(n), np.zeros(m)
    lo = int(np.diff(rp).max()) + 3
    for limit in (lo, lo + 1, lo + 2, 2 * lo, len(ci) // 7):
        p = E.Spmv64Plan(window=limit)
        E.spmv64(p, "N", m, n, rp, ci, v, x, y, 1.0, 0.0)
        assert p.windows() == expected_windows(rp, limit), limit
        p.close()


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("col_bits", [32, 64])
@pytest.mark.parametrize("window", [None, 40000, 2000])
def test_matches_the_32_bit_path(emu, oracle, dtype, col_bits, window):
    m, n = 6000, 5000
    rp64, ci32, v = random_crs(m, n, 9.0, seed=11, long_rows=3)
    v = v.astype(dtype)
    ci = ci32.astype(np.int64) if col_bits == 64 else ci32
    rp32 = rp64.astype(np.int32)
    rng = np.random.default_rng(5)
    tol = 1e-13 if dtype == np.float64 else 1e-5
    for mode, alpha, beta in (("N", 1.0, 0.0), ("N", -0.7, 1.3), ("C", 2.0, 1.0), ("T", 1.0, 0.0), ("H", 0.5, -2.0)):
        trans = mode in "TH"
        x = rng.uniform(-1, 1, m if trans else n).astype(dtype)
        y0 = rng.uniform(-1, 1, n if trans else m).astype(dtype)
        if beta == 0.0:
            y0[::7] = np.nan  # beta == 0 never reads y
        p32, p64 = E.SpmvPlan(), E.Spmv64Plan(window=window)
        y32, y64 = y0.copy(), y0.copy()
        for _ in range(4):  # through the plan's self-tuning phases (tile, tile timed, vector timed, choice)
            y32[:], y64[:] = y0, y0
            E.spmv(p32, mode, m, n, rp32, ci32, v, x, y32, alpha, beta)
            E.spmv64(p64, mode, m, n, rp64, ci, v, x, y64, alpha, beta)
            if not trans:
                # same lanes per row, same order: equal bits -- except that a window of fewer than 32768 entries (in
                # production only the last one can be that small) sums its rows of more than 512 entries with the row's
                # lanes instead of a CTA
                short = np.diff(rp64) <= 512
                assert np.array_equal(y32[short], y64[short]), (mode, p32.kernel(), p64.kernel())
                assert np.allclose(y32, y64, rtol=0, atol=tol * 50)
                if window is None:
                    assert np.array_equal(y32, y64)
            else:  # atomic scatters: same sums, another order
                assert np.allclose(y32, y64, rtol=0, atol=tol * 50)
        if window is None:
            assert p64.windows() == 1
        else:
            assert p64.windows() >= len(ci) // window
        assert "window" in p64.kernel()
        # and the oracle (CPU restatement of the reference) within the reference's own tolerance law
        yo = np.where(np.isnan(y0), 0, y0).astype(dtype) if beta == 0.0 else y0.copy()
        if trans:
            import scipy.sparse as sps

            A = sps.csr_matrix((v.astype(np.float64), ci32, rp32), shape=(m, n))
            yo = (beta * yo.astype(np.float64) + alpha * (A.T @ x.astype(np.float64))).astype(dtype)
        else:
            oracle.spmv_serial(rp32, ci32, v, x, yo, alpha, beta)
        assert np.max(np.abs(y64.astype(np.float64) - yo.astype(np.float64))) <= tol * 100 * max(1.0, np.max(np.abs(yo)))
        p32.close()
        p64.close()


def test_window_boundaries_and_corner_cases(emu, oracle):
    rng = np.random.default_rng(1)
    # every row exactly 7 entries: window bases fall on all residues mod 4
    m, n = 900, 64
    rp = np.arange(m + 1, dtype=np.int64) * 7
    ci = np.concatenate([np.sort(rng.choice(n, 7, replace=False)) for _ in range(m)]).astype(np.int64)
    v = rng.uniform(-1, 1, len(ci))
    x = rng.uniform(-1, 1, n)
    y = np.full(m, np.nan)
    p = E.Spmv64Plan(window=53)  # 7 rows per window
    E.spmv64(p, "N", m, n, rp, ci, v, x, y, 1.0, 0.0)
    assert p.windows() == (m + 6) // 7
    yo = np.zeros(m)
    oracle.spmv_serial(rp.astype(np.int32), ci.astype(np.int32), v, x, yo, 1.0, 0.0)
    assert np.allclose(y, yo, rtol=0, atol=1e-13)
    # same plan, same pointers: no second analysis (windows kept); new window size: analysed again
    E.spmv64(p, "N", m, n, rp, ci, v, x, y, 1.0, 0.0)
    assert E.lib().b200sp_spmv64_plan_set_window(p.h, 700) == 0
    E.spmv64(p, "N", m, n, rp, ci, v, x, y, 1.0, 0.0)
    assert p.windows() == (m + 99) // 100 and np.allclose(y, yo, rtol=0, atol=1e-13)
    # a row longer than the window: refused, nothing written
    assert E.lib().b200sp_spmv64_plan_set_window(p.h, 8) == 0
    y[:] = 5.0
    assert E.spmv64_rc(p, "N", m, n, rp, ci, v, x, y, 1.0, 0.0) == 4  # B200SP_ERR_OVERFLOW
    assert b"window" in E.lib().b200sp_last_error_string() and np.all(y == 5.0)
    # a column index that does not fit 31 bits
    assert E.lib().b200sp_spmv64_plan_set_window(p.h, 700) == 0
    bad = ci.copy()
    bad[100] = 2**31
    assert E.spmv64_rc(p, "N", m, n, rp, bad, v, x, y, 1.0, 0.0) == 4
    # the plan still works afterwards
    E.spmv64(p, "N", m, n, rp, ci, v, x, y, 1.0, 0.0)
    assert np.allclose(y, yo, rtol=0, atol=1e-13)
    # leading / trailing empty rows, an empty matrix, alpha == 0, bad arguments
    rp2 = np.concatenate([np.zeros(50, np.int64), rp, np.full(30, rp[-1], np.int64)])
    m2 = len(rp2) - 1
    y2 = np.full(m2, np.nan)
    E.spmv64(p, "N", m2, n, rp2, ci, v, x, y2, 1.0, 0.0)
    assert np.all(y2[:50] == 0) and np.all(y2[-30:] == 0) and np.allclose(y2[50:50 + m], yo, rtol=0, atol=1e-13)
    ye = np.array([1.0, 2.0, 3.0])
    E.spmv64(p, "N", 3, 4, np.zeros(4, np.int64), np.zeros(0, np.int64), np.zeros(0), np.ones(4), ye, 1.0, 2.0)
    assert np.array_equal(ye, [2.0, 4.0, 6.0])
    y3 = yo.copy()
    E.spmv64(p, "N", m, n, rp, ci, v, x, y3, 0.0, -1.0)
    assert np.array_equal(y3, -yo)
    assert E.spmv64_rc(p, "X", m, n, rp, ci, v, x, y, 1.0, 0.0) == 1
    assert E.spmv64_rc(p, "N", 2**31 + 5, n, rp, ci, v, x, y, 1.0, 0.0) == 4
    assert E.spmv64_rc(p, "N", -1, n, rp, ci, v, x, y, 1.0, 0.0) == 1
    none = E.Spmv64Plan()
    none.close()
    assert E.spmv64_rc(none, "N", m, n, rp, ci, v, x, y, 1.0, 0.0) == 1  # a plan is required
    assert E.lib().b200sp_spmv64_plan_set_window(p.h, 3) == 1
    p.close()


def test_transposed_accumulates_over_windows(emu):
    import scipy.sparse as sps

    m, n = 3000, 800
    rp, ci, v = random_crs(m, n, 12.0, seed=4)
    A = sps.csr_matrix((v, ci, rp.astype(np.int32)), shape=(m, n))
    rng = np.random.default_rng(2)
    x = rng.uniform(-1, 1, m)
    y0 = rng.uniform(-1, 1, n)
    p = E.Spmv64Plan(window=1500)
    for beta in (0.0, 1.0, -0.25):
        y = y0.copy()
        E.spmv64(p, "T", m, n, rp, ci, v, x, y, 1.5, beta)
        assert p.windows() > 10
        assert np.allclose(y, beta * y0 + 1.5 * (A.T @ x), rtol=0, atol=1e-12)
    p.close()


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("layouts", ["CC", "FF", "CF"])
def test_rank2_over_windows(emu, dtype, layouts):
    """Multivectors: every window shifts the rows of Y (N / C) or of X (T / H) by its first row, in either layout; equal
    bits to the 32-bit entry point in the non-transposed modes."""
    m, n, k = 2500, 1800, 5
    rp64, ci32, v = random_crs(m, n, 10.0, seed=21)
    v = v.astype(dtype)
    rp32 = rp64.astype(np.int32)
    rng = np.random.default_rng(9)
    tol = 1e-12 if dtype == np.float64 else 2e-5
    for mode, alpha, beta in (("N", 1.0, 0.0), ("N", 0.5, -1.5), ("T", 2.0, 0.0), ("T", -1.0, 1.0)):
        trans = mode == "T"
        xr, yr = (m, n) if trans else (n, m)
        X = np.asarray(rng.uniform(-1, 1, (xr, k)).astype(dtype), order=layouts[0])
        Y0 = np.asarray(rng.uniform(-1, 1, (yr, k)).astype(dtype), order=layouts[1])
        p32, p64 = E.SpmvPlan(), E.Spmv64Plan(window=3000)
        Y32, Y64 = Y0.copy(order="K"), Y0.copy(order="K")
        E.spmm(p32, mode, m, n, rp32, ci32, v, X, Y32, alpha, beta)
        E.spmm64(p64, mode, m, n, rp64, ci32.astype(np.int64), v, X, Y64, alpha, beta)
        assert p64.windows() >= 8
        if trans:
            assert np.allclose(Y32, Y64, rtol=0, atol=tol * 20)
        else:
            assert np.array_equal(Y32, Y64)
        p32.close()
        p64.close()
