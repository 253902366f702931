"""The exact rank-2 SpMV reference and its per-entry bound (tests/exact_ref.py): the reference is exact enough, the bound
holds for a correct implementation (the oracle's, in the kernel's precision) and fails for subtly wrong ones."""
from fractions import Fraction

import numpy as np
import pytest

import exact_ref as R
import spmm_cases

DTYPES = [np.float64, np.float32]


def _oracle_mv(oracle, rp, ci, v, ncols, X, Y0, alpha, beta, trans):
    Y = Y0.copy()
    if trans:
        return oracle.spmv_mv_transpose(rp, ci, v, ncols, X, Y, alpha, beta)
    if beta == 0:
        Y = np.zeros_like(Y0)  # the oracle's functor scales a NaN by 0; the library overwrites
    return oracle.spmv_mv(rp, ci, v, ncols, X, Y, alpha, beta)


def _random_case(rng, dtype):
    m, n = int(rng.integers(1, 60)), int(rng.integers(1, 60))
    lens = rng.integers(0, 3 * n, m) * (rng.random(m) < 0.85)
    rp, ci, v = spmm_cases.from_lengths(lens, n, rng, dtype)
    for i in np.flatnonzero(rng.random(m) < 0.2):  # cancelling rows: +a and -a at one column, a up to 2^12
        s, e = rp[i], rp[i + 1]
        h = (e - s) // 2
        if h:
            ci[s + h:s + 2 * h] = ci[s:s + h]
            v[s:s + h] *= dtype(4096.0)
            v[s + h:s + 2 * h] = -v[s:s + h]
    return rp, ci, v, n


def test_exact_matches_rational_arithmetic():
    """The reference against Fractions on small cases: within its own stated error (len*2^-53 resp. 2^-64 relative)."""
    rng = np.random.default_rng(3)
    for dtype in DTYPES:
        for trans in (False, True):
            rp, ci, v, n = _random_case(rng, dtype)
            m = len(rp) - 1
            rows_out, rows_in = (n, m) if trans else (m, n)
            X = spmm_cases.dense_operands(rng, rows_in, 3, dtype)
            Y0 = spmm_cases.dense_operands(rng, rows_out, 3, dtype)
            alpha, beta = -1.5, 0.25
            got = R.spmm_exact(rp, ci, v, X, Y0, alpha, beta, trans)
            assert got.dtype == R.wide(dtype)
            scale = R.spmm_scale(rp, ci, v, X, Y0, alpha, beta, trans)
            lens = R.op_row_lengths(rp, ci, rows_out, trans)
            arow = np.repeat(np.arange(m), np.diff(rp))
            orow, xrow = (ci, arow) if trans else (arow, ci)
            ex = [[Fraction(beta) * Fraction(float(Y0[i, c])) for c in range(3)] for i in range(rows_out)]
            for e in range(len(ci)):
                for c in range(3):
                    ex[orow[e]][c] += Fraction(alpha) * Fraction(float(v[e])) * Fraction(float(X[xrow[e], c]))
            for i in range(rows_out):
                for c in range(3):
                    err = abs(Fraction(*got[i, c].as_integer_ratio()) - ex[i][c])
                    assert err <= float(R.gamma(lens[i] + 2, R.unit_roundoff(R.wide(dtype)))) * scale[i, c], (dtype, trans, i, c)


def test_exact_special_scalars():
    rp, ci, v, n = spmm_cases.small(1, np.float64)
    m = len(rp) - 1
    X = np.full((n, 2), np.nan)
    Y0 = np.full((m, 2), 3.0)
    assert np.array_equal(R.spmm_exact(rp, ci, v, X, Y0, 0.0, 2.5), np.full((m, 2), 7.5))  # X never read
    Y0[::3] = np.nan
    X = np.ones((n, 2))
    out = R.spmm_exact(rp, ci, v, X, Y0, 1.0, 0.0)  # Y0 ignored
    assert np.isfinite(out).all()
    assert not R.spmm_exact(rp, ci, v, X, Y0, 0.0, 0.0).any()
    # empty rows give 0 (np.add.reduceat would repeat the next element)
    empty = np.diff(rp) == 0
    assert empty.any() and not out[empty].any()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("trans", [False, True])
def test_bound_holds_for_the_oracle(oracle, dtype, trans):
    """A few hundred random products in the kernel's own precision, mixed signs, cancelling rows: all within the bound."""
    rng = np.random.default_rng(20 + trans)
    worst = 0.0
    for _ in range(150):
        rp, ci, v, n = _random_case(rng, dtype)
        m = len(rp) - 1
        k = int(rng.integers(1, 6))
        rows_out, rows_in = (n, m) if trans else (m, n)
        X = spmm_cases.dense_operands(rng, rows_in, k, dtype)
        Y0 = spmm_cases.dense_operands(rng, rows_out, k, dtype)
        alpha, beta = [(1.0, 0.0), (-1.0, 1.0), (2.5, -0.5), (0.0, 2.5), (1.0, 1.0), (0.0, 0.0)][int(rng.integers(0, 6))]
        got = _oracle_mv(oracle, rp, ci, v, n, X, Y0, alpha, beta, trans)
        exact = R.spmm_exact(rp, ci, v, X, Y0, alpha, beta, trans)
        bound = R.spmm_bound(rp, ci, v, X, Y0, alpha, beta, trans)
        R.assert_within(got, exact, bound, f"oracle {dtype.__name__} trans={trans}")
        with np.errstate(invalid="ignore", divide="ignore"):
            r = np.abs(got.astype(exact.dtype) - exact) / bound
        worst = max(worst, float(np.nanmax(np.where(bound > 0, r, 0))))
    assert worst > 0.01  # the bound is not vacuous either: real rounding errors use a visible part of it


@pytest.mark.parametrize("trans", [False, True])
def test_bound_catches_a_dropped_term(oracle, trans):
    """Removing one entry whose |alpha*a*x| exceeds 64u of its row's scale, in a row of at most 12 entries."""
    rng = np.random.default_rng(7)
    caught = 0
    for dtype in DTYPES:
        u = R.unit_roundoff(dtype)
        for _ in range(80):
            rp, ci, v, n = _random_case(rng, dtype)
            m = len(rp) - 1
            rows_out, rows_in = (n, m) if trans else (m, n)
            X = spmm_cases.dense_operands(rng, rows_in, 2, dtype)
            Y0 = spmm_cases.dense_operands(rng, rows_out, 2, dtype)
            alpha, beta = 1.5, -0.5
            lens = R.op_row_lengths(rp, ci, rows_out, trans)
            scale = R.spmm_scale(rp, ci, v, X, Y0, alpha, beta, trans)
            arow = np.repeat(np.arange(m), np.diff(rp))
            orow, xrow = (ci, arow) if trans else (arow, ci)
            term = np.abs(alpha * v.astype(np.float64) * X[xrow, 0].astype(np.float64))
            ok = (lens[orow] <= 12) & (term > 64 * u * scale[orow, 0])
            if not ok.any():
                continue
            e = int(np.flatnonzero(ok)[0])
            keep = np.ones(len(ci), bool)
            keep[e] = False
            rp2 = rp.copy()
            rp2[arow[e] + 1:] -= 1
            got = _oracle_mv(oracle, rp2, ci[keep], v[keep], n, X, Y0, alpha, beta, trans)
            with pytest.raises(AssertionError, match=f"row {orow[e]}, column 0"):
                R.assert_within(got, R.spmm_exact(rp, ci, v, X, Y0, alpha, beta, trans), R.spmm_bound(rp, ci, v, X, Y0, alpha, beta, trans), "dropped")
            caught += 1
    assert caught >= 20


def test_bound_catches_fp32_accumulation_of_fp64_data(oracle):
    """One row of an fp64 product computed from fp32-rounded data."""
    rng = np.random.default_rng(9)
    for _ in range(20):
        rp, ci, v, n = _random_case(rng, np.float64)
        m = len(rp) - 1
        X = spmm_cases.dense_operands(rng, n, 2, np.float64) * (1 + rng.random((n, 2)))
        Y0 = spmm_cases.dense_operands(rng, m, 2, np.float64)
        got = _oracle_mv(oracle, rp, ci, v, n, X, Y0, 1.0, 1.0, False)
        got32 = _oracle_mv(oracle, rp, ci, v.astype(np.float32), n, X.astype(np.float32), Y0.astype(np.float32), 1.0, 1.0, False)
        i = int(np.argmax(np.diff(rp)))
        got[i] = got32[i]
        with pytest.raises(AssertionError, match=f"row {i}, "):
            R.assert_within(got, R.spmm_exact(rp, ci, v, X, Y0, 1.0, 1.0), R.spmm_bound(rp, ci, v, X, Y0, 1.0, 1.0), "fp32 row")


@pytest.mark.parametrize("dtype", DTYPES)
def test_bound_catches_swapped_columns(oracle, dtype):
    rng = np.random.default_rng(11)
    rp, ci, v, n = spmm_cases.small(2, dtype)
    m = len(rp) - 1
    X = spmm_cases.dense_operands(rng, n, 4, dtype)
    Y0 = spmm_cases.dense_operands(rng, m, 4, dtype)
    got = _oracle_mv(oracle, rp, ci, v, n, np.ascontiguousarray(X[:, [0, 2, 1, 3]]), Y0, 1.0, 0.0, False)
    with pytest.raises(AssertionError, match="column 1"):
        R.assert_within(got, R.spmm_exact(rp, ci, v, X, Y0, 1.0, 0.0), R.spmm_bound(rp, ci, v, X, Y0, 1.0, 0.0), "swapped")


def _bsr_dense(bs, mb, nb, rp, ci, v):
    D = np.zeros((mb * bs, nb * bs), dtype=np.float64)
    blocks = v.reshape(-1, bs, bs)
    for br in range(mb):
        for k in range(rp[br], rp[br + 1]):
            D[br * bs:(br + 1) * bs, ci[k] * bs:(ci[k] + 1) * bs] += blocks[k]
    return D


@pytest.mark.parametrize("bs", [1, 2, 3, 7])
def test_bsr_to_point_crs_matches_a_dense_product(bs):
    """The expansion against a dense matrix assembled block by block (row-major blocks), rank 1 and 2, N and T; point rows
    hold bs * (block degree) entries; an empty block row gives empty point rows."""
    from bsr_cases import bsr_random

    rng = np.random.default_rng(bs)
    mb, nb = 9, 11
    rp, ci, v = bsr_random(bs, mb, nb, seed=bs, min_blocks=0, max_blocks=5, sort=False)
    v = spmm_cases._values(rng, len(v), np.float64)
    prp, pci, pv = R.bsr_to_point_crs(bs, rp, ci, v)
    assert np.array_equal(np.diff(prp), np.repeat(np.diff(rp) * bs, bs))
    D = _bsr_dense(bs, mb, nb, rp, ci, v)
    P = np.zeros_like(D)
    np.add.at(P, (np.repeat(np.arange(mb * bs), np.diff(prp)), pci), pv)
    assert np.array_equal(P, D)
    for trans in (False, True):
        rows_out, rows_in = (nb * bs, mb * bs) if trans else (mb * bs, nb * bs)
        for X in (spmm_cases.dense_operands(rng, rows_in, 3, np.float64), spmm_cases.dense_operands(rng, rows_in, 1, np.float64)[:, 0]):
            Y0 = np.ones((rows_out,) + X.shape[1:])
            got = R.spmm_exact(prp, pci, pv, X, Y0, 1.5, -0.5, trans)
            ref = 1.5 * ((D.T if trans else D) @ X) - 0.5 * Y0
            R.assert_within(ref, got.reshape(ref.shape), R.spmm_bound(prp, pci, pv, X, Y0, 1.5, -0.5, trans), f"bs={bs} trans={trans}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_bound_rejects_a_transposed_block(dtype):
    """A kernel that reads a block column-major instead of row-major: caught in the point rows of that block."""
    from bsr_cases import bsr_random

    bs, mb, nb = 4, 12, 10
    rng = np.random.default_rng(5)
    rp, ci, v = bsr_random(bs, mb, nb, seed=5, min_blocks=1, max_blocks=4, sort=False)
    v = spmm_cases._values(rng, len(v), dtype)
    x = spmm_cases.dense_operands(rng, nb * bs, 1, dtype)[:, 0]
    y0 = spmm_cases.dense_operands(rng, mb * bs, 1, dtype)[:, 0]
    prp, pci, pv = R.bsr_to_point_crs(bs, rp, ci, v)
    exact = R.spmm_exact(prp, pci, pv, x, y0, 1.0, 1.0)
    bound = R.spmm_bound(prp, pci, pv, x, y0, 1.0, 1.0)
    good = (_bsr_dense(bs, mb, nb, rp, ci, v.astype(np.float64)) @ x.astype(np.float64) + y0).astype(dtype)
    R.assert_within(good, exact, bound, "row-major blocks")
    vt = v.reshape(-1, bs, bs).copy()
    k = int(rp[3])  # the first block of block row 3
    vt[k] = vt[k].T
    bad = (_bsr_dense(bs, mb, nb, rp, ci, vt.reshape(-1).astype(np.float64)) @ x.astype(np.float64) + y0).astype(dtype)
    with pytest.raises(AssertionError, match=r"first at row 1[2-5], column 0"):
        R.assert_within(bad, exact, bound, "one block transposed")


def test_assert_within_special_values():
    exact = np.array([[1.0, np.inf, np.nan]], dtype=np.longdouble)
    bound = np.zeros((1, 3))
    R.assert_within(np.array([[1.0, np.inf, np.nan]]), exact, bound, "ok")
    for bad in ([[np.nan, np.inf, np.nan]], [[1.0, -np.inf, np.nan]], [[1.0, np.inf, 0.0]], [[np.inf, np.inf, np.nan]]):
        with pytest.raises(AssertionError, match="row 0"):
            R.assert_within(np.array(bad), exact, bound, "special")


# ---- SpGEMM and spgemm_jacobi ---------------------------------------------------------------------------------------------
def _spgemm_pair(rng, dtype, square=False, cancel=True):
    """A (m x n) and B (n x k) with distinct sorted columns per row, mixed-sign values; a few pairs of equal B rows that A
    weights +a and -a (entries that cancel exactly)."""
    m, n, k = (int(rng.integers(5, 40)),) * 3 if square else tuple(int(x) for x in rng.integers(5, 40, 3))
    if square:
        n = k = m

    def rows(nr, nc, lo, hi):
        cols = [np.sort(rng.choice(nc, min(nc, int(rng.integers(lo, hi))), replace=False)) for _ in range(nr)]
        rp = np.concatenate([[0], np.cumsum([len(c) for c in cols])]).astype(np.int32)
        ci = np.concatenate(cols).astype(np.int32) if cols else np.zeros(0, np.int32)
        return rp, ci, spmm_cases._values(rng, len(ci), dtype)

    A = rows(m, n, 0, 9)
    B = rows(n, k, 0, 9)
    if square:  # the whole diagonal
        cols = [np.union1d(A[1][A[0][i]:A[0][i + 1]], [i]) for i in range(m)]
        rp = np.concatenate([[0], np.cumsum([len(c) for c in cols])]).astype(np.int32)
        A = (rp, np.concatenate(cols).astype(np.int32), spmm_cases._values(rng, int(rp[-1]), dtype))
    if cancel and n >= 2:  # B row 1 = B row 0; every row of A holding both weights them +a, -a
        rpB, ciB, vB = B
        r0 = (ciB[rpB[0]:rpB[1]], vB[rpB[0]:rpB[1]])
        cols = [r0[0] if j == 1 else ciB[rpB[j]:rpB[j + 1]] for j in range(n)]
        vals = [r0[1] if j == 1 else vB[rpB[j]:rpB[j + 1]] for j in range(n)]
        B = (np.concatenate([[0], np.cumsum([len(c) for c in cols])]).astype(np.int32), np.concatenate(cols).astype(np.int32),
             np.concatenate(vals).astype(dtype))
        rpA, ciA, vA = A
        vA = vA.copy()
        for i in range(m):
            seg = slice(rpA[i], rpA[i + 1])
            c = ciA[seg]
            if 0 in c and 1 in c:
                vA[seg][np.flatnonzero(c == 1)[0]] = -vA[seg][np.flatnonzero(c == 0)[0]]
        A = (rpA, ciA, vA)
    return A, B, m, n, k


def _kernel_like(A, B, dtype, rng, omega=None, dinv=None, mutate=None):
    """C in the data's own precision the way a kernel may compute it: every product rounded, each entry's products added
    in a random order from +0.  mutate(i, j, terms) may change one entry's list of (kind, value) terms."""
    rp, ci, _ = R.spgemm_exact(A, B)
    out = np.zeros(len(ci), dtype=dtype)
    rpA, ciA, vA = A
    rpB, ciB, vB = B
    for i in range(len(rpA) - 1):
        terms = {}
        mult = None if omega is None else dtype(-dtype(omega) * dinv[i])
        for e in range(rpA[i], rpA[i + 1]):
            a = vA[e] if mult is None else dtype(vA[e] * mult)
            for f in range(rpB[ciA[e]], rpB[ciA[e] + 1]):
                terms.setdefault(int(ciB[f]), []).append(("p", dtype(vB[f] * a)))
        if omega is not None:
            for f in range(rpB[i], rpB[i + 1]):
                if int(ciB[f]) in terms:
                    terms[int(ciB[f])].append(("b", vB[f]))
        for q in range(rp[i], rp[i + 1]):
            t = terms[int(ci[q])]
            if mutate is not None:
                t = mutate(i, int(ci[q]), list(t))
            acc = dtype(0)
            for j in rng.permutation(len(t)):
                acc = dtype(acc + t[j][1])
            out[q] = acc
    return out


@pytest.mark.parametrize("dtype", DTYPES)
def test_spgemm_exact_structure_and_values(oracle, dtype):
    """Structure equal to the oracle's SpGEMM and spgemm_jacobi; fp32 values equal scipy's float64 product of the same data
    (every fp32 product is exact in float64)."""
    import scipy.sparse as ss

    rng = np.random.default_rng(31)
    for it in range(40):
        square = it % 2 == 1
        A, B, m, n, k = _spgemm_pair(rng, dtype, square)
        rp, ci, v = R.spgemm_exact(A, B)
        assert v.dtype == R.wide(dtype)
        exp = oracle.spgemm(*A, *B, k)
        assert np.array_equal(exp[0], rp) and np.array_equal(exp[1], ci)
        if dtype == np.float32:
            sA = ss.csr_matrix((A[2].astype(np.float64), A[1], A[0]), shape=(m, n))
            sB = ss.csr_matrix((B[2].astype(np.float64), B[1], B[0]), shape=(n, k))
            S, M = (sA @ sB).toarray(), (abs(sA) @ abs(sB)).toarray()  # scipy's float64 sums, and their scale
            D = np.zeros((m, k))
            D[np.repeat(np.arange(m), np.diff(rp)), ci] = v
            assert (np.abs(D - S) <= 1e-14 * M).all()
        if square:
            dinv = spmm_cases._values(rng, m, dtype)
            rpj, cij, vj = R.jacobi_exact(A, B, 0.7, dinv)
            expj = oracle.spgemm_jacobi(*A, *B, k, dtype(0.7), dinv)
            assert np.array_equal(expj[0], rpj) and np.array_equal(expj[1], cij)


def test_spgemm_exact_keeps_cancelled_entries():
    rng = np.random.default_rng(4)
    A = (np.array([0, 2], np.int32), np.array([0, 1], np.int32), np.array([1.5, -1.5]))
    v = spmm_cases._values(rng, 3, np.float64)
    B = (np.array([0, 3, 6], np.int32), np.array([2, 5, 9, 2, 5, 9], np.int32), np.concatenate([v, v]))
    rp, ci, val = R.spgemm_exact(A, B)
    assert list(rp) == [0, 3] and list(ci) == [2, 5, 9] and not val.any()
    assert (R.spgemm_bound(A, B) > 0).all()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("jacobi", [False, True])
def test_spgemm_bound_holds_and_catches(dtype, jacobi):
    """A kernel-like computation (rounded products, random addition order) stays within the bound; the same with one
    product dropped, one product added twice, one product's sign flipped, or (jacobi) dinv[0] read for every row is
    caught."""
    rng = np.random.default_rng(17 + jacobi)
    caught = dict(drop=0, twice=0, sign=0, dinv0=0)
    for _ in range(25):
        A, B, m, n, k = _spgemm_pair(rng, dtype, square=jacobi)
        omega, dinv = (0.7, spmm_cases._values(rng, m, dtype)) if jacobi else (None, None)
        if jacobi:
            rp, ci, ex, bound = R.jacobi_ref(A, B, omega, dinv)
        else:
            rp, ci, ex, bound = R.spgemm_ref(A, B)
        for _ in range(2):  # re-summed in other orders: within the bound
            R.assert_within(_kernel_like(A, B, dtype, rng, omega, dinv), ex, bound, "kernel-like")
        # the entry with the largest product relative to its scale: a single product there exceeds the bound
        target = {}

        def pick(i, j, t):
            big = max(range(len(t)), key=lambda x: abs(float(t[x][1])))
            if t[big][0] == "p":
                target.setdefault((i, j), (big, abs(float(t[big][1]))))
            return t

        _kernel_like(A, B, dtype, rng, omega, dinv, pick)
        q_of = {(i, int(c)): q for i in range(m) for q, c in zip(range(rp[i], rp[i + 1]), ci[rp[i]:rp[i + 1]])}
        cand = [(ij, b) for ij, (b, mag) in target.items() if mag > 8 * bound[q_of[ij]]]
        if not cand:
            continue
        (ti, tj), big = cand[0]
        muts = {"drop": lambda t: t[:big] + t[big + 1:], "twice": lambda t: t + [t[big]],
                "sign": lambda t: t[:big] + [("p", -t[big][1])] + t[big + 1:]}
        for kind, f in muts.items():
            bad = _kernel_like(A, B, dtype, rng, omega, dinv, lambda i, j, t: f(t) if (i, j) == (ti, tj) else t)
            with pytest.raises(AssertionError, match=f"row {q_of[(ti, tj)]}, "):
                R.assert_within(bad, ex, bound, kind)
            caught[kind] += 1
        if jacobi and m > 1 and not np.all(dinv == dinv[0]):
            bad = _kernel_like(A, B, dtype, rng, omega, np.full(m, dinv[0], dtype))
            with pytest.raises(AssertionError):
                R.assert_within(bad, ex, bound, "dinv[0]")
            caught["dinv0"] += 1
    assert min(caught["drop"], caught["twice"], caught["sign"]) >= 10, caught
    assert not jacobi or caught["dinv0"] >= 10, caught


# ---- Gauss-Seidel -------------------------------------------------------------------------------------------------------
def _greedy_coloring(c):
    """A proper colouring of A + A^T (square part), natural order, as (colors, color_ptr, color_rows)."""
    import gs_cases as G

    P = G._pattern(c)
    P = (P + P.T).tocsr()
    n = c["n"]
    col = np.full(n, -1)
    for i in range(n):
        used = set(col[P.indices[P.indptr[i]:P.indptr[i + 1]]].tolist())
        k = 0
        while k in used:
            k += 1
        col[i] = k
    nc = col.max() + 1
    cptr = np.zeros(nc + 1, np.int32)
    np.cumsum(np.bincount(col, minlength=nc), out=cptr[1:])
    return col, cptr, np.argsort(col, kind="stable").astype(np.int32)


def _gs_case(dtype, cancel=False):
    import gs_cases as G

    c = G.nonsymmetric_case(0.1, ghosts=7)
    v = c["v"].astype(dtype)
    y, x0 = G.vectors(c, dtype, 1)
    if cancel:  # y = A x0 on every third row: the residual of those rows cancels
        n = c["n"]
        Ax = np.zeros(n, dtype)
        rows = np.repeat(np.arange(n), np.diff(c["rp"]))
        np.add.at(Ax, rows, (v.astype(np.float64) * x0[c["ci"]]).astype(dtype))
        y[::3] = Ax[::3]
    return c, v, y, x0


def _dinv(c, v):
    n = c["n"]
    rows = np.repeat(np.arange(n), np.diff(c["rp"]))
    d = rows == c["ci"]
    return (1.0 / np.bincount(rows[d], weights=v[d].astype(np.float64), minlength=n)).astype(v.dtype)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("cancel", [False, True])
def test_gs_sweep_bound_holds_for_the_oracle(oracle, dtype, cancel):
    c, v, y, x0 = _gs_case(dtype, cancel)
    colors, cptr, crows = _greedy_coloring(c)
    for direction in (1, 2):
        x = x0.copy()
        oracle.gs_apply(c["rp"], c["ci"], v, cptr, crows, _dinv(c, v), y, x, False, dtype(0.9), 1, direction)
        ex = R.gs_sweep_exact(c["rp"], c["ci"], v, colors, x0, x, y, 0.9, direction)
        R.assert_within(x[:c["n"]], ex, R.gs_sweep_bound(c["rp"], c["ci"], v, colors, x0, x, y, 0.9, direction), f"direction {direction}")


def test_gs_sweep_bound_rejects_a_dropped_entry_and_a_wrong_colour_order(oracle):
    c, v, y, x0 = _gs_case(np.float64)
    colors, cptr, crows = _greedy_coloring(c)
    n, rp, ci = c["n"], c["rp"], c["ci"]
    rows = np.repeat(np.arange(n), np.diff(rp))
    ex_bd = lambda x, d: (R.gs_sweep_exact(rp, ci, v, colors, x0, x, y, 0.9, d), R.gs_sweep_bound(rp, ci, v, colors, x0, x, y, 0.9, d))
    # a dropped entry: the largest off-diagonal term of a row
    off = np.flatnonzero(rows != ci)
    e = off[np.argmax(np.abs(v[off] * x0[ci[off]]))]
    vd = v.copy()
    vd[e] = 0
    x = x0.copy()
    oracle.gs_apply(rp, ci, vd, cptr, crows, _dinv(c, v), y, x, False, 0.9, 1, 1)
    with pytest.raises(AssertionError):
        R.assert_within(x[:n], *ex_bd(x, 1), "dropped entry")
    # one row swept in the wrong colour order: moved behind every other set of a forward sweep
    sq = (rows != ci) & (ci < n)
    r = next(i for i in range(n) if np.any(sq[rp[i]:rp[i + 1]] & (colors[np.minimum(ci[rp[i]:rp[i + 1]], n - 1)] > colors[i])))
    late = np.concatenate([crows[crows != r], [r]]).astype(np.int32)
    lptr = np.concatenate([cptr, [n]]).astype(np.int32)
    lptr[colors[r] + 1:len(cptr)] = cptr[colors[r] + 1:] - 1  # r's own set ends one row earlier, r alone in a last set
    x = x0.copy()
    oracle.gs_apply(rp, ci, v, lptr, late, _dinv(c, v), y, x, False, 0.9, 1, 1)
    with pytest.raises(AssertionError, match=f"row {r},"):
        R.assert_within(x[:n], *ex_bd(x, 1), "wrong colour order")


GS2_OPTS = [dict(compact=False, inner=2, gamma=0.7, outer=1, omega=0.9, given=False, direction=0, init_zero=False, num_iter=2),
            dict(compact=True, inner=3, gamma=1.0, outer=3, omega=0.9, given=True, direction=2, init_zero=True, num_iter=1),
            dict(compact=True, inner=0, gamma=0.7, outer=1, omega=1.0, given=False, direction=1, init_zero=False, num_iter=1)]


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_gs2_bound_holds_for_the_oracle(oracle, dtype):
    import gs_cases as G

    c = G.gs2_case(0.1)
    v = c["v"].astype(dtype)
    b, x0 = G.vectors(c, dtype, 2)
    b[::4] = 0  # rows whose update is pure cancellation of the current x
    for g in GS2_OPTS:
        dinv = G.given_dinv(c, dtype) if g["given"] else None
        x = x0.copy()
        oracle.gs2_apply(c["rp"], c["ci"], v, c["ncols"], x, b, g["init_zero"], dtype(g["omega"]), g["num_iter"], g["direction"], compact=g["compact"],
                         inner_sweeps=g["inner"], outer_sweeps=g["outer"], gamma=dtype(g["gamma"]), inverse_diagonal=dinv)
        ex, bd = R.gs2_ref(c["rp"], c["ci"], v, c["ncols"], x0, b, g["init_zero"], g["omega"], g["num_iter"], g["direction"], g["compact"], g["inner"],
                           g["outer"], g["gamma"], True, dinv)
        R.assert_within(x, ex, bd, str(g))
    for given, compact, direction in ((False, False, 0), (True, True, 1), (True, False, 2)):
        dinv = G.given_dinv(c, dtype) if given else None
        x = x0.copy()
        oracle.gs2_classic_apply(c["rp"], c["ci"], v, c["ncols"], x, b, False, 2, direction, compact=compact, inverse_diagonal=dinv)
        ex, bd = R.gs2_ref(c["rp"], c["ci"], v, c["ncols"], x0, b, False, 1.0, 2, direction, compact, 0, 1, 1.0, False, dinv)
        R.assert_within(x, ex, bd, f"classic {given} {compact} {direction}")
        z = np.zeros(c["ncols"], dtype)
        oracle.gs2_classic_apply(c["rp"], c["ci"], v, c["ncols"], z, b, True, 1, 1 + (direction == 2), compact=compact, inverse_diagonal=dinv)
        ex, bd = R.trsv_row_bound(c["rp"], c["ci"], v, b, z[:c["n"]], direction != 2, dinv)
        R.assert_within(z[:c["n"]], ex, bd, "classic local")


def test_gs2_bound_rejects_wrong_programs(oracle):
    """A dropped entry, (1 - gamma) * Z for (1 - gamma) * R, and x += omega Z where the compact form needs x = omega Z, each
    computed in the data's own precision, fall outside the bound; the same program without the change stays inside."""
    import gs_cases as G

    c = G.gs2_case(0.1)
    v = c["v"]
    b, x0 = G.vectors(c, np.float64, 2)
    args = (c["rp"], c["ci"], v, c["ncols"], x0, b)
    plain = lambda variant, **k: R._gs2_run(*args, **k, dt=np.float64, variant=variant).val
    opts = dict(init_zero=False, omega=0.9, num_iter=1, direction=1, compact=True, inner=2, outer=1, gamma_=0.7, two_stage=True, dinv=None)
    ex, bd = R.gs2_ref(*args, False, 0.9, 1, 1, True, 2, 1, 0.7)
    R.assert_within(plain(None, **opts), ex, bd, "plain run")
    for variant in ("damp_z", "accumulate"):
        with pytest.raises(AssertionError):
            R.assert_within(plain(variant, **opts), ex, bd, variant)
    rows = np.repeat(np.arange(c["n"]), np.diff(c["rp"]))
    off = np.flatnonzero(rows != c["ci"])
    vd = v.copy()
    vd[off[len(off) // 2]] = 0
    x = x0.copy()
    oracle.gs2_apply(c["rp"], c["ci"], vd, c["ncols"], x, b, False, 0.9, 1, 1, compact=True, inner_sweeps=2, gamma=0.7)
    with pytest.raises(AssertionError):
        R.assert_within(x, ex, bd, "dropped entry")
