"""SpGEMM and spgemm_jacobi inputs built to reach each kernel path of csrc/spgemm.cu and csrc/spgemm_esc.cuh, shared by the
GPU and the emulated path tests.  Values are mixed-sign over several binades (spmm_cases._values), and some rows are made
of pairs of equal B rows weighted +a and -a, so that every entry of those rows cancels exactly to 0.

The paths, and the bounds the rows are placed on (the library reports which path every row took through
b200sp_spgemm_plan_paths; `intended_paths` below is what the cases were built for, so a bound that moves shows up as a
mismatch between the two):
  * symbolic and numeric: rows binned by key = max(products, 2 nnz(A_i)): expand / sort / compress (ESC) bins of <= 256,
    1024, 4096 and 8192, then the symbolic hash kernel (<= 16384) and the global bitmap (above);
  * numeric rows with key > 8192: hash kernels binned by nnz(C_i) <= 64, 256, 1024, 4096, 8192, each with a dense
    accumulator when the row's column span fits KSLOTS and a monotone multiplicative map otherwise; rows with more
    columns go to the global fallback, and so do rows whose ordered probe runs off the table's pad (overflow);
  * spgemm_jacobi: every row in the hash kernels by nnz(C_i), the same bounds.

Every case is a dict: name, A, B (row_map, entries, values), m, n, k, targets (paths the case must reach), overflow (rows
expected to overflow at run time, None = not checked), oracle (k small enough for the oracle's k-sized accumulators),
square (A is n x n with its whole diagonal, B n x n: a spgemm_jacobi case) and no_diag (rows of A built without their
diagonal, whose row of B leaves the pattern)."""
import numpy as np

import exact_ref as R
from spmm_cases import _values

ESC_BOUNDS = (256, 1024, 4096, 8192)   # kEscThr
SYM_HASH_MAX = 16384                   # the symbolic hash bin above the ESC bins
NUM_BOUNDS = (64, 256, 1024, 4096, 8192)  # kNumThr
KSLOTS = (256, 1024, 4096, 16384, 32768)  # key slots of the numeric hash bins
PADS = (32, 64, 128, 256, 512)
PATHS = ("esc0", "esc1", "esc2", "esc3", "sym_hash", "sym_bitmap", "hash0", "hash1", "hash2", "hash3", "hash4", "fallback",
         "overflow")


def _bin(x, bounds):
    return int(np.searchsorted(np.asarray(bounds), x, side="left"))


def intended_paths(products, nnz_a, nnz_c, jacobi=False):
    """Counts per path (PATHS, "overflow" left at 0) of rows with the given products, entries of A and entries of C."""
    key = np.maximum(products, 2 * nnz_a)
    out = dict.fromkeys(PATHS, 0)
    sym = np.array([_bin(x, ESC_BOUNDS + (SYM_HASH_MAX,)) for x in key])
    for b in range(6):
        out[PATHS[b]] = int((sym == b).sum())
    num_rows = np.ones(len(key), bool) if jacobi else key > ESC_BOUNDS[-1]
    nb = np.array([_bin(x, NUM_BOUNDS) for x in nnz_c[num_rows]], dtype=np.int64)
    for b in range(5):
        out["hash%d" % b] = int((nb == b).sum())
    out["fallback"] = int((nb == 5).sum())
    return out


class Builder:
    """A product made row by row.  Each row of A gets B rows of its own, so that its products, its distinct columns and
    their span are what the row asks for.  square=True: A and B are N x N, row i of A holds its diagonal (its first B row
    is row i of B) and rows past the built ones are empty."""

    def __init__(self, seed, dtype, square=False, blen=16):
        self.rng = np.random.default_rng(seed)
        self.dtype = dtype
        self.square = square
        self.blen = blen
        self.rows = []  # per row of A: (list of (cols, vals) B rows, A values, extra entries on empty B rows, diag, own B row)

    def _brows(self, cols_multiset_rows):
        return [(np.asarray(c, dtype=np.int64), _values(self.rng, len(c), self.dtype)) for c in cols_multiset_rows]

    def row(self, products, cols, n_a=None, cancel=False, blen=None, diag=True, own=None):
        """A row of A whose products cover the distinct columns `cols` (every column at least once) and number `products`
        in all, in B rows of at most `blen` distinct columns.  n_a > B rows: the extra entries of A point at empty rows of
        B.  cancel: every B row comes twice, weighted +a and -a (products doubles, every value of the row is 0).
        diag=False (square): row i of A does not reference row i of B, which holds the columns `own` instead."""
        cols = np.asarray(cols, dtype=np.int64)
        nz = len(cols)
        assert products >= nz or nz == 0
        L = max(1, min(blen or self.blen, nz)) if nz else 1
        perm = self.rng.permutation(cols)
        brows = [perm[j:j + L] for j in range(0, nz, L)]
        left = products - nz
        while left > 0:
            t = min(L, left)
            brows.append(self.rng.choice(cols, t, replace=False))
            left -= t
        br = self._brows(brows)
        av = _values(self.rng, len(br), self.dtype)
        if cancel:
            br = [x for b in br for x in (b, b)]
            av = np.stack([av, -av], axis=1).reshape(-1)
        extra = 0 if n_a is None else n_a - len(br)
        assert extra >= 0
        self.rows.append((br, av, extra, diag, None if own is None else self._brows([own])[0]))
        return self

    def empty(self, count=1):
        for _ in range(count):
            self.rows.append(([], np.zeros(0, self.dtype), 0, True, None))
        return self

    def build(self, k=None, sort=True):
        """(A, B, m, n, k).  Rows of A and B come out sorted unless sort=False (then shuffled)."""
        m = len(self.rows)
        ncols = max([int(c.max()) + 1 for r in self.rows for c, _ in r[0] if len(c)] + [int(r[4][0].max()) + 1 for r in self.rows
                                                                                        if r[4] is not None and len(r[4][0])] + [1])
        nB = sum(len(r[0]) + r[2] for r in self.rows)
        if self.square:
            N = max(m + nB, ncols, k or 0)
            m = n = k = N
            Brows = [None] * N
            nxt = len(self.rows)
        else:
            k = max(ncols, k or 0)
            n = nB
            Brows = [None] * n
            nxt = 0
        a_ent, a_val = [], []
        for i, (br, av, extra, diag, own) in enumerate(self.rows):
            idx = []
            for j, b in enumerate(br):
                if self.square and diag and j == 0:
                    Brows[i] = b
                    idx.append(i)
                else:
                    Brows[nxt] = b
                    idx.append(nxt)
                    nxt += 1
            if self.square and own is not None:
                Brows[i] = own
            for _ in range(extra):
                if self.square and diag and not idx:
                    idx.append(i)  # the diagonal points at an empty row of B
                    continue
                idx.append(nxt)
                nxt += 1
            ent = np.asarray(idx, dtype=np.int64)
            vals = np.concatenate([av, _values(self.rng, len(ent) - len(av), self.dtype)])
            if self.square and diag and i not in idx:  # a row without B rows: its diagonal alone
                ent, vals = np.append(ent, i), np.append(vals, _values(self.rng, 1, self.dtype))
            a_ent.append(ent)
            a_val.append(vals)
        for i in range(len(a_ent), m):  # square: the rows past the built ones hold their diagonal only
            a_ent.append(np.array([i], dtype=np.int64))
            a_val.append(_values(self.rng, 1, self.dtype))
        A = _csr(list(zip(a_ent, a_val)), self.dtype, sort, self.rng)
        empty = (np.zeros(0, np.int64), np.zeros(0, self.dtype))
        B = _csr([b if b is not None else empty for b in Brows], self.dtype, sort, self.rng)
        return A, B, m, n, k


def _csr(rows, dtype, sort, rng):
    lens = np.array([len(c) for c, _ in rows], dtype=np.int64)
    rp = np.concatenate([[0], np.cumsum(lens)])
    assert rp[-1] < 2**31
    ci = np.empty(int(rp[-1]), dtype=np.int32)
    v = np.empty(int(rp[-1]), dtype=dtype)
    for r, (c, val) in enumerate(rows):
        o = np.argsort(c, kind="stable") if sort else rng.permutation(len(c))
        ci[rp[r]:rp[r + 1]] = np.asarray(c)[o]
        v[rp[r]:rp[r + 1]] = np.asarray(val)[o]
    return rp.astype(np.int32), ci, v


def dense_cols(rng, nz, span, lo=0):
    """nz distinct columns in [lo, lo + span), both ends included."""
    assert span >= nz
    if nz <= 2:
        return np.array([lo, lo + span - 1][:nz])
    mid = rng.choice(np.arange(1, span - 1), nz - 2, replace=False)
    return np.concatenate([[lo], lo + mid, [lo + span - 1]])


def spread_cols(nz, span, lo=0):
    """nz columns spread evenly over [lo, lo + span), both ends included: no probe cluster under the multiplicative map."""
    return lo + np.unique(np.round(np.linspace(0, span - 1, nz)).astype(np.int64))


def cluster_cols(nz, span, lo=0):
    """One column at lo and nz - 1 consecutive ones at the top of the span: the ordered probe of a hashed row runs
    past the pad."""
    return np.concatenate([[lo], lo + span - nz + 1 + np.arange(nz - 1)])


def _case(name, built, targets, overflow=0, oracle=True, square=False, no_diag=0):
    A, B, m, n, k = built
    return dict(name=name, A=A, B=B, m=m, n=n, k=k, targets=tuple(targets), overflow=overflow, oracle=oracle and k <= 1 << 21,
                square=square, no_diag=no_diag)


def esc_bounds(dtype, square=False, seed=1):
    """Rows at both sides of every ESC bound by their products, and by 2 nnz(A_i) (long rows of A over empty or short B
    rows), cancelling rows, empty rows."""
    b = Builder(seed, dtype, square)
    rng = b.rng
    for P in (256, 257, 1024, 1025, 4096, 4097, 8192):
        b.row(P, dense_cols(rng, P // 2, P, lo=int(rng.integers(0, 3000))))
    for na in (128, 129, 512, 513, 2048, 2049, 4096, 4097):
        nz = na // 8
        b.row(nz * 2, dense_cols(rng, nz, 4 * nz), n_a=na, blen=4)
    b.row(600, dense_cols(rng, 150, 400), cancel=True)
    b.row(3000, spread_cols(900, 9000), cancel=True)
    b.empty(3)
    return _case("esc_bounds", b.build(), ["esc0", "esc1", "esc2", "esc3"], square=square)


def sym_bounds(dtype, square=False, seed=2):
    """Keys 16384 and 16385 by products and 16384 / 16386 by entries of A: the symbolic hash bin and the bitmap."""
    b = Builder(seed, dtype, square)
    rng = b.rng
    b.row(16384, dense_cols(rng, 3000, 3500), blen=32)
    b.row(16385, spread_cols(3000, 40000), blen=32)
    b.row(300, dense_cols(rng, 100, 300), n_a=8192, blen=4)
    b.row(300, dense_cols(rng, 100, 300), n_a=8193, blen=4)
    return _case("sym_bounds", b.build(), ["sym_hash", "sym_bitmap"], square=square)


NZ_BOUNDS = (64, 65, 256, 257, 1024, 1025, 4096, 4097, 8192)


def hash_bins(dtype, square=False, seed=3):
    """Rows of more than 8192 products with nnz(C_i) at both sides of every numeric bound, each once with a span that fits
    the bin's KSLOTS (dense accumulator) and once with a wider one (multiplicative map); one row above 8192 columns."""
    b = Builder(seed, dtype, square)
    rng = b.rng
    for nz in NZ_BOUNDS:
        ks = KSLOTS[_bin(nz, NUM_BOUNDS)]
        P = nz + 8300
        b.row(P, dense_cols(rng, nz, min(ks, 2 * nz + 7)), blen=32)
        b.row(P, spread_cols(nz, 2 * ks + 11, lo=5), blen=32)
    b.row(8193 + 8300, spread_cols(8193, 50000), blen=32)
    b.row(9000, dense_cols(rng, 80, 200), cancel=True, blen=32)
    return _case("hash_bins", b.build(), ["hash0", "hash1", "hash2", "hash3", "hash4", "fallback"], square=square)


def overflow(dtype, square=False, seed=4, bins=(0, 1, 2, 3, 4)):
    """One hashed row per numeric bin whose columns are one far column and a dense cluster at the top of the span: the
    ordered probe runs past KSLOTS + PAD and the row is handed to the fallback at run time."""
    b = Builder(seed, dtype, square)
    for bn in bins:
        nz = (NUM_BOUNDS[bn] * 15) // 16
        assert nz - nz // 4 > PADS[bn]
        b.row(nz + 8300, cluster_cols(nz, 4 * KSLOTS[bn]), blen=32)
    return _case("overflow", b.build(), ["hash%d" % x for x in bins] + ["overflow"], overflow=len(bins), square=square)


def fallback(dtype, square=False, seed=5):
    """Rows of more than 8192 distinct columns: the global hash and bitonic sort (row lengths not powers of two)."""
    b = Builder(seed, dtype, square)
    rng = b.rng
    b.row(8193 + 9000, dense_cols(rng, 8193, 8193 + 500), blen=32)
    b.row(12000 + 5000, spread_cols(12000, 90000), blen=32)
    b.row(500, dense_cols(rng, 200, 400))
    return _case("fallback", b.build(), ["fallback"], square=square)


def lanes(dtype, lb, seed=6):
    """B's mean row length set for `lb` lanes per B row (4, 8, 16, 32), B rows of up to 4x the mean (longer than the
    sub-warp), A mostly short rows plus long ones for the hash kernels and the symbolic hash bin."""
    rng = np.random.default_rng(seed + lb)
    mean = {4: 3, 8: 6, 16: 12, 32: 24}[lb]
    nB, k, m = 3000, 3000, 400
    lensB = rng.integers(mean - 2, mean + 3, nB)
    lensB[rng.permutation(nB)[:nB // 20]] = 0
    lensB[rng.permutation(nB)[:nB // 20]] = 4 * mean  # longer than the lb lanes of a sub-warp
    Bc = [rng.choice(k, int(l), replace=False) for l in lensB]
    lensA = rng.integers(0, 40, m)
    lensA[:2] = [int(9000 / mean), int(2200 / mean)]  # the hash kernels (nnz(C_i) near k), ESC bin 2
    Ac = [rng.choice(nB, int(l), replace=False) for l in lensA]
    A = _csr([(c, _values(rng, len(c), dtype)) for c in Ac], dtype, True, rng)
    B = _csr([(c, _values(rng, len(c), dtype)) for c in Bc], dtype, True, rng)
    avg = len(B[1]) / nB
    assert lb // 2 < avg <= lb or (lb == 4 and avg <= 4), (lb, avg)
    return _case("lanes_lb%d" % lb, (A, B, m, nB, k), ["esc0", "esc2", "sym_hash", "hash3"], overflow=None)


def layout(dtype, seed=7):
    """Unsorted rows of A and B, empty rows in both, a rectangular product with a row of A longer than half its bin."""
    rng = np.random.default_rng(seed)
    m, n, k = 900, 700, 1100
    lensA = rng.integers(0, 12, m)
    lensA[::17] = 0
    lensA[10] = 300
    lensA[11] = 650  # 2 nnz(A_i) = 1300: ESC bin 2 by its entries
    lensB = rng.integers(0, 9, n)
    lensB[:20] = 0
    lensB[20:40] = 60
    A = _csr([(rng.choice(n, int(l), replace=False), _values(rng, int(l), dtype)) for l in lensA], dtype, False, rng)
    B = _csr([(rng.choice(k, int(l), replace=False), _values(rng, int(l), dtype)) for l in lensB], dtype, False, rng)
    return _case("layout_unsorted_rect", (A, B, m, n, k), ["esc0", "esc2"], overflow=None)


def wide_columns(dtype, seed=8):
    """k = 2^30 - 3: columns across the whole range, so the multiplicative map and (c - cmin) run on spans near 2^30; a dense
    row at the top of the range.  No bitmap row (it allocates k bits per CTA) and no oracle (k-sized accumulators)."""
    b = Builder(seed, dtype)
    rng = b.rng
    k = (1 << 30) - 3
    b.row(500, np.sort(rng.choice(k, 300, replace=False)))
    b.row(5000, np.sort(rng.choice(k, 2000, replace=False)))
    b.row(8192 + 900, spread_cols(900, k))
    b.row(8192 + 3000, spread_cols(3000, k - 7, lo=7))
    b.row(8192 + 200, dense_cols(rng, 200, 250, lo=k - 250))
    b.row(9000 + 4000, spread_cols(9000, k))
    return _case("wide_columns", b.build(k=k), ["esc1", "esc3", "sym_hash", "hash1", "hash2", "hash3", "fallback"], oracle=False)


def no_diagonal(dtype, seed=9):
    """spgemm_jacobi rows of A without their diagonal whose row of B brings columns outside the pattern: in a shared-memory
    bin (handed to the fallback at run time), with one pattern column (a 2-slot table in the fallback), and in the
    static fallback; plus a row whose pattern is empty and an ordinary row."""
    b = Builder(seed, dtype, square=True)
    rng = b.rng
    b.row(40, dense_cols(rng, 20, 30), diag=False, own=[2000, 2001, 7])
    b.row(1, [100], diag=False, own=[3000, 3001, 3002])
    b.row(8193 + 9000, dense_cols(rng, 8193, 8500, lo=10000), diag=False, own=[10000, 30000, 30001])
    b.row(0, [], diag=False, own=[5, 6])
    b.row(300, dense_cols(rng, 100, 200))
    return _case("no_diagonal", b.build(), ["hash0", "fallback", "overflow"], overflow=2, square=True, no_diag=4)


def spgemm_cases(dtype):
    """The A*B cases."""
    out = [esc_bounds(dtype), sym_bounds(dtype), hash_bins(dtype), overflow(dtype), fallback(dtype)]
    out += [lanes(dtype, lb) for lb in (4, 8, 16, 32)]
    out += [layout(dtype), wide_columns(dtype)]
    return out


def jacobi_cases(dtype):
    """Square versions with the whole diagonal (every row in the jacobi hash bins by nnz(C_i)), and the rows without it."""
    out = [esc_bounds(dtype, True), hash_bins(dtype, True), overflow(dtype, True, bins=(0, 1, 2, 3)), fallback(dtype, True),
           no_diagonal(dtype)]
    return out


def jacobi_operands(case, dtype, seed=11):
    """dinv per row, mixed sign over several binades, and omega != 1."""
    rng = np.random.default_rng(seed)
    return 0.7, _values(rng, case["m"], dtype)


# ---- checks shared by the GPU and the emulated tests ----
def expected_paths(case, rp_exact, jacobi):
    """What `case` was built for, from its structure and the exact row map of C (jacobi: every row by nnz(C_i))."""
    A, B = case["A"], case["B"]
    return intended_paths(R.product_rows(A, B), np.diff(A[0].astype(np.int64)), np.diff(rp_exact.astype(np.int64)), jacobi)


def check_paths(got, case, rp_exact, jacobi, what):
    """The witness of a run equals the rows the case was built for, and every targeted path was reached."""
    exp = expected_paths(case, rp_exact, jacobi)
    if case["overflow"] is None:
        got = dict(got, overflow=0)
    else:
        exp["overflow"] = case["overflow"]
    assert got == exp, f"{what}: paths {got} != built for {exp}"
    for t in case["targets"]:
        assert got[t] > 0, f"{what}: path {t} not reached"


def check_addressing(case, rp, ci):
    """Every hash bin the case targets gets a row whose span fits the bin's KSLOTS and one whose span does not."""
    if case["name"] != "hash_bins":
        return
    nz = np.diff(rp)
    prods = R.product_rows(case["A"], case["B"])
    for b, ks in enumerate(KSLOTS):
        rows = [i for i in range(len(nz)) if nz[i] and _bin(nz[i], NUM_BOUNDS) == b and prods[i] > ESC_BOUNDS[-1]]
        spans = [int(ci[rp[i + 1] - 1]) - int(ci[rp[i]]) + 1 for i in rows]
        assert any(s <= ks for s in spans) and any(s > ks for s in spans), (b, spans)


def new_values(case, dtype, seed):
    """A and B of the case with new values (the same structure): a second numeric on the same handle."""
    rng = np.random.default_rng(seed)
    A, B = case["A"], case["B"]
    return (A[0], A[1], _values(rng, len(A[1]), dtype)), (B[0], B[1], _values(rng, len(B[1]), dtype))
