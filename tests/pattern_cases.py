"""Inputs for the tests of the tiled SpMV kernel's pattern form (DESIGN.md section 3.6), and the rule that picks a matrix's
column form, restated in Python: the pattern form when every row of 1..LMAX entries has one of a few patterns (its columns
minus its first column) that together hold at most DCAP offsets; else the delta form when every in-row delta of those rows
lies in [0, 65535]; else the 32-bit columns."""
import numpy as np

from kokkos_kernels_b200 import matgen

DCAP = 1024
AB = ((1.0, 0.0), (-0.7, 1.3), (2.5, -0.5))  # beta == 0 is run with NaN in y, which must not survive
LMAX = {0: 512, 1: 1024, 2: 1024, 3: 256, 4: 512, 8: 512}  # CAP / 4 of the ring configurations the tests use
LONG = 1100  # longer than LMAX of every ring configuration


def lap27(nx, ny, nz, ndof=2, row_begin=0, row_end=None):
    """the bench family; row_begin/row_end: the shard of rows bench.py gives one of several GPUs (global columns)"""
    rp, ci, v = matgen.lap27(nx, ny, nz, ndof=ndof, row_begin=row_begin, row_end=row_end, noise=0.5)
    return rp, ci, v, nx * ny * nz * ndof


LAP_CASES = {
    "dof1": (9, 8, 7, 1),
    "dof2": (10, 9, 8, 2),
    "dof3": (7, 6, 5, 3),
    "flat2": (2, 9, 8, 2),   # one axis of two nodes: no interior along x
    "flat3": (9, 3, 7, 2),
}


def lap_case(name):
    if name == "shard":
        n = 10 * 9 * 8 * 2
        return lap27(10, 9, 8, 2, row_begin=n // 3, row_end=2 * n // 3)
    return lap27(*LAP_CASES[name])


def expected_cols(A, lmax):
    """'pat', 'delta' or 'i32': the form the plan picks for A under a ring configuration with row limit lmax"""
    rp, ci = A[0], A[1].astype(np.int64)
    pats, deltas_ok = set(), True
    for r in range(len(rp) - 1):
        c = ci[rp[r]:rp[r + 1]]
        if 1 <= len(c) <= lmax:
            pats.add(tuple(c - c[0]))
            d = np.diff(c)
            deltas_ok &= bool(np.all((d >= 0) & (d <= 65535)))
    if sum(len(p) for p in pats) <= DCAP:
        return "pat"
    return "delta" if deltas_ok else "i32"


def _assemble(rows, ncols, seed):
    rp = np.zeros(len(rows) + 1, np.int32)
    rp[1:] = np.cumsum([len(r) for r in rows])
    ci = np.concatenate([np.asarray(r, np.int64) for r in rows]).astype(np.int32) if rp[-1] else np.zeros(0, np.int32)
    v = np.random.default_rng(seed).uniform(-1, 1, len(ci))
    return rp, ci, v, ncols


def _from_patterns(patterns, m, ncols, seed, empty_every=0):
    """row r: a random anchor plus patterns[r % len(patterns)] (rows every empty_every-th are empty)"""
    rng = np.random.default_rng(seed)
    span = max(int(np.max(p)) for p in patterns) + 1
    rows = []
    for r in range(m):
        if empty_every and r % empty_every == 0:
            rows.append(np.zeros(0, np.int64))
            continue
        p = np.asarray(patterns[r % len(patterns)], np.int64)
        rows.append(int(rng.integers(0, ncols - span)) + p)
    return rows


def dict_matrix(total, m=2000, seed=11):
    """distinct patterns that hold `total` >= 1024 offsets: 32 patterns of 32 offsets (the same first 31, a different last
    one), plus one of total - 1024 offsets.  total = DCAP qualifies, DCAP + 1 does not."""
    pats = [list(range(31)) + [31 + p] for p in range(32)]
    if total > 32 * 32:
        pats.append(list(range(total - 32 * 32)))
    return _assemble(_from_patterns(pats, m, 5000, seed), 5000, seed)


def near_patterns_matrix(m=3000, seed=12):
    """patterns that differ only in length ({0,1,2} / {0,1,2,3}) or only in their last offset ({0,1,2,5})"""
    return _assemble(_from_patterns([[0, 1, 2], [0, 1, 2, 3], [0, 1, 2, 5], [0, 1, 2, 3]], m, 4000, seed), 4000, seed)


def diagonal_matrix(m=5000, seed=13):
    """one entry per row: more rows per tile than a stage stages, so rows past it read anchor and pid from global memory"""
    return _assemble([np.array([r]) for r in range(m)], m, seed)


def long_rows_matrix(m=3000, seed=14):
    """regular rows (two patterns) plus rows longer than any LMAX with unsorted columns and wide jumps: the tiled kernel
    never reads them, so the matrix still takes the pattern form"""
    ncols = 300000
    rows = _from_patterns([[0, 1, 7, 40], [0, 2, 3, 100, 101, 102]], m, ncols, seed)
    rng = np.random.default_rng(seed)
    rows[7] = rng.permutation(ncols)[:LONG]
    rows[2000] = np.arange(LONG)[::-1] * 250
    return _assemble(rows, ncols, seed)


def empty_rows_matrix(m=5000, seed=15):
    """every third row empty, the others one of three patterns, nnz not a multiple of 8"""
    rows = _from_patterns([[0, 1, 2, 9], [0, 5], [0, 1, 2, 3, 4, 5, 6]], m, 20000, seed, empty_every=3)
    while sum(len(r) for r in rows) % 8 == 0:
        rows[1] = rows[1][:1]
    return _assemble(rows, 20000, seed)


def random_rows(rp, ncols, seed=16):
    """sorted random columns with small gaps under the given row_ptr: no repeated patterns, the delta form"""
    rng = np.random.default_rng(seed)
    rows = []
    for r in range(len(rp) - 1):
        n = rp[r + 1] - rp[r]
        rows.append(int(rng.integers(0, ncols - 3 * n)) + np.cumsum(rng.integers(1, 4, n)) - 1)
    return _assemble(rows, ncols, seed)[1]
