"""Matrices for rank-1 SpMV (csrc/spmv.cu) at the row lengths and row positions where its kernels change behaviour, shared
by the emulated-kernel tests and the GPU tests.  Every builder returns (rp, ci, v, ncols); values are mixed-sign over
several binades (spmm_cases._values), so that dropping, repeating or misplacing a term shows.

The thresholds (csrc/spmv.cu, kCfgs and plan_analyse): a ring configuration of stage capacity CAP has the row limit
LMAX = CAP/4 and the tile size T = CAP - LMAX - 8.  Tile b owns the rows whose first entry lies in [b*T, (b+1)*T); rows
longer than LMAX go to the long-row kernels; build_tiles_kernel clamps a tile's staged end to (s & ~3) + CAP - 4 when its
last row is long.  The segmented long-row kernels (B200SP_SPMV_LONGROWS=seg) cut rows into segments of SEG entries."""
import numpy as np

from spmm_cases import _values, from_lengths

# ring configurations of the tiled kernel (kCfgs in csrc/spmv.cu and the template arguments launch_tile_cfg gives them):
# cfg -> (consumer warps NW, STAGES, CAP, UNR)
CFGS = {0: (8, 4, 2048, 8), 1: (16, 4, 4096, 8), 2: (8, 3, 4096, 8), 3: (8, 6, 1024, 8), 4: (16, 3, 2048, 8),
        5: (24, 3, 2048, 8), 6: (31, 3, 2048, 8), 7: (16, 5, 1024, 8), 8: (16, 4, 2048, 8), 9: (16, 3, 2048, 4),
        10: (31, 3, 4096, 8)}
CAPS = (1024, 2048, 4096)
LPRS = (2, 4, 8, 16, 32)
SEG = 4096
LONG_LENGTHS = (4095, 4096, 4097, 2 * 4096 + 1)  # one, one, two and three segments


def limits(cap):
    """(LMAX, T) of a ring configuration of stage capacity cap"""
    lmax = cap // 4
    return lmax, cap - lmax - 8


def tile_label(dtype, cfg, lpr, cols):
    """the part of last_kernel() a tiled launch reports, up to the grid: cols is 'IDX=i32', 'IDX=u16,COLS=delta' or
    'IDX=u16,COLS=pat'"""
    nw, stages, cap, unr = CFGS[cfg]
    prec = "f64" if np.dtype(dtype) == np.float64 else "f32"
    return f"tile<{prec},LPR={lpr},NW={nw},STAGES={stages},CAP={cap},UNR={unr},{cols}>"


def threshold_lengths(seed, nnz_mod4):
    """Row lengths that put, for every CAP: rows of LMAX-1, LMAX and LMAX+1 entries; rows starting at b*T - 1, b*T and
    b*T + 1 for several tiles b, with lengths 1, LMAX-1, LMAX, LMAX+1 and short ones; a long row as a tile's last row (far
    enough past the tile's end that its staged end is clamped); a run of empty rows longer than a tile; empty first and last
    rows; nnz % 4 == nnz_mod4.  Short random rows (0..40 entries) fill the gaps."""
    rng = np.random.default_rng(seed)
    lens = [0]  # empty first row

    def nnz():
        return sum(lens)

    def fill_to(target):
        while nnz() < target:
            lens.append(min(target - nnz(), int(rng.integers(0, 41))))

    for cap in CAPS:
        lmax, _ = limits(cap)
        for L in (lmax - 1, lmax, lmax + 1):
            lens.append(L)
            lens.extend(rng.integers(0, 41, 3).tolist())
    # row starts at tile boundaries: (position, length) wanted, in increasing position
    wants = []
    # one region of the matrix per CAP, so that no row placed for one CAP covers a boundary wanted for another
    for cap, tiles in ((1024, range(6, 25, 3)), (2048, range(13, 26, 2)), (4096, range(13, 26, 2))):
        lmax, T = limits(cap)
        kinds = [(-1, lmax), (0, 1), (1, lmax - 1), (-2, cap // 2 + lmax),  # a long last row of tile b-1: end clamped
                 (-1, 1), (0, lmax + 1), (1, int(rng.integers(2, 40)))]
        for i, b in enumerate(tiles):
            d, L = kinds[i % len(kinds)]
            wants.append((b * T + d, L, cap, d))
    assert [w[2] for w in sorted(wants)] == [w[2] for w in wants]
    placed = set()
    for pos, L, cap, d in wants:
        if pos < nnz():
            continue  # covered by the row before; coverage is checked below
        fill_to(pos)
        lens.append(L)
        placed.add((cap, d, L > limits(cap)[0]))
        if len(lens) % 5 == 0:
            lens.extend([0] * int(rng.integers(1, 4)))
    for cap in CAPS:
        for d in (-1, 0, 1):
            assert any(c == cap and dd == d for c, dd, _ in placed), (cap, d)
        assert (cap, -2, True) in placed, cap
    lens.extend([0] * (max(CAPS) + 300))  # empty rows: more rows than any tile has entries
    lens.extend(rng.integers(0, 41, 200).tolist())
    lens.append((nnz_mod4 - nnz()) % 4 + 4)
    lens.append(0)  # empty last row
    assert nnz() % 4 == nnz_mod4
    return np.asarray(lens, dtype=np.int64)


def thresholds(seed, dtype, nnz_mod4=3):
    """threshold_lengths with uniform random columns (unsorted, duplicates possible): the 32-bit column form"""
    rng = np.random.default_rng(seed + 100)
    ncols = 9000
    return (*from_lengths(threshold_lengths(seed, nnz_mod4), ncols, rng, dtype), ncols)


def thresholds_sorted(seed, dtype, nnz_mod4=3):
    """The same row lengths with sorted columns whose in-row gaps lie in [0, 65535] (0: a repeated column), so the matrix
    qualifies for the delta form under every ring configuration and has far too many patterns for the pattern form.  One
    short row has a gap of exactly 65535; one row of 1,100 entries (longer than every LMAX, so the long-row kernel reads
    it from col_idx) has a gap of 65536."""
    rng = np.random.default_rng(seed + 200)
    lens = threshold_lengths(seed, nnz_mod4)
    short = np.flatnonzero((lens >= 2) & (lens <= 40))
    lens[short[-1]] += 1100 - lens[short[-1]]
    lens[-2] += (nnz_mod4 - int(lens.sum())) % 4  # keep nnz % 4 (the row before the empty last row)
    ncols = 200000
    rows = []
    for L in lens:
        L = int(L)
        gaps = rng.integers(0, 24, L)
        gaps[:1] = 0
        rows.append(int(rng.integers(0, ncols - 24 * max(L, 1) - 70000)) + np.cumsum(gaps))
    r65535 = int(short[0])
    rows[r65535][-1] = rows[r65535][-2] + 65535
    rl = int(short[-1])
    rows[rl][600:] += 65536 - (rows[rl][600] - rows[rl][599])
    assert rows[rl][-1] < ncols and rows[r65535][-1] < ncols
    rp = np.zeros(len(lens) + 1, dtype=np.int64)
    np.cumsum(lens, out=rp[1:])
    ci = np.concatenate(rows).astype(np.int32)
    assert int(rp[-1]) % 4 == nnz_mod4
    return rp.astype(np.int32), ci, _values(rng, len(ci), dtype), ncols


def long_rows(seed, dtype, m=6000):
    """Rows of LONG_LENGTHS entries (one to three segments of the segmented path) and a few other long rows, first, inside
    and last, between short and empty rows; nnz % 4 == 1."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 30, m)
    lens[rng.integers(0, m, m // 6)] = 0
    at = [0, 77, 1500, 1501, 3000, m - 1]
    for r, L in zip(at, LONG_LENGTHS + (1025, 2 * SEG)):
        lens[r] = L
    lens[m - 2] += (1 - int(lens.sum())) % 4
    ncols = 12000
    return (*from_lengths(lens, ncols, rng, dtype), ncols)


def hostvec_big(seed, dtype=np.float64, m=260000):
    """More than 2^22 entries (the pipelined host-vector path), with long rows in every 24th of the rows, so that every
    piece of every B200SP_HOSTVEC_PIECES setting (1, 2, 3, 4, 6 or 8 pieces), the last one included, holds long rows."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 40, m)
    lens[rng.integers(0, m, m // 10)] = 0
    for k in range(24):
        lens[(k * m) // 24 + int(rng.integers(0, m // 30))] = int(rng.integers(600, 6000))
    lens[m - 3] = 5000
    lens[m - 1] = 4097
    assert lens.sum() >= (1 << 22)
    ncols = m
    return (*from_lengths(lens, ncols, rng, dtype), ncols)


def with_values(A, seed, dtype):
    """(rp, ci, ncols) of A with fresh mixed-sign values of dtype"""
    rp, ci, _, ncols = A
    return rp, ci, _values(np.random.default_rng(seed), len(ci), dtype), ncols


def vector_operand(rng, n, dtype):
    """Mixed-sign x / y entries over 2^-2 .. 2^2, no zeros."""
    return (rng.uniform(0.5, 1.0, n) * rng.choice([-1.0, 1.0], n) * np.exp2(rng.integers(-2, 3, n))).astype(dtype)
