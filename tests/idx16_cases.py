"""Inputs for the tests of the tiled SpMV kernel's 16-bit column form (DESIGN.md section 3.5): a matrix qualifies when every
in-row column delta of its rows of at most LMAX entries lies in [0, 65535]; the others run on the 32-bit columns."""
import numpy as np

from kokkos_kernels_b200 import matgen

# (alpha, beta) pairs; beta == 0 is run with NaN in y, which must not survive
AB = ((1.0, 0.0), (-0.7, 1.3), (2.5, -0.5))
LONG = 1100  # longer than LMAX of every ring configuration (cfg 1: 1024)


def lap27(nx, ny, nz):
    """the bench family: 27-point Laplacian, 2 unknowns per node (in-row gaps 1, 2*nx+1.., 2*nx*ny..)"""
    rp, ci, v = matgen.lap27(nx, ny, nz, ndof=2, noise=0.5)
    return rp, ci, v, len(rp) - 1


def _assemble(rows, ncols, seed):
    rp = np.zeros(len(rows) + 1, np.int32)
    rp[1:] = np.cumsum([len(r) for r in rows])
    ci = np.concatenate([np.asarray(r, np.int64) for r in rows]).astype(np.int32) if rp[-1] else np.zeros(0, np.int32)
    v = np.random.default_rng(seed).uniform(-1, 1, len(ci))
    return rp, ci, v, ncols


def _base_rows(m, ncols, seed, max_len=20, empty_every=0):
    rng = np.random.default_rng(seed)
    rows = []
    for r in range(m):
        n = 0 if (empty_every and r % empty_every == 0) else int(rng.integers(0, max_len + 1))
        start = int(rng.integers(0, ncols - 21 * max_len))
        rows.append(start + np.cumsum(rng.integers(1, 21, n)) - 1)
    return rows


def gap_matrix(gap, m=3000, seed=3):
    """sorted rows with small gaps, and row 17 = {5, 5 + gap}: qualifies iff gap <= 65535"""
    ncols = gap + 1000
    rows = _base_rows(m, ncols, seed)
    rows[17] = np.array([5, 5 + gap])
    return _assemble(rows, ncols, seed)


def unsorted_matrix(m=3000, seed=4):
    """one row of ordinary length with two columns swapped: a negative delta, does not qualify"""
    rows = _base_rows(m, 70000, seed)
    rows[1234] = np.array([10, 900, 400, 1000])
    return _assemble(rows, 70000, seed)


def long_wide_matrix(m=3000, seed=5):
    """rows longer than any LMAX whose columns fall and jump by more than 65535: the tiled kernel never reads them, so the
    matrix still qualifies (the long-row kernel reads col_idx)"""
    ncols = 300000
    rows = _base_rows(m, ncols, seed)
    rows[7] = np.arange(LONG)[::-1] * 250                            # descending: gaps of -250
    rows[2000] = np.concatenate([np.arange(LONG // 2), 100000 + np.arange(LONG - LONG // 2)])  # one gap of about 100000
    return _assemble(rows, ncols, seed)


def empty_rows_matrix(m=5000, seed=6):
    """every third row empty, others up to 20 entries, nnz not a multiple of 8"""
    rows = _base_rows(m, 20000, seed, empty_every=3)
    while sum(len(r) for r in rows) % 8 == 0:
        rows[-1] = rows[-1][:-1] if len(rows[-1]) else np.array([3])
    return _assemble(rows, 20000, seed)
