"""Matrices for rank-2 SpMV (csrc/spmm.cu) at the row lengths, shapes and values where its kernels change behaviour,
shared by the emulated-kernel tests and the GPU tests.  Every builder takes a seed and a dtype and returns
(rp, ci, v, ncols); values are mixed-sign and span a few binades, so that dropping, repeating or misplacing a term shows.

The thresholds (csrc/spmm.cu):
  * cooperative item kernel: batches of EB = 4 entries, then a remainder of 0..EB-1;
  * items of LMAX entries (B200SP_SPMM_ITEM_LMAX, 16..256, default 64): longer rows are split into pieces;
  * rows of more than MMI_LONG_PIECES = 64 pieces are reduced by a CTA instead of a warp."""
import numpy as np

# row lengths straddling every threshold above, at the default LMAX values
THRESHOLD_LENGTHS = [0, 1, 3, 4, 5, 7, 8, 9,          # EB = 4 batch remainders
                     15, 16, 17, 255, 256, 257,       # item LMAX extremes
                     63, 64, 65, 127, 128, 129,       # item pieces at LMAX = 64
                     2047, 2048, 2049, 4097,          # long rows of many pieces
                     4096]                            # exactly 64 pieces of 64 (warp reduce); 4097 is the CTA reduce


def _values(rng, n, dtype):
    """Mixed signs over 2^-4 .. 2^4 in magnitude."""
    return (rng.uniform(0.5, 1.0, n) * rng.choice([-1.0, 1.0], n) * np.exp2(rng.integers(-4, 5, n))).astype(dtype)


def from_lengths(lens, ncols, rng, dtype, dup_pool=None):
    """CSR with the given row lengths; columns uniform over [0, ncols) (duplicates possible) or, with dup_pool, drawn from
    that many columns per row (heavy duplication)."""
    lens = np.asarray(lens, dtype=np.int64)
    rp = np.zeros(len(lens) + 1, dtype=np.int64)
    np.cumsum(lens, out=rp[1:])
    assert rp[-1] < 2**31
    nnz = int(rp[-1])
    if ncols == 0:
        assert nnz == 0
        ci = np.zeros(0, dtype=np.int32)
    elif dup_pool is None:
        ci = rng.integers(0, ncols, nnz).astype(np.int32)
    else:
        row = np.repeat(np.arange(len(lens)), lens)
        pool = rng.integers(0, ncols, (len(lens), dup_pool))
        ci = pool[row, rng.integers(0, dup_pool, nnz)].astype(np.int32)
    return rp.astype(np.int32), ci, _values(rng, nnz, dtype)


def thresholds(seed, dtype):
    """Every length of THRESHOLD_LENGTHS twice, between random short rows, runs of empty rows, a long first and last row;
    nnz % 4 == 3."""
    rng = np.random.default_rng(seed)
    ncols = 6000
    parts = [[2100]]  # long first row
    for L in THRESHOLD_LENGTHS * 2:
        parts.append(rng.integers(0, 12, rng.integers(1, 6)).tolist())
        parts.append([L])
    parts.append([0] * 300)  # a long run of empty rows
    parts.append(rng.integers(0, 12, 400).tolist())
    lens = [x for p in parts for x in p]
    lens.append(0)
    lens.append(0)
    tail = 4100  # long last row
    lens.append(tail + (3 - (sum(lens) + tail)) % 4)
    return (*from_lengths(lens, ncols, rng, dtype), ncols)


def small(seed, dtype, nnz_mod4=1):
    """A few hundred short and medium rows (every batch remainder, one and two items at LMAX = 16 and 64) with a given
    nnz % 4; rectangular."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 70, 500)
    lens[rng.integers(0, 500, 20)] = 0
    lens[-1] += (nnz_mod4 - int(lens.sum())) % 4
    ncols = 350
    return (*from_lengths(lens, ncols, rng, dtype), ncols)


def duplicates(seed, dtype):
    """Rows whose columns repeat many times (legal for SpMV: the terms add up)."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 300, 400)
    return (*from_lengths(lens, 900, rng, dtype, dup_pool=3), 900)


def cancelling(seed, dtype):
    """Rows whose terms come in pairs +-a at one column, a up to 2^20, spread over the row: the exact product is 0 (or the
    few small terms left) while the partial sums are large; plus ordinary rows."""
    rng = np.random.default_rng(seed)
    ncols = 1000
    m = 300
    rows_c, rows_v = [], []
    for i in range(m):
        if i % 3 == 0:
            npairs = int(rng.integers(1, 150))
            c = rng.integers(0, ncols, npairs)
            a = _values(rng, npairs, np.float64) * 2.0**20
            cc = np.concatenate([c, c])
            vv = np.concatenate([a, -a])
            if i % 2 == 0:  # a few small terms that survive the cancellation
                extra = int(rng.integers(1, 4))
                cc = np.concatenate([cc, rng.integers(0, ncols, extra)])
                vv = np.concatenate([vv, _values(rng, extra, np.float64)])
            p = rng.permutation(len(cc))
            rows_c.append(cc[p])
            rows_v.append(vv[p])
        else:
            L = int(rng.integers(0, 200))
            rows_c.append(rng.integers(0, ncols, L))
            rows_v.append(_values(rng, L, np.float64))
    lens = [len(c) for c in rows_c]
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    ci = np.concatenate(rows_c).astype(np.int32)
    v = np.concatenate(rows_v).astype(dtype)
    return rp, ci, v, ncols


def no_columns(seed, dtype):
    """m x 0: no entries; Y = beta*Y."""
    return np.zeros(41, dtype=np.int32), np.zeros(0, dtype=np.int32), np.zeros(0, dtype=dtype), 0


def wide_short(seed, dtype):
    """Few rows, many columns (the transpose has many short rows)."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 600, 30)
    return (*from_lengths(lens, 20000, rng, dtype), 20000)


# cases the emulated tests can afford (small m, tens of thousands of entries)
SMALL_CASES = {"thresholds": thresholds, "small_mod1": lambda s, d: small(s, d, 1), "small_mod2": lambda s, d: small(s, d, 2),
               "small_mod3": lambda s, d: small(s, d, 3), "duplicates": duplicates, "cancelling": cancelling,
               "no_columns": no_columns, "wide_short": wide_short}


# ---- large cases: the grid-stride loops of the reduce, relayout and scale kernels wrap on 132 SMs (GPU only) ----
def many_multi_piece_rows(seed, dtype):
    """17,500 rows of 2..3 pieces of 64 (> 132 SMs * 16 blocks * 8 warps = 16,896 rows for spmm_item_reduce_kernel)
    between empty and short rows."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 8, 40000)
    lens[rng.permutation(40000)[:17500]] = rng.integers(65, 190, 17500)
    return (*from_lengths(lens, 50000, rng, dtype), 50000)


def many_long_rows(seed, dtype):
    """1,100 rows of 4,097..4,160 entries (more than 64 pieces of 64: > 132 SMs * 8 CTAs = 1,056 rows for
    spmm_item_reduce_long_kernel), about 4.5 M entries."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 6, 3000)
    lens[rng.permutation(3000)[:1100]] = rng.integers(4097, 4161, 1100)
    return (*from_lengths(lens, 30000, rng, dtype), 30000)


def tall(seed, dtype):
    """300,000 rows (> 132 SMs * 16 CTAs * 128 rows = 270,336 for relayout_kernel; with k >= 2, rows * k > 540,672 for
    scale2d_kernel) of 0..5 entries."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 6, 300000)
    return (*from_lengths(lens, 7000, rng, dtype), 7000)


def dense_operands(rng, rows, k, dtype):
    """Mixed-sign X / Y0 entries over 2^-2 .. 2^2, no zeros."""
    return (rng.uniform(0.5, 1.0, (rows, k)) * rng.choice([-1.0, 1.0], (rows, k)) * np.exp2(rng.integers(-2, 3, (rows, k)))).astype(dtype)
