"""Block SpGEMM test support: the block checker (oracle/libkkoracle_bspgemm.so, restatement of the reference's
bspgemm_debug_numeric, and oracle/_ref/libkkref_bspgemm.so, the reference compiled in place when it was built), inputs,
and the comparisons shared by the oracle, emulated and GPU tests.

A case is (name, bs, (rpA, ciA, vA), (rpB, ciB, vB), mb, nb, kb): A is mb x nb blocks, B is nb x kb blocks, values hold
bs*bs entries per block, row-major within the block."""
import ctypes as C
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ODIR = os.path.join(ROOT, "oracle")

# the reference's sweep (sparse/unit_test/Test_Sparse_bspgemm.hpp:232-242): (m, n, k, nnz, bandwidth, row size variance);
# A is m x k blocks, B is k x n
REF_SWEEP = [(50, 50, 50, 2000, 50, 5), (50, 50, 50, 1000, 50, 5), (500, 500, 500, 32000, 500, 500), (2, 3, 4, 2, 2, 0),
             (0, 0, 0, 0, 10, 10), (0, 12, 5, 0, 10, 0), (10, 10, 0, 0, 10, 10)]
BLOCK_SIZES = [1, 2, 3, 4, 5, 8, 16, 17]


def _p(a):
    return C.c_void_p(a.ctypes.data) if a is not None and a.size else C.c_void_p(0)


def _sfx(dtype):
    return "f64" if np.dtype(dtype) == np.float64 else "f32"


class BlockOracle:
    """kko_bspgemm_* (the restatement; rows come out sorted) and, when present, kkref_bspgemm_numeric_* (the reference
    in place; first-touch column order, sorted here the way sort_bsr_matrix does)."""

    def __init__(self):
        self.lib = C.CDLL(os.path.join(ODIR, "libkkoracle_bspgemm.so"))
        self.lib.kko_bspgemm_symbolic.restype = C.c_int64
        rpath = os.path.join(ODIR, "_ref", "libkkref_bspgemm.so")
        self.ref = C.CDLL(rpath) if os.path.exists(rpath) else None

    def symbolic(self, mb, nb, kb, rpA, ciA, rpB, ciB):
        rpC = np.zeros(mb + 1, dtype=np.int32)
        nnz = self.lib.kko_bspgemm_symbolic(mb, nb, kb, _p(rpA), _p(ciA), _p(rpB), _p(ciB), _p(rpC))
        return rpC, int(nnz)

    def bspgemm(self, bs, A, B, mb, nb, kb):
        """(rpC, ciC, vC) of the restatement"""
        rpC, nnz = self.symbolic(mb, nb, kb, A[0], A[1], B[0], B[1])
        dt = A[2].dtype
        ciC = np.zeros(nnz, dtype=np.int32)
        vC = np.zeros(nnz * bs * bs, dtype=dt)
        getattr(self.lib, "kko_bspgemm_numeric_" + _sfx(dt))(mb, nb, kb, bs, _p(A[0]), _p(A[1]), _p(A[2]), _p(B[0]), _p(B[1]),
                                                                _p(B[2]), _p(rpC), _p(ciC), _p(vC))
        return rpC, ciC, vC

    def bspgemm_ref(self, bs, A, B, mb, nb, kb):
        """(rpC, ciC, vC) of the reference's bspgemm_debug_numeric, each row's blocks then sorted by column"""
        assert self.ref is not None
        rpC, nnz = self.symbolic(mb, nb, kb, A[0], A[1], B[0], B[1])
        dt = A[2].dtype
        ciC = np.zeros(nnz, dtype=np.int32)
        vC = np.zeros(nnz * bs * bs, dtype=dt)
        rpA, ciA, vA = (np.ascontiguousarray(x) for x in A)
        rpB, ciB, vB = (np.ascontiguousarray(x) for x in B)
        getattr(self.ref, "kkref_bspgemm_numeric_" + _sfx(dt))(mb, nb, kb, bs, _p(rpA), len(ciA), _p(ciA), _p(vA), _p(rpB), len(ciB),
                                                                 _p(ciB), _p(vB), _p(rpC), nnz, _p(ciC), _p(vC))
        blocks = vC.reshape(max(nnz, 0), bs * bs)
        for i in range(mb):
            s, e = rpC[i], rpC[i + 1]
            order = np.argsort(ciC[s:e], kind="stable")
            ciC[s:e] = ciC[s:e][order]
            blocks[s:e] = blocks[s:e][order]
        return rpC, ciC, vC


def same_bits(a, b):
    """Bit-identical, NaN compared as NaN (the NaN payload and sign are not part of the contract: x86 and the GPU
    propagate different payloads)."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    na, nb_ = np.isnan(a), np.isnan(b)
    if not np.array_equal(na, nb_):
        return False
    it = np.uint64 if a.dtype == np.float64 else np.uint32
    return bool(np.array_equal(a[~na].view(it), b[~nb_].view(it)))


def random_bsr(mb, nbc, nnz, bandwidth, variance, bs, seed, dtype=np.float64, sort=True, signed=True):
    """block graph from the reference's generator (kk_generate_sparse_matrix's CRS part: matgen.kk_generate), values
    uniform in [-1, 1] (or [0.1, 1]) scaled over several binades"""
    from kokkos_kernels_b200 import matgen

    if mb == 0 or nbc == 0 or nnz == 0:
        rp = np.zeros(mb + 1, dtype=np.int32)
        ci = np.zeros(0, dtype=np.int32)
    else:
        rp, ci = matgen.kk_generate(mb, nbc, nnz, variance, bandwidth)
        rp, ci = np.asarray(rp, dtype=np.int32), np.asarray(ci, dtype=np.int32)
        if sort:
            ci = ci.copy()
            for i in range(mb):
                ci[rp[i]:rp[i + 1]] = np.sort(ci[rp[i]:rp[i + 1]])
    rng = np.random.default_rng(seed)
    n = len(ci) * bs * bs
    v = rng.uniform(-1.0, 1.0, n) if signed else rng.uniform(0.1, 1.0, n)
    v = v * np.exp2(rng.integers(-6, 7, n))
    return rp, ci, v.astype(dtype)


def ref_sweep_cases(bs, dtype=np.float64, seed=5):
    out = []
    for t, (m, n, k, nnz, bw, var) in enumerate(REF_SWEEP):
        if bs >= 8 and m >= 500:
            continue  # the 500-row case at large blocks is covered at bs <= 5 (keeps the CPU checkers quick)
        A = random_bsr(m, k, nnz, bw, var, bs, seed + 2 * t, dtype)
        B = random_bsr(k, n, nnz, bw, var, bs, seed + 2 * t + 1, dtype)
        out.append((f"sweep{t}_bs{bs}", bs, A, B, m, k, n))
    return out


def _from_rows(rows, ncols, bs, rng, dtype):
    rp = np.zeros(len(rows) + 1, dtype=np.int32)
    rp[1:] = np.cumsum([len(r) for r in rows])
    ci = np.array([c for r in rows for c in r], dtype=np.int32)
    v = (rng.uniform(-1.0, 1.0, len(ci) * bs * bs) * np.exp2(rng.integers(-4, 5, len(ci) * bs * bs))).astype(dtype)
    return rp, ci, v


def special_cases(bs, dtype=np.float64, seed=11):
    """unsorted rows, repeated columns in a row, explicit zero blocks, signed zeros, NaN and Inf in A"""
    rng = np.random.default_rng(seed)
    out = []
    m, n, k = 40, 30, 35
    rowsA = [list(rng.permutation(n)[: rng.integers(0, 9)]) for _ in range(m)]
    rowsB = [list(rng.permutation(k)[: rng.integers(0, 9)]) for _ in range(n)]
    out.append(("unsorted", bs, _from_rows(rowsA, n, bs, rng, dtype), _from_rows(rowsB, k, bs, rng, dtype), m, n, k))
    rowsA2 = [r + r[:2] for r in rowsA]  # the first two columns of each row again
    rowsB2 = [r[:1] + r for r in rowsB]
    out.append(("repeated_cols", bs, _from_rows(rowsA2, n, bs, rng, dtype), _from_rows(rowsB2, k, bs, rng, dtype), m, n, k))
    A = _from_rows(rowsA, n, bs, rng, dtype)
    B = _from_rows(rowsB, k, bs, rng, dtype)
    vA, vB = A[2].copy(), B[2].copy()
    bb = bs * bs
    vA[: bb * 3] = 0.0                      # explicit zero blocks
    vA[bb * 3: bb * 5] = -0.0               # negative zero blocks
    vB[::7] = -0.0
    vB[1::11] = 0.0
    out.append(("zeros_signed", bs, (A[0], A[1], vA), (B[0], B[1], vB), m, n, k))
    vA2 = A[2].copy()
    vA2[5::97] = np.nan
    vA2[13::89] = np.inf
    vA2[29::83] = -np.inf
    out.append(("nan_inf", bs, (A[0], A[1], vA2), B, m, n, k))
    return out


def long_row_case(bs, dtype=np.float64, seed=13, products=6000):
    """one block row with more products than the shared-memory bins hold (> 4096): the long-row path; other rows short"""
    rng = np.random.default_rng(seed)
    m, n, k = 6, 120, 400
    per_b = products // n + 1
    rowsA = [list(range(n))] + [list(rng.permutation(n)[:4]) for _ in range(m - 1)]
    rowsB = [list(rng.permutation(k)[:per_b]) for _ in range(n)]
    return ("long_row", bs, _from_rows(rowsA, n, bs, rng, dtype), _from_rows(rowsB, k, bs, rng, dtype), m, n, k)


def dense_bound_ok(bs, A, B, mb, nb, kb, rpC, ciC, vC):
    """|C - A*B| within gamma(bs * products of the block + 1) * (|A| |B|) per entry, against a dense float64 (fp32 inputs) /
    long double (fp64 inputs) product of the point forms"""
    from exact_ref import bsr_to_point_crs, gamma, unit_roundoff

    wide = np.longdouble if A[2].dtype == np.float64 else np.float64
    u = unit_roundoff(A[2].dtype)

    def dense(rp, ci, v, nr, nc):
        prp, pci, pv = bsr_to_point_crs(bs, rp, ci, v)
        D = np.zeros((nr * bs, nc * bs), dtype=wide)
        for r in range(nr * bs):
            np.add.at(D[r], pci[prp[r]:prp[r + 1]], pv[prp[r]:prp[r + 1]].astype(wide))
        return D

    Da, Db = dense(A[0], A[1], A[2], mb, nb), dense(B[0], B[1], B[2], nb, kb)
    Dc = dense(rpC, ciC, vC, mb, kb)
    exact = Da @ Db
    scale = np.abs(Da) @ np.abs(Db)
    # products per point entry <= bs * (products of the block row); a row-uniform bound is enough here
    prods = np.zeros(mb, dtype=np.int64)
    for i in range(mb):
        prods[i] = sum(B[0][c + 1] - B[0][c] for c in A[1][A[0][i]:A[0][i + 1]])
    g = np.repeat(np.array([gamma(int(p) * bs + 1, u) for p in prods], dtype=wide), bs) if mb else np.zeros(0, dtype=wide)
    err = np.abs(Dc - exact)
    return bool(np.all(err <= g[:, None] * scale))
