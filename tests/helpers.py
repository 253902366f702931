"""Shared test helpers: inputs as the reference's tests define them, and its
acceptance laws."""
import hashlib
import json
import os

import numpy as np

from kokkos_kernels_b200 import matgen

REFERENCE_DIGESTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_digests.json")


class ReferenceOutputs:
    """Arrays a test requires to be, bit for bit, what the reference's own code returns on the same inputs.  What the
    reference returned is stored as one SHA-256 digest per test under `key` in tests/golden/reference_digests.json, so the
    comparison needs no reference build: add() every result in order, then check().  With KKREF_RECORD=1 (and oracle/_ref
    built from the reference tree, see oracle/Makefile) add() also runs `ref()`, the reference's code, compares its arrays
    with the results directly, and check() records the digest.  Without KKREF_RECORD the reference library is never called,
    even where oracle/_ref exists: the digests stand for its outputs, bit for bit."""

    def __init__(self, key):
        self.key = key
        self.hash = hashlib.sha256()
        self.record = os.environ.get("KKREF_RECORD") == "1"

    def add(self, got, ref, what=""):
        if self.record:
            want = ref()
            assert len(want) == len(got), (self.key, what)
            for a, b in zip(got, want):
                a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
                assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), (self.key, what)
        for a in got:
            a = np.ascontiguousarray(a)
            self.hash.update(f"{a.dtype.str}{a.shape}".encode())
            self.hash.update(a.tobytes())

    def check(self):
        digest = self.hash.hexdigest()
        stored = json.load(open(REFERENCE_DIGESTS)) if os.path.exists(REFERENCE_DIGESTS) else {}
        if self.record:
            stored[self.key] = digest
            with open(REFERENCE_DIGESTS, "w") as f:
                json.dump(stored, f, indent=0, sort_keys=True)
                f.write("\n")
            return
        assert self.key in stored, f"no stored reference output for {self.key}"
        assert digest == stored[self.key], f"{self.key}: differs from the reference's output"


def kk_matrix(nrows, ncols, nnz, variance, bandwidth, dtype=np.float64, seed=13718, lo=0.0, hi=1.0, sort=False, oracle=None):
    """kk_generate_sparse_matrix structure + seeded uniform values (the
    reference re-draws values in [0, max_val) with its own RNG, Test_Sparse_spmv.hpp:413)."""
    rp, ci = matgen.kk_generate(nrows, ncols, nnz, variance, bandwidth)
    v = matgen.fill(len(ci), lo, hi, seed, dtype=dtype)
    if sort:
        oracle.sort_crs(rp, ci, v)
    return rp, ci, v


def spmv_tolerance(eps, alpha, beta, max_nnz_per_row, max_val=1.0, max_x=1.0, max_y=1.0):
    """|expected - actual| <= 10*eps*(beta*max_y + alpha*max_row*max_val*max_x)
    (Test_Sparse_spmv.hpp:67-104,181,432).  abs() guards negative alpha/beta as
    the functor takes AT::abs(max_val)."""
    return 10.0 * eps * abs(beta * max_y + alpha * max_nnz_per_row * max_val * max_x)


def rowwise_scale(rp, ci, v, x, y0, alpha, beta, ncols_out=None, trans=False):
    """|alpha| * sum_j |a_ij||x_j| + |beta||y0_i|  (SURVEY.md section 8d parity criterion)."""
    m = len(rp) - 1
    rows = np.repeat(np.arange(m), np.diff(rp))
    av = np.abs(v.astype(np.float64))
    if not trans:
        s = np.bincount(rows, weights=av * np.abs(x[ci].astype(np.float64)), minlength=m)
    else:
        s = np.bincount(ci, weights=av * np.abs(x[rows].astype(np.float64)), minlength=ncols_out)
    out = abs(alpha) * s
    if beta != 0:
        out = out + abs(beta) * np.abs(np.nan_to_num(y0.astype(np.float64)))
    return out


def dense_from_csr(rp, ci, v, ncols):
    m = len(rp) - 1
    A = np.zeros((m, ncols), dtype=np.float64)
    rows = np.repeat(np.arange(m), np.diff(rp))
    np.add.at(A, (rows, ci), v)
    return A
