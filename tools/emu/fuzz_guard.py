#!/usr/bin/env python
"""Memory-safety + parity fuzzing of the library's kernels under the CUDA-on-CPU emulation (TEST INFRASTRUCTURE).

Every input and output array of every call lives in a block that ends at an inaccessible page (tests/emu_lib.guarded), and
the emulated library runs with B200EMU_GUARD=1 so its own temporaries do too: a kernel (or host routine) that touches one
element outside any array faults, with the seed printed just before.  Results are compared with the oracle.  On a GPU the
same over-read is silent whenever the neighbouring bytes belong to the same allocation granule or pool -- this is the
compute-sanitizer memcheck the round had no GPU minutes for, over a wider input space than the GPU tests.

  python tools/emu/fuzz_guard.py --seeds 0:200            # all operations
  python tools/emu/fuzz_guard.py --seeds 17:18 --ops spgemm -v
"""
import argparse
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests"))
os.environ.setdefault("B200EMU_GUARD", "1")

import emu_lib as E  # noqa: E402
import oracle_lib  # noqa: E402

TOL = {np.dtype(np.float64): 1e-10, np.dtype(np.float32): 1e-4}


def rand_csr(rng, m, n, dtype, sort=False, distinct=False, long_rows=True):
    """Row lengths from a mixture: empty, short, medium and (sometimes) a few very long rows."""
    kind = rng.integers(0, 4)
    if m == 0:
        lens = np.zeros(0, np.int64)
    elif kind == 0:
        lens = rng.integers(0, 4, m)
    elif kind == 1:
        lens = rng.integers(0, 40, m)
    elif kind == 2:
        lens = np.where(rng.random(m) < 0.5, 0, rng.integers(1, 12, m))
    else:
        lens = rng.integers(3, 9, m)
    if long_rows and m > 0 and rng.random() < 0.5:
        for _ in range(int(rng.integers(1, 4))):
            lens[rng.integers(0, m)] = int(rng.integers(200, 6000))
    if distinct:
        lens = np.minimum(lens, n)
    if n == 0:
        lens[:] = 0
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    cols = []
    for l in lens:
        c = rng.choice(n, int(l), replace=False) if distinct else rng.integers(0, max(n, 1), int(l))
        cols.append(np.sort(c) if sort else c)
    ci = (np.concatenate(cols) if cols else np.zeros(0)).astype(np.int32)
    v = rng.uniform(-1, 1, len(ci)).astype(dtype)
    return rp, ci, v


def g(a, rng):
    """Guard an array; half the time with a 16-byte aligned start (TMA-eligible), else exact end."""
    return E.guarded(a, 16 if rng.random() < 0.6 else None)


def scaled_ok(got, exp, scale, tol):
    return bool(np.all(np.abs(got.astype(np.float64) - exp.astype(np.float64)) <= tol * scale + 1e-300))


def row_scale(rp, ci, v, x, y0, alpha, beta, n_out=None, trans=False):
    m = len(rp) - 1
    rows = np.repeat(np.arange(m), np.diff(rp))
    av = np.abs(v.astype(np.float64))
    if not trans:
        s = np.bincount(rows, weights=av * np.abs(x[ci].astype(np.float64)), minlength=m)
    else:
        s = np.bincount(ci, weights=av * np.abs(x[rows].astype(np.float64)), minlength=n_out)
    return abs(alpha) * s + abs(beta) * np.abs(np.nan_to_num(y0.astype(np.float64)))


def op_spmv(rng, orc, verbose):
    dtype = [np.float64, np.float32][rng.integers(0, 2)]
    big = rng.random() < 0.25
    m, n = int(rng.integers(0, 30000 if big else 4000)), int(rng.integers(1, 30000 if big else 4000))
    rp, ci, v = rand_csr(rng, m, n, dtype)
    mode = "NNNCTH"[rng.integers(0, 6)]
    trans = mode in "TH"
    nx, ny = (m, n) if trans else (n, m)
    x = rng.uniform(-1, 1, nx).astype(dtype)
    y0 = rng.uniform(-1, 1, ny).astype(dtype)
    alpha, beta = [(1.0, 0.0), (2.5, -0.5), (-1.0, 1.0), (1.0, 0.0), (-0.3, 2.0), (2.5, 0.0), (1.0, 1.0), (0.0, 2.0)][rng.integers(0, 8)]
    grp, gci, gv, gx, gy = g(rp, rng), g(ci, rng), g(v, rng), g(x, rng), g(y0, rng)
    plan = E.SpmvPlan(int(rng.integers(0, 3)))
    if trans and rng.random() < 0.4:
        E.ok(E.lib().b200sp_spmv_plan_set_option(plan.h, 1, 1))
    if not trans and rng.random() < 0.6:  # force the TMA tile kernel in one of its configurations, whatever the size
        E.ok(E.lib().b200sp_spmv_plan_tune(plan.h, int(rng.integers(0, 11)), int(2 ** rng.integers(1, 6)), 0))
    if not trans and rng.random() < 0.3:
        os.environ["B200SP_SPMV_LONGROWS"] = "seg"
    for _ in range(4 if rng.random() < 0.3 else 2):  # later calls: cached analysis, self-tuning phases
        gy[...] = y0
        E.spmv(plan, mode, m, n, grp, gci, gv, gx, gy, alpha, beta)
    kern = plan.kernel()
    plan.close()
    os.environ.pop("B200SP_SPMV_LONGROWS", None)
    exp = orc.spmv_transpose(rp, ci, v, n, x, y0.copy(), alpha, beta) if trans else orc.spmv_serial(rp, ci, v, x, y0.copy(), alpha, beta)
    ok = scaled_ok(gy, exp, row_scale(rp, ci, v, x, y0, alpha, beta, n, trans), TOL[np.dtype(dtype)])
    return ok, f"spmv {mode} {np.dtype(dtype).name} {m}x{n} nnz={len(ci)} {kern}"


def op_gs2(rng, orc, verbose):
    """two-stage Gauss-Seidel (gs2.cu): random options, ghost columns, directions."""
    import scipy.sparse as sps

    dtype = [np.float64, np.float32][rng.integers(0, 2)]
    n = int(rng.integers(1, 3000))
    ghosts = int(rng.integers(0, 50)) if rng.random() < 0.5 else 0
    rp, ci, v = rand_csr(rng, n, n + ghosts, np.float64)
    A = sps.csr_matrix((v, ci, rp), shape=(n, n + ghosts)).tolil()
    rowsum = np.asarray(abs(sps.csr_matrix((v, ci, rp), shape=(n, n + ghosts))).sum(axis=1)).ravel()
    A.setdiag(rowsum + 1.0 + rng.random(n))  # diagonally dominant, every row has its diagonal
    A = A.tocsr()
    if rng.random() < 0.5:
        A.sort_indices()
    rp, ci, v = A.indptr.astype(np.int32), A.indices.astype(np.int32), A.data.astype(dtype)
    ncols = n + ghosts
    compact, inner, outer = bool(rng.integers(0, 2)), int(rng.integers(0, 4)), int(rng.integers(1, 3))
    gamma = [1.0, 0.9][rng.integers(0, 2)]
    omega = [1.0, 0.9, 1.1][rng.integers(0, 3)]
    direction, init_zero, num_iter = int(rng.integers(0, 3)), bool(rng.integers(0, 2)), int(rng.integers(1, 3))
    b = rng.uniform(-1, 1, n).astype(dtype)
    x0 = rng.uniform(-1, 1, ncols).astype(dtype)
    grp, gci, gv, gb, gx = g(rp, rng), g(ci, rng), g(v, rng), g(b, rng), g(x0, rng)
    classic = rng.random() < 0.35  # the sptrsv form: triangular solves on A's own triangles (level sets), omega = 1 only
    plan = E.Gs2Plan(compact=compact, inner=inner, outer=outer, gamma=gamma)
    if classic:
        omega = 1.0
        E.ok(plan.set(5, 0.0))
        os.environ["B200SP_SPTRSV_GROUP"] = str([8, 16, 32][rng.integers(0, 3)])
    E.ok(plan.symbolic(n, ncols, grp, gci))
    E.ok(plan.numeric(n, ncols, grp, gci, gv))
    E.ok(plan.apply(n, ncols, grp, gci, gv, gx, gb, init_zero, omega, num_iter, direction))
    plan.close()
    os.environ.pop("B200SP_SPTRSV_GROUP", None)
    xo = x0.copy()
    if classic:
        orc.gs2_classic_apply(rp, ci, v, ncols, xo, b, init_zero, num_iter, direction, compact=compact, outer_sweeps=outer)
    else:
        orc.gs2_apply(rp, ci, v, ncols, xo, b, init_zero, dtype(omega), num_iter, direction, compact=compact, inner_sweeps=inner,
                      outer_sweeps=outer, gamma=dtype(gamma))
    tol = 1e-12 if dtype == np.float64 else 5e-5
    ok = bool(np.max(np.abs(gx.astype(np.float64) - xo.astype(np.float64)), initial=0.0) <= tol * max(1.0, np.max(np.abs(xo), initial=0.0)))
    return ok, f"gs2 {'classic ' if classic else ''}{np.dtype(dtype).name} n={n}+{ghosts} nnz={len(ci)} compact={compact} inner={inner} outer={outer} gamma={gamma} omega={omega} dir={direction}"


def op_spmv64(rng, orc, verbose):
    """64-bit offsets (spmv64.cu): random window limits, 32- or 64-bit columns, rank 1."""
    dtype = [np.float64, np.float32][rng.integers(0, 2)]
    big = rng.random() < 0.25
    m, n = int(rng.integers(0, 30000 if big else 4000)), int(rng.integers(1, 30000 if big else 4000))
    rp, ci, v = rand_csr(rng, m, n, dtype)
    rp64 = rp.astype(np.int64)
    ci_in = ci.astype(np.int64) if rng.random() < 0.5 else ci
    mode = "NNNCTH"[rng.integers(0, 6)]
    trans = mode in "TH"
    nx, ny = (m, n) if trans else (n, m)
    x = rng.uniform(-1, 1, nx).astype(dtype)
    y0 = rng.uniform(-1, 1, ny).astype(dtype)
    alpha, beta = [(1.0, 0.0), (2.5, -0.5), (-1.0, 1.0), (1.0, 0.0), (-0.3, 2.0), (2.5, 0.0), (1.0, 1.0), (0.0, 2.0)][rng.integers(0, 8)]
    longest = int(np.diff(rp).max()) if m > 0 else 0
    window = None
    if rng.random() < 0.8:  # at least the longest row (+3: the window's base is rounded down to a multiple of 4)
        window = int(max(8, longest + 3, len(ci) // 2000 + 8, rng.integers(8, max(9, len(ci) // int(rng.integers(1, 40)) + 9))))  # <= 4096 windows
    grp, gci, gv, gx, gy = g(rp64, rng), g(ci_in, rng), g(v, rng), g(x, rng), g(y0, rng)
    plan = E.Spmv64Plan(int(rng.integers(0, 3)), window=window)
    for _ in range(4 if rng.random() < 0.3 else 2):
        gy[...] = y0
        E.spmv64(plan, mode, m, n, grp, gci, gv, gx, gy, alpha, beta)
    kern, nw = plan.kernel(), plan.windows()
    plan.close()
    exp = orc.spmv_transpose(rp, ci, v, n, x, y0.copy(), alpha, beta) if trans else orc.spmv_serial(rp, ci, v, x, y0.copy(), alpha, beta)
    ok = scaled_ok(gy, exp, row_scale(rp, ci, v, x, y0, alpha, beta, n, trans), TOL[np.dtype(dtype)])
    return ok, f"spmv64 {mode} {np.dtype(dtype).name} {m}x{n} nnz={len(ci)} cols{8 * ci_in.dtype.itemsize} window={window} -> {nw}: {kern}"


def op_spmm(rng, orc, verbose):
    dtype = [np.float64, np.float32][rng.integers(0, 2)]
    m, n = int(rng.integers(0, 2500)), int(rng.integers(1, 2500))
    rp, ci, v = rand_csr(rng, m, n, dtype)
    k = int(rng.integers(1, 20))
    order = "CF"[rng.integers(0, 2)]
    mode = "NT"[rng.integers(0, 2)] if rng.random() < 0.3 else "N"
    trans = mode == "T"
    nx, ny = (m, n) if trans else (n, m)
    X = np.asarray(rng.uniform(-1, 1, (nx, k)).astype(dtype), order=order)
    Y0 = np.asarray(rng.uniform(-1, 1, (ny, k)).astype(dtype), order=order)
    alpha, beta = [(1.0, 0.0), (-2.0, 0.5), (1.0, 1.0)][rng.integers(0, 3)]
    grp, gci, gv = g(rp, rng), g(ci, rng), g(v, rng)
    gX, gY = E.guarded(X, 16 if rng.random() < 0.6 else None), E.guarded(Y0, 16 if rng.random() < 0.6 else None)
    plan = E.SpmvPlan()
    E.spmm(plan, mode, m, n, grp, gci, gv, gX, gY, alpha, beta)
    kern = plan.kernel()
    plan.close()
    Yc = Y0.copy(order=order)
    exp = orc.spmv_mv_transpose(rp, ci, v, n, X, Yc, alpha, beta) if trans else orc.spmv_mv(rp, ci, v, n, X, Yc, alpha, beta)
    ok = True
    for j in range(k):
        ok &= scaled_ok(gY[:, j], exp[:, j], row_scale(rp, ci, v, X[:, j], Y0[:, j], alpha, beta, n, trans), TOL[np.dtype(dtype)])
    return ok, f"spmm {mode} {np.dtype(dtype).name} {m}x{n} k={k} {order} kernel={kern}"


def op_spgemm(rng, orc, verbose):
    dtype = [np.float64, np.float32][rng.integers(0, 2)]
    m, k, n = int(rng.integers(0, 400)), int(rng.integers(1, 400)), int(rng.integers(1, 3000))
    A = rand_csr(rng, m, k, dtype, distinct=True, long_rows=False)
    B = rand_csr(rng, k, n, dtype, distinct=True, long_rows=bool(rng.random() < 0.3))
    A = (A[0], A[1], np.abs(A[2]) + dtype(0.5))
    B = (B[0], B[1], np.abs(B[2]) + dtype(0.5))
    num, sym = int(rng.integers(1, 7)), int(rng.integers(1, 3))
    os.environ["B200SP_SPGEMM_NUMERIC"], os.environ["B200SP_SPGEMM_SYMBOLIC"] = str(num), str(sym)
    gA = tuple(g(a, rng) for a in A)
    gB = tuple(g(b, rng) for b in B)
    L = E.lib()
    h = C.c_void_p()
    E.ok(L.b200sp_spgemm_plan_create(C.byref(h)))
    rpC = E.guarded(np.full(m + 1, 123, np.int32))
    nnz, mx = C.c_int64(), C.c_int()
    E.ok(L.b200sp_spgemm_symbolic_i32(h, None, m, k, n, E.ptr(gA[0]), E.ptr(gA[1]), E.ptr(gB[0]), E.ptr(gB[1]), E.ptr(rpC), C.byref(nnz), C.byref(mx)))
    ciC = E.guarded(np.full(nnz.value, -1, np.int32), 16 if rng.random() < 0.5 else None)
    vC = E.guarded(np.full(nnz.value, np.nan, dtype), 16 if rng.random() < 0.5 else None)
    fn = getattr(L, "b200sp_spgemm_numeric_%s_i32" % E.sfx(dtype))
    E.ok(fn(h, None, m, k, n, E.ptr(gA[0]), E.ptr(gA[1]), E.ptr(gA[2]), E.ptr(gB[0]), E.ptr(gB[1]), E.ptr(gB[2]), E.ptr(rpC), E.ptr(ciC), E.ptr(vC)))
    E.ok(L.b200sp_spgemm_plan_destroy(h, None))
    os.environ.pop("B200SP_SPGEMM_NUMERIC", None)
    os.environ.pop("B200SP_SPGEMM_SYMBOLIC", None)
    exp = orc.spgemm(*A, *B, n)
    eps = 1e-7 if dtype == np.float64 else 3.7e-3
    ok = np.array_equal(rpC, exp[0]) and np.array_equal(ciC, exp[1]) and orc.rel_mismatch(vC.astype(np.float64), exp[2].astype(np.float64), eps) == 0
    return ok, f"spgemm {np.dtype(dtype).name} {m}x{k}x{n} c_nnz={nnz.value} numeric_v{num} symbolic_v{sym}"


def op_crs(rng, orc, verbose):
    dtype = [np.float64, np.float32][rng.integers(0, 2)]
    m, n = int(rng.integers(0, 1500)), int(rng.integers(1, 800))
    L = E.lib()
    which = rng.integers(0, 4)
    s = E.sfx(dtype)
    if which == 0:  # sort
        rp, ci, v = rand_csr(rng, m, n, dtype)
        grp, gci, gv = g(rp, rng), g(ci, rng), g(v, rng)
        E.ok(getattr(L, f"b200sp_sort_crs_{s}_i32")(None, m, E.ptr(grp), E.ptr(gci), E.ptr(gv)))
        eci, ev = ci.copy(), v.copy()
        orc.sort_crs_stable(rp, eci, ev)
        return np.array_equal(gci, eci) and np.array_equal(gv, ev), f"sort_crs {s} {m}x{n} nnz={len(ci)}"
    if which == 1:  # sort_and_merge
        rp, ci, v = rand_csr(rng, max(m, 1), n, dtype)
        m = len(rp) - 1
        grp, gci, gv = g(rp, rng), g(ci, rng), g(v, rng)
        orp = E.guarded(np.zeros(m + 1, np.int32))
        nnz = C.c_int64()
        E.ok(getattr(L, f"b200sp_sort_and_merge_count_{s}_i32")(None, m, E.ptr(grp), E.ptr(gci), E.ptr(gv), E.ptr(orp), C.byref(nnz)))
        oci, ov = E.guarded(np.zeros(nnz.value, np.int32)), E.guarded(np.zeros(nnz.value, dtype))
        E.ok(getattr(L, f"b200sp_sort_and_merge_fill_{s}_i32")(None, m, E.ptr(grp), E.ptr(gci), E.ptr(gv), E.ptr(orp), E.ptr(oci), E.ptr(ov)))
        exp = orc.sort_and_merge(rp.copy(), ci.copy(), v.copy())
        return np.array_equal(orp, exp[0]) and np.array_equal(oci, exp[1]) and np.array_equal(ov, exp[2]), f"sort_and_merge {s} {m}x{n} nnz={len(ci)}->{nnz.value}"
    if which == 2:  # transpose (f64 oracle)
        rp, ci, v = rand_csr(rng, m, n, np.float64)
        grp, gci, gv = g(rp, rng), g(ci, rng), g(v, rng)
        trp, tci, tv = E.guarded(np.zeros(n + 1, np.int32)), E.guarded(np.zeros(len(ci), np.int32)), E.guarded(np.zeros(len(ci)))
        E.ok(L.b200sp_transpose_f64_i32(None, m, n, E.ptr(grp), E.ptr(gci), E.ptr(gv), E.ptr(trp), E.ptr(tci), E.ptr(tv)))
        e = orc.transpose(rp, ci, v, n)
        return np.array_equal(trp, e[0]) and np.array_equal(tci, e[1]) and np.array_equal(tv, e[2]), f"transpose {m}x{n} nnz={len(ci)}"
    sorted_in = bool(rng.integers(0, 2))  # spadd
    A = rand_csr(rng, m, n, dtype, sort=sorted_in, distinct=sorted_in, long_rows=False)
    B = rand_csr(rng, m, n, dtype, sort=sorted_in, distinct=sorted_in, long_rows=False)
    gA, gB = tuple(g(a, rng) for a in A), tuple(g(b, rng) for b in B)
    h = C.c_void_p()
    E.ok(L.b200sp_spadd_plan_create(C.byref(h), int(sorted_in), 0))
    rpC = E.guarded(np.zeros(m + 1, np.int32))
    nnz = C.c_int64()
    E.ok(L.b200sp_spadd_symbolic_i32(h, None, m, n, E.ptr(gA[0]), E.ptr(gA[1]), E.ptr(gB[0]), E.ptr(gB[1]), E.ptr(rpC), C.byref(nnz)))
    ciC, vC = E.guarded(np.zeros(nnz.value, np.int32)), E.guarded(np.zeros(nnz.value, dtype))
    E.ok(getattr(L, f"b200sp_spadd_numeric_{s}_i32")(h, None, m, n, E.ptr(gA[0]), E.ptr(gA[1]), E.ptr(gA[2]), E.scalar(dtype, 0.3), E.ptr(gB[0]),
                                                    E.ptr(gB[1]), E.ptr(gB[2]), E.scalar(dtype, -1.7), E.ptr(rpC), E.ptr(ciC), E.ptr(vC)))
    E.ok(L.b200sp_spadd_plan_destroy(h, None))
    exp = orc.spadd(*A, 0.3, *B, -1.7, sorted_in)
    return np.array_equal(rpC, exp[0]) and np.array_equal(ciC, exp[1]) and np.array_equal(vC, exp[2]), f"spadd sorted={sorted_in} {s} {m}x{n} c_nnz={nnz.value}"


def op_bsr(rng, orc, verbose):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from bsr_cases import bsr_random, op_max_nnz_per_row, tolerance

    dtype = [np.float64, np.float32][rng.integers(0, 2)]
    bs = int(rng.integers(1, 19))
    mb, nb = int(rng.integers(0, 2500 // bs + 2)), int(rng.integers(1, 2500 // bs + 2))
    rp, ci, v = bsr_random(bs, mb, nb, seed=int(rng.integers(0, 1 << 30)), dtype=dtype, max_blocks=int(rng.integers(1, 30)), sort=False)
    if mb > 3 and nb > 40 and rng.random() < 0.4:  # a long block row
        lens = np.diff(rp)
        lens[rng.integers(0, mb)] = min(nb, int(rng.integers(60, 900)))
        rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
        ci = np.concatenate([rng.choice(nb, int(l), replace=False) for l in lens]).astype(np.int32)
        v = rng.uniform(0, 10, len(ci) * bs * bs).astype(dtype)
    mode = "NNNNCTH"[rng.integers(0, 7)]
    trans = mode in "TH"
    nx, ny = (mb * bs, nb * bs) if trans else (nb * bs, mb * bs)
    alpha, beta = [(1.0, 0.0), (3.7, -1.5), (-1.0, 1.0), (3.7, 0.0), (1.0, 1.0), (-1.0, -1.5), (1.0, 0.0), (0.0, -1.0)][rng.integers(0, 8)]
    grp, gci, gv = g(rp, rng), g(ci, rng), g(v, rng)
    plan = E.BsrPlan()
    knob = [None, None, "walk", "vector"][rng.integers(0, 4)]
    if knob:
        os.environ["B200SP_BSR_KERNEL"] = knob
    k = 1 if rng.random() < 0.6 else int(rng.integers(1, 9))
    if k == 1 and rng.random() < 0.8:
        x, y0 = rng.uniform(0, 10, nx).astype(dtype), rng.uniform(0, 10, ny).astype(dtype)
        gx, gy = g(x, rng), g(y0, rng)
        E.bsr_spmv(plan, mode, mb, nb, bs, grp, gci, gv, gx, gy, alpha, beta)
        X, Y0, got = x, y0, gy
    else:
        order = "CF"[rng.integers(0, 2)]
        X = np.asarray(rng.uniform(0, 10, (nx, k)).astype(dtype), order=order)
        Y0 = np.asarray(rng.uniform(0, 10, (ny, k)).astype(dtype), order=order)
        gX, gY = E.guarded(X), E.guarded(Y0)
        E.bsr_spmm(plan, mode, mb, nb, bs, grp, gci, gv, gX, gY, alpha, beta)
        got = gY
    kern = plan.kernel()
    plan.close()
    os.environ.pop("B200SP_BSR_KERNEL", None)
    Yc = Y0.copy(order="K")
    exp = orc.bsr_spmv_v41(mode, bs, nb, rp, ci, v, X, Yc, alpha, beta) if trans else orc.bsr_spmv_v42(bs, rp, ci, v, X, Yc, alpha, beta)
    tol = tolerance(dtype, alpha, beta, op_max_nnz_per_row(bs, rp, ci, nb, trans))
    ok = bool(np.max(np.abs(got - exp), initial=0.0) <= tol)
    return ok, f"bsr {mode} {np.dtype(dtype).name} bs={bs} {mb}x{nb} nnzb={len(ci)} k={k} {kern}"


def op_gs(rng, orc, verbose):
    """Point Gauss-Seidel: colouring (symmetric or not), inverse diagonal, sweeps in every direction against the oracle over the
    library's own colour sets."""
    dtype = [np.float64, np.float32][rng.integers(0, 2)]
    n = int(rng.integers(1, 1500))
    rp, ci, v = rand_csr(rng, n, n, np.float64, sort=True, distinct=True, long_rows=bool(rng.random() < 0.3))
    # put a dominant diagonal into every row (merge it into the sorted row)
    rows = []
    for i in range(n):
        c = set(ci[rp[i]:rp[i + 1]].tolist()) | {i}
        rows.append(np.array(sorted(c), dtype=np.int32))
    rp = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
    ci = np.concatenate(rows).astype(np.int32)
    rid = np.repeat(np.arange(n), np.diff(rp))
    v = rng.uniform(-1, 1, len(ci))
    v[rid == ci] = np.bincount(rid, weights=np.abs(v), minlength=n) + 1.0
    v = v.astype(dtype)
    grp, gci, gv = g(rp, rng), g(ci, rng), g(v, rng)
    plan = E.GsPlan()
    plan.symbolic(n, grp, gci, False)
    nc, colors, cptr, crows = plan.coloring(n)
    ok = not np.any((colors[rid] == colors[ci]) & (rid != ci)) and cptr[-1] == n and np.array_equal(np.sort(crows), np.arange(n))
    # symmetrised check: colours of (j, i) for every (i, j) differ as well
    ok &= E.lib().b200sp_gs_numeric_f64_i32(plan.h, None, n, E.ptr(grp), E.ptr(gci), E.ptr(gv)) == 0 if dtype == np.float64 else plan.numeric(n, grp, gci, gv) == 0
    y = rng.uniform(-1, 1, n).astype(dtype)
    gy = g(y, rng)
    direction, sweeps = int(rng.integers(0, 3)), int(rng.integers(1, 4))
    omega = [1.0, 0.9, 1.3][rng.integers(0, 3)]
    x = E.guarded(rng.uniform(-1, 1, n).astype(dtype))
    x0 = x.copy()
    init_zero = bool(rng.integers(0, 2))
    ok &= plan.apply(n, grp, gci, gv, x, gy, init_zero, omega, sweeps, direction) == 0
    plan.close()
    dinv = (1.0 / v[rid == ci].astype(np.float64)).astype(dtype)
    xo = orc.gs_apply(rp, ci, v, cptr, crows, dinv, y, x0.copy(), init_zero, dtype(omega), sweeps, direction)
    tol = 1e-11 if dtype == np.float64 else 5e-5
    ok &= bool(np.max(np.abs(x.astype(np.float64) - xo.astype(np.float64)), initial=0.0) <= tol * max(1.0, float(np.max(np.abs(xo), initial=0.0))))
    return ok, f"gs {np.dtype(dtype).name} n={n} nnz={len(ci)} colors={nc} dir={direction} sweeps={sweeps}"


def op_sptrsv(rng, orc, verbose):
    """Level-set triangular solve: a random lower / upper triangular matrix (unsorted rows, the diagonal anywhere in its row, long
    dependency chains or wide levels, sometimes a hub row), lane groups of 8 / 16 / 32 and chaining on / off, bit for bit against
    the oracle's serial substitution."""
    dtype = [np.float64, np.float32][rng.integers(0, 2)]
    n = int(rng.integers(1, 1200))
    lower = bool(rng.integers(0, 2))
    band = int(rng.integers(1, max(2, n)))  # narrow band: long chains of small levels; wide: few large levels
    rows = []
    for i in range(n):
        k = int(rng.integers(0, 6)) if rng.random() < 0.9 else int(rng.integers(20, 90))
        lo, hi = (max(0, i - band), i) if lower else (i + 1, min(n, i + 1 + band))
        cand = np.arange(lo, hi)
        deps = rng.choice(cand, min(k, len(cand)), replace=False) if len(cand) else np.zeros(0, np.int64)
        cols = np.concatenate([deps, [i]]).astype(np.int32)
        rows.append(cols[rng.permutation(len(cols))])
    rp = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
    ci = np.concatenate(rows).astype(np.int32)
    rid = np.repeat(np.arange(n), np.diff(rp))
    v = rng.uniform(-0.5, 0.5, len(ci))
    v[rid == ci] = rng.uniform(1.0, 2.0, n) * np.where(rng.random(n) < 0.5, 1.0, -1.0)
    v = v.astype(dtype)
    b = rng.uniform(-1, 1, n).astype(dtype)
    os.environ["B200SP_SPTRSV_GROUP"] = str([8, 16, 32][rng.integers(0, 3)])
    os.environ["B200SP_SPTRSV_CHAIN"] = str(int(rng.integers(0, 2)))
    L = E.lib()
    grp, gci, gv, gb = g(rp, rng), g(ci, rng), g(v, rng), g(b, rng)
    x = E.guarded(np.full(n, np.nan, dtype))
    h = C.c_void_p()
    E.ok(L.b200sp_sptrsv_plan_create(C.byref(h)))
    E.ok(L.b200sp_sptrsv_symbolic_i32(h, None, n, E.ptr(grp), E.ptr(gci), int(lower)))
    levels, launches = L.b200sp_sptrsv_levels(h), L.b200sp_sptrsv_launches(h)
    E.ok(getattr(L, f"b200sp_sptrsv_solve_{E.sfx(dtype)}_i32")(h, None, n, E.ptr(grp), E.ptr(gci), E.ptr(gv), E.ptr(gb), E.ptr(x)))
    E.ok(L.b200sp_sptrsv_plan_destroy(h, None))
    os.environ.pop("B200SP_SPTRSV_GROUP", None)
    os.environ.pop("B200SP_SPTRSV_CHAIN", None)
    exp = orc.sptrsv(rp, ci, v, b, lower)
    ok = np.array_equal(np.asarray(x).view(np.uint8), exp.view(np.uint8)) and 1 <= levels <= n and 1 <= launches <= levels
    return ok, f"sptrsv {np.dtype(dtype).name} n={n} nnz={len(ci)} lower={lower} band={band} levels={levels} launches={launches}"


OPS = {"gs": op_gs, "gs2": op_gs2, "spmv": op_spmv, "spmv64": op_spmv64, "spmm": op_spmm, "spgemm": op_spgemm, "crs": op_crs, "bsr": op_bsr,
       "sptrsv": op_sptrsv}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seeds", default="0:50")
    ap.add_argument("--ops", default=",".join(OPS))
    ap.add_argument("-v", action="store_true")
    a = ap.parse_args()
    lo, hi = (int(t) for t in a.seeds.split(":"))
    ops = a.ops.split(",")
    orc = oracle_lib.Oracle()
    bad = 0
    L = E.lib()
    L.b200emu_live_allocations.restype = C.c_longlong
    L.b200emu_live_allocations.argtypes = [C.c_void_p]
    for seed in range(lo, hi):
        for name in ops:
            rng = np.random.default_rng([seed, sorted(OPS).index(name)])
            print(f"[fuzz] seed {seed} {name} ...", end=" ", flush=True)  # printed BEFORE the call: a fault names its seed
            live0 = L.b200emu_live_allocations(None)
            ok, what = OPS[name](rng, orc, a.v)
            E.guarded_release()
            leaked = L.b200emu_live_allocations(None) - live0  # plans are closed inside the op: nothing may stay allocated
            if leaked:
                ok, what = False, what + f"  LEAK: {leaked} device blocks still allocated"
            print(("ok   " if ok else "MISMATCH ") + what, flush=True)
            bad += 0 if ok else 1
    print(f"[fuzz] seeds {lo}:{hi} ops {','.join(ops)}: {bad} mismatches")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
