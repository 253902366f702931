"""Device-memory accounting under the CPU emulation (tools/emu counts live cudaMalloc / cudaMallocAsync / cudaMallocHost blocks):
whatever a call sequence allocates -- plan analyses, windows, cached transposes, solver work vectors, temporaries of the
stateless entry points, also on the error paths -- is given back when the plans are destroyed.  A leak here is HBM a
long-running solver never gets back; no GPU tool in this image reports it."""
import ctypes as C

import numpy as np
import pytest

import emu_lib as E
from bsr_cases import bsr_random
from gmres_cases import gmres_matrix
from test_emulated_spmv64 import random_crs


@pytest.fixture(scope="module")
def emu():
    return E.lib()


def live(emu):
    emu.b200emu_live_allocations.restype = C.c_longlong
    emu.b200emu_live_allocations.argtypes = [C.POINTER(C.c_longlong)]
    b = C.c_longlong(0)
    n = emu.b200emu_live_allocations(C.byref(b))
    return n, b.value


class balanced:
    def __init__(self, emu, what):
        self.emu, self.what = emu, what

    def __enter__(self):
        self.before = live(self.emu)

    def __exit__(self, et, ev, tb):
        if et is None:
            after = live(self.emu)
            assert after == self.before, f"{self.what}: {after[0] - self.before[0]} blocks / {after[1] - self.before[1]} bytes still allocated"


def test_spmv_plans_give_everything_back(emu):
    m, n = 9000, 7000
    rp64, ci, v = random_crs(m, n, 9.0, seed=3, long_rows=3)
    rp = rp64.astype(np.int32)
    rng = np.random.default_rng(0)
    x, xt = rng.random(n), rng.random(m)
    with balanced(emu, "rank-1 plan (tile analysis, long rows, self-tuning, segments)"):
        p = E.SpmvPlan()
        y = np.zeros(m)
        for _ in range(5):
            E.spmv(p, "N", m, n, rp, ci, v, x, y, 1.0, 0.0)
        p.close()
    with balanced(emu, "cached transpose"):
        p = E.SpmvPlan()
        E.ok(emu.b200sp_spmv_plan_set_option(p.h, 1, 1))
        yt = np.zeros(n)
        for _ in range(2):
            E.spmv(p, "T", m, n, rp, ci, v, xt, yt, 1.0, 0.0)
        p.close()
    with balanced(emu, "rank-2 plan (relayout scratch, tile analysis, chunk table)"):
        p = E.SpmvPlan()
        for order in "CF":
            X = np.asarray(rng.random((n, 5)), order=order)
            Y = np.asarray(np.zeros((m, 5)), order=order)
            E.spmm(p, "N", m, n, rp, ci, v, X, Y, 1.0, 0.0)
        p.close()
    with balanced(emu, "64-bit offsets: windows, relative row maps, narrowed columns, one plan per window; re-analysis; error paths"):
        p = E.Spmv64Plan(window=20000)
        y = np.zeros(m)
        c64 = ci.astype(np.int64)
        E.spmv64(p, "N", m, n, rp64, c64, v, x, y, 1.0, 0.0)
        E.ok(emu.b200sp_spmv64_plan_set_window(p.h, 5000))
        E.spmv64(p, "N", m, n, rp64, c64, v, x, y, 1.0, 0.0)  # analysed again: the old windows are released
        E.ok(emu.b200sp_spmv64_plan_set_window(p.h, 8))
        assert E.spmv64_rc(p, "N", m, n, rp64, c64, v, x, y, 1.0, 0.0) == 4  # a row does not fit: refused
        bad = c64.copy()
        bad[5] = 2**40
        E.ok(emu.b200sp_spmv64_plan_set_window(p.h, 5000))
        assert E.spmv64_rc(p, "N", m, n, rp64, bad, v, x, y, 1.0, 0.0) == 4
        p.close()


def test_spgemm_crs_utilities_and_bsr(emu):
    m = 3000
    rp64, ci, v = random_crs(m, m, 8.0, seed=5)
    rp = rp64.astype(np.int32)
    with balanced(emu, "spgemm symbolic + numeric (handle created and destroyed inside)"):
        E.spgemm((rp, ci, v), (rp, ci, v), m, m, m, np.float64)
    with balanced(emu, "BsrMatrix plan (tile analysis, long block rows, transposed, multivector)"):
        bs, mb, nb = 3, 900, 700
        brp, bci, bv = bsr_random(bs, mb, nb, seed=2, dtype=np.float64, sort=True)
        p = E.BsrPlan()
        rng = np.random.default_rng(1)
        y = np.zeros(mb * bs)
        E.bsr_spmv(p, "N", mb, nb, bs, brp, bci, bv, rng.random(nb * bs), y, 1.0, 0.0)
        yt = np.zeros(nb * bs)
        E.bsr_spmv(p, "T", mb, nb, bs, brp, bci, bv, rng.random(mb * bs), yt, 1.0, 0.0)
        Y = np.zeros((mb * bs, 4))
        E.bsr_spmm(p, "N", mb, nb, bs, brp, bci, bv, rng.random((nb * bs, 4)), Y, 1.0, 0.0)
        p.close()


def test_solvers(emu):
    n = 2500
    rp, ci, v = gmres_matrix(n, 1.0, seed=7)
    import scipy.sparse as sps

    S = sps.csr_matrix((v, ci, rp), shape=(n, n))
    S = ((S + S.T) * 0.5 + sps.identity(n) * 2.0).tocsr()
    S.sort_indices()
    srp, sci, sv = S.indptr.astype(np.int32), S.indices.astype(np.int32), S.data.copy()
    b = np.ones(n)
    with balanced(emu, "CG (device-resident state, work vectors)"):
        p = E.SpmvPlan()
        E.cg_solve(p, srp, sci, sv, b, np.zeros(n), 50, 1e-10)
        p.close()
    with balanced(emu, "Gauss-Seidel plan (colouring, row lists, inverse diagonal) and PCG"):
        g, p = E.GsPlan(), E.SpmvPlan()
        g.symbolic(n, srp, sci, True)
        assert g.numeric(n, srp, sci, sv) == 0
        x = np.zeros(n)
        assert g.apply(n, srp, sci, sv, x, b, True, 1.0, 2, 0) == 0
        g.symbolic(n, srp, sci, True)  # a second symbolic replaces the first
        assert g.numeric(n, srp, sci, sv) == 0
        E.pcg_solve(p, g, srp, sci, sv, b, np.zeros(n), 50, 1e-10)
        g.close()
        p.close()
    with balanced(emu, "two-stage Gauss-Seidel plan (L, U, La, Ua, diagonals, work vectors, five SpMV plans); re-symbolic; error path"):
        g2 = E.Gs2Plan(compact=True, inner=2)
        assert g2.symbolic(n, n, srp, sci) == 0 and g2.numeric(n, n, srp, sci, sv) == 0
        assert g2.apply(n, n, srp, sci, sv, np.zeros(n), b, True, 0.9, 2, 0) == 0
        assert g2.set(1, 0.0) == 0  # classic form: symbolic again
        assert g2.symbolic(n, n, srp, sci) == 0 and g2.numeric(n, n, srp, sci, sv.astype(np.float32)) == 0
        assert g2.symbolic(3, 3, np.array([0, 1, 2, 3], np.int32), np.array([0, 0, 2], np.int32)) == 1  # no diagonal in row 1
        g2.close()
    with balanced(emu, "GMRES (Krylov basis, Hessenberg scratch)"):
        p = E.SpmvPlan()
        E.gmres(p, (rp, ci, v), b, np.zeros(n), m=15, tol=1e-8, max_restart=5, ortho=0)
        E.gmres(p, (rp, ci, v), b, np.zeros(n), m=15, tol=1e-8, max_restart=5, ortho=1)
        p.close()


def test_stateless_entry_points_and_pipelines(emu, oracle):
    """The cases of tests/test_emulated_kernels.py once more, each bracketed by the accounting (their plans are closed inside)."""
    import test_emulated_kernels as K

    with balanced(emu, "sort_and_merge"):
        for case in range(len(K.MERGE_CASES)):
            try:
                K.test_sort_and_merge_golden(emu, case)
            except pytest.skip.Exception:
                pass
    with balanced(emu, "sort_crs / transpose"):
        K.test_sort_transpose(emu, oracle)
    for sorted_input in (True, False):
        with balanced(emu, f"spadd sorted={sorted_input}"):
            K.test_spadd(emu, oracle, sorted_input, np.float64)
    with balanced(emu, "spgemm_jacobi"):
        K.test_spgemm_jacobi(emu, oracle)
    with balanced(emu, "spgemm, rows wider than the shared-memory tables (global scratch)"):
        K.test_spgemm_wide_rows_global_fallback(emu, oracle)
    with balanced(emu, "host-vector pipeline (double-buffered staging vectors)"):
        K.test_hostvec_pipeline_logic(emu, oracle, 4)
    with balanced(emu, "multi-GPU kernels in one process"):
        K.test_multi_gpu_kernels_single_process(emu, oracle)


def hostvec(emu, p, mode, m, n, rp, ci, v, x, y, alpha, beta):
    E.ok(emu.b200sp_spmv_hostvec_f64_i32(p.h, None, mode.encode(), m, n, len(ci), alpha, E.ptr(rp), E.ptr(ci), E.ptr(v), E.ptr(x), beta,
                                         E.ptr(y)))


def test_spmv_plan_parts_give_everything_back(emu):
    """each part of the SpMV plan that no bracket above reaches: long-row segments, the pattern form's tile table and the cfg's
    cut again, the simple host-vector path, and every part built again after invalidate"""
    from test_emulated_kernels import env
    import pattern_cases as PC

    m, n = 9000, 7000
    rp64, ci, v = random_crs(m, n, 9.0, seed=3, long_rows=3)
    rp = rp64.astype(np.int32)
    rng = np.random.default_rng(4)
    x, xt = rng.random(n), rng.random(m)
    with balanced(emu, "long-row segments (B200SP_SPMV_LONGROWS=seg)"), env(B200SP_SPMV_LONGROWS="seg"):
        p = E.SpmvPlan()
        y = np.zeros(m)
        for _ in range(4):
            E.spmv(p, "N", m, n, rp, ci, v, x, y, 1.0, 0.0)
            assert p.kernel().endswith("+seg"), p.kernel()
        p.close()
    with balanced(emu, "pattern tile table -> cfg tile table -> pattern tile table on one plan"):
        A = PC.lap_case("dof2")
        ya = np.zeros(len(A[0]) - 1)
        p = E.SpmvPlan()
        for idx16 in (None, "0", None):
            with env(B200SP_SPMV_IDX16=idx16, B200SP_NO_AUTOTUNE=1):
                E.spmv(p, "N", len(A[0]) - 1, A[3], A[0], A[1], A[2], np.ones(A[3]), ya, 1.0, 0.0)
            assert ("COLS=pat" in p.kernel()) == (idx16 is None), p.kernel()
        p.close()
    with balanced(emu, "simple host-vector path (staging vectors)"):
        p = E.SpmvPlan()
        for mode, xv, ylen in (("N", x, m), ("T", xt, n), ("N", x, m)):
            hostvec(emu, p, mode, m, n, rp, ci, v, xv, np.zeros(ylen), 1.0, 0.0)
        p.close()
    with balanced(emu, "invalidate, then every part built again"):
        p = E.SpmvPlan()
        E.ok(emu.b200sp_spmv_plan_set_option(p.h, 1, 1))
        for _ in range(2):
            with env(B200SP_SPMV_LONGROWS="seg"):
                for _ in range(4):
                    E.spmv(p, "N", m, n, rp, ci, v, x, np.zeros(m), 1.0, 0.0)
            E.spmv(p, "T", m, n, rp, ci, v, xt, np.zeros(n), 1.0, 0.0)
            for order in "CF":
                E.spmm(p, "N", m, n, rp, ci, v, np.asarray(rng.random((n, 5)), order=order), np.zeros((m, 5), order=order), 1.0, 0.0)
            hostvec(emu, p, "N", m, n, rp, ci, v, x, np.zeros(m), 1.0, 0.0)
            E.ok(emu.b200sp_spmv_plan_invalidate(p.h, None))
        p.close()


def test_hostvec_pipeline_follows_col_idx(emu):
    """one plan, one structure, three col_idx arrays: the pattern form, a copy of it at another address, and columns that only
    qualify for the deltas; and a call on the 32-bit columns between two pattern calls, after which the plan holds both tile
    tables.  The piece bounds follow the table each call launches on."""
    from test_emulated_kernels import env
    import pattern_cases as PC

    rp, ci, v, ncols = PC.lap27(36, 36, 36, 2)
    m = len(rp) - 1
    assert len(ci) >= (1 << 22)  # the pipeline
    assert PC.expected_cols((rp, ci, v, ncols), 512) == "pat"
    ci_delta = PC.random_rows(rp, ncols)
    assert PC.expected_cols((rp, ci_delta, v, ncols), 512) == "delta"
    x = np.random.default_rng(5).uniform(-1, 1, ncols)
    with balanced(emu, "host-vector pipeline over changing col_idx"):
        p = E.SpmvPlan()
        for cols, idx16 in ((ci, None), (ci, None), (ci, "0"), (ci, None), (ci.copy(), None), (ci_delta, None), (ci, None)):
            y = np.full(m, np.nan)
            with env(B200SP_SPMV_IDX16=idx16):
                hostvec(emu, p, "N", m, ncols, rp, cols, v, x, y, 1.0, 0.0)
            ref = E.SpmvPlan()
            yr = np.full(m, np.nan)
            E.spmv(ref, "N", m, ncols, rp, cols, v, x, yr, 1.0, 0.0)
            ref.close()
            assert np.array_equal(y, yr), idx16
        p.close()
