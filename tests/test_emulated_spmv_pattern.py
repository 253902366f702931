"""The tiled SpMV kernel's pattern form (one 16-bit pattern start per row into a dictionary of in-row column offsets, plus one
anchor column per row, DESIGN.md section 3.6) under the CPU emulation: which matrices take it, that it gives the same bits as
the 32-bit columns, the delta form and the row-vector kernel, and what the plan holds.  Every call that picks a form asserts
it through last_kernel()."""
import ctypes as C

import numpy as np
import pytest

import emu_lib as E
import pattern_cases as K
from helpers import rowwise_scale
from test_emulated_kernels import env
from test_emulated_leaks import live


@pytest.fixture(scope="module")
def emu():
    return E.lib()


def plan(cfg=-1, lpr=-1, ctas=-1, algo=0):
    p = E.SpmvPlan(algo)
    E.ok(E.lib().b200sp_spmv_plan_tune(p.h, cfg, lpr, ctas))
    return p


def call(p, A, x, y0, alpha, beta):
    rp, ci, v, ncols = A
    y = y0.copy()
    E.spmv(p, "N", len(rp) - 1, ncols, rp, ci, v.astype(x.dtype), x, y, alpha, beta)
    return y, p.kernel()


def inputs(A, beta, seed=0, dtype=np.float64):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-1, 1, A[3]).astype(dtype)
    y0 = rng.uniform(-1, 1, len(A[0]) - 1).astype(dtype)
    if beta == 0.0:
        y0[::7] = np.nan
    return x, y0


def check_oracle(oracle, A, x, y0, alpha, beta, y):
    rp, ci, v, _ = A
    v = v.astype(x.dtype)
    exp = oracle.spmv_serial(rp, ci, v, x, y0.copy(), alpha, beta)
    scale = rowwise_scale(rp, ci, v, x, y0, alpha, beta)
    tol = 1e-10 if x.dtype == np.float64 else 1e-4
    assert not np.isnan(y).any()
    assert np.all(np.abs(y - exp) <= tol * scale + 1e-300)


def three_forms(p, A, x, y0, alpha, beta):
    """the pattern handle's result, and those of the 32-bit columns and of a handle built under B200SP_SPMV_PATTERN=0"""
    y, k = call(p, A, x, y0, alpha, beta)
    with env(B200SP_SPMV_IDX16="0"):
        y32, k32 = call(p, A, x, y0, alpha, beta)
    assert "IDX=i32" in k32, k32
    with env(B200SP_SPMV_PATTERN="0"):
        pd = plan(p.cfg, p.lpr, 1)
        yd, kd = call(pd, A, x, y0, alpha, beta)
        pd.close()
    return y, k, y32, yd, kd


def tuned(cfg, lpr=-1, ctas=1):
    p = plan(cfg, lpr, ctas)
    p.cfg, p.lpr = cfg, lpr
    return p


@pytest.mark.parametrize("case", ["dof1", "dof2", "dof3", "flat2", "flat3", "shard"])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_lap27_pattern_same_bits(emu, oracle, case, dtype):
    A = K.lap_case(case)
    assert K.expected_cols(A, 512) == "pat"
    for alpha, beta in K.AB:
        x, y0 = inputs(A, beta, dtype=dtype)
        pv = plan(lpr=4, algo=1)
        yv, kv = call(pv, A, x, y0, alpha, beta)
        pv.close()
        assert kv.startswith("vector"), kv
        p = tuned(8, 4)
        y, k, y32, yd, kd = three_forms(p, A, x, y0, alpha, beta)
        p.close()
        assert "IDX=u16,COLS=pat" in k, k
        assert "IDX=u16,COLS=delta" in kd, kd
        check_oracle(oracle, A, x, y0, alpha, beta, y)
        assert np.array_equal(y, y32) and np.array_equal(y, yd) and np.array_equal(y, yv), (alpha, beta)


@pytest.mark.parametrize("lpr", [2, 4, 8, 16, 32])
def test_lap27_every_lpr_and_ring(emu, oracle, lpr):
    A = K.lap_case("dof2")
    x, y0 = inputs(A, 1.3)
    ref = None
    for cfg in (0, 1, 2, 3, 4, 8):
        p = tuned(cfg, lpr)
        y, k, y32, yd, kd = three_forms(p, A, x, y0, -0.7, 1.3)
        p.close()
        assert "COLS=pat" in k and f"LPR={lpr}," in k, k
        assert "COLS=delta" in kd, kd
        assert np.array_equal(y, y32) and np.array_equal(y, yd), cfg
        ref = y if ref is None else ref
        assert np.array_equal(y, ref), cfg
    check_oracle(oracle, A, x, y0, -0.7, 1.3, ref)


@pytest.mark.parametrize("total,form", [(K.DCAP, "pat"), (K.DCAP + 1, "delta")])
def test_dictionary_boundary(emu, oracle, total, form):
    A = K.dict_matrix(total)
    assert K.expected_cols(A, 512) == form
    x, y0 = inputs(A, 0.0)
    p = tuned(8)
    y, k, y32, yd, _ = three_forms(p, A, x, y0, 1.0, 0.0)
    p.close()
    assert f"COLS={form}" in k, k
    check_oracle(oracle, A, x, y0, 1.0, 0.0, y)
    assert np.array_equal(y, y32) and np.array_equal(y, yd)


@pytest.mark.parametrize("name", ["near_patterns_matrix", "diagonal_matrix", "long_rows_matrix", "empty_rows_matrix"])
@pytest.mark.parametrize("cfg", [3, 8])
def test_special_matrices(emu, oracle, name, cfg):
    A = getattr(K, name)()
    assert K.expected_cols(A, K.LMAX[cfg]) == "pat"
    for lpr in (2, 8):
        for alpha, beta in K.AB:
            x, y0 = inputs(A, beta, seed=1)
            p = tuned(cfg, lpr)
            y, k, y32, yd, _ = three_forms(p, A, x, y0, alpha, beta)
            p.close()
            assert "COLS=pat" in k, k
            check_oracle(oracle, A, x, y0, alpha, beta, y)
            assert np.array_equal(y, y32) and np.array_equal(y, yd), (lpr, alpha, beta)


def test_new_col_idx_same_row_ptr(emu, oracle):
    """the streams are keyed on col_idx: lap27, the shifted lap27, random rows and lap27 again under one row_ptr array"""
    rp, ci, v, n = A1 = K.lap27(8, 7, 6)
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    ci2 = ((ci.astype(np.int64) + 2 * rows) % n).astype(np.int32)
    for r in range(len(rp) - 1):
        ci2[rp[r]:rp[r + 1]].sort()
    ci3 = K.random_rows(rp, n)
    x, y0 = inputs(A1, 0.0)
    p = tuned(8)
    for A in (A1, (rp, ci2, v, n), (rp, ci3, v, n), A1):
        form = K.expected_cols(A, 512)
        y, k = call(p, A, x, y0, 1.0, 0.0)
        assert f"IDX=u16,COLS={form}" in k, (form, k)
        check_oracle(oracle, A, x, y0, 1.0, 0.0, y)
    assert [K.expected_cols(A, 512) for A in (A1, (rp, ci3, v, n))] == ["pat", "delta"]
    p.close()


def test_plan_memory(emu):
    """the deltas go once the pattern form is chosen (on the next call); invalidate and destroy release everything"""
    A = K.lap27(8, 7, 6)
    m, nnz = len(A[0]) - 1, len(A[1])
    x, y0 = inputs(A, 0.0)
    before = live(emu)[1]
    with env(B200SP_SPMV_IDX16="0"):
        p = tuned(8)
        call(p, A, x, y0, 1.0, 0.0)
        held32 = live(emu)[1] - before
        p.close()
    p = tuned(8)
    for i in range(3):
        y, k = call(p, A, x, y0, 1.0, 0.0)
        assert "COLS=pat" in k, k
        held = live(emu)[1] - before - held32
        if i == 0:
            assert held >= 2 * nnz + 4 * m  # the deltas are still there after the call that built them
        else:
            # anchors (4 B/row), pattern starts (2 B/row, padded), dictionary, flags and their pinned mirror
            assert 6 * m <= held <= 6 * m + 64 + 4 * (K.DCAP + 1) + 64, held
    E.ok(emu.b200sp_spmv_plan_invalidate(p.h, None))
    assert live(emu)[1] - before < 64  # the pinned mirrors of the counters
    y2, k = call(p, A, x, y0, 1.0, 0.0)
    assert "COLS=pat" in k and np.array_equal(y, y2), k
    p.close()
    assert live(emu)[1] == before


def test_forward_and_hostvec_entries(emu):
    """the fused all-gather entry and the host-vector entry take the pattern form and give the 32-bit form's bits"""
    A = K.lap_case("dof2")
    rp, ci, v, n = A
    x, y0 = inputs(A, 1.3)
    outs = {}
    for form in ("pat", "i32"):
        with env(B200SP_SPMV_IDX16="0" if form == "i32" else "1"):
            p = tuned(8, 4, 0)
            loc, fwd = np.full(n, np.nan), np.full(n, np.nan)
            E.ok(emu.b200sp_spmv_forward_f64_i32(p.h, None, n, n, len(ci), 1.0, E.ptr(rp), E.ptr(ci), E.ptr(v), E.ptr(x),
                                                 E.ptr(loc), C.c_void_p(fwd.ctypes.data)))
            kf = p.kernel()
            hv = y0.copy()
            E.ok(emu.b200sp_spmv_hostvec_f64_i32(p.h, None, b"N", n, n, len(ci), -0.7, E.ptr(rp), E.ptr(ci), E.ptr(v), E.ptr(x),
                                                 1.3, E.ptr(hv)))
            kh = p.kernel()
            p.close()
        want = "IDX=u16,COLS=pat" if form == "pat" else "IDX=i32"
        assert want in kf and want in kh, (kf, kh)
        assert np.array_equal(loc, fwd)
        outs[form] = (loc, hv)
    assert np.array_equal(outs["pat"][0], outs["i32"][0]) and np.array_equal(outs["pat"][1], outs["i32"][1])
