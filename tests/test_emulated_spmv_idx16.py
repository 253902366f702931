"""The tiled SpMV kernel's 16-bit column form (in-row column deltas + one anchor per row, DESIGN.md section 3.5) under the
CPU emulation: which matrices take it, that it gives the same bits as the 32-bit columns and the row-vector kernel, and that
the plan keys and releases the stream.  Every call that picks a form asserts it through last_kernel()."""
import numpy as np
import pytest

import emu_lib as E
import idx16_cases as K
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
    E.spmv(p, "N", len(rp) - 1, ncols, rp, ci, v, x, y, alpha, beta)
    return y, p.kernel()


def inputs(A, beta, seed=0):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-1, 1, A[3])
    y0 = rng.uniform(-1, 1, len(A[0]) - 1)
    if beta == 0.0:
        y0[::7] = np.nan
    return x, y0


def check_oracle(oracle, A, x, y0, alpha, beta, y):
    rp, ci, v, _ = A
    exp = oracle.spmv_serial(rp, ci, v, x, y0.copy(), alpha, beta)
    scale = rowwise_scale(rp, ci, v, x, y0, alpha, beta)
    assert not np.isnan(y).any()
    assert np.all(np.abs(y - exp) <= 1e-10 * scale + 1e-300)


@pytest.mark.parametrize("lpr", [2, 4, 8, 16, 32])
def test_lap27_u16_same_bits_as_i32_and_vector(emu, oracle, lpr):
    # ctas_per_sm 1: 8 CTAs on the emulated device, every ring wraps several times
    A = K.lap27(10, 9, 8)
    for alpha, beta in K.AB:
        x, y0 = inputs(A, beta)
        pv = plan(lpr=lpr, algo=1)
        yv, kv = call(pv, A, x, y0, alpha, beta)
        pv.close()
        assert kv.startswith("vector"), kv
        check_oracle(oracle, A, x, y0, alpha, beta, yv)
        for cfg in range(5):
            p = plan(cfg, lpr, 1)
            y16, k16 = call(p, A, x, y0, alpha, beta)
            assert "IDX=u16" in k16 and f"LPR={lpr}," in k16, k16
            with env(B200SP_SPMV_IDX16="0"):
                y32, k32 = call(p, A, x, y0, alpha, beta)
            assert "IDX=i32" in k32, k32
            y16b, k16b = call(p, A, x, y0, alpha, beta)  # the stream is kept across the 32-bit call
            assert "IDX=u16" in k16b, k16b
            p.close()
            assert np.array_equal(y16, y32) and np.array_equal(y16, yv) and np.array_equal(y16, y16b), (cfg, alpha, beta)


@pytest.mark.parametrize("gap,form", [(65535, "u16"), (65536, "i32")])
def test_gap_boundary(emu, oracle, gap, form):
    A = K.gap_matrix(gap)
    x, y0 = inputs(A, 0.0)
    p = plan(8)
    y, k = call(p, A, x, y0, 1.0, 0.0)
    assert f"IDX={form}" in k, k
    check_oracle(oracle, A, x, y0, 1.0, 0.0, y)
    with env(B200SP_SPMV_IDX16="0"):
        y32, _ = call(p, A, x, y0, 1.0, 0.0)
    assert np.array_equal(y, y32)
    p.close()


def test_unsorted_row_keeps_i32(emu, oracle):
    A = K.unsorted_matrix()
    x, y0 = inputs(A, 0.5)
    p = plan(8)
    for _ in range(2):
        y, k = call(p, A, x, y0, -1.0, 0.5)
        assert "IDX=i32" in k, k
        check_oracle(oracle, A, x, y0, -1.0, 0.5, y)
    p.close()


@pytest.mark.parametrize("cfg", [0, 1, 3, 8])
def test_long_rows_with_wide_gaps_still_qualify(emu, oracle, cfg):
    A = K.long_wide_matrix()
    x, y0 = inputs(A, 0.0)
    p = plan(cfg)
    y, k = call(p, A, x, y0, 2.0, 0.0)
    assert "IDX=u16" in k, k
    check_oracle(oracle, A, x, y0, 2.0, 0.0, y)
    with env(B200SP_SPMV_IDX16="0"):
        y32, k32 = call(p, A, x, y0, 2.0, 0.0)
    assert "IDX=i32" in k32 and np.array_equal(y, y32)
    p.close()


@pytest.mark.parametrize("lpr", [2, 8, 32])
def test_empty_rows_and_ragged_nnz(emu, oracle, lpr):
    A = K.empty_rows_matrix()
    assert len(A[1]) % 8 != 0
    for alpha, beta in K.AB:
        x, y0 = inputs(A, beta, seed=1)
        p = plan(8, lpr)
        y, k = call(p, A, x, y0, alpha, beta)
        assert "IDX=u16" in k, k
        check_oracle(oracle, A, x, y0, alpha, beta, y)
        with env(B200SP_SPMV_IDX16="0"):
            y32, _ = call(p, A, x, y0, alpha, beta)
        p.close()
        assert np.array_equal(y, y32)


def test_new_col_idx_same_row_ptr(emu, oracle):
    """the stream is keyed on col_idx: a second matrix with the same row_ptr array gets its own"""
    rp, ci, v, n = A1 = K.lap27(8, 7, 6)
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    ci2 = ((ci.astype(np.int64) + 2 * rows) % n).astype(np.int32)
    for r in range(len(rp) - 1):
        ci2[rp[r]:rp[r + 1]].sort()
    A2 = (rp, ci2, v, n)
    x, y0 = inputs(A1, 0.0)
    p = plan(8)
    for A in (A1, A2, A1):
        y, k = call(p, A, x, y0, 1.0, 0.0)
        assert "IDX=u16" in k, k
        check_oracle(oracle, A, x, y0, 1.0, 0.0, y)
    p.close()


def test_invalidate_releases_the_stream(emu):
    A = K.lap27(8, 7, 6)
    m, nnz = len(A[0]) - 1, len(A[1])
    x, y0 = inputs(A, 0.0)
    before = live(emu)[1]
    with env(B200SP_SPMV_IDX16="0"):
        p = plan(8)
        call(p, A, x, y0, 1.0, 0.0)
        held32 = live(emu)[1] - before
        p.close()
    p = plan(8)
    call(p, A, x, y0, 1.0, 0.0)
    held16 = live(emu)[1] - before
    # on top of the analysis: the deltas (2 B/entry, padded to 8 entries), the anchors (4 B/row, padded to 4 rows), the flag
    # and its pinned mirror
    assert held16 - held32 >= 2 * nnz + 4 * m
    E.ok(emu.b200sp_spmv_plan_invalidate(p.h, None))
    assert live(emu)[1] - before < 64  # what remains are the pinned mirrors of the counters
    y, k = call(p, A, x, y0, 1.0, 0.0)  # built again
    assert "IDX=u16" in k, k
    p.close()
    assert live(emu)[1] == before
