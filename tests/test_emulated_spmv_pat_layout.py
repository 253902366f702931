"""The pattern form's own stage layout (DESIGN.md section 3.6: stages of PAT_CAP values and PAT_RCAP row slots, on a tile table
of its own cut with the cfg's LMAX) under the CPU emulation, against the 32-bit columns on the cfg's tiles: the same bits on
every matrix, every entry point and every switch between the two."""
import ctypes as C

import numpy as np
import pytest

import emu_lib as E
import pattern_cases as K
import test_emulated_spmv_pattern as P
from test_emulated_kernels import env
from test_emulated_leaks import live

PAT_CAP, PAT_TILE_CAP, PAT_RCAP = 4096, 4040, 256
LAYOUT = f"pat<STAGES=3,CAP={PAT_CAP},RCAP={PAT_RCAP}>"


@pytest.fixture(scope="module")
def emu():
    return E.lib()


def pat_tiles(A, lmax=512):
    return len(A[1]) // (PAT_TILE_CAP - lmax - 8) + 1


def same_as_i32(A, dtype=np.float64, cfg=8, lpr=4, alpha=-0.7, beta=1.3, ctas=1):
    """the pattern form's y and that of the 32-bit columns, on one plan"""
    x, y0 = P.inputs(A, beta, dtype=dtype)
    p = P.tuned(cfg, lpr, ctas)
    y, k = P.call(p, A, x, y0, alpha, beta)
    with env(B200SP_SPMV_IDX16="0"):
        y32, k32 = P.call(p, A, x, y0, alpha, beta)
    p.close()
    assert "IDX=u16,COLS=pat>" + LAYOUT in k, k
    assert "IDX=i32>grid" in k32, k32
    assert np.array_equal(y, y32), (k, k32)
    return x, y0, y


@pytest.mark.parametrize("case", ["dof1", "dof2", "dof3"])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_lap27_dof(emu, oracle, case, dtype):
    A = K.lap_case(case)
    assert pat_tiles(A) > 2
    for alpha, beta in K.AB:
        x, y0, y = same_as_i32(A, dtype, alpha=alpha, beta=beta)
        P.check_oracle(oracle, A, x, y0, alpha, beta, y)


@pytest.mark.parametrize("name", ["diagonal_matrix", "near_patterns_matrix", "empty_rows_matrix"])
@pytest.mark.parametrize("lpr", [2, 8])
def test_rows_past_the_row_slots(emu, oracle, name, lpr):
    """short rows: a tile holds more rows than a stage has row slots, and the rest read row_ptr, anchor and pattern start
    from global memory"""
    A = getattr(K, name)()
    rp = A[0]
    first = np.searchsorted(rp, np.arange(pat_tiles(A)) * (PAT_TILE_CAP - 512 - 8), side="right") - 1
    assert np.max(np.diff(first)) > PAT_RCAP
    x, y0, y = same_as_i32(A, lpr=lpr)
    P.check_oracle(oracle, A, x, y0, -0.7, 1.3, y)


def lmax_rows_matrix(m=3000, seed=21):
    """lap-like rows of 27 entries, rows of exactly LMAX = 512 entries (one pattern) and of LMAX + 1 (long rows: the
    long-row kernel's), spread over the pattern tiles"""
    rows = K._from_patterns([list(range(9)) + list(range(40, 49)) + list(range(80, 89))], m, 200000, seed)
    for r in range(5, m, 50):
        rows[r] = rows[r][0] % 190000 + np.arange(512)
    for r in range(30, m, 77):
        rows[r] = rows[r][0] % 190000 + 2 * np.arange(513)
    return K._assemble(rows, 200000, seed)


@pytest.mark.parametrize("cfg", [0, 8])
def test_rows_of_lmax_and_lmax_plus_one(emu, oracle, cfg):
    A = lmax_rows_matrix()
    assert K.expected_cols(A, 512) == "pat"
    lens = np.diff(A[0])
    assert (lens == 512).sum() > 10 and (lens == 513).sum() > 10
    for alpha, beta in K.AB:
        x, y0, y = same_as_i32(A, cfg=cfg, alpha=alpha, beta=beta)
        P.check_oracle(oracle, A, x, y0, alpha, beta, y)


def test_switching_tables_on_one_plan(emu):
    """the cfg's tiles (32-bit columns), then the pattern tiles, and back, on one plan: every call the same bits"""
    A = K.lap_case("dof2")
    x, y0 = P.inputs(A, 1.3)
    p = P.tuned(8, 4)
    ys = []
    for i32 in (True, False, True, False):
        with env(B200SP_SPMV_IDX16="0" if i32 else None):
            y, k = P.call(p, A, x, y0, -0.7, 1.3)
        assert (LAYOUT in k) != i32, k
        ys.append(y)
    p.close()
    assert all(np.array_equal(ys[0], y) for y in ys[1:])


def test_forward_tiles_over_64_rows(emu):
    """the fused all-gather form on pattern tiles of more than 64 rows (its producer forwards them with forward_rows), with
    more tiles per CTA than stages"""
    A = K.lap27(16, 16, 16, ndof=1)
    rp, ci, v, n = A
    first = np.searchsorted(rp, np.arange(pat_tiles(A)) * (PAT_TILE_CAP - 512 - 8), side="right") - 1
    assert np.min(np.diff(first)) > 64 and pat_tiles(A) > 4 * 4
    x, _ = P.inputs(A, 0.0)
    outs = {}
    for form in ("pat", "i32"):
        with env(B200SP_SPMV_IDX16="0" if form == "i32" else None):
            p = P.tuned(8, 4, 1)
            loc, fwd = np.full(n, np.nan), np.full(n, np.nan)
            for _ in range(2):
                E.ok(E.lib().b200sp_spmv_forward_f64_i32(p.h, None, n, n, len(ci), 1.0, E.ptr(rp), E.ptr(ci), E.ptr(v), E.ptr(x),
                                                         E.ptr(loc), C.c_void_p(fwd.ctypes.data)))
            k = p.kernel()
            p.close()
        assert (LAYOUT in k) == (form == "pat"), k
        assert np.array_equal(loc, fwd)
        outs[form] = loc
    assert np.array_equal(outs["pat"], outs["i32"])


def test_hostvec_after_the_switch(emu):
    A = K.lap_case("dof2")
    rp, ci, v, n = A
    x, y0 = P.inputs(A, 1.3)
    outs = {}
    for form in ("pat", "i32"):
        with env(B200SP_SPMV_IDX16="0" if form == "i32" else None):
            p = P.tuned(8, 4)
            for _ in range(3):
                hv = y0.copy()
                E.ok(E.lib().b200sp_spmv_hostvec_f64_i32(p.h, None, b"N", n, n, len(ci), -0.7, E.ptr(rp), E.ptr(ci), E.ptr(v),
                                                         E.ptr(x), 1.3, E.ptr(hv)))
                assert (LAYOUT in p.kernel()) == (form == "pat"), p.kernel()
            p.close()
        outs[form] = hv
    assert np.array_equal(outs["pat"], outs["i32"])


def test_plan_memory(emu):
    """the pattern form holds its tile table instead of the cfg's; invalidate and destroy release it"""
    A = K.lap_case("dof2")
    m, nnz = len(A[0]) - 1, len(A[1])
    x, y0 = P.inputs(A, 0.0)
    before = live(emu)[1]
    with env(B200SP_SPMV_IDX16="0"):
        p = P.tuned(8)
        P.call(p, A, x, y0, 1.0, 0.0)
        held32 = live(emu)[1] - before
        p.close()
    p = P.tuned(8)
    for _ in range(2):
        y, k = P.call(p, A, x, y0, 1.0, 0.0)
        assert LAYOUT in k, k
    held = live(emu)[1] - before - held32
    tiles = 16 * pat_tiles(A) - 16 * (nnz // (2048 - 512 - 8) + 1)
    # anchors (4 B/row), pattern starts (2 B/row, padded), dictionary, flags and their pinned mirror, the pattern tiles
    # instead of the cfg's
    assert 6 * m + tiles <= held <= 6 * m + tiles + 64 + 4 * (K.DCAP + 1) + 64, held
    E.ok(emu.b200sp_spmv_plan_invalidate(p.h, None))
    assert live(emu)[1] - before < 64
    y2, k = P.call(p, A, x, y0, 1.0, 0.0)
    assert LAYOUT in k and np.array_equal(y, y2), k
    p.close()
    assert live(emu)[1] == before
