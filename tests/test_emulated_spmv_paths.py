"""The rank-1 SpMV kernel paths EXECUTED on the CPU (tools/emu) on the shared cases of spmv_cases.py, each result checked
entry by entry against the exact product within the per-entry rounding bound (tests/exact_ref.py) -- the same inputs and
the same check as tests/test_gpu_spmv_paths.py, through the C ABI.  Every call that selects a path asserts last_kernel()."""
import ctypes as C

import numpy as np
import pytest

import emu_lib as E
import exact_ref as R
import pattern_cases
import spmm_cases
import spmv_cases as S
from test_emulated_kernels import env

DTYPES = [np.float64, np.float32]
AB = ((1.0, 0.0), (2.5, -1.0))


@pytest.fixture(scope="module")
def emu():
    return E.lib()


_MATS = {}


def matrix(name, dtype):
    key = (name, np.dtype(dtype).name)
    if key not in _MATS:
        if name.startswith("thresholds"):
            base, _, mod = name.partition("_mod")
            _MATS[key] = (S.thresholds_sorted if base == "thresholds_sorted" else S.thresholds)(5, dtype, int(mod or 3))
        elif name == "long_rows":
            _MATS[key] = S.long_rows(5, dtype)
        elif name == "lap27":
            _MATS[key] = S.with_values(pattern_cases.lap_case("dof2"), 5, dtype)
        else:
            _MATS[key] = spmm_cases.SMALL_CASES[name](5, dtype)
    return _MATS[key]


_REFS = {}


def reference(name, dtype, trans, alpha, beta, special=False):
    key = (name, np.dtype(dtype).name, trans, alpha, beta, special)
    if key not in _REFS:
        rp, ci, v, ncols = matrix(name, dtype)
        rng = np.random.default_rng(0)
        x = S.vector_operand(rng, len(rp) - 1 if trans else ncols, dtype)
        y0 = S.vector_operand(rng, ncols if trans else len(rp) - 1, dtype)
        if special:
            x[int(ci[len(ci) // 3]) if not trans else 7] = np.inf
            x[int(ci[len(ci) // 2]) if not trans else 11] = np.nan
        if beta == 0:
            y0[::3] = np.nan
        _REFS[key] = (x, y0, R.spmm_exact(rp, ci, v, x, y0, alpha, beta, trans), R.spmm_bound(rp, ci, v, x, y0, alpha, beta, trans))
    return _REFS[key]


def plan(cfg=-1, lpr=-1, algo=0, cache_transpose=False):
    p = E.SpmvPlan(algo)
    E.ok(E.lib().b200sp_spmv_plan_tune(p.h, cfg, lpr, -1))
    if cache_transpose:
        E.ok(E.lib().b200sp_spmv_plan_set_option(p.h, 1, 1))
    return p


def checked(p, name, dtype, mode, alpha, beta, arrays=None, special=False):
    rp, ci, v, ncols = matrix(name, dtype) if arrays is None else arrays
    x, y0, exact, bound = reference(name, dtype, mode in "TH", alpha, beta, special)
    y = y0.copy()
    E.spmv(p, mode, len(rp) - 1, ncols, rp, ci, v, x, y, alpha, beta)
    k = p.kernel()
    R.assert_within(y, exact, bound, f"{k} {name} {np.dtype(dtype).name} mode {mode} a={alpha} b={beta}")
    return y, k


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("form", ["i32", "delta", "pat"])
def test_tile_forms_every_cfg(emu, dtype, form):
    """Every ring configuration at LPR 4 and configuration 8 at every LPR, on the threshold matrix (32-bit columns), its
    sorted variant (delta form) and a lap27 matrix (pattern form)."""
    name = {"i32": "thresholds", "delta": "thresholds_sorted", "pat": "lap27"}[form]
    cols = {"i32": "IDX=i32", "delta": "IDX=u16,COLS=delta", "pat": "IDX=u16,COLS=pat"}[form]
    with env(B200SP_SPMV_IDX16="0" if form == "i32" else None):
        for cfg, lpr in [(c, 4) for c in sorted(S.CFGS)] + [(8, l) for l in S.LPRS if l != 4]:
            p = plan(cfg, lpr)
            checked(p, name, dtype, "N", 1.0, 0.0)  # the emulated plan has its verdict after the first call
            for alpha, beta in AB:
                y, k = checked(p, name, dtype, "N", alpha, beta)
                assert k.startswith(S.tile_label(dtype, cfg, lpr, cols)), (k, cfg, lpr)
            p.close()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("nnz_mod4", [1, 2])
def test_tile_ragged_nnz(emu, dtype, nnz_mod4):
    name = f"thresholds_mod{nnz_mod4}"
    with env(B200SP_SPMV_IDX16="0"):
        for cfg in (3, 6, 9, 10):
            p = plan(cfg, 8)
            _, k = checked(p, name, dtype, "N", -1.0, 1.0)
            assert k.startswith(S.tile_label(dtype, cfg, 8, "IDX=i32")), k
            p.close()


@pytest.mark.parametrize("dtype", DTYPES)
def test_vector_kernel(emu, dtype):
    prec = "f64" if dtype == np.float64 else "f32"
    for lpr in S.LPRS:
        p = plan(-1, lpr)
        _, k = checked(p, "small_mod1", dtype, "N", 2.5, -1.0)
        assert k.startswith(f"vector<{prec},LPR={lpr}>"), k
        p.close()
    p = plan(algo=1)
    _, k = checked(p, "thresholds", dtype, "N", 1.0, 0.0)
    assert k.startswith(f"vector<{prec},"), k
    p.close()
    rp, ci, v, ncols = matrix("thresholds", dtype)
    for which in ("ci", "v"):
        a = ci if which == "ci" else v
        buf = np.concatenate([a[:1], a])
        arrays = (rp, buf[1:], v, ncols) if which == "ci" else (rp, ci, buf[1:], ncols)
        p = plan(8, 4)
        _, k = checked(p, "thresholds", dtype, "N", 2.5, -1.0, arrays=arrays)
        assert k.startswith(f"vector<{prec},LPR=4>"), k
        p.close()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("longrows", [None, "seg"])
def test_long_rows(emu, dtype, longrows):
    with env(B200SP_SPMV_LONGROWS=longrows):
        for cfg in (3, 8):
            p = plan(cfg, 8)
            y1, k = checked(p, "long_rows", dtype, "N", 1.0, 0.0)
            checked(p, "long_rows", dtype, "N", 2.5, -1.0)
            y3, _ = checked(p, "long_rows", dtype, "N", 1.0, 0.0)
            assert k.startswith("tile<") and k.endswith("+seg") == (longrows == "seg"), k
            assert np.array_equal(y1.view(np.uint8), y3.view(np.uint8))
            p.close()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", ["duplicates", "cancelling", "wide_short"])
def test_transpose_modes(emu, dtype, name):
    prec = "f64" if dtype == np.float64 else "f32"
    for mode in "TH":
        for alpha, beta in AB:
            p = plan()
            _, k = checked(p, name, dtype, mode, alpha, beta)
            assert k.startswith(f"transpose<{prec},"), k
            p.close()
            p = plan(cache_transpose=True)
            _, k = checked(p, name, dtype, mode, alpha, beta)
            assert k.startswith("cached_transpose+"), k
            p.close()


@pytest.mark.parametrize("dtype", DTYPES)
def test_alpha_beta_grid(emu, dtype):
    coefs = [0.0, 1.0, -1.0, 2.5]
    for alpha in coefs:
        for beta in coefs:
            for mode, kw in (("N", {"cfg": 8, "lpr": 4}), ("N", {"algo": 1}), ("T", {}), ("H", {"cache_transpose": True})):
                for special in (False, True):
                    p = plan(**kw)
                    _, k = checked(p, "thresholds", dtype, mode, alpha, beta, special=special)
                    p.close()
                    assert (k == "scale") == (alpha == 0), k


def _entry(fn, p, name, x, y, *tail):
    rp, ci, v, ncols = matrix(name, np.float64)
    E.ok(fn(p.h, None, len(rp) - 1, ncols, len(ci), 1.5, E.ptr(rp), E.ptr(ci), E.ptr(v), E.ptr(x), E.ptr(y), *tail))


@pytest.mark.parametrize("name", ["thresholds", "long_rows"])
def test_scatter_and_forward(emu, name):
    """spmv_scatter with 1 and 7 local extra buffers and spmv_forward at configurations 8 (forwarding form) and 3 (direct
    stores): y within the bound, every other destination with y's bits."""
    x, _, exact, bound = reference(name, np.float64, False, 1.5, 0.0)
    m = len(matrix(name, np.float64)[0]) - 1
    for n_extra in (1, 7):
        p = plan()
        y = np.full(m, np.nan)
        extra = [np.full(m, np.nan) for _ in range(n_extra)]
        arr = (C.c_void_p * n_extra)(*[e.ctypes.data for e in extra])
        _entry(emu.b200sp_spmv_scatter_f64_i32, p, name, x, y, n_extra, arr)
        k = p.kernel()
        p.close()
        assert k.startswith("tile<f64,"), k
        R.assert_within(y, exact, bound, f"{k} scatter {n_extra}")
        for e in extra:
            assert np.array_equal(e.view(np.uint8), y.view(np.uint8))
    for cfg in (8, 3):
        p = plan(cfg, 4)
        y = np.full(m, np.nan)
        fwd = np.full(m, np.nan)
        _entry(emu.b200sp_spmv_forward_f64_i32, p, name, x, y, E.ptr(fwd))
        k = p.kernel()
        p.close()
        assert k.startswith(S.tile_label(np.float64, cfg, 4, "")[:-1]), k
        R.assert_within(y, exact, bound, f"{k} forward")
        assert np.array_equal(fwd.view(np.uint8), y.view(np.uint8))
