"""Every rank-1 SpMV kernel path and entry point (csrc/spmv.cu) on the GPU, each call checked entry by entry against the
exact product (tests/exact_ref.py) within a rigorous per-entry rounding bound, in fp32 and fp64.  Paths are selected with
SPMVHandle.tune, the handle's algorithm, operand alignment and the library's B200SP_* variables (read by getenv on every
call); every call that selects a path asserts the handle's last_kernel(), so a dispatcher that quietly falls back cannot
make a test vacuous.  The exact reference is computed once per operand set and reused across the paths that share it.

With B200SP_TEST_EMULATED=1 the module runs on the CPU emulation; it then skips the host-vector tests, which need pinned
memory."""
import os

import numpy as np
import pytest
import torch

import exact_ref as R
import pattern_cases
import spmm_cases
import spmv_cases as S

pytestmark = pytest.mark.gpu

EMULATED = os.environ.get("B200SP_TEST_EMULATED") == "1"
DTYPES = [np.float64, np.float32]
SPMV_VARS = ["B200SP_SPMV_IDX16", "B200SP_SPMV_PATTERN", "B200SP_SPMV_LONGROWS", "B200SP_HOSTVEC_PIECES",
             "B200SP_HOSTVEC_SIMPLE", "B200SP_NO_AUTOTUNE"]
needs_pinned = pytest.mark.skipif(EMULATED, reason="pinned host memory needs the real CUDA runtime")


@pytest.fixture(autouse=True)
def _clean_env(monkeypatch):
    for k in SPMV_VARS:
        monkeypatch.delenv(k, raising=False)


# ---- matrices, operands and exact references, built once per session ------------------------------------------------
_MATS = {}


def matrix(name, dtype, seed=5):
    key = (name, np.dtype(dtype).name, seed)
    if key not in _MATS:
        if name.startswith("thresholds"):
            base, _, mod = name.partition("_mod")
            builder = S.thresholds_sorted if base == "thresholds_sorted" else S.thresholds
            _MATS[key] = builder(seed, dtype, int(mod or 3))
        elif name in ("long_rows", "hostvec_big"):
            _MATS[key] = getattr(S, name)(seed, dtype)
        elif name == "lap27":
            _MATS[key] = S.with_values(pattern_cases.lap_case("dof2"), seed, dtype)
        elif name == "dictionary":
            _MATS[key] = S.with_values(pattern_cases.dict_matrix(pattern_cases.DCAP), seed, dtype)
        else:
            _MATS[key] = spmm_cases.SMALL_CASES[name](seed, dtype)
    return _MATS[key]


_REFS = {}


def reference(name, dtype, trans, alpha, beta, seed=0, special=False):
    """(x, y0, exact, bound) of one operand set; special: an Inf and a NaN in x (they reach exactly the rows whose exact
    value is not finite)"""
    key = (name, np.dtype(dtype).name, trans, alpha, beta, seed, special)
    if key not in _REFS:
        rp, ci, v, ncols = matrix(name, dtype)
        m = len(rp) - 1
        rng = np.random.default_rng(seed)
        x = S.vector_operand(rng, m if trans else ncols, dtype)
        y0 = S.vector_operand(rng, ncols if trans else m, dtype)
        if special:
            x[int(ci[len(ci) // 3]) if not trans else 7] = np.inf
            x[int(ci[len(ci) // 2]) if not trans else 11] = np.nan
        if beta == 0:
            y0[::3] = np.nan  # must not survive
        _REFS[key] = (x, y0, R.spmm_exact(rp, ci, v, x, y0, alpha, beta, trans), R.spmm_bound(rp, ci, v, x, y0, alpha, beta, trans))
    return _REFS[key]


_DEV = {}


def dev_matrix(cuda, name, dtype):
    from kokkos_kernels_b200 import sparse as sp

    key = (name, np.dtype(dtype).name)
    if key not in _DEV:
        rp, ci, v, ncols = matrix(name, dtype)
        _DEV[key] = sp.CrsMatrix(torch.from_numpy(rp).to(cuda), torch.from_numpy(ci).to(cuda), torch.from_numpy(v).to(cuda), ncols)
    return _DEV[key]


def call(cuda, h, mode, alpha, A, x, beta, y0):
    from kokkos_kernels_b200 import sparse as sp

    y = torch.from_numpy(y0.copy()).to(cuda)
    sp.spmv(h, mode, alpha, A, torch.from_numpy(x).to(cuda), beta, y)
    torch.cuda.synchronize()
    return y.cpu().numpy(), (h.last_kernel() if h is not None else "no plan")


def checked(cuda, h, name, dtype, mode, alpha, beta, A=None, seed=0, special=False, what=""):
    """one call on matrix `name`, checked against the bound; returns (y, last_kernel)"""
    trans = mode in "TH"
    x, y0, exact, bound = reference(name, dtype, trans, alpha, beta, seed, special)
    y, k = call(cuda, h, mode, alpha, dev_matrix(cuda, name, dtype) if A is None else A, x, beta, y0)
    R.assert_within(y, exact, bound, f"{k} {name} {np.dtype(dtype).name} mode {mode} a={alpha} b={beta} {what}")
    return y, k


def handle(cfg=-1, lpr=-1, algo=None):
    from kokkos_kernels_b200 import sparse as sp

    h = sp.SPMVHandle(sp.SPMV_DEFAULT if algo is None else algo)
    h.tune(cfg, lpr, -1)
    return h


def same_bits(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


AB = ((1.0, 0.0), (2.5, -1.0))


# ---- tiled kernel -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lpr", S.LPRS)
@pytest.mark.parametrize("cfg", sorted(S.CFGS))
@pytest.mark.parametrize("dtype", DTYPES)
def test_tile_every_cfg_and_lpr(cuda, monkeypatch, dtype, cfg, lpr):
    """The threshold matrix (rows at LMAX-1/LMAX/LMAX+1 and at tile boundaries of every CAP, a clamped tile end, empty
    runs; nnz % 4 = 1, 2, 3 across the configurations) on the 32-bit columns, through every ring configuration and
    lanes-per-row; a second call gives the same bits."""
    monkeypatch.setenv("B200SP_SPMV_IDX16", "0")
    name = f"thresholds_mod{cfg % 3 + 1}"
    h = handle(cfg, lpr)
    want = S.tile_label(dtype, cfg, lpr, "IDX=i32")
    for alpha, beta in AB:
        y, k = checked(cuda, h, name, dtype, "N", alpha, beta)
        assert k.startswith(want), (k, want)
        y2, _ = checked(cuda, h, name, dtype, "N", alpha, beta)
        assert same_bits(y, y2), k


FORM_RUNS = [(c, 4) for c in sorted(S.CFGS)] + [(8, l) for l in S.LPRS if l != 4]


@pytest.mark.parametrize("cfg,lpr", FORM_RUNS)
@pytest.mark.parametrize("form", ["delta", "pat"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_tile_column_forms(cuda, dtype, form, cfg, lpr):
    """The delta form on the sorted threshold matrix, the pattern form on a lap27 matrix and at the dictionary's capacity:
    every configuration at one lanes-per-row, configuration 8 at every lanes-per-row.  The form is known once the plan's
    verdict has reached the host, so each handle is called and synchronised once before the checked calls."""
    names = ["thresholds_sorted"] if form == "delta" else ["lap27", "dictionary"]
    for name in names:
        h = handle(cfg, lpr)
        checked(cuda, h, name, dtype, "N", 1.0, 0.0, what="(first call)")
        want = S.tile_label(dtype, cfg, lpr, f"IDX=u16,COLS={form}")
        for alpha, beta in AB:
            y, k = checked(cuda, h, name, dtype, "N", alpha, beta)
            assert k.startswith(want), (k, want)


# ---- vector kernel ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_vector_kernel(cuda, dtype):
    """SPMV_FAST_SETUP, no handle, an untuned handle under 32768 entries, every lanes-per-row, and matrices whose col_idx
    or values start one element into their buffer (the TMA kernel needs 16-byte alignment) on a tuned handle."""
    from kokkos_kernels_b200 import sparse as sp

    prec = "f64" if dtype == np.float64 else "f32"
    for name in ("small_mod1", "small_mod2", "thresholds"):
        for alpha, beta in AB:
            _, k = checked(cuda, handle(algo=sp.SPMV_FAST_SETUP), name, dtype, "N", alpha, beta)
            assert k.startswith(f"vector<{prec},"), k
            checked(cuda, None, name, dtype, "N", alpha, beta)
    for name in ("small_mod1", "small_mod2", "small_mod3"):
        assert len(matrix(name, dtype)[1]) < 32768
        _, k = checked(cuda, handle(), name, dtype, "N", -1.0, 1.0)
        assert k.startswith(f"vector<{prec},"), k
        for lpr in S.LPRS:
            _, k = checked(cuda, handle(-1, lpr), name, dtype, "N", 2.5, 0.0)
            assert k.startswith(f"vector<{prec},LPR={lpr}>"), k
    rp, ci, v, ncols = matrix("thresholds", dtype)
    A = dev_matrix(cuda, "thresholds", dtype)
    for which in ("col_idx", "values"):
        src = ci if which == "col_idx" else v
        buf = torch.from_numpy(np.concatenate([src[:1], src])).to(cuda)
        shifted = buf[1:]
        assert shifted.data_ptr() % 16 != 0
        Au = sp.CrsMatrix(A.row_map, shifted if which == "col_idx" else A.entries, shifted if which == "values" else A.values, ncols)
        for alpha, beta in AB:
            _, k = checked(cuda, handle(8, 4), "thresholds", dtype, "N", alpha, beta, A=Au, what=f"unaligned {which}")
            assert k.startswith(f"vector<{prec},LPR=4>"), k


@pytest.mark.parametrize("dtype", DTYPES)
def test_self_tuning_handle(cuda, dtype):
    """Six calls on one untuned handle pass through the self-tuning phases (tiled kernel, timed tiled kernel, timed vector
    kernel, choice): every call meets the bound, and all give the same bits."""
    for name in ("thresholds", "long_rows"):
        assert len(matrix(name, dtype)[1]) >= 32768
        h = handle()
        outs = [checked(cuda, h, name, dtype, "N", -0.5, 2.5) for _ in range(6)]
        assert any(k.startswith("tile<") for _, k in outs), [k for _, k in outs]
        for y, k in outs[1:]:
            assert same_bits(y, outs[0][0]), k


# ---- long rows --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("longrows", ["cta", "seg"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_long_rows(cuda, monkeypatch, dtype, longrows):
    """Rows of 4095, 4096, 4097 and 8193 entries (one to three segments of 4096) and others longer than every LMAX, first
    and last rows included: the CTA-per-row kernel and the segmented kernels, at two ring configurations."""
    if longrows == "seg":
        monkeypatch.setenv("B200SP_SPMV_LONGROWS", "seg")
    for cfg in (3, 8):
        h = handle(cfg, 8)
        outs = []
        for alpha, beta in AB + ((1.0, 0.0),):
            y, k = checked(cuda, h, "long_rows", dtype, "N", alpha, beta)
            assert k.startswith("tile<") and k.endswith("+seg") == (longrows == "seg"), k
            outs.append(y)
        assert same_bits(outs[0], outs[2]), k
    for name in ("thresholds", "thresholds_sorted"):
        _, k = checked(cuda, handle(1, 16), name, dtype, "N", 2.5, -1.0)
        assert k.endswith("+seg") == (longrows == "seg"), k


# ---- transposed modes -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["duplicates", "cancelling", "wide_short", "thresholds"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_transpose_modes(cuda, dtype, name):
    """T and H through the atomics kernel and through the plan's cached transpose, beta = 0 over a NaN-filled y included;
    the cached transpose gives the same bits from call to call."""
    prec = "f64" if dtype == np.float64 else "f32"
    for mode in "TH":
        h = handle()
        hc = handle()
        hc.cache_transpose(True)
        for alpha, beta in AB + ((-1.0, 1.0),):
            _, k = checked(cuda, h, name, dtype, mode, alpha, beta)
            assert k.startswith(f"transpose<{prec},"), k
            yc, kc = checked(cuda, hc, name, dtype, mode, alpha, beta)
            assert kc.startswith("cached_transpose+"), kc
            yc2, _ = checked(cuda, hc, name, dtype, mode, alpha, beta)
            assert same_bits(yc, yc2), kc


# ---- alpha and beta ---------------------------------------------------------------------------------------------------
COEFS = [0.0, 1.0, -1.0, 2.5]


@pytest.mark.parametrize("dtype", DTYPES)
def test_alpha_beta_grid(cuda, dtype):
    """alpha, beta over {0, 1, -1, 2.5}^2 in every mode, through the tiled, the vector and the transpose kernels, with an
    Inf and a NaN in x: they reach exactly the rows whose exact value is not finite, and alpha = 0 never reads x."""
    from kokkos_kernels_b200 import sparse as sp

    name = "thresholds"
    tiled = handle(8, 4)
    vec = handle(algo=sp.SPMV_FAST_SETUP)
    cached = handle()
    cached.cache_transpose(True)
    for alpha in COEFS:
        for beta in COEFS:
            for mode in "NCTH":
                hs = (tiled, vec) if mode in "NC" else (handle(), cached)
                for h in hs:
                    for special in (False, True):
                        _, k = checked(cuda, h, name, dtype, mode, alpha, beta, special=special)
                        if alpha == 0:
                            assert k == "scale", k
                        else:
                            assert k.startswith(("tile<", "vector<", "transpose<", "cached_transpose+tile<",
                                                 "cached_transpose+vector<")), k


# ---- entry points -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_extra", [1, 7])
@pytest.mark.parametrize("name", ["thresholds", "long_rows"])
def test_scatter_to_local_buffers(cuda, name, n_extra):
    """spmv_scatter (fp64, beta = 0) with 1 and 7 extra destinations on this device: y meets the bound and every extra
    buffer holds y's bits, long rows included."""
    from kokkos_kernels_b200 import sparse as sp

    dtype = np.float64
    x, _, exact, bound = reference(name, dtype, False, 1.5, 0.0)
    A = dev_matrix(cuda, name, dtype)
    m = A.numRows()
    for cfg in (-1, 3):
        h = handle(cfg)
        for _ in range(2):
            y = torch.full((m,), float("nan"), dtype=torch.float64, device=cuda)
            extra = [torch.full((m,), float("nan"), dtype=torch.float64, device=cuda) for _ in range(n_extra)]
            sp.spmv_scatter(h, 1.5, A, torch.from_numpy(x).to(cuda), y, [e.data_ptr() for e in extra])
            torch.cuda.synchronize()
            k = h.last_kernel()
            assert k.startswith("tile<f64,"), k
            got = y.cpu().numpy()
            R.assert_within(got, exact, bound, f"{k} scatter {name} cfg {cfg}")
            for e in extra:
                assert same_bits(e.cpu().numpy(), got), k


@pytest.mark.parametrize("cfg", [8, 3])
@pytest.mark.parametrize("form", ["i32", "delta"])
def test_forward(cuda, monkeypatch, form, cfg):
    """spmv_forward (fp64, beta = 0) on the 32-bit and the delta column forms: configuration 8 runs the forwarding
    instantiation, configuration 3 stores to the destination from the consumers.  The destination holds y's bits."""
    from kokkos_kernels_b200 import sparse as sp

    if form == "i32":
        monkeypatch.setenv("B200SP_SPMV_IDX16", "0")
    name = "thresholds_sorted"
    dtype = np.float64
    x, _, exact, bound = reference(name, dtype, False, -2.5, 0.0)
    A = dev_matrix(cuda, name, dtype)
    m = A.numRows()
    h = handle(cfg, 4)
    want = S.tile_label(dtype, cfg, 4, "IDX=i32" if form == "i32" else "IDX=u16,COLS=delta")
    for i in range(3):
        y = torch.full((m,), float("nan"), dtype=torch.float64, device=cuda)
        fwd = torch.full((m,), float("nan"), dtype=torch.float64, device=cuda)
        sp.spmv_forward(h, -2.5, A, torch.from_numpy(x).to(cuda), y, fwd.data_ptr())
        torch.cuda.synchronize()
        k = h.last_kernel()
        got = y.cpu().numpy()
        R.assert_within(got, exact, bound, f"{k} forward cfg {cfg}")
        assert same_bits(fwd.cpu().numpy(), got), k
        if i > 0:  # the first call cannot know the delta form's verdict yet
            assert k.startswith(want), (k, want)


def _pinned(a):
    return torch.from_numpy(a.copy()).pin_memory()


@needs_pinned
@pytest.mark.parametrize("variant", ["default", "fast_setup", "simple_env"])
def test_hostvec_simple_path(cuda, monkeypatch, variant):
    """spmv_hostvec below 2^22 entries, with SPMV_FAST_SETUP, or under B200SP_HOSTVEC_SIMPLE: upload, one device call,
    download, in every mode."""
    from kokkos_kernels_b200 import sparse as sp

    if variant == "simple_env":
        monkeypatch.setenv("B200SP_HOSTVEC_SIMPLE", "1")
    dtype = np.float64
    for name in ("thresholds", "long_rows"):
        A = dev_matrix(cuda, name, dtype)
        h = handle(algo=sp.SPMV_FAST_SETUP) if variant == "fast_setup" else handle()
        for mode in "NCTH":
            for alpha, beta in AB:
                x, y0, exact, bound = reference(name, dtype, mode in "TH", alpha, beta)
                xh, yh = _pinned(x), _pinned(y0)  # both held until the stream is synchronised: they are read asynchronously
                sp.spmv_hostvec(h, mode, alpha, A, xh, beta, yh)
                torch.cuda.synchronize()
                R.assert_within(yh.numpy(), exact, bound, f"{h.last_kernel()} hostvec {variant} {name} mode {mode} a={alpha} b={beta}")


@needs_pinned
@pytest.mark.parametrize("pieces", ["1", "3", "8"])
def test_hostvec_pipeline(cuda, monkeypatch, pieces):
    """The pipelined host-vector path on more than 2^22 entries with long rows in every piece (the last one included):
    three calls with beta = 0 over NaN and beta != 0, queued before one synchronise, each within the bound."""
    from kokkos_kernels_b200 import sparse as sp

    monkeypatch.setenv("B200SP_HOSTVEC_PIECES", pieces)
    name, dtype = "hostvec_big", np.float64
    A = dev_matrix(cuda, name, dtype)
    assert A.nnz() >= (1 << 22)
    h = handle()
    runs = [(1.0, 0.0, 0), (-0.5, 2.5, 1), (2.5, 0.0, 2)]
    refs = [reference(name, dtype, False, a, b, seed) for a, b, seed in runs]
    xs = [_pinned(r[0]) for r in refs]  # held until the synchronise: the uploads are asynchronous
    ys = [_pinned(r[1]) for r in refs]
    for (alpha, beta, _), xh, yh in zip(runs, xs, ys):
        sp.spmv_hostvec(h, "N", alpha, A, xh, beta, yh)
    torch.cuda.synchronize()
    k = h.last_kernel()
    assert k.startswith("tile<f64,"), k
    for (alpha, beta, _), r, yh in zip(runs, refs, ys):
        R.assert_within(yh.numpy(), r[2], r[3], f"{k} hostvec pipeline pieces={pieces} a={alpha} b={beta}")
