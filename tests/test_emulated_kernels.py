"""The library's CUDA kernels EXECUTED on the CPU (tools/emu: the .cu sources compiled by g++ against a
CUDA-on-CPU emulation layer) and checked against the oracle through the same C ABI the GPU tests use.

What this covers: kernel logic -- indexing, warp/group collectives, block barriers, the mbarrier/TMA ring
protocol, hash tables, the host-side planning and launch configuration -- including the opt-in variants
(DESIGN.md section 9) that have not had a GPU run yet.  What it does not cover: real concurrency (fibers run one
at a time), the memory model, PTX, performance.  `-m gpu` stays the parity gate; this is the guard that keeps
a logic bug from costing a GPU call.

Shapes follow the reference's unit tests (Test_Sparse_spmv.hpp:1060-1068, Test_Sparse_spgemm.hpp:483-511,
Test_Sparse_SortCrs.hpp, Test_Sparse_spadd.hpp) at the small end so the file runs in about a minute."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import emu_lib as E
from crs_cases import MERGE_CASES, random_matrix, spadd_dense_check
from helpers import kk_matrix, rowwise_scale

TOL = {np.dtype(np.float64): 1e-10, np.dtype(np.float32): 1e-4}


@pytest.fixture(scope="module")
def emu():
    return E.lib()


class env:
    """Set library knobs (read by getenv at call time) for one block."""

    def __init__(self, **kv):
        self.kv = kv

    def __enter__(self):
        self.old = {k: os.environ.get(k) for k in self.kv}
        for k, v in self.kv.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = str(v)

    def __exit__(self, *a):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def check_spmv(oracle, plan, mode, rp, ci, v, ncols, x, y0, alpha, beta):
    nrows = len(rp) - 1
    trans = mode in "TH"
    y = y0.copy()
    E.spmv(plan, mode, nrows, ncols, rp, ci, v, x, y, alpha, beta)
    if not trans:
        exp = oracle.spmv_serial(rp, ci, v, x, y0.copy(), alpha, beta)
    else:
        exp = oracle.spmv_transpose(rp, ci, v, ncols, x, y0.copy(), alpha, beta)
    assert not np.isnan(y).any(), "NaN survived beta == 0"
    scale = rowwise_scale(rp, ci, v, x, y0, alpha, beta, ncols_out=ncols, trans=trans)
    err = np.abs(y.astype(np.float64) - exp.astype(np.float64))
    bad = err > TOL[v.dtype] * scale + 1e-300
    assert not bad.any(), f"{plan.kernel()} mode {mode} a={alpha} b={beta}: {bad.sum()} entries off"


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_spmv_modes_and_kernels(emu, oracle, dtype):
    rows, cols = 30000, 25000  # enough tiles per CTA (emulated device: 8 SMs) to wrap the TMA ring several times
    rp, ci, v = kk_matrix(rows, cols, rows * 12, 10, 200, dtype=dtype)
    rng = np.random.default_rng(13718)
    seen = set()
    for algo in (0, 1, 2):  # DEFAULT, NATIVE, MERGE_PATH (include/b200sparse.h)
        plan = E.SpmvPlan(algo)
        for mode in "NCTH":
            nx, ny = (cols, rows) if mode in "NC" else (rows, cols)
            x = rng.random(nx).astype(dtype)
            y0 = rng.random(ny).astype(dtype)
            y0[::17] = np.nan
            check_spmv(oracle, plan, mode, rp, ci, v, cols, x, y0, 2.5, 0.0)
            seen.add(plan.kernel().split("<")[0])
            y0 = rng.random(ny).astype(dtype)
            check_spmv(oracle, plan, mode, rp, ci, v, cols, x, y0, -1.0, 0.5)
        plan.close()
    assert any(k.startswith("tile") for k in seen) and any(k.startswith("transpose") for k in seen), seen


def test_spmv_unaligned_and_degenerate(emu, oracle):
    # CSR arrays at odd offsets: the TMA ring needs 16-byte alignment, the library must pick another kernel
    rp, ci, v = kk_matrix(2000, 2000, 30000, 5, 100)
    cib = np.empty(len(ci) + 1, np.int32)
    cib[1:] = ci
    vb = np.empty(len(v) + 1, np.float64)
    vb[1:] = v
    x = np.random.default_rng(1).random(2000)
    plan = E.SpmvPlan()
    check_spmv(oracle, plan, "N", rp, cib[1:], vb[1:], 2000, x, np.zeros(2000), 1.0, 0.0)
    assert not plan.kernel().startswith("tile"), plan.kernel()
    plan.close()
    # no rows / no entries
    plan = E.SpmvPlan()
    y = np.full(5, 3.0)
    E.spmv(plan, "N", 5, 4, np.zeros(6, np.int32), np.zeros(0, np.int32), np.zeros(0), np.ones(4), y, 1.0, 2.0)
    assert np.array_equal(y, np.full(5, 6.0))
    E.spmv(plan, "N", 0, 4, np.zeros(1, np.int32), np.zeros(0, np.int32), np.zeros(0), np.ones(4), np.zeros(0), 1.0, 0.0)
    plan.close()


def test_spmv_long_rows_both_strategies(emu, oracle):
    # a few rows far beyond the tile capacity: CTA-per-row kernel (default) and the opt-in segment path
    rng = np.random.default_rng(5)
    rows = cols = 6000
    lens = rng.integers(0, 8, rows)
    lens[[7, 3000, 5999]] = [5000, 2049, 6000]
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    ci = np.concatenate([np.sort(rng.choice(cols, l, replace=False)) for l in lens]).astype(np.int32)
    v = rng.uniform(-1, 1, len(ci))
    x, y0 = rng.random(cols), rng.random(rows)
    for knob in (None, "seg"):
        with env(B200SP_SPMV_LONGROWS=knob):
            plan = E.SpmvPlan()
            check_spmv(oracle, plan, "N", rp, ci, v, cols, x, y0, 1.5, -0.5)
            assert ("+seg" in plan.kernel()) == (knob == "seg"), plan.kernel()
            plan.close()


def test_spmv_self_tuning_never_changes_a_bit(emu):
    """An untuned plan runs the tiled kernel, times it, times the row-vector kernel and keeps the faster one: whichever it
    settles on (a matter of timing, so it may differ from run to run), every call must return the same bits -- also for the
    rows beyond the tile capacity, which both kernels leave to the CTA-per-row kernel."""
    rng = np.random.default_rng(8)
    rows = cols = 9000
    lens = rng.integers(0, 12, rows)
    lens[[5, 4000, 8999]] = [3000, 513, 700]
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    ci = np.concatenate([np.sort(rng.choice(cols, l, replace=False)) for l in lens]).astype(np.int32)
    assert len(ci) >= 32768  # large enough for the tiled path
    v = rng.uniform(-1, 1, len(ci))
    x, y0 = rng.uniform(-1, 1, cols), rng.uniform(-1, 1, rows)
    plan = E.SpmvPlan()
    seen, kernels = [], set()
    for _ in range(6):
        y = y0.copy()
        E.spmv(plan, "N", rows, cols, rp, ci, v, x, y, -0.7, 1.3)
        seen.append(y)
        kernels.add(plan.kernel().split("<")[0])
    assert kernels == {"tile", "vector"}
    for y in seen[1:]:
        assert np.array_equal(y, seen[0])
    plan.close()


def test_spmv_cached_transpose(emu, oracle):
    rp, ci, v = kk_matrix(2500, 1500, 30000, 10, 300)
    rng = np.random.default_rng(2)
    x, y0 = rng.random(2500), rng.random(1500)
    plan = E.SpmvPlan()
    E.ok(emu.b200sp_spmv_plan_set_option(plan.h, 1, 1))  # B200SP_SPMV_OPT_CACHE_TRANSPOSE
    for _ in range(2):  # second call reuses the cached transpose
        check_spmv(oracle, plan, "T", rp, ci, v, 1500, x, y0, 2.0, 0.25)
        assert plan.kernel().startswith("cached_transpose"), plan.kernel()
    plan.close()


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("lmax", [None, "16"], ids=["items", "items16"])
def test_spmm_kernels_layouts(emu, oracle, dtype, lmax):
    rng = np.random.default_rng(11)
    rows, cols = 1500, 1300
    lens = rng.integers(0, 30, rows)
    lens[[3, 700]] = [1200, 1100]  # long rows -> rows of many pieces
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    ci = np.concatenate([np.sort(rng.choice(cols, l, replace=False)) for l in lens]).astype(np.int32)
    v = rng.uniform(-1, 1, len(ci)).astype(dtype)
    with env(B200SP_SPMM_ITEM_LMAX=lmax):
        for k in (1, 3, 8, 17, 16, 40):
            for order in "CF":
                X = np.asarray(rng.random((cols, k)).astype(dtype), order=order)
                Y0 = np.asarray(rng.random((rows, k)).astype(dtype), order=order)
                for alpha, beta in ((1.0, 0.0), (-2.0, 0.5)):
                    Y = Y0.copy(order=order)
                    if beta == 0.0:
                        Y[::13] = np.nan
                    plan = E.SpmvPlan()
                    E.spmm(plan, "N", rows, cols, rp, ci, v, X, Y, alpha, beta)
                    plan.close()
                    exp = oracle.spmv_mv(rp, ci, v, cols, X, np.zeros_like(Y0) if beta == 0.0 else Y0.copy(order=order), alpha, beta)
                    assert not np.isnan(Y).any()
                    for j in range(k):
                        scale = rowwise_scale(rp, ci, v, X[:, j], Y0[:, j], alpha, beta)
                        err = np.abs(Y[:, j].astype(np.float64) - exp[:, j].astype(np.float64))
                        assert not (err > TOL[v.dtype] * scale + 1e-300).any(), (lmax, k, order, alpha, beta, j)


def gen_ab(oracle, m, k, n, nnz, dtype):
    A = kk_matrix(m, k, nnz, 10, 200, dtype=dtype, lo=1.0, hi=50.0, seed=1, sort=True, oracle=oracle)
    B = kk_matrix(k, n, nnz, 10, 200, dtype=dtype, lo=1.0, hi=50.0, seed=2, sort=True, oracle=oracle)
    return A, B


@pytest.mark.parametrize("dtype,eps", [(np.float64, 1e-7), (np.float32, 3.7e-3)])
def test_spgemm_all_variants(emu, oracle, dtype, eps):
    m, k, n = 1000, 500, 1600  # Test_Sparse_spgemm.hpp:483-511's small shape
    A, B = gen_ab(oracle, m, k, n, 20000, dtype)
    exp = oracle.spgemm(*A, *B, n)
    for sym in (3, 1, 2):
        for num in (7, 1, 2, 3, 4, 5, 6):
            if sym == 2 and num not in (1, 6):
                continue
            if sym == 1 and num == 7:
                continue
            with env(B200SP_SPGEMM_SYMBOLIC=sym, B200SP_SPGEMM_NUMERIC=num):
                rpC, ciC, vC, mx = E.spgemm(A, B, m, k, n, dtype)
            assert np.array_equal(rpC, exp[0]), (sym, num)
            assert mx == int(np.diff(exp[0]).max())
            assert np.array_equal(ciC, exp[1]), (sym, num)
            assert oracle.rel_mismatch(vC.astype(np.float64), exp[2].astype(np.float64), eps) == 0, (sym, num)


def test_spgemm_wide_rows_global_fallback(emu, oracle):
    # C rows beyond every shared-memory table: the global-memory accumulator
    rng = np.random.default_rng(9)
    m, k, n = 200, 3000, 40000
    lens = rng.integers(1, 4, m)
    lens[5] = 900
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    ci = np.concatenate([rng.choice(k, l, replace=False) for l in lens]).astype(np.int32)  # unsorted input rows
    v = rng.uniform(1, 50, len(ci))
    lensB = np.full(k, 40)
    rpB = np.concatenate([[0], np.cumsum(lensB)]).astype(np.int32)
    ciB = np.concatenate([rng.choice(n, 40, replace=False) for _ in range(k)]).astype(np.int32)
    vB = rng.uniform(1, 50, len(ciB))
    exp = oracle.spgemm(rp, ci, v, rpB, ciB, vB, n)
    assert np.diff(exp[0]).max() > 16384
    for num in (7, 1, 6):
        with env(B200SP_SPGEMM_NUMERIC=num):
            rpC, ciC, vC, _ = E.spgemm((rp, ci, v), (rpB, ciB, vB), m, k, n, np.float64)
        assert np.array_equal(rpC, exp[0]) and np.array_equal(ciC, exp[1])
        assert oracle.rel_mismatch(vC, exp[2], 1e-7) == 0


def test_spgemm_jacobi(emu, oracle):
    rng = np.random.default_rng(3)
    m = 800
    rp, ci, v = kk_matrix(m, m, 16000, 5, 100, lo=-1.0, hi=1.0, sort=True, oracle=oracle)
    # A must hold its diagonal (KokkosSparse_spgemm_jacobi.hpp): add it through the oracle's own spadd
    rpI = np.arange(m + 1, dtype=np.int32)
    ciI = np.arange(m, dtype=np.int32)
    rpA, ciA, vA = oracle.spadd(rp, ci, v, 1.0, rpI, ciI, np.full(m, 10.0), 1.0, True)
    rpB, ciB, vB = rpA, ciA, rng.uniform(-1, 1, len(ciA))
    dinv = rng.uniform(0.5, 1.5, m)
    exp = oracle.spgemm_jacobi(rpA, ciA, vA, rpB, ciB, vB, m, 0.7, dinv)
    L = emu
    h = C.c_void_p()
    E.ok(L.b200sp_spgemm_plan_create(C.byref(h)))
    rpC = np.zeros(m + 1, np.int32)
    nnz, mx = C.c_int64(), C.c_int()
    E.ok(L.b200sp_spgemm_symbolic_i32(h, None, m, m, m, E.ptr(rpA), E.ptr(ciA), E.ptr(rpB), E.ptr(ciB), E.ptr(rpC), C.byref(nnz), C.byref(mx)))
    ciC = np.full(nnz.value, -1, np.int32)
    vC = np.full(nnz.value, np.nan)
    E.ok(L.b200sp_spgemm_jacobi_f64_i32(h, None, m, m, m, E.ptr(rpA), E.ptr(ciA), E.ptr(vA), E.ptr(rpB), E.ptr(ciB), E.ptr(vB), E.ptr(rpC),
                                        E.ptr(ciC), E.ptr(vC), 0.7, E.ptr(dinv)))
    E.ok(L.b200sp_spgemm_plan_destroy(h, None))
    assert np.array_equal(rpC, exp[0]) and np.array_equal(ciC, exp[1])
    assert oracle.rel_mismatch(vC, exp[2], 1e-7) == 0


@pytest.mark.parametrize("case", sorted(MERGE_CASES))
def test_sort_and_merge_golden(emu, case):
    c = MERGE_CASES[case]
    if c["nrows"] == 0 and len(c["rowmap"]) == 0:
        pytest.skip("no row map at all: handled above the C ABI")
    rp, ci, v = c["rowmap"].copy(), c["entries"].copy(), c["values"].copy()
    out_rp = np.zeros_like(rp)
    nnz = C.c_int64()
    E.ok(emu.b200sp_sort_and_merge_count_f64_i32(None, c["nrows"], E.ptr(rp), E.ptr(ci), E.ptr(v), E.ptr(out_rp), C.byref(nnz)))
    assert nnz.value == len(c["gold_entries"]) and np.array_equal(out_rp, c["gold_rowmap"])
    oci, ov = np.zeros(nnz.value, np.int32), np.zeros(nnz.value)
    E.ok(emu.b200sp_sort_and_merge_fill_f64_i32(None, c["nrows"], E.ptr(rp), E.ptr(ci), E.ptr(v), E.ptr(out_rp), E.ptr(oci), E.ptr(ov)))
    assert np.array_equal(oci, c["gold_entries"]) and np.array_equal(ov, c["gold_values"])


def test_sort_transpose(emu, oracle):
    rp, ci, v = random_matrix(700, 90, 0, 200, False, seed=4)  # rows longer than ncols: repeated columns (ties)
    eci, ev = ci.copy(), v.copy()
    oracle.sort_crs_stable(rp, eci, ev)
    ci2, v2 = ci.copy(), v.copy()
    E.ok(emu.b200sp_sort_crs_f64_i32(None, 700, E.ptr(rp), E.ptr(ci2), E.ptr(v2)))
    assert np.array_equal(ci2, eci) and np.array_equal(v2, ev)
    t_rp, t_ci, t_v = np.zeros(91, np.int32), np.zeros(len(ci), np.int32), np.zeros(len(ci))
    E.ok(emu.b200sp_transpose_f64_i32(None, 700, 90, E.ptr(rp), E.ptr(ci), E.ptr(v), E.ptr(t_rp), E.ptr(t_ci), E.ptr(t_v)))
    e_rp, e_ci, e_v = oracle.transpose(rp, ci, v, 90)
    assert np.array_equal(t_rp, e_rp) and np.array_equal(t_ci, e_ci) and np.array_equal(t_v, e_v)


@pytest.mark.parametrize("sorted_input", [True, False])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_spadd(emu, oracle, sorted_input, dtype):
    m, n = 600, 400
    A = random_matrix(m, n, 0, 60, sorted_input, seed=1, dtype=dtype)
    B = random_matrix(m, n, 0, 60, sorted_input, seed=2, dtype=dtype)
    h = C.c_void_p()
    E.ok(emu.b200sp_spadd_plan_create(C.byref(h), int(sorted_input), 0))
    rpC = np.zeros(m + 1, np.int32)
    nnz = C.c_int64()
    E.ok(emu.b200sp_spadd_symbolic_i32(h, None, m, n, E.ptr(A[0]), E.ptr(A[1]), E.ptr(B[0]), E.ptr(B[1]), E.ptr(rpC), C.byref(nnz)))
    ciC, vC = np.zeros(nnz.value, np.int32), np.zeros(nnz.value, dtype)
    fn = getattr(emu, "b200sp_spadd_numeric_%s_i32" % E.sfx(dtype))
    E.ok(fn(h, None, m, n, E.ptr(A[0]), E.ptr(A[1]), E.ptr(A[2]), E.scalar(dtype, 0.3), E.ptr(B[0]), E.ptr(B[1]), E.ptr(B[2]),
            E.scalar(dtype, -1.7), E.ptr(rpC), E.ptr(ciC), E.ptr(vC)))
    E.ok(emu.b200sp_spadd_plan_destroy(h, None))
    exp = oracle.spadd(*A, 0.3, *B, -1.7, sorted_input)
    assert np.array_equal(rpC, exp[0]) and np.array_equal(ciC, exp[1]) and np.array_equal(vC, exp[2])
    spadd_dense_check(A, B, (rpC, ciC, vC), n, 0.3, -1.7)


_HARNESS_RUNS = [("spmv_t", "random:5"), ("crs", "reverse"), ("spmv_longrows", "reverse")]
if os.environ.get("B200SP_TEST_FULL") == "1":  # these two take another ~70 s; their kernels have ctypes tests of their own below
    _HARNESS_RUNS += [("jacobi", "random:11"), ("spmv64", "random:3")]


@pytest.mark.parametrize("suite,order", _HARNESS_RUNS)
def test_harness_runs_emulated(suite, order):
    """tools/gpu_check.cpp -- the torch-free harness of the GPU calls -- linked against the emulated library: the
    suite EXECUTES (not --dry) and every check is ok.  B200EMU_GUARD puts every device allocation of the harness
    between inaccessible pages (an out-of-bounds access of a kernel is a fault, not a silent read); B200EMU_ORDER runs
    the threads of a block in another order (a missing barrier that forward order hides shows up)."""
    envv = dict(os.environ, B200EMU_GUARD="1", B200EMU_ORDER=order)
    out = subprocess.run([E.harness(), "--timeout-scale", "40", "--suite", suite, "--out", os.devnull], capture_output=True, text=True,
                         timeout=900, env=envv)
    log = out.stdout + out.stderr
    assert out.returncode == 0, log[-3000:]
    assert "[summary] " + suite in log and " FAIL" not in log, log[-3000:]


def test_kokkos_shim_driver_emulated():
    """tests/shim_mock/shim_driver.cpp -- the Kokkos TPL specialisations of kokkos_shim/ instantiated as KokkosSparse::spmv /
    spgemm / spadd would -- built against the emulated library: SPMV, SPMV_MV, SPGEMM_*, SPADD_* and (--bsr, --jacobi) the
    BsrMatrix, SPGEMM_JACOBI, GAUSS_SEIDEL_*, GMRES and SPTRSV_* specialisations run end to end on the host."""
    E.harness()  # builds everything under tools/emu/_build
    drv = os.path.join(os.path.dirname(E.harness()), "shim_driver_emu")
    out = subprocess.run([drv, "--bsr", "--jacobi", "--gs", "--gmres", "--spmv64", "--sptrsv", "--n", "12000"], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "SHIM DRIVER OK" in out.stdout and out.stdout.count(" 0 mismatches") == 14, out.stdout


@pytest.mark.skipif(os.environ.get("B200EMU_NESTED") == "1", reason="this is the nested run")
@pytest.mark.parametrize("order", ["random:9"])  # `reverse` is covered by the harness runs above
def test_kernels_under_other_schedules(order):
    """The ctypes tests of this file once more with the threads of every block scheduled differently: `reverse`
    runs high thread ids first; `random` shuffles every pass and gives each warp its own speed, so producer warps run
    ahead of (or behind) the consumers.  Correct kernels do not care.  (Checked by mutation when this was written:
    removing the consumers' wait on the `full` barrier of the SpMV tile ring fails under every order, removing the
    producer's wait on the `empty` barrier fails under `random` only.)"""
    envv = dict(os.environ, B200EMU_ORDER=order, B200EMU_NESTED="1")
    # the default CPU suite re-runs the kernels with producer / consumer rings and cross-warp hand-offs (where a schedule can
    # matter); B200SP_TEST_FULL=1 re-runs every ctypes test of the file (about two minutes more)
    sel = ("(spmv or spmm or spgemm or sort or spadd) and not harness" if os.environ.get("B200SP_TEST_FULL") == "1"
           else "(spmv or spmm or multi_gpu) and not harness and not spgemm and not sort")
    out = subprocess.run([os.sys.executable, "-m", "pytest", os.path.abspath(__file__), "-x", "-q", "-k", sel],
                         capture_output=True, text=True, timeout=1500, env=envv,
                         cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    assert out.returncode == 0, (out.stdout + out.stderr)[-3000:]


def test_cg_driver(emu, oracle):
    """b200sp_cg_solve (device-resident CG, the reference's pcgsolve without preconditioner) against the oracle's
    restatement: same iteration count up to the rounding of the dots (+-2), same residual bound, same solution."""
    from test_oracle_cg import spd_lap27

    rp, ci, v = spd_lap27(14, shift=0.5)
    n = len(rp) - 1
    rng = np.random.default_rng(0)
    xs = rng.uniform(-1, 1, n)
    b = np.zeros(n)
    oracle.spmv_serial(rp, ci, v, xs, b, 1.0, 0.0)
    xo = np.zeros(n)
    it_o, nr_o = oracle.cg(rp, ci, v, b, xo, 100000, 1e-7)
    for check_every in (1, 8):
        plan = E.SpmvPlan()
        x = np.zeros(n)
        it, nr = E.cg_solve(plan, rp, ci, v, b, x, 100000, 1e-7, check_every)
        plan.close()
        assert abs(it - it_o) <= 2 and nr <= 1e-7, (it, it_o, nr)
        assert np.linalg.norm(x - xo) / np.linalg.norm(xo) < 1e-8
    plan = E.SpmvPlan()
    x = np.zeros(n)
    it, nr = E.cg_solve(plan, rp, ci, v, b, x, 7, 1e-7, 3)  # the limit stops it (7 is not a multiple of the polling interval)
    xo7 = np.zeros(n)
    it7, nr7 = oracle.cg(rp, ci, v, b, xo7, 7, 1e-7)
    assert it == 7 == it7 and abs(nr - nr7) <= 1e-9 * nr7 and np.allclose(x, xo7, rtol=1e-10, atol=1e-12)
    it0, _ = E.cg_solve(plan, rp, ci, v, b, xo.copy(), 100, 1e-5, 4)  # converged start: no iteration
    assert it0 == 0
    plan.close()


def test_multi_gpu_kernels_single_process(emu, oracle):
    """The device side of the row-block operator (kokkos-kernels_b200/multigpu.py) with the ranks played one after the other in
    one process: every rank's SpMV stores its block of y into its own buffer AND into the slots of the other ranks' next-x
    buffers (b200sp_spmv_scatter_*, the fused all-gather; peer pointers are plain pointers here), then the copy kernel of the
    multicast mode (b200sp_multicast_push) for every size / alignment class it distinguishes.  Needs no NVLink: logic only."""
    L = emu
    n, P = 9000, 3
    rp, ci, v = kk_matrix(n, n, n * 9, 5, 400)
    x = np.random.default_rng(4).uniform(-1, 1, n)
    exp = oracle.spmv_serial(rp, ci, v, x, np.zeros(n), 1.0, 0.0)
    bounds = [0, 2999, 6001, n]  # ragged blocks, odd offsets (8-byte aligned slots only)
    nxt = [np.full(n, np.nan) for _ in range(P)]  # every rank's buffer for the next x
    for r in range(P):
        lo, hi = bounds[r], bounds[r + 1]
        rpl = (rp[lo:hi + 1] - rp[lo]).astype(np.int32)  # row block with rebased row map; columns stay global
        cil, vl = ci[rp[lo]:rp[hi]].copy(), v[rp[lo]:rp[hi]].copy()
        plan = E.SpmvPlan()
        E.ok(L.b200sp_spmv_plan_tune(plan.h, 8, 4, 0))  # the tile kernel, as at bench size
        extra = [nxt[q][lo:hi] for q in range(P) if q != r]
        arr = (C.c_void_p * len(extra))(*[C.c_void_p(a.ctypes.data) for a in extra])
        E.ok(L.b200sp_spmv_scatter_f64_i32(plan.h, None, hi - lo, n, len(cil), 1.0, E.ptr(rpl), E.ptr(cil), E.ptr(vl), E.ptr(x),
                                           E.ptr(nxt[r][lo:hi]), len(extra), arr))
        assert plan.kernel().startswith("tile"), plan.kernel()
        plan.close()
    scale = rowwise_scale(rp, ci, v, x, np.zeros(n), 1.0, 0.0)
    for q in range(P):
        assert not np.isnan(nxt[q]).any()
        assert np.array_equal(nxt[q], nxt[0])  # every replica bit-identical
        assert np.all(np.abs(nxt[q] - exp) <= 1e-10 * scale + 1e-300)
    # forward mode: finished tiles go on to ONE destination from the producer warp (the multicast mapping on a GPU)
    fwd = np.full(n, np.nan)
    loc = np.full(n, np.nan)
    for r in range(P):
        lo, hi = bounds[r], bounds[r + 1]
        rpl = (rp[lo:hi + 1] - rp[lo]).astype(np.int32)
        cil, vl = ci[rp[lo]:rp[hi]].copy(), v[rp[lo]:rp[hi]].copy()
        plan = E.SpmvPlan()
        E.ok(L.b200sp_spmv_plan_tune(plan.h, 8, 4, 0))
        E.ok(L.b200sp_spmv_forward_f64_i32(plan.h, None, hi - lo, n, len(cil), 1.0, E.ptr(rpl), E.ptr(cil), E.ptr(vl), E.ptr(x),
                                           E.ptr(loc[lo:hi]), C.c_void_p(fwd[lo:hi].ctypes.data)))
        assert plan.kernel().startswith("tile"), plan.kernel()
        plan.close()
    assert np.array_equal(fwd, nxt[0]) and np.array_equal(loc, nxt[0])
    # ... and on ~55 entries per row (tiles of ~37 rows, the config-2 shape): the forwarding is software-pipelined by one tile there
    rp2, ci2, v2 = kk_matrix(4000, 4000, 4000 * 55, 5, 600)
    x2 = np.random.default_rng(6).uniform(-1, 1, 4000)
    exp2 = oracle.spmv_serial(rp2, ci2, v2, x2, np.zeros(4000), 1.0, 0.0)
    fwd2, loc2 = np.full(4000, np.nan), np.full(4000, np.nan)
    plan = E.SpmvPlan()
    E.ok(L.b200sp_spmv_plan_tune(plan.h, 8, 4, 0))
    E.ok(L.b200sp_spmv_forward_f64_i32(plan.h, None, 4000, 4000, len(ci2), 1.0, E.ptr(rp2), E.ptr(ci2), E.ptr(v2), E.ptr(x2), E.ptr(loc2),
                                       C.c_void_p(fwd2.ctypes.data)))
    assert plan.kernel().startswith("tile"), plan.kernel()
    plan.close()
    scale2 = rowwise_scale(rp2, ci2, v2, x2, np.zeros(4000), 1.0, 0.0)
    assert np.array_equal(fwd2, loc2) and np.all(np.abs(loc2 - exp2) <= 1e-10 * scale2 + 1e-300)
    # multicast push: 16-byte stores with a one-element head / tail when the 16-byte phase asks for it
    src_all = np.random.default_rng(5).uniform(-1, 1, 5000)
    for off in (0, 1):  # 8-byte phase of both pointers (they must agree)
        for cnt in (0, 1, 2, 3, 255, 256, 257, 4097):
            src = src_all[off:off + cnt]
            dst_all = np.full(5000, -7.0)
            dst = dst_all[2 + off:2 + off + cnt]
            assert ((src.ctypes.data ^ dst.ctypes.data) & 15) == 0 or cnt == 0
            E.ok(L.b200sp_multicast_push(None, E.ptr(src) if cnt else None, E.ptr(dst) if cnt else None, cnt * 8, 3))
            assert np.array_equal(dst, src)
            assert np.all(dst_all[:2 + off] == -7.0) and np.all(dst_all[2 + off + cnt:] == -7.0)  # nothing outside
    y = np.zeros(4)
    assert L.b200sp_multicast_push(None, E.ptr(src_all[0:4]), E.ptr(y[1:]), 24, 1) != 0  # different 16-byte phase: refused


@pytest.mark.parametrize("pieces", [None, "3"])
def test_hostvec_pipeline_logic(emu, oracle, pieces):
    """b200sp_spmv_hostvec_* (host x / y, double-buffered upload, piecewise compute + download): the piece arithmetic for
    every piece count, incl. the B200SP_HOSTVEC_PIECES override; streams and copies are synchronous under the emulation."""
    n = 70000  # nnz >= 2^22 switches the pipeline on
    rp, ci, v = kk_matrix(n, n, n * 64, 3, 2000)
    assert len(ci) >= (1 << 22)
    rng = np.random.default_rng(8)
    x, y0 = rng.uniform(-1, 1, n), rng.uniform(-1, 1, n)
    with env(B200SP_HOSTVEC_PIECES=pieces):
        for alpha, beta in ((1.0, 0.0), (2.0, -0.5)):
            plan = E.SpmvPlan()
            y = y0.copy()
            for _ in range(2):  # second call: staging buffers and analysis reused
                y[:] = y0
                E.ok(emu.b200sp_spmv_hostvec_f64_i32(plan.h, None, b"N", n, n, len(ci), alpha, E.ptr(rp), E.ptr(ci), E.ptr(v), E.ptr(x), beta,
                                                     E.ptr(y)))
            plan.close()
            exp = oracle.spmv_serial(rp, ci, v, x, y0.copy(), alpha, beta)
            assert np.all(np.abs(y - exp) <= 1e-10 * rowwise_scale(rp, ci, v, x, y0, alpha, beta) + 1e-300)


def test_hostvec_deferred_completion_logic(emu, oracle):
    """B200SP_SPMV_OPT_HOSTVEC_DEFER: calls stop waiting for their own download; b200sp_spmv_hostvec_flush closes the sequence.
    Under the emulation the copies are synchronous, so this checks the bookkeeping (buffers alternate, flush resets, the option
    cannot be switched off with downloads outstanding), not the overlap."""
    n = 70000
    rp, ci, v = kk_matrix(n, n, n * 64, 3, 2000)
    rng = np.random.default_rng(8)
    xs = [rng.uniform(-1, 1, n) for _ in range(5)]
    ys = [np.full(n, np.nan) for _ in range(5)]
    plan = E.SpmvPlan()
    E.ok(emu.b200sp_spmv_plan_set_option(plan.h, 2, 1))
    for x, y in zip(xs, ys):
        E.ok(emu.b200sp_spmv_hostvec_f64_i32(plan.h, None, b"N", n, n, len(ci), 1.0, E.ptr(rp), E.ptr(ci), E.ptr(v), E.ptr(x), 0.0, E.ptr(y)))
    assert emu.b200sp_spmv_plan_set_option(plan.h, 2, 0) == 3  # B200SP_ERR_STATE: downloads outstanding
    E.ok(emu.b200sp_spmv_hostvec_flush(plan.h, None))
    E.ok(emu.b200sp_spmv_hostvec_flush(plan.h, None))  # idempotent
    E.ok(emu.b200sp_spmv_plan_set_option(plan.h, 2, 0))
    for x, y in zip(xs, ys):
        exp = oracle.spmv_serial(rp, ci, v, x, np.zeros(n), 1.0, 0.0)
        assert np.all(np.abs(y - exp) <= 1e-10 * rowwise_scale(rp, ci, v, x, np.zeros(n), 1.0, 0.0) + 1e-300)
    plan.close()
    assert emu.b200sp_spmv_hostvec_flush(None, None) == 1


@pytest.mark.parametrize("dtype,tol", [(np.float64, 1e-8), (np.float32, 1e-5)])
@pytest.mark.parametrize("variant", ["cgs2", "mgs", "matrixprec"])
def test_gmres(emu, oracle, dtype, tol, variant):
    """b200sp_gmres_* on the reference's own unit test (sparse/unit_test/Test_Sparse_gmres.hpp:86-170: n = 5000, m = 15, B = 1,
    X = 0, CGS2 / MGS / MatrixPrec(A), double 1e-8 and float 1e-5): true relative residual below the tolerance, flag Conv, and
    the same iteration count as the oracle's restatement of the reference algorithm."""
    from gmres_cases import gmres_matrix, true_rel_res

    n, m = (5000 if (variant == "cgs2" and dtype == np.float64) else 2000), 15  # the reference's size once, smaller for the rest
    A = gmres_matrix(n, 1.0, dtype=dtype)
    b = np.ones(n, dtype=dtype)
    prec = A if variant == "matrixprec" else None
    ortho = 1 if variant == "mgs" else 0
    xo = np.zeros(n, dtype=dtype)
    st_o, it_o, res_o, flag_o = oracle.gmres(A, b, xo, m=m, tol=tol, ortho=ortho, prec=prec)
    pa, pm = E.SpmvPlan(), (E.SpmvPlan() if prec is not None else None)
    x = np.zeros(n, dtype=dtype)
    rc, it, res, flag = E.gmres(pa, A, b, x, m=m, tol=tol, ortho=ortho, prec=prec, plan_m=pm)
    pa.close()
    if pm:
        pm.close()
    assert rc == 0 and flag == 0 == flag_o, (rc, it, res, flag)
    assert true_rel_res(oracle, A, b, x) < tol and res < tol
    assert abs(it - it_o) <= 1, (it, it_o)
    assert np.linalg.norm(x.astype(np.float64) - xo.astype(np.float64)) / np.linalg.norm(xo.astype(np.float64)) < 50 * tol


def test_gmres_corner_cases(emu, oracle):
    from gmres_cases import gmres_matrix

    n = 300
    A = gmres_matrix(n, 2.0)
    pa = E.SpmvPlan()
    x = np.ones(n)
    rc, it, res, flag = E.gmres(pa, A, np.zeros(n), x, m=10)  # zero rhs: X reset to 0
    assert rc == 0 and it == 0 and res == 0 and np.all(x == 0) and flag == 0
    xs = np.random.default_rng(1).uniform(-1, 1, n)
    b = np.zeros(n)
    oracle.spmv_serial(A[0], A[1], A[2], xs, b, 1.0, 0.0)
    x = xs.copy()
    rc, it, res, flag = E.gmres(pa, A, b, x, m=10)  # exact guess
    assert rc == 0 and it == 0 and flag == 0 and np.array_equal(x, xs)
    hard = gmres_matrix(n, 0.02)
    x, xo = np.zeros(n), np.zeros(n)
    rc, it, res, flag = E.gmres(pa, hard, np.ones(n), x, m=2, tol=1e-13, max_restart=1)  # restart limit: never Conv
    st_o, it_o, res_o, flag_o = oracle.gmres(hard, np.ones(n), xo, m=2, tol=1e-13, max_restart=1)
    assert rc == 0 and flag == flag_o != 0 and it == it_o and abs(res - res_o) <= 1e-8 * abs(res_o)
    assert emu.b200sp_gmres_f64_i32(pa.h, None, n, len(A[1]), E.ptr(A[0]), E.ptr(A[1]), E.ptr(A[2]), None, 0, None, None, None, E.ptr(b), E.ptr(x), 10,
                                    1e-8, 50, 7, C.byref(C.c_int()), C.byref(C.c_double()), C.byref(C.c_int())) != 0  # ortho
    pa.close()


@pytest.mark.parametrize("variant", ["cgs2", "matrixprec"])
def test_gmres_bsr(emu, oracle, variant):
    """The BsrMatrix half of the reference's GMRES test (Test_Sparse_gmres.hpp:86-101: the same matrix as 10 x 10 blocks)."""
    from gmres_cases import crs_to_bsr, gmres_matrix, true_rel_res

    n, m, bs, tol = 2000, 15, 10, 1e-8
    A = gmres_matrix(n, 1.0)
    Ab = crs_to_bsr(*A, bs)
    b = np.ones(n)
    prec = Ab if variant == "matrixprec" else None
    pa, pm = E.BsrPlan(), (E.BsrPlan() if prec is not None else None)
    x = np.zeros(n)
    rc, it, res, flag = E.gmres_bsr(pa, bs, Ab, b, x, m=m, tol=tol, prec=prec, plan_m=pm)
    pa.close()
    if pm:
        pm.close()
    xo = np.zeros(n)
    st_o, it_o, _, flag_o = oracle.gmres(A, b, xo, m=m, tol=tol, prec=A if prec is not None else None)
    assert rc == 0 and flag == 0 == flag_o and abs(it - it_o) <= 1, (rc, it, it_o, flag)
    assert true_rel_res(oracle, A, b, x) < tol and res < tol


def test_plan_invalidate_drops_stale_analysis(emu, oracle):
    """A different matrix at the SAME row_map address with the same shape and nnz finds the cached tiles of the first one
    (the cache key is pointer + shape); b200sp_spmv_plan_invalidate is the documented way out (ADVICE round 1)."""
    rng = np.random.default_rng(5)
    m = n = 900
    lens1 = rng.integers(1, 12, m)
    lens2 = lens1[::-1].copy()  # same nnz, other row boundaries
    rp = np.concatenate([[0], np.cumsum(lens1)]).astype(np.int32)
    nnz = int(rp[-1])
    ci = rng.integers(0, n, nnz).astype(np.int32)
    v = rng.uniform(-1, 1, nnz)
    x = rng.random(n)
    plan = E.SpmvPlan()
    check_spmv(oracle, plan, "N", rp, ci, v, n, x, np.zeros(m), 1.0, 0.0)
    rp[:] = np.concatenate([[0], np.cumsum(lens2)]).astype(np.int32)  # edited in place: same pointer, m, nnz
    E.ok(emu.b200sp_spmv_plan_invalidate(plan.h, None))
    check_spmv(oracle, plan, "N", rp, ci, v, n, x, np.zeros(m), 1.0, 0.0)
    plan.close()
