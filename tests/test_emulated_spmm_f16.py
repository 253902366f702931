"""Half-precision rank-2 SpMV (b200sp_spmm_f16_i32) EXECUTED on the CPU (tools/emu) on the shared cases of spmm_cases.py in
float16: every path with its last_kernel(), the bit identity with the fp32 entry point on the item paths
(Y16 == round_fp16(Y32 on the widened inputs)), fp32 accumulation, special values, strided and misaligned operands, and the
memory a plan gives back."""
import ctypes as C

import numpy as np
import pytest

import emu_lib as E
import half_ref as H
import spmm_cases as cases
from test_emulated_kernels import env

F16 = np.float16


@pytest.fixture(scope="module")
def emu():
    return E.lib()


def _lay(a):
    it = a.dtype.itemsize
    if a.strides[1] == it:  # row-major: leading dimension = row stride
        return a.strides[0] // it, 1
    assert a.strides[0] == it
    return a.strides[1] // it, 0


def spmm16(plan, mode, m, n, rp, ci, v, X, Y, alpha, beta):
    """The fp16 entry point on numpy float16 arrays (C- or F-ordered 2-D views); plan None runs without a plan."""
    ldx, rmx = _lay(X)
    ldy, rmy = _lay(Y)
    E.ok(E.lib().b200sp_spmm_f16_i32(plan.h if plan else None, None, mode.encode(), m, n, len(ci), X.shape[1], C.c_float(alpha),
                                     E.ptr(rp), E.ptr(ci), E.ptr(v), E.ptr(X), ldx, rmx, C.c_float(beta), E.ptr(Y), ldy, rmy))


def run16(A, X, Y0, alpha, beta, mode="N", plan=True, y_nan=False):
    rp, ci, v, ncols = A
    Y = Y0.copy(order="K")
    if y_nan:
        Y[...] = np.nan
    p = E.SpmvPlan() if plan else None
    try:
        spmm16(p, mode, len(rp) - 1, ncols, rp, ci, v, X, Y, alpha, beta)
        return Y, (p.kernel() if p else None)
    finally:
        if p:
            p.close()


def run32(A, X, Y0, alpha, beta, mode="N"):
    """The fp32 entry point on the widened inputs, same layouts."""
    rp, ci, v, ncols = A
    w = lambda a: np.asarray(a.astype(np.float32), order="F" if (a.flags.f_contiguous and not a.flags.c_contiguous) else "C")
    Y = w(Y0)
    p = E.SpmvPlan()
    try:
        E.spmm(p, mode, len(rp) - 1, ncols, rp, ci, v.astype(np.float32), w(X), Y, alpha, beta)
        return Y, p.kernel()
    finally:
        p.close()


def case16(name, seed=5):
    rp, ci, v, ncols = cases.SMALL_CASES[name](seed, np.float32)
    if name == "cancelling":  # pairs +-a with a up to 2^24: scaled into the fp16 range (by a power of two, so they still cancel)
        v = v * np.float32(2.0**-10)
    return rp, ci, v.astype(F16), ncols


def operands16(A, k, order, mode="N", seed=None):
    rp, ci, v, ncols = A
    rng = np.random.default_rng(k if seed is None else seed)
    xr, yr = (len(rp) - 1, ncols) if mode in "TH" else (ncols, len(rp) - 1)
    return (np.asarray(cases.dense_operands(rng, xr, k, F16), order=order), np.asarray(cases.dense_operands(rng, yr, k, F16), order=order))


def check_bound(A, X, Y0, got, alpha, beta, mode, what):
    rp, ci, v, _ = A
    t = mode in "TH"
    H.assert_within16(got, H.spmm_exact16(rp, ci, v, X, Y0, alpha, beta, t), H.spmm_bound16(rp, ci, v, X, Y0, alpha, beta, t), what)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint16)


# (X order, Y order, k) -> label of the path
PATHS = [("C", "C", 16, "spmm_items_vec"), ("C", "C", 5, "spmm_items"), ("F", "F", 16, "spmm_relayout+items"),
         ("C", "F", 16, "spmm_relayout+items"), ("F", "C", 8, "spmm_relayout+items"), ("F", "F", 3, "spmm_general"),
         ("C", "C", 24, "spmm_items_vec")]


@pytest.mark.parametrize("xo,yo,k,label", PATHS)
@pytest.mark.parametrize("case", ["thresholds", "small_mod3", "cancelling"])
def test_paths_within_bound(emu, case, xo, yo, k, label):
    A = case16(case)
    X, Y0 = operands16(A, k, "C")
    X, Y0 = np.asarray(X, order=xo), np.asarray(Y0, order=yo)
    for alpha, beta in ((1.5, -0.5), (1.0, 0.0)):
        got, kern = run16(A, X, Y0, alpha, beta, y_nan=beta == 0)
        assert kern == label, (kern, label)
        check_bound(A, X, Y0, got, alpha, beta, "N", f"{kern} {case} k={k} {xo}{yo} a={alpha} b={beta}")


@pytest.mark.parametrize("mode", ["N", "T", "H", "C"])
@pytest.mark.parametrize("order", ["C", "F"])
def test_no_plan_and_transpose(emu, mode, order):
    """Without a plan: spmm_general (N/C) or the fp32-scratch transpose (T/H); with a plan, T/H report spmm_transpose."""
    A = case16("small_mod1")
    for k in (1, 5, 16):
        X, Y0 = operands16(A, k, order, mode)
        for alpha, beta in ((-1.5, 0.5), (1.0, 0.0), (0.0, 2.5)):
            got, _ = run16(A, X, Y0, alpha, beta, mode, plan=False, y_nan=beta == 0)
            check_bound(A, X, Y0, got, alpha, beta, mode, f"no plan {mode} k={k} {order} a={alpha} b={beta}")
            if mode in "TH":
                got, kern = run16(A, X, Y0, alpha, beta, mode, y_nan=beta == 0)
                if alpha != 0:
                    assert kern == "spmm_transpose", kern
                check_bound(A, X, Y0, got, alpha, beta, mode, f"{kern} {mode} k={k} {order} a={alpha} b={beta}")


IDENTITY = [("C", "C", 16, {}), ("C", "C", 5, {}), ("F", "F", 16, {}), ("C", "F", 5, {}), ("F", "C", 8, {}),
            ("C", "C", 16, {"B200SP_SPMM_ITEM_LMAX": "16"}), ("C", "C", 16, {"B200SP_SPMM_ITEM_LMAX": "256"}),
            ("F", "F", 4, {"B200SP_SPMM_ITEM_LMAX": "16"})]


@pytest.mark.parametrize("xo,yo,k,envs", IDENTITY)
def test_bit_identity_with_fp32(emu, xo, yo, k, envs):
    """Y16 == round_fp16(fp32 call on the widened inputs) on every item path, multi-piece rows of both reduce kernels
    included (the thresholds case has rows of more than 64 pieces at LMAX 16 and 64)."""
    A = case16("thresholds")
    X, Y0 = operands16(A, k, "C")
    X, Y0 = np.asarray(X, order=xo), np.asarray(Y0, order=yo)
    with env(**envs):
        for alpha, beta in ((1.5, -0.5), (1.0, 0.0), (-0.75, 1.0)):
            got, kern = run16(A, X, Y0, alpha, beta)
            y32, kern32 = run32(A, X, Y0, alpha, beta)
            assert kern.startswith("spmm_items") or kern == "spmm_relayout+items", kern
            assert kern32.split("_vec")[0] == kern.split("_vec")[0], (kern, kern32)
            assert np.array_equal(bits(got), bits(H.round16(y32))), f"{kern} k={k} {xo}{yo} {envs} a={alpha} b={beta}"


def one_row(vals, k=8, ncols=None):
    """A 1-row matrix over len(vals) columns (or ncols, cycling) and X of ones."""
    vals = np.asarray(vals, dtype=np.float64)
    nc = ncols or len(vals)
    rp = np.array([0, len(vals)], dtype=np.int32)
    ci = (np.arange(len(vals)) % nc).astype(np.int32)
    return (rp, ci, vals.astype(F16), nc), np.ones((nc, k), dtype=F16), np.zeros((1, k), dtype=F16)


ACCUMULATION = [([2048, 1, -2048], 1.0, 1.0), ([60000, 60000, -60000], 1.0, 60000.0), ([60000, 60000], 0.5, 60000.0),
                ([60000, 60000], 1.0, np.inf), ([-60000, -60000], 1.0, -np.inf)]


@pytest.mark.parametrize("vals,alpha,want", ACCUMULATION)
@pytest.mark.parametrize("xo,yo,k,plan", [("C", "C", 8, True), ("C", "C", 3, True), ("F", "F", 8, True), ("C", "C", 8, False)])
def test_fp32_accumulation(emu, vals, alpha, want, xo, yo, k, plan):
    A, X, Y0 = one_row(vals, k)
    got, kern = run16(A, np.asarray(X, order=xo), np.asarray(Y0, order=yo), alpha, 0.0, plan=plan)
    assert np.all(got.astype(np.float64) == want), (got, want, kern)


@pytest.mark.parametrize("vals,alpha,want", ACCUMULATION)
def test_fp32_accumulation_transpose(emu, vals, alpha, want):
    """The same rows as columns of A, through mode T (fp32 scratch, one rounding)."""
    vals = np.asarray(vals, dtype=np.float64)
    n = len(vals)
    A = (np.arange(n + 1, dtype=np.int32), np.zeros(n, dtype=np.int32), vals.astype(F16), 1)
    X, Y0 = np.ones((n, 8), dtype=F16), np.zeros((1, 8), dtype=F16)
    for plan in (True, False):
        got, _ = run16(A, X, Y0, alpha, 0.0, "T", plan=plan)
        assert np.all(got.astype(np.float64) == want), (got, want, plan)


def test_special_values(emu):
    # subnormal results: 2^-24 exactly; 3 * 2^-25 = 1.5 * 2^-24, a tie rounded to even (2^-23); 2^-25, a tie between 0 and
    # 2^-24 rounded to 0
    for vals, x, want in (([2.0**-14], 2.0**-10, 2.0**-24), ([2.0**-13] * 3, 2.0**-12, 2.0**-23),
                          ([2.0**-14, -2.0**-15], 2.0**-10, 0.0)):
        A, X, Y0 = one_row(vals, 8)
        X[...] = x
        for plan, order in ((True, "C"), (True, "F"), (False, "C")):
            got, kern = run16(A, np.asarray(X, order=order), np.asarray(Y0, order=order), 1.0, 0.0, plan=plan)
            assert np.all(got.astype(np.float64) == want), (vals, got, want, kern)
    # NaN / Inf propagation and NaN in Y with beta == 0
    A = case16("small_mod1")
    X, Y0 = operands16(A, 8, "C")
    X[3, :] = np.inf
    X[7, 2] = np.nan
    for order in "CF":
        Xo, Yo = np.asarray(X, order=order), np.asarray(Y0, order=order)
        for alpha, beta in ((1.0, 0.0), (2.0, -1.0)):
            got, kern = run16(A, Xo, Yo, alpha, beta, y_nan=beta == 0)
            check_bound(A, Xo, Yo, got, alpha, beta, "N", f"{kern} inf/nan {order}")
    Yn = np.full_like(Y0, np.nan)
    got, _ = run16(A, np.ones_like(X), Yn, 1.0, 0.0)
    assert not np.isnan(got).any()


def test_strided_and_misaligned(emu):
    """Odd leading dimensions and X / Y one element off 16-byte alignment give the bits of the aligned vector kernel."""
    A = case16("thresholds")
    k = 16
    X, Y0 = operands16(A, k, "C")
    ref, kern = run16(A, X, Y0, 1.5, -0.5)
    assert kern == "spmm_items_vec", kern
    # odd leading dimension: views into wider buffers
    bx = np.zeros((X.shape[0], k + 1), dtype=F16)
    by = np.zeros((Y0.shape[0], k + 1), dtype=F16)
    bx[:, :k], by[:, :k] = X, Y0
    got, kern = run16(A, bx[:, :k], by[:, :k], 1.5, -0.5)
    assert kern == "spmm_items", kern
    assert np.array_equal(bits(got), bits(ref))
    # misaligned: one element past a 16-byte boundary
    bx = np.zeros(X.size + 8, dtype=F16)
    by = np.zeros(Y0.size + 8, dtype=F16)
    off_x = (8 - (bx.ctypes.data % 16) // 2 + 1) % 8 or 8
    off_y = (8 - (by.ctypes.data % 16) // 2 + 1) % 8 or 8
    Xo = bx[off_x:off_x + X.size].reshape(X.shape)
    Yo = by[off_y:off_y + Y0.size].reshape(Y0.shape)
    Xo[...], Yo[...] = X, Y0
    assert (Xo.ctypes.data % 16) and (Yo.ctypes.data % 16)
    p = E.SpmvPlan()
    spmm16(p, "N", len(A[0]) - 1, A[3], *A[:3], Xo, Yo, 1.5, -0.5)
    assert p.kernel() == "spmm_items", p.kernel()
    p.close()
    assert np.array_equal(bits(Yo), bits(ref))


def test_plan_returns_every_allocation(emu):
    live = emu.b200emu_live_allocations
    live.restype, live.argtypes = C.c_longlong, [C.c_void_p]
    A = case16("thresholds")
    base = live(None)
    p = E.SpmvPlan()
    for xo, yo, k, mode in (("C", "C", 16, "N"), ("F", "F", 8, "N"), ("C", "F", 5, "N"), ("C", "C", 8, "T"), ("F", "F", 16, "H")):
        X, Y0 = operands16(A, k, "C", mode)
        X, Y = np.asarray(X, order=xo), np.asarray(Y0, order=yo).copy(order="K")
        spmm16(p, mode, len(A[0]) - 1, A[3], *A[:3], X, Y, 1.0, 0.5)
    assert live(None) > base  # the plan holds items, partial sums and scratch
    p.close()
    assert live(None) == base
    # without a plan the T-mode scratch is a temporary of the call
    X, Y0 = operands16(A, 4, "C", "T")
    spmm16(None, "T", len(A[0]) - 1, A[3], *A[:3], X, Y0.copy(), 1.0, 0.0)
    assert live(None) == base


def test_errors(emu):
    A = case16("small_mod1")
    X, Y0 = operands16(A, 4, "C")
    rp, ci, v, nc = A
    L = E.lib()
    args = lambda mode, ldx: (None, None, mode, len(rp) - 1, nc, len(ci), 4, C.c_float(1.0), E.ptr(rp), E.ptr(ci), E.ptr(v), E.ptr(X), ldx, 1,
                              C.c_float(0.0), E.ptr(Y0), 4, 1)
    assert L.b200sp_spmm_f16_i32(*args(b"Q", 4)) == 1
    assert L.b200sp_spmm_f16_i32(*args(b"N", 3)) == 1  # leading dimension below k
