"""SpGEMM and spgemm_jacobi kernel paths EXECUTED on the CPU (tools/emu) on the cases of spgemm_path_cases.py, with the
checks of tests/test_gpu_spgemm_paths.py: the plan's path witness (b200sp_spgemm_plan_paths) equals the rows each case was
built for, row_map and entries equal the exact structure (and the oracle's), and every value is within the per-entry
rounding bound of the exact product (tests/exact_ref.py).  The emulation affords the whole case list."""
import ctypes as C

import numpy as np
import pytest

import emu_lib as E
import exact_ref as R
import spgemm_path_cases as P

DTYPES = [np.float64, np.float32]


@pytest.fixture(scope="module")
def emu():
    return E.lib()


class Plan:
    def __init__(self, window=None):
        self.h = C.c_void_p()
        E.ok(E.lib().b200sp_spgemm_plan_create(C.byref(self.h)))
        if window is not None:
            E.ok(E.lib().b200sp_spgemm_plan_set_window(self.h, C.c_int64(window)))

    def close(self):
        E.ok(E.lib().b200sp_spgemm_plan_destroy(self.h, None))

    def symbolic(self, case, bits=32):
        A, B, m, n, k = case["A"], case["B"], case["m"], case["n"], case["k"]
        it = np.int32 if bits == 32 else np.int64
        rpC = np.full(m + 1, -7, dtype=it)
        nnz, mx = C.c_int64(), C.c_int()
        fn = E.lib().b200sp_spgemm_symbolic_i32 if bits == 32 else E.lib().b200sp_spgemm_symbolic_i64
        rpA, rpB = A[0].astype(it), B[0].astype(it)  # held until the call returns
        E.ok(fn(self.h, None, m, n, k, E.ptr(rpA), E.ptr(A[1]), E.ptr(rpB), E.ptr(B[1]), E.ptr(rpC), C.byref(nnz), C.byref(mx)))
        self.rpC, self.nnz, self.bits = rpC, nnz.value, bits
        return rpC

    def numeric(self, case, A, B, dtype):
        it = np.int32 if self.bits == 32 else np.int64
        ciC = np.full(self.nnz, -1, dtype=np.int32)
        vC = np.full(self.nnz, np.nan, dtype=dtype)
        fn = getattr(E.lib(), "b200sp_spgemm_numeric_%s_i%d" % (E.sfx(dtype), self.bits))
        rpA, rpB = A[0].astype(it), B[0].astype(it)
        E.ok(fn(self.h, None, case["m"], case["n"], case["k"], E.ptr(rpA), E.ptr(A[1]), E.ptr(A[2]), E.ptr(rpB), E.ptr(B[1]), E.ptr(B[2]),
                E.ptr(self.rpC), E.ptr(ciC), E.ptr(vC)))
        return ciC, vC

    def jacobi(self, case, A, B, dtype, omega, dinv):
        ciC = np.full(self.nnz, -1, dtype=np.int32)
        vC = np.full(self.nnz, np.nan, dtype=dtype)
        fn = getattr(E.lib(), "b200sp_spgemm_jacobi_%s_i32" % E.sfx(dtype))
        E.ok(fn(self.h, None, case["m"], case["n"], case["k"], E.ptr(A[0]), E.ptr(A[1]), E.ptr(A[2]), E.ptr(B[0]), E.ptr(B[1]),
                E.ptr(B[2]), E.ptr(self.rpC), E.ptr(ciC), E.ptr(vC), E.scalar(dtype, omega), E.ptr(dinv)))
        return ciC, vC

    def paths(self):
        return E.spgemm_paths(self.h)


def _case_ids(cases):
    return [c["name"] for c in cases]


SPGEMM = P.spgemm_cases(np.float64)
JACOBI = P.jacobi_cases(np.float64)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", _case_ids(SPGEMM))
def test_spgemm_paths(emu, oracle, name, dtype):
    case = next(c for c in P.spgemm_cases(dtype) if c["name"] == name)
    A, B = case["A"], case["B"]
    rp, ci, v, bound = R.spgemm_ref(A, B)
    if case["oracle"]:
        exp = oracle.spgemm(*A, *B, case["k"])
        assert np.array_equal(exp[0], rp) and np.array_equal(exp[1], ci), f"{name}: exact structure != oracle's"
    P.check_addressing(case, rp, ci)
    p = Plan()
    try:
        rpC = p.symbolic(case)
        assert np.array_equal(rpC, rp), f"{name}: row_map"
        ciC, vC = p.numeric(case, A, B, dtype)
        P.check_paths(p.paths(), case, rp, False, name)
        assert np.array_equal(ciC, ci), f"{name}: entries"
        R.assert_within(vC, v, bound, f"{name} {dtype.__name__}")
        # reuse: a second numeric on the same handle with new values
        A2, B2 = P.new_values(case, dtype, 5)
        rp2, ci2, v2, bound2 = R.spgemm_ref(A2, B2)
        ciC, vC = p.numeric(case, A2, B2, dtype)
        assert np.array_equal(ciC, ci2), f"{name}: entries (reuse)"
        R.assert_within(vC, v2, bound2, f"{name} {dtype.__name__} reuse")
        P.check_paths(p.paths(), case, rp, False, name + " reuse")
    finally:
        p.close()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", _case_ids(JACOBI))
def test_jacobi_paths(emu, oracle, name, dtype):
    case = next(c for c in P.jacobi_cases(dtype) if c["name"] == name)
    A, B = case["A"], case["B"]
    omega, dinv = P.jacobi_operands(case, dtype)
    rp, ci, v, bound = R.jacobi_ref(A, B, omega, dinv)
    if case["oracle"] and not case["no_diag"]:
        exp = oracle.spgemm_jacobi(*A, *B, case["k"], dtype(omega), dinv)
        assert np.array_equal(exp[0], rp) and np.array_equal(exp[1], ci), f"{name}: exact structure != oracle's"
    p = Plan()
    try:
        rpC = p.symbolic(case)
        assert np.array_equal(rpC, rp), f"{name}: row_map"
        ciC, vC = p.jacobi(case, A, B, dtype, omega, dinv)
        P.check_paths(p.paths(), case, rp, True, name)
        assert np.array_equal(ciC, ci), f"{name}: entries"
        R.assert_within(vC, v, bound, f"{name} {dtype.__name__} jacobi")
    finally:
        p.close()


@pytest.mark.parametrize("dtype", DTYPES)
def test_i64_windows(emu, dtype):
    """The _i64 entry points with a window limit that puts rows of different paths in different windows: the same
    structure, values within the bound, and the witness summed over the windows equal to the 32-bit one."""
    for case in P.spgemm_cases(dtype)[:5]:
        A, B = case["A"], case["B"]
        rp, ci, v, bound = R.spgemm_ref(A, B)
        limit = max(int(R.product_rows(A, B).max()), int(np.diff(A[0]).max()), 8)
        p = Plan(limit)
        try:
            rpC = p.symbolic(case, 64)
            assert E.lib().b200sp_spgemm_plan_windows(p.h) > 1, case["name"]
            assert np.array_equal(rpC, rp.astype(np.int64)), case["name"]
            ciC, vC = p.numeric(case, A, B, dtype)
            assert np.array_equal(ciC, ci), case["name"]
            R.assert_within(vC, v, bound, f"{case['name']} {dtype.__name__} i64")
            P.check_paths(p.paths(), case, rp, False, case["name"] + " i64")
        finally:
            p.close()


def test_paths_accessor_before_numeric(emu):
    """Before any numeric call only the symbolic counters are set; counters past the 13th read 0; a null plan is refused."""
    case = P.esc_bounds(np.float64)
    p = Plan()
    try:
        counts = (C.c_int64 * 16)(*([-1] * 16))
        E.ok(E.lib().b200sp_spgemm_plan_paths(p.h, counts, 16))
        assert list(counts) == [0] * 16
        rp = p.symbolic(case)
        got = p.paths()
        exp = P.expected_paths(case, rp, False)
        assert all(got[k] == exp[k] for k in P.PATHS[:6]) and not any(got[k] for k in P.PATHS[6:])
    finally:
        p.close()
    assert E.lib().b200sp_spgemm_plan_paths(C.c_void_p(0), counts, 16) != 0
