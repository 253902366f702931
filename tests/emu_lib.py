"""ctypes view of the EMULATED library (tools/emu: the product's .cu sources compiled by g++ against a
CUDA-on-CPU emulation layer -- fibers for threads, warp/block collectives, mbarrier/TMA, a fake runtime).
"Device" pointers of that build are host pointers, so numpy arrays go straight through the C ABI.

TEST INFRASTRUCTURE: this is how kernel LOGIC (indexing, collectives, barrier protocols, launch
configuration, host-side planning) is exercised without a GPU.  It says nothing about memory-model races or
speed; the `-m gpu` parity tests remain the real gate."""
import ctypes as C
import importlib.util
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "kokkos-kernels_b200"))


def _builder():
    spec = importlib.util.spec_from_file_location("build_emu", os.path.join(ROOT, "tools", "emu", "build_emu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


_LIB = None


def lib():
    """The emulated libb200sparse, built on demand (about 20 s) and bound with the product's signature table."""
    global _LIB
    if _LIB is None:
        b = _builder()
        if not b.up_to_date():
            b.build(verbose=False)
        import _lib as product_binding  # kokkos-kernels_b200/_lib.py: only its SPARSE_API table is used

        so = C.CDLL(os.path.join(b.OUT, "libb200sparse_emu.so"))
        for name, (res, args) in product_binding.SPARSE_API.items():
            fn = getattr(so, name)
            fn.restype, fn.argtypes = res, args
        _LIB = so
    return _LIB


def harness():
    b = _builder()
    if not b.up_to_date():
        b.build(verbose=False)
    return os.path.join(b.OUT, "gpu_check_emu")


def ptr(a):
    return C.c_void_p(a.ctypes.data) if a is not None else C.c_void_p(0)


def ok(rc):
    if rc != 0:
        raise RuntimeError("b200sp status %d: %s" % (rc, lib().b200sp_last_error_string().decode()))


def sfx(dtype):
    return "f64" if np.dtype(dtype) == np.float64 else "f32"


def scalar(dtype, x):
    return C.c_double(x) if np.dtype(dtype) == np.float64 else C.c_float(x)


class SpmvPlan:
    def __init__(self, algo=0):
        self.h = C.c_void_p()
        ok(lib().b200sp_spmv_plan_create(C.byref(self.h), algo))

    def close(self):
        if self.h:
            ok(lib().b200sp_spmv_plan_destroy(self.h, None))
            self.h = C.c_void_p()

    def kernel(self):
        return lib().b200sp_spmv_last_kernel(self.h).decode()


def spmv(plan, mode, nrows, ncols, rp, ci, v, x, y, alpha, beta):
    fn = getattr(lib(), "b200sp_spmv_%s_i32" % sfx(v.dtype))
    ok(fn(plan.h, None, mode.encode(), nrows, ncols, len(ci), scalar(v.dtype, alpha), ptr(rp), ptr(ci), ptr(v), ptr(x),
          scalar(v.dtype, beta), ptr(y)))


class Spmv64Plan:
    def __init__(self, algo=0, window=None):
        self.h = C.c_void_p()
        ok(lib().b200sp_spmv64_plan_create(C.byref(self.h), algo))
        if window is not None:
            ok(lib().b200sp_spmv64_plan_set_window(self.h, C.c_int64(window)))

    def close(self):
        if self.h:
            ok(lib().b200sp_spmv64_plan_destroy(self.h, None))
            self.h = C.c_void_p()

    def windows(self):
        return lib().b200sp_spmv64_plan_windows(self.h)

    def kernel(self):
        return lib().b200sp_spmv64_last_kernel(self.h).decode()


def spmv64_rc(plan, mode, nrows, ncols, rp64, ci, v, x, y, alpha, beta):
    """64-bit offsets (rp64: int64), 32- or 64-bit columns by ci.dtype; returns the status code."""
    assert rp64.dtype == np.int64 and ci.dtype in (np.int32, np.int64)
    fn = getattr(lib(), "b200sp_spmv_%s_i64" % sfx(v.dtype))
    return fn(plan.h, None, mode.encode(), C.c_int64(nrows), C.c_int64(ncols), C.c_int64(len(ci)), scalar(v.dtype, alpha), ptr(rp64),
              ptr(ci), 8 * ci.dtype.itemsize, ptr(v), ptr(x), scalar(v.dtype, beta), ptr(y))


def spmv64(plan, *a):
    ok(spmv64_rc(plan, *a))


def spmm64(plan, mode, nrows, ncols, rp64, ci, v, X, Y, alpha, beta):
    fn = getattr(lib(), "b200sp_spmm_%s_i64" % sfx(v.dtype))
    it = v.dtype.itemsize

    def lay(a):
        if a.strides[1] == it:
            return a.strides[0] // it, 1
        assert a.strides[0] == it
        return a.strides[1] // it, 0

    ldx, rmx = lay(X)
    ldy, rmy = lay(Y)
    ok(fn(plan.h, None, mode.encode(), C.c_int64(nrows), C.c_int64(ncols), C.c_int64(len(ci)), X.shape[1], scalar(v.dtype, alpha),
          ptr(rp64), ptr(ci), 8 * ci.dtype.itemsize, ptr(v), ptr(X), C.c_int64(ldx), rmx, scalar(v.dtype, beta), ptr(Y), C.c_int64(ldy), rmy))


def spmm(plan, mode, nrows, ncols, rp, ci, v, X, Y, alpha, beta):
    """X, Y: 2-D numpy arrays, either C- or F-ordered (LayoutRight / LayoutLeft); strides are passed in elements."""
    fn = getattr(lib(), "b200sp_spmm_%s_i32" % sfx(v.dtype))
    it = v.dtype.itemsize

    def lay(a):
        if a.strides[1] == it:  # row-major: leading dimension = row stride
            return a.strides[0] // it, 1
        assert a.strides[0] == it
        return a.strides[1] // it, 0

    ldx, rmx = lay(X)
    ldy, rmy = lay(Y)
    ok(fn(plan.h, None, mode.encode(), nrows, ncols, len(ci), X.shape[1], scalar(v.dtype, alpha), ptr(rp), ptr(ci), ptr(v), ptr(X),
          ldx, rmx, scalar(v.dtype, beta), ptr(Y), ldy, rmy))


def spgemm(A, B, m, n, k, dtype):
    """symbolic + numeric; returns (rowmapC, entriesC, valuesC)."""
    L = lib()
    h = C.c_void_p()
    ok(L.b200sp_spgemm_plan_create(C.byref(h)))
    try:
        rpC = np.full(m + 1, 123, dtype=np.int32)
        nnz, mx = C.c_int64(), C.c_int()
        ok(L.b200sp_spgemm_symbolic_i32(h, None, m, n, k, ptr(A[0]), ptr(A[1]), ptr(B[0]), ptr(B[1]), ptr(rpC), C.byref(nnz), C.byref(mx)))
        ciC = np.full(nnz.value, -1, dtype=np.int32)
        vC = np.full(nnz.value, np.nan, dtype=dtype)
        fn = getattr(L, "b200sp_spgemm_numeric_%s_i32" % sfx(dtype))
        ok(fn(h, None, m, n, k, ptr(A[0]), ptr(A[1]), ptr(A[2]), ptr(B[0]), ptr(B[1]), ptr(B[2]), ptr(rpC), ptr(ciC), ptr(vC)))
        return rpC, ciC, vC, mx.value
    finally:
        ok(L.b200sp_spgemm_plan_destroy(h, None))


PATHS = ("esc0", "esc1", "esc2", "esc3", "sym_hash", "sym_bitmap", "hash0", "hash1", "hash2", "hash3", "hash4", "fallback",
         "overflow")


def spgemm_paths(h):
    """b200sp_spgemm_plan_paths of a plan handle (c_void_p) as a dict keyed by PATHS (kokkos_kernels_b200.sparse's
    SPGEMMHandle.PATHS)."""
    counts = (C.c_int64 * len(PATHS))()
    ok(lib().b200sp_spgemm_plan_paths(h, counts, len(PATHS)))
    return dict(zip(PATHS, counts))


class BsrPlan:
    def __init__(self):
        self.h = C.c_void_p()
        ok(lib().b200sp_bsr_plan_create(C.byref(self.h)))

    def close(self):
        if self.h:
            ok(lib().b200sp_bsr_plan_destroy(self.h, None))
            self.h = C.c_void_p()

    def kernel(self):
        return lib().b200sp_bsr_last_kernel(self.h).decode()


def bsr_spmv(plan, mode, mb, nb, bs, rp, ci, v, x, y, alpha, beta):
    fn = getattr(lib(), "b200sp_bsr_spmv_%s_i32" % sfx(v.dtype))
    ok(fn(plan.h, None, mode.encode(), mb, nb, len(ci), bs, scalar(v.dtype, alpha), ptr(rp), ptr(ci), ptr(v), ptr(x), scalar(v.dtype, beta),
          ptr(y)))


def bsr_spmm(plan, mode, mb, nb, bs, rp, ci, v, X, Y, alpha, beta):
    fn = getattr(lib(), "b200sp_bsr_spmm_%s_i32" % sfx(v.dtype))
    it = v.dtype.itemsize

    def lay(a):
        if a.shape[1] == 1 or a.strides[0] == it:  # column-major (LayoutLeft)
            return max(a.strides[1] // it, a.shape[0]), 0
        return a.strides[0] // it, 1

    ldx, rmx = lay(X)
    ldy, rmy = lay(Y)
    ok(fn(plan.h, None, mode.encode(), mb, nb, len(ci), bs, X.shape[1], scalar(v.dtype, alpha), ptr(rp), ptr(ci), ptr(v), ptr(X), ldx, rmx,
          scalar(v.dtype, beta), ptr(Y), ldy, rmy))


# ---- guarded inputs: numpy views over blocks that end right before an inaccessible page (tools/emu/emu_runtime.cpp) ----
_GUARDED = []


def guarded(a, align=None):
    """Copy `a` (1-D or contiguous 2-D) into a guarded block and return an ndarray view of it.  align = element size
    (default): the byte after the array faults, the start is aligned to the element only (the library's unaligned
    paths); align = 16: the start is 16-byte aligned (TMA paths) and up to 15 bytes of slack precede the guard page."""
    L = lib()
    L.b200emu_guarded_alloc.restype = C.c_void_p
    L.b200emu_guarded_alloc.argtypes = [C.c_size_t, C.c_size_t]
    a = np.ascontiguousarray(a) if not a.flags.f_contiguous or a.ndim == 1 else a
    al = a.dtype.itemsize if align is None else align
    p = L.b200emu_guarded_alloc(a.nbytes, al)
    assert p, "guarded allocation failed"
    _GUARDED.append(p)
    buf = (C.c_char * max(a.nbytes, 1)).from_address(p)
    v = np.frombuffer(buf, dtype=a.dtype, count=a.size).reshape(a.shape, order="F" if (a.ndim == 2 and a.flags.f_contiguous and not a.flags.c_contiguous) else "C")
    v[...] = a
    return v


def guarded_release():
    L = lib()
    L.b200emu_guarded_free.argtypes = [C.c_void_p]
    while _GUARDED:
        L.b200emu_guarded_free(_GUARDED.pop())


def cg_solve(plan, rp, ci, v, b, x, maximum_iteration, tolerance, check_every=0):
    it, nr = C.c_int(), C.c_double()
    ok(lib().b200sp_cg_solve_f64_i32(plan.h, None, len(rp) - 1, len(ci), ptr(rp), ptr(ci), ptr(v), ptr(b), ptr(x), maximum_iteration,
                                     C.c_double(tolerance), check_every, C.byref(it), C.byref(nr)))
    return it.value, nr.value


def gmres(plan_a, A, b, x, m=50, tol=1e-8, max_restart=50, ortho=0, prec=None, plan_m=None):
    """b200sp_gmres_*: returns (status, num_iters, end_rel_res, conv_flag); x updated in place."""
    rp, ci, v = A
    f64 = v.dtype == np.float64
    fn = lib().b200sp_gmres_f64_i32 if f64 else lib().b200sp_gmres_f32_i32
    it, flag = C.c_int(), C.c_int()
    res = C.c_double() if f64 else C.c_float()
    pr = prec if prec is not None else (None, None, None)
    rc = fn(plan_a.h, None, len(rp) - 1, len(ci), ptr(rp), ptr(ci), ptr(v), plan_m.h if plan_m else None, len(pr[1]) if prec is not None else 0,
            ptr(pr[0]), ptr(pr[1]), ptr(pr[2]), ptr(b), ptr(x), m, scalar(v.dtype, tol), max_restart, ortho, C.byref(it), C.byref(res),
            C.byref(flag))
    return rc, it.value, res.value, flag.value


def gmres_bsr(plan_a, bs, A, b, x, m=50, tol=1e-8, max_restart=50, ortho=0, prec=None, plan_m=None):
    """b200sp_gmres_bsr_*: A (and prec) = (block row map, block columns, values); plans are BsrPlan."""
    rp, ci, v = A
    f64 = v.dtype == np.float64
    fn = lib().b200sp_gmres_bsr_f64_i32 if f64 else lib().b200sp_gmres_bsr_f32_i32
    it, flag = C.c_int(), C.c_int()
    res = C.c_double() if f64 else C.c_float()
    pr = prec if prec is not None else (None, None, None)
    rc = fn(plan_a.h, None, len(rp) - 1, len(ci), bs, ptr(rp), ptr(ci), ptr(v), plan_m.h if plan_m else None, len(pr[1]) if prec is not None else 0,
            ptr(pr[0]), ptr(pr[1]), ptr(pr[2]), ptr(b), ptr(x), m, scalar(v.dtype, tol), max_restart, ortho, C.byref(it), C.byref(res),
            C.byref(flag))
    return rc, it.value, res.value, flag.value


class GsPlan:
    def __init__(self):
        self.h = C.c_void_p()
        ok(lib().b200sp_gs_plan_create(C.byref(self.h)))

    def close(self):
        if self.h:
            ok(lib().b200sp_gs_plan_destroy(self.h, None))
            self.h = C.c_void_p()

    def symbolic(self, n, rp, ci, symmetric, ncols=None):
        if ncols is None:
            ok(lib().b200sp_gs_symbolic_i32(self.h, None, n, ptr(rp), ptr(ci), int(symmetric)))
        else:
            ok(lib().b200sp_gs_symbolic_nc_i32(self.h, None, n, ncols, ptr(rp), ptr(ci), int(symmetric)))

    def numeric(self, n, rp, ci, v):
        return getattr(lib(), "b200sp_gs_numeric_%s_i32" % sfx(v.dtype))(self.h, None, n, ptr(rp), ptr(ci), ptr(v))

    def apply(self, n, rp, ci, v, x, y, init_zero_x, omega, sweeps, direction):
        return getattr(lib(), "b200sp_gs_apply_%s_i32" % sfx(v.dtype))(self.h, None, n, ptr(rp), ptr(ci), ptr(v), ptr(x), ptr(y), int(init_zero_x),
                                                                       scalar(v.dtype, omega), sweeps, direction)

    def coloring(self, n):
        """(num_colors, colors[n], color_ptr[nc+1], color_rows[n]) copied out of the plan ("device" memory is host memory here)."""
        nc = C.c_int()
        pc, pp, pr = C.c_void_p(), C.c_void_p(), C.c_void_p()
        ok(lib().b200sp_gs_get_coloring(self.h, C.byref(nc), C.byref(pc), C.byref(pp), C.byref(pr)))
        arr = lambda p, cnt: np.ctypeslib.as_array((C.c_int * cnt).from_address(p.value)).copy() if cnt else np.zeros(0, np.int32)
        return nc.value, arr(pc, n), arr(pp, nc.value + 1), arr(pr, n)

    def kernel(self):
        return lib().b200sp_gs_last_kernel(self.h).decode()


def pcg_solve(plan, gs_plan, rp, ci, v, b, x, maximum_iteration, tolerance, check_every=0):
    it, nr = C.c_int(), C.c_double()
    ok(lib().b200sp_pcg_solve_f64_i32(plan.h, gs_plan.h, None, len(rp) - 1, len(ci), ptr(rp), ptr(ci), ptr(v), ptr(b), ptr(x), maximum_iteration,
                                      C.c_double(tolerance), check_every, C.byref(it), C.byref(nr)))
    return it.value, nr.value


def pcg_solve_gs2(plan, gs2_plan, rp, ci, v, b, x, maximum_iteration, tolerance, check_every=0):
    it, nr = C.c_int(), C.c_double()
    ok(lib().b200sp_pcg_solve_gs2_f64_i32(plan.h, gs2_plan.h, None, len(rp) - 1, len(ci), ptr(rp), ptr(ci), ptr(v), ptr(b), ptr(x), maximum_iteration,
                                          C.c_double(tolerance), check_every, C.byref(it), C.byref(nr)))
    return it.value, nr.value


class Gs2Plan:
    """b200sp_gs2_*: two-stage Gauss-Seidel (inner Jacobi-Richardson sweeps)."""

    def __init__(self, compact=False, inner=1, outer=1, gamma=1.0):
        self.h = C.c_void_p()
        ok(lib().b200sp_gs2_plan_create(C.byref(self.h)))
        for opt, val in ((1, float(compact)), (2, float(inner)), (3, float(outer)), (4, float(gamma))):
            ok(lib().b200sp_gs2_plan_set(self.h, opt, C.c_double(val)))

    def close(self):
        if self.h:
            ok(lib().b200sp_gs2_plan_destroy(self.h, None))
            self.h = C.c_void_p()

    def set(self, option, value):
        return lib().b200sp_gs2_plan_set(self.h, option, C.c_double(value))

    def symbolic(self, n, ncols, rp, ci):
        return lib().b200sp_gs2_symbolic_i32(self.h, None, n, ncols, ptr(rp), ptr(ci))

    def numeric(self, n, ncols, rp, ci, v, dinv=None):
        return getattr(lib(), "b200sp_gs2_numeric_%s_i32" % sfx(v.dtype))(self.h, None, n, ncols, ptr(rp), ptr(ci), ptr(v), ptr(dinv))

    def apply(self, n, ncols, rp, ci, v, x, b, init_zero_x, omega, num_iter, direction):
        """x: (ncols,) or (ncols, nrhs) F-ordered; b likewise with n rows."""
        nrhs = 1 if x.ndim == 1 else x.shape[1]
        ldx = ncols if x.ndim == 1 else x.strides[1] // x.itemsize
        ldb = n if b.ndim == 1 else b.strides[1] // b.itemsize
        return getattr(lib(), "b200sp_gs2_apply_%s_i32" % sfx(v.dtype))(self.h, None, n, ncols, ptr(rp), ptr(ci), ptr(v), ptr(x), C.c_int64(ldx), ptr(b),
                                                                       C.c_int64(ldb), nrhs, int(init_zero_x), scalar(v.dtype, omega), num_iter, direction)
