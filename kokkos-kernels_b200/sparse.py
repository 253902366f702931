"""Host-side mirror of the reference's public sparse API for the hot path
(names, argument meaning and error behaviour follow the reference; storage is
torch CUDA tensors, compute is libb200sparse through the C ABI):

  CrsMatrix                      sparse/src/KokkosSparse_CrsMatrix.hpp:317-388
  SPMVAlgorithm / SPMVHandle     sparse/src/KokkosSparse_spmv_handle.hpp:32-47,217-349
  spmv(handle, mode, alpha, A, x, beta, y)
                                 sparse/src/KokkosSparse_spmv.hpp:77-375,440-474
  SPGEMMAlgorithm / KokkosKernelsHandle / SPGEMMHandle
                                 sparse/src/KokkosSparse_spgemm_handle.hpp:44-87,94-747
  spgemm_symbolic / spgemm_numeric / spgemm
                                 sparse/src/KokkosSparse_spgemm.hpp:40-61,119-129,170-218
  sort_crs_matrix / sort_crs_graph / sort_and_merge_matrix / sort_and_merge_graph
                                 sparse/src/KokkosSparse_SortCrs.hpp:43-146,209-300,303-537
  SPADDHandle / spadd_symbolic / spadd_numeric
                                 sparse/src/KokkosSparse_spadd_handle.hpp:24-137, KokkosSparse_spadd.hpp:29-319
  transpose_matrix               sparse/src/KokkosSparse_Utils.hpp:338-398
  BsrMatrix (spmv accepts it)    sparse/src/KokkosSparse_BsrMatrix.hpp:317-520, KokkosSparse_spmv.hpp:113,169-185,322-375

PyTorch is plumbing here (device memory + streams); there is no torch compute
on this path and no CPU fallback.
"""
import ctypes as C

import torch

from . import _lib
from ._lib import B200SparseError, B200SparseInvalidArgument, check

# SPMVAlgorithm (spmv_handle.hpp:32-47)
SPMV_DEFAULT, SPMV_FAST_SETUP, SPMV_NATIVE, SPMV_MERGE_PATH, SPMV_NATIVE_MERGE_PATH, SPMV_BSR_V41, SPMV_BSR_V42, SPMV_BSR_TC = range(8)
# GSAlgorithm (sparse/src/KokkosSparse_gauss_seidel_handle.hpp:29): the point (multicolour) algorithm serves GS_DEFAULT / PERMUTED / TEAM,
# GS_TWOSTAGE is the SpMV-based two-stage method; GS_CLUSTER is not provided
GS_DEFAULT, GS_PERMUTED, GS_TEAM, GS_CLUSTER, GS_TWOSTAGE = range(5)
# SPGEMMAlgorithm subset that matters here (spgemm_handle.hpp:44-87)
SPGEMM_KK, SPGEMM_KK_MEMORY, SPGEMM_KK_SPEED, SPGEMM_KK_LP, SPGEMM_DEBUG, SPGEMM_SERIAL = range(6)

# the BsrMatrix-only algorithm requests (V41 / V42 / tensor cores) name reference-native kernels; here they select the one
# BsrMatrix path (DESIGN.md section 7c) and, on a CrsMatrix, the default
_ALGO_TO_C = {SPMV_DEFAULT: 0, SPMV_FAST_SETUP: 1, SPMV_NATIVE: 1, SPMV_MERGE_PATH: 2, SPMV_NATIVE_MERGE_PATH: 2, SPMV_BSR_V41: 0,
              SPMV_BSR_V42: 0, SPMV_BSR_TC: 0}


def _idx(t):
    """Device pointer of a 32-bit index array: every entry point but spmv's and spgemm's 64-bit ones reads int32 ordinals and
    offsets."""
    if t is not None and t.dtype != torch.int32:
        raise B200SparseError(f"b200sparse: this operation takes int32 row maps / entries, got {t.dtype} "
                              "(only spmv and spgemm accept 64-bit offsets)")
    return _ptr(t)


def _spgemm_wide(row_maps, entries):
    """True when a point SpGEMM runs on 64-bit offsets (spgemm64.cu): the row maps of A, B and C share one dtype, int32 or
    int64, and the entries are int32 (the (int, size_t) instantiation; 64-bit ordinals are not provided)."""
    dts = {t.dtype for t in row_maps if t is not None}
    if len(dts) > 1:
        raise B200SparseError(f"KokkosSparse::spgemm: the row maps of A, B and C must share one dtype, got {sorted(map(str, dts))}")
    if dts - {torch.int32, torch.int64}:
        raise B200SparseError(f"KokkosSparse::spgemm: row maps must be int32 or int64, got {dts.pop()}")
    for t in entries:
        if t is not None and t.dtype != torch.int32:
            raise B200SparseError(f"KokkosSparse::spgemm: 64-bit ordinals are not provided (entries must be int32, got {t.dtype})")
    return dts == {torch.int64}


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None and t.numel() > 0 else C.c_void_p(0)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class CrsMatrix:
    """graph.row_map / graph.entries / values / numCols (0-based CSR; rows need
    not be sorted, duplicates are legal for spmv).  Ordinal / offset types: (int32, int32) everywhere; spmv also takes 64-bit
    offsets -- row_map int64 with int32 or int64 entries, the (int64_t, size_t) instantiation of the reference's cuSPARSE slot
    (sparse/tpls/KokkosSparse_spmv_tpl_spec_decl.hpp:246-257) -- for matrices past 2^31 entries, and spgemm takes row_map
    int64 with int32 entries, Kokkos' (int, size_t), for products past 2^31 entries."""

    def __init__(self, row_map, entries, values, ncols):
        assert (row_map.dtype == torch.int32 and entries.dtype == torch.int32) or (
            row_map.dtype == torch.int64 and entries.dtype in (torch.int32, torch.int64))
        self.row_map, self.entries, self.values = row_map, entries, values
        self._ncols = int(ncols)

    def numRows(self):
        return max(self.row_map.numel() - 1, 0)

    def numCols(self):
        return self._ncols

    def nnz(self):
        return self.entries.numel()


class BsrMatrix:
    """KokkosSparse::Experimental::BsrMatrix: graph.row_map / graph.entries over BLOCKS, values =
    nnzb*blockDim*blockDim with every block row-major (BsrMatrix.hpp:355-370); numRows()/numCols() count
    block rows / block columns, numPointRows()/numPointCols() the point dimensions (:880-900)."""

    def __init__(self, row_map, entries, values, ncols_blocks, block_dim):
        assert row_map.dtype == torch.int32 and entries.dtype == torch.int32
        if int(block_dim) < 1:  # BsrMatrix.hpp:429-433
            raise B200SparseError(f"KokkosSparse::Experimental::BsrMatrix: Inappropriate block size: {block_dim}")
        if values.numel() != entries.numel() * int(block_dim) ** 2:
            raise B200SparseError("BsrMatrix: values must hold nnz*blockDim*blockDim entries")
        self.row_map, self.entries, self.values = row_map, entries, values
        self._ncols = int(ncols_blocks)
        self._bs = int(block_dim)

    def blockDim(self):
        return self._bs

    def numRows(self):
        return max(self.row_map.numel() - 1, 0)

    def numCols(self):
        return self._ncols

    def numPointRows(self):
        return self.numRows() * self._bs

    def numPointCols(self):
        return self._ncols * self._bs

    def nnz(self):
        return self.entries.numel()


class SPMVHandle:
    """Owns the per-matrix plan like SPMVHandle owns tpl_rank1/tpl_rank2; all
    calls through one handle must use the same matrix (spmv_handle.hpp:276-277)."""

    def __init__(self, algo=SPMV_DEFAULT):
        if algo not in _ALGO_TO_C:
            raise B200SparseInvalidArgument(f"unknown SPMVAlgorithm {algo}")
        self.algo = algo
        self._plan = C.c_void_p(0)
        self._bsr_plan = C.c_void_p(0)  # created by the first BsrMatrix call (the handle then only ever sees that matrix)
        self._plan64 = C.c_void_p(0)    # created by the first call with 64-bit offsets
        check(_lib.sparse().b200sp_spmv_plan_create(C.byref(self._plan), _ALGO_TO_C[algo]))

    def _p64(self):
        if not self._plan64:
            check(_lib.sparse().b200sp_spmv64_plan_create(C.byref(self._plan64), _ALGO_TO_C[self.algo]))
        return self._plan64

    def set_window(self, max_entries):
        """64-bit offsets only: entries per 32-bit window (default 2^31 - 65537; smaller values are for tests)."""
        check(_lib.sparse().b200sp_spmv64_plan_set_window(self._p64(), int(max_entries)))

    def windows(self):
        return _lib.sparse().b200sp_spmv64_plan_windows(self._plan64) if self._plan64 else 0

    def _bsr(self):
        if not self._bsr_plan:
            check(_lib.sparse().b200sp_bsr_plan_create(C.byref(self._bsr_plan)))
            # spmv_bsrmatrix_spec.hpp:176-177: SPMV_BSR_TC asks for tensor cores, V41 / V42 for the scalar functors; the
            # library's default uses tensor cores where they are faster
            a = {SPMV_BSR_TC: 1, SPMV_BSR_V41: 2, SPMV_BSR_V42: 2}.get(self.algo, 0)
            if a:
                check(_lib.sparse().b200sp_bsr_plan_set_algorithm(self._bsr_plan, a))
        return self._bsr_plan

    def get_algorithm(self):
        return self.algo

    def cache_transpose(self, enable=True):
        """Modes T / H through an explicit transpose kept in the plan (deterministic, no atomics)."""
        check(_lib.sparse().b200sp_spmv_plan_set_option(self._plan, 1, int(bool(enable))))

    def hostvec_defer(self, enable=True):
        """spmv_hostvec calls stop making the stream wait for their own download of y: consecutive calls overlap upload, kernel and
        download; y_host is valid after hostvec_flush() + a stream synchronisation (B200SP_SPMV_OPT_HOSTVEC_DEFER)."""
        check(_lib.sparse().b200sp_spmv_plan_set_option(self._plan, 2, int(bool(enable))))

    def hostvec_flush(self):
        check(_lib.sparse().b200sp_spmv_hostvec_flush(self._plan, _stream()))

    def tune(self, cfg=-1, lanes_per_row=-1, ctas_per_sm=-1):
        check(_lib.sparse().b200sp_spmv_plan_tune(self._plan, cfg, lanes_per_row, ctas_per_sm))

    def invalidate(self):
        """Drop the cached analysis of the matrix this handle last saw (b200sp_spmv_plan_invalidate).  The cache is keyed on
        (row_map pointer, shape, nnz); call this when a DIFFERENT matrix may sit at the same address with the same shape
        (an in-place edit of row_map, or a caching allocator reusing the block) -- the reference's contract is one matrix
        per handle (sparse/src/KokkosSparse_spmv_handle.hpp:276-277)."""
        if self._plan:
            check(_lib.sparse().b200sp_spmv_plan_invalidate(self._plan, _stream()))

    def last_kernel(self):
        if self._bsr_plan:
            return _lib.sparse().b200sp_bsr_last_kernel(self._bsr_plan).decode()
        if self._plan64:
            return _lib.sparse().b200sp_spmv64_last_kernel(self._plan64).decode()
        return _lib.sparse().b200sp_spmv_last_kernel(self._plan).decode()

    def __del__(self):
        try:
            st = _stream() if torch.cuda.is_available() else C.c_void_p(0)
            if self._bsr_plan:
                _lib.sparse().b200sp_bsr_plan_destroy(self._bsr_plan, st)
                self._bsr_plan = C.c_void_p(0)
            if self._plan64:
                _lib.sparse().b200sp_spmv64_plan_destroy(self._plan64, st)
                self._plan64 = C.c_void_p(0)
            if self._plan:
                _lib.sparse().b200sp_spmv_plan_destroy(self._plan, st)
                self._plan = C.c_void_p(0)
        except Exception:
            pass


def _mode_char(mode):
    if not isinstance(mode, str) or len(mode) < 1:
        raise B200SparseError(f"Invalid transpose mode {mode!r} for KokkosSparse::spmv()")
    return mode[0]


def spmv(handle, mode, alpha, A, x, beta, y):
    """y = beta*y + alpha*Op(A)*x, rank-1 or rank-2 (x.dim()); handle may be None
    (the convenience overload builds a throw-away SPMV_FAST_SETUP handle,
    KokkosSparse_spmv.hpp:465-474)."""
    m0 = _mode_char(mode)
    is_bsr = isinstance(A, BsrMatrix)
    m, n = (A.numPointRows(), A.numPointCols()) if is_bsr else (A.numRows(), A.numCols())
    if x.dim() != y.dim() or x.dim() not in (1, 2):
        raise B200SparseError("KokkosSparse::spmv: x and y must both be rank 1 or both rank 2")
    xcols = x.shape[1] if x.dim() == 2 else 1
    ycols = y.shape[1] if y.dim() == 2 else 1
    if m0 in "NnCc":
        bad = xcols != ycols or n != x.shape[0] or m != y.shape[0]
    elif m0 in "TtHh":
        bad = xcols != ycols or m != x.shape[0] or n != y.shape[0]
    else:
        raise B200SparseError(f"Invalid transpose mode {mode} for KokkosSparse::spmv()")
    if bad:  # KokkosSparse_spmv.hpp:126-142
        raise B200SparseError(
            f"KokkosSparse::spmv: Dimensions do not match: , A: {m} x {n}, x: {x.shape[0]} x {xcols}, "
            f"y: {y.shape[0]} x {ycols}"
        )
    if torch.float16 in (A.values.dtype, x.dtype, y.dtype):
        return _spmm_f16(handle, m0, alpha, A, x, beta, y, m, n, xcols)
    if A.values.dtype != x.dtype or x.dtype != y.dtype:
        raise B200SparseError("b200sparse: A.values, x and y must share one scalar type (f64 or f32)")
    lib = _lib.sparse()
    plan = handle._plan if handle is not None else C.c_void_p(0)
    f64 = x.dtype == torch.float64
    if not f64 and x.dtype != torch.float32:
        raise B200SparseError("b200sparse: only double and float are instantiated")
    mc = m0.encode()
    if is_bsr:
        tmp = handle if handle is not None else SPMVHandle(SPMV_FAST_SETUP)
        return _spmv_bsr(lib, tmp._bsr(), mc, alpha, A, x, beta, y, f64, xcols)
    wide = A.row_map.dtype == torch.int64  # 64-bit offsets: the plan's 32-bit windows (spmv64.cu)
    if wide:
        owner = handle if handle is not None else SPMVHandle(SPMV_FAST_SETUP)  # kept alive until the call returns
        plan = owner._p64()
        bits = 64 if A.entries.dtype == torch.int64 else 32
    if x.dim() == 1:
        if x.stride(0) != 1 or y.stride(0) != 1:
            raise B200SparseError("b200sparse: rank-1 x and y must be contiguous")
        if wide:
            fn = lib.b200sp_spmv_f64_i64 if f64 else lib.b200sp_spmv_f32_i64
            check(fn(plan, _stream(), mc, m, n, A.nnz(), alpha, _ptr(A.row_map), _ptr(A.entries), bits, _ptr(A.values),
                     _ptr(x), beta, _ptr(y)))
            return y
        fn = lib.b200sp_spmv_f64_i32 if f64 else lib.b200sp_spmv_f32_i32
        check(fn(plan, _stream(), mc, m, n, A.nnz(), alpha, _idx(A.row_map), _idx(A.entries), _ptr(A.values),
                 _ptr(x), beta, _ptr(y)))
        return y

    def layout(t):
        # LayoutRight: (ld,1); LayoutLeft: (1,ld)
        if t.shape[1] == 1 or t.stride(1) == 1:
            return max(t.stride(0), 1) if t.shape[0] > 1 else max(t.shape[1], 1), 1
        if t.stride(0) == 1:
            return t.stride(1), 0
        raise B200SparseError("b200sparse: X/Y must be LayoutLeft or LayoutRight")

    ldx, xrm = layout(x)
    ldy, yrm = layout(y)
    if wide:
        fn = lib.b200sp_spmm_f64_i64 if f64 else lib.b200sp_spmm_f32_i64
        check(fn(plan, _stream(), mc, m, n, A.nnz(), xcols, alpha, _ptr(A.row_map), _ptr(A.entries), bits, _ptr(A.values),
                 _ptr(x), ldx, xrm, beta, _ptr(y), ldy, yrm))
        return y
    fn = lib.b200sp_spmm_f64_i32 if f64 else lib.b200sp_spmm_f32_i32
    check(fn(plan, _stream(), mc, m, n, A.nnz(), xcols, alpha, _idx(A.row_map), _idx(A.entries), _ptr(A.values),
             _ptr(x), ldx, xrm, beta, _ptr(y), ldy, yrm))
    return y


def _half_coefficient(c):
    """A coefficient as the half_t it is in Kokkos (coefficient_type of a half_t multivector): rounded to binary16, to
    nearest even; beyond +-65504 it is +-inf."""
    import numpy as np

    with np.errstate(over="ignore"):
        return float(np.float16(c))


def _spmm_f16(handle, m0, alpha, A, x, beta, y, m, n, xcols):
    """Rank-2 SpMV on float16 A, X and Y with fp32 products, sums and epilogue (b200sp_spmm_f16_i32; the reference's half_t
    SPMV_MV slot, sparse/tpls/KokkosSparse_spmv_mv_tpl_spec_avail.hpp:93-104)."""
    if not (A.values.dtype == x.dtype == y.dtype == torch.float16):
        raise B200SparseError(f"b200sparse: half precision needs A.values, x and y all float16, got {A.values.dtype}, {x.dtype}, "
                              f"{y.dtype} (mixed precision is not provided)")
    if isinstance(A, BsrMatrix):
        raise B200SparseError("b200sparse: half precision is provided for CrsMatrix only, not BsrMatrix")
    if x.dim() != 2:
        raise B200SparseError("b200sparse: half precision is provided for rank-2 x and y only, not rank 1")
    if A.row_map.dtype != torch.int32 or A.entries.dtype != torch.int32:
        raise B200SparseError("b200sparse: half precision takes int32 row maps and entries, not 64-bit offsets")
    ldx, xrm = _mv_layout(x)
    ldy, yrm = _mv_layout(y)
    plan = handle._plan if handle is not None else C.c_void_p(0)
    check(_lib.sparse().b200sp_spmm_f16_i32(plan, _stream(), m0.encode(), m, n, A.nnz(), xcols, _half_coefficient(alpha),
                                            _idx(A.row_map), _idx(A.entries), _ptr(A.values), _ptr(x), ldx, xrm,
                                            _half_coefficient(beta), _ptr(y), ldy, yrm))
    return y


def _mv_layout(t):
    # LayoutRight: (ld, 1); LayoutLeft: (ld, 0)
    if t.shape[1] == 1 or t.stride(1) == 1:
        return (max(t.stride(0), 1) if t.shape[0] > 1 else max(t.shape[1], 1)), 1
    if t.stride(0) == 1:
        return t.stride(1), 0
    raise B200SparseError("b200sparse: X/Y must be LayoutLeft or LayoutRight")


def _spmv_bsr(lib, plan, mc, alpha, A, x, beta, y, f64, xcols):
    """SPMV_BSRMATRIX / SPMV_MV_BSRMATRIX (sparse/impl/KokkosSparse_spmv_bsrmatrix_spec.hpp:165-283) on the
    b200sp_bsr_* entries; every mode and blockDim() == 1 are accepted."""
    mb, nb, bs = A.numRows(), A.numCols(), A.blockDim()
    if x.dim() == 1:
        if x.stride(0) != 1 or y.stride(0) != 1:
            raise B200SparseError("b200sparse: rank-1 x and y must be contiguous")
        fn = lib.b200sp_bsr_spmv_f64_i32 if f64 else lib.b200sp_bsr_spmv_f32_i32
        check(fn(plan, _stream(), mc, mb, nb, A.nnz(), bs, alpha, _idx(A.row_map), _idx(A.entries), _ptr(A.values), _ptr(x), beta,
                 _ptr(y)))
        return y
    ldx, xrm = _mv_layout(x)
    ldy, yrm = _mv_layout(y)
    fn = lib.b200sp_bsr_spmm_f64_i32 if f64 else lib.b200sp_bsr_spmm_f32_i32
    check(fn(plan, _stream(), mc, mb, nb, A.nnz(), bs, xcols, alpha, _idx(A.row_map), _idx(A.entries), _ptr(A.values), _ptr(x), ldx,
             xrm, beta, _ptr(y), ldy, yrm))
    return y


class SPTRSVHandle:
    """KokkosSparse::Experimental::SPTRSVHandle as far as sptrsv_symbolic / sptrsv_solve need it (sparse/src/KokkosSparse_sptrsv_handle.hpp:
    is_lower_tri, nrows, the level sets): owns a b200sp_sptrsv_plan."""

    def __init__(self, nrows, lower_tri):
        self.nrows, self.lower_tri = int(nrows), bool(lower_tri)
        self._plan = C.c_void_p(0)
        check(_lib.sparse().b200sp_sptrsv_plan_create(C.byref(self._plan)))
        self._symbolic = False

    def is_lower_tri(self): return self.lower_tri
    def get_nrows(self): return self.nrows
    def get_num_levels(self): return _lib.sparse().b200sp_sptrsv_levels(self._plan)
    def get_num_launches(self): return _lib.sparse().b200sp_sptrsv_launches(self._plan)  # kernel launches of one solve
    def is_symbolic_complete(self): return self._symbolic

    def __del__(self):
        try:
            if self._plan:
                st = _stream() if torch.cuda.is_available() else C.c_void_p(0)
                _lib.sparse().b200sp_sptrsv_plan_destroy(self._plan, st)
                self._plan = C.c_void_p(0)
        except Exception:
            pass


def sptrsv_symbolic(handle, row_map, entries):
    """KokkosSparse::sptrsv_symbolic(handle, rowmap, entries) (sparse/src/KokkosSparse_sptrsv.hpp:40-170): the dependency levels of a
    lower / upper triangular matrix whose diagonal is stored."""
    if row_map.numel() != handle.nrows + 1:
        raise B200SparseError("sptrsv_symbolic: row map does not match the handle's number of rows")
    check(_lib.sparse().b200sp_sptrsv_symbolic_i32(handle._plan, _stream(), handle.nrows, _idx(row_map), _idx(entries), int(handle.lower_tri)))
    handle._symbolic = True


def sptrsv_solve(handle, row_map, entries, values, b, x):
    """KokkosSparse::sptrsv_solve(handle, rowmap, entries, values, b, x) (sparse/src/KokkosSparse_sptrsv.hpp:290-480): x = T^{-1} b."""
    if not handle._symbolic:
        raise B200SparseError("sptrsv_solve: sptrsv_symbolic was not called on this handle")
    if b.numel() != handle.nrows or x.numel() != handle.nrows:
        raise B200SparseError("sptrsv_solve: vector lengths do not match the handle's number of rows")
    fn = getattr(_lib.sparse(), f"b200sp_sptrsv_solve_{_sfx(values)}_i32")
    check(fn(handle._plan, _stream(), handle.nrows, _idx(row_map), _idx(entries), _ptr(values), _ptr(b), _ptr(x)))
    return x


class GMRESHandle:
    """sparse/src/KokkosSparse_gmres_handle.hpp:66-186: options (m, tol, max_restart, ortho, verbose) and the statistics of the
    last run (num_iters, end_rel_res, conv_flag_val)."""

    CGS2, MGS = 0, 1  # Ortho (:76-79)
    Conv, NoConv, LOA, NotRun = 0, 1, 2, 3  # Flag (:84-89)

    def __init__(self, m=50, tol=1e-8, max_restart=50):
        self.reset_handle(m, tol, max_restart)

    def reset_handle(self, m=50, tol=1e-8, max_restart=50):
        self.m, self.tol, self.max_restart = int(m), float(tol), int(max_restart)
        self.ortho, self.verbose = GMRESHandle.CGS2, False
        self.num_iters, self.end_rel_res, self.conv_flag_val = -1, 0.0, GMRESHandle.NotRun

    def set_m(self, m): self.m = int(m)
    def set_tol(self, tol): self.tol = float(tol)
    def set_max_restart(self, r): self.max_restart = int(r)
    def set_ortho(self, o): self.ortho = o
    def set_verbose(self, v): self.verbose = bool(v)
    def get_m(self): return self.m
    def get_tol(self): return self.tol
    def get_max_restart(self): return self.max_restart
    def get_ortho(self): return self.ortho
    def get_num_iters(self): return self.num_iters
    def get_end_rel_res(self): return self.end_rel_res
    def get_conv_flag_val(self): return self.conv_flag_val


class MatrixPrec:
    """KokkosSparse::Experimental::MatrixPrec (sparse/src/KokkosSparse_MatrixPrec.hpp:33-96): a preconditioner whose apply is
    an spmv with the given matrix."""

    def __init__(self, A):
        self.A = A
        self._handle = SPMVHandle(SPMV_DEFAULT)


def gmres(handle, A, B, X, precond=None, spmv_handle=None):
    """KokkosSparse::Experimental::gmres(handle, A, B, X, precond) (sparse/src/KokkosSparse_gmres.hpp:60-160): `handle` is a
    GMRESHandle (or a KokkosKernelsHandle carrying one); A a CrsMatrix or a BsrMatrix; X is the
    initial guess and receives the solution.  Statistics land on the handle (set_stats, gmres_handle.hpp:175)."""
    gh = handle.get_gmres_handle() if hasattr(handle, "get_gmres_handle") else handle
    is_bsr = isinstance(A, BsrMatrix)
    n = A.numPointRows() if is_bsr else A.numRows()
    ncols = A.numPointCols() if is_bsr else A.numCols()
    if ncols != n:  # gmres.hpp:84-90
        raise B200SparseError(f"KokkosSparse::gmres: A must be a square matrix: numRows: {n}  numCols: {ncols}")
    if X.dim() != 1 or B.dim() != 1 or X.shape[0] != n or B.shape[0] != n:  # :92-101
        raise B200SparseError(f"KokkosSparse::gmres: Dimensions do not match: X: {X.shape[0]} B: {B.shape[0]} A: {n}")
    if not (A.values.dtype == X.dtype == B.dtype) or X.dtype not in (torch.float64, torch.float32):
        raise B200SparseError("b200sparse: gmres needs A, B, X of one scalar type (double or float)")
    if gh.ortho not in (GMRESHandle.CGS2, GMRESHandle.MGS):
        raise B200SparseInvalidArgument("Invalid argument for 'ortho'.  Please use 'CGS2' or 'MGS'.")
    f64 = X.dtype == torch.float64
    lib = _lib.sparse()
    ha = spmv_handle if spmv_handle is not None else SPMVHandle(SPMV_DEFAULT)
    it, flag = C.c_int(0), C.c_int(0)
    res = C.c_double(0.0) if f64 else C.c_float(0.0)
    tol = C.c_double(gh.tol) if f64 else C.c_float(gh.tol)
    null = C.c_void_p(0)
    if precond is not None:
        M = precond.A
        if isinstance(M, BsrMatrix) != is_bsr or M.values.dtype != X.dtype or (is_bsr and M.blockDim() != A.blockDim()) or \
                M.numRows() != A.numRows() or M.numCols() != A.numCols():
            raise B200SparseError("gmres: the MatrixPrec matrix must have A's type, size and scalar")
        pm = precond._handle._bsr() if is_bsr else precond._handle._plan
        nnzm, rpm, cim, vm = M.nnz(), _idx(M.row_map), _idx(M.entries), _ptr(M.values)
    else:
        pm, nnzm, rpm, cim, vm = null, 0, null, null, null
    if is_bsr:
        fn = lib.b200sp_gmres_bsr_f64_i32 if f64 else lib.b200sp_gmres_bsr_f32_i32
        check(fn(ha._bsr(), _stream(), A.numRows(), A.nnz(), A.blockDim(), _idx(A.row_map), _idx(A.entries), _ptr(A.values), pm, nnzm, rpm, cim, vm,
                 _ptr(B), _ptr(X), gh.m, tol, gh.max_restart, gh.ortho, C.byref(it), C.byref(res), C.byref(flag)))
    else:
        fn = lib.b200sp_gmres_f64_i32 if f64 else lib.b200sp_gmres_f32_i32
        check(fn(ha._plan, _stream(), n, A.nnz(), _idx(A.row_map), _idx(A.entries), _ptr(A.values), pm, nnzm, rpm, cim, vm, _ptr(B), _ptr(X),
                 gh.m, tol, gh.max_restart, gh.ortho, C.byref(it), C.byref(res), C.byref(flag)))
    gh.num_iters, gh.end_rel_res, gh.conv_flag_val = it.value, float(res.value), flag.value
    return gh


class GaussSeidelHandle:
    """The point Gauss-Seidel handle (sparse/src/KokkosSparse_gauss_seidel_handle.hpp:37-330; GS_DEFAULT): owns the colouring and
    the inverse diagonal (b200sp_gs_plan)."""

    def __init__(self):
        self._plan = C.c_void_p(0)
        check(_lib.sparse().b200sp_gs_plan_create(C.byref(self._plan)))
        self._symbolic = self._numeric = False

    def is_symbolic_called(self): return self._symbolic
    def is_numeric_called(self): return self._numeric

    def get_num_colors(self):
        nc = C.c_int(0)
        check(_lib.sparse().b200sp_gs_get_coloring(self._plan, C.byref(nc), None, None, None))
        return nc.value

    def get_coloring(self, n):
        """(colors[n], color_ptr[num_colors + 1], color_rows[n]) as host numpy arrays."""
        import numpy as np

        nc = self.get_num_colors()
        colors, cptr, crows = np.zeros(n, np.int32), np.zeros(nc + 1, np.int32), np.zeros(n, np.int32)
        check(_lib.sparse().b200sp_gs_copy_coloring(self._plan, _stream(), C.c_void_p(colors.ctypes.data), C.c_void_p(cptr.ctypes.data),
                                                    C.c_void_p(crows.ctypes.data)))
        return colors, cptr, crows

    def __del__(self):
        try:
            if self._plan:
                st = _stream() if torch.cuda.is_available() else C.c_void_p(0)
                _lib.sparse().b200sp_gs_plan_destroy(self._plan, st)
                self._plan = C.c_void_p(0)
        except Exception:
            pass


class TwoStageGaussSeidelHandle:
    """TwoStageGaussSeidelHandle (sparse/src/KokkosSparse_gauss_seidel_handle.hpp:513-673) with inner Jacobi-Richardson sweeps: owns
    L, U (and La, Ua in the compact form), the scaled diagonal, the work vectors and the SpMV plans (b200sp_gs2_plan)."""

    def __init__(self):
        self._plan = C.c_void_p(0)
        check(_lib.sparse().b200sp_gs2_plan_create(C.byref(self._plan)))
        self._symbolic = self._numeric = False
        self.two_stage, self.compact_form, self.num_inner_sweeps, self.num_outer_sweeps, self.inner_omega = True, False, 1, 1, 1.0

    def is_symbolic_called(self): return self._symbolic
    def is_numeric_called(self): return self._numeric

    def _set(self, option, value):
        check(_lib.sparse().b200sp_gs2_plan_set(self._plan, option, C.c_double(float(value))))

    def setTwoStage(self, two_stage):
        """False selects the classic form (gauss_seidel_handle.hpp:560-566): triangular solves (b200sp_sptrsv level sets on the
        triangles of A) instead of inner Jacobi-Richardson sweeps; omega must be 1 then."""
        self.two_stage = bool(two_stage)
        self._set(5, self.two_stage)
        self._symbolic = self._numeric = False

    def isTwoStage(self): return self.two_stage

    def setCompactForm(self, compact_form):
        self.compact_form = bool(compact_form)
        self._set(1, self.compact_form)
        self._symbolic = self._numeric = False

    def isCompactForm(self): return self.compact_form

    def setNumInnerSweeps(self, n):
        self.num_inner_sweeps = int(n)
        self._set(2, n)

    def getNumInnerSweeps(self): return self.num_inner_sweeps

    def setNumOuterSweeps(self, n):
        self.num_outer_sweeps = int(n)
        self._set(3, n)

    def getNumOuterSweeps(self): return self.num_outer_sweeps

    def setInnerDampFactor(self, g):
        self.inner_omega = float(g)
        self._set(4, g)

    def getInnerDampFactor(self): return self.inner_omega

    def __del__(self):
        try:
            if self._plan:
                st = _stream() if torch.cuda.is_available() else C.c_void_p(0)
                _lib.sparse().b200sp_gs2_plan_destroy(self._plan, st)
                self._plan = C.c_void_p(0)
        except Exception:
            pass


def _gs_handle(handle):
    gh = handle.get_gs_handle() if hasattr(handle, "get_gs_handle") else handle
    if gh is None:
        raise B200SparseInvalidArgument("Gauss-Seidel handle has not been created (create_gs_handle)")
    return gh


def gauss_seidel_symbolic(handle, num_rows, num_cols, row_map, entries, is_graph_symmetric=True):
    """KokkosSparse::gauss_seidel_symbolic (sparse/src/KokkosSparse_gauss_seidel.hpp:49-110)."""
    gh = _gs_handle(handle)
    if isinstance(gh, TwoStageGaussSeidelHandle):
        check(_lib.sparse().b200sp_gs2_symbolic_i32(gh._plan, _stream(), int(num_rows), int(num_cols), _idx(row_map), _idx(entries)))
        gh._symbolic, gh._numeric = True, False
        return
    if num_cols < num_rows:
        raise B200SparseError("b200sparse: Gauss-Seidel needs num_cols >= num_rows (columns beyond num_rows are ghost entries of x)")
    check(_lib.sparse().b200sp_gs_symbolic_nc_i32(gh._plan, _stream(), int(num_rows), int(num_cols), _idx(row_map), _idx(entries),
                                                  int(bool(is_graph_symmetric))))
    gh._symbolic, gh._numeric = True, False


def gauss_seidel_numeric(handle, num_rows, num_cols, row_map, entries, values, is_graph_symmetric=True, given_inverse_diagonal=None):
    """KokkosSparse::gauss_seidel_numeric (:223-290, and the overload taking the inverse diagonal :118-221 -- used by the two-stage
    method only here); is_graph_symmetric only matters to symbolic."""
    gh = _gs_handle(handle)
    if isinstance(gh, TwoStageGaussSeidelHandle):
        fn = _lib.sparse().b200sp_gs2_numeric_f64_i32 if values.dtype == torch.float64 else _lib.sparse().b200sp_gs2_numeric_f32_i32
        check(fn(gh._plan, _stream(), int(num_rows), int(num_cols), _idx(row_map), _idx(entries), _ptr(values), _ptr(given_inverse_diagonal)))
        gh._numeric = True
        return
    fn = _lib.sparse().b200sp_gs_numeric_f64_i32 if values.dtype == torch.float64 else _lib.sparse().b200sp_gs_numeric_f32_i32
    check(fn(gh._plan, _stream(), int(num_rows), _idx(row_map), _idx(entries), _ptr(values)))
    gh._numeric = True


def _gs2_apply(gh, num_rows, num_cols, row_map, entries, values, x_lhs, y_rhs, init_zero_x_vector, omega, numIter, direction):
    """rank-1 or rank-2 (columns contiguous: LayoutLeft, the reference's default_layout on the GPU) x (num_cols rows) and y (num_rows)."""
    if values.dtype != x_lhs.dtype or x_lhs.dtype != y_rhs.dtype or x_lhs.dim() != y_rhs.dim() or x_lhs.dim() not in (1, 2):
        raise B200SparseError("b200sparse: gauss_seidel_apply needs x, y of the matrix' scalar type, both rank 1 or both rank 2")
    if x_lhs.shape[0] != num_cols or y_rhs.shape[0] != num_rows:
        raise B200SparseError("b200sparse: gauss_seidel_apply: x needs num_cols rows, y num_rows")
    nrhs, ldx, ldy = 1, int(num_cols), int(num_rows)
    if x_lhs.dim() == 2:
        nrhs = x_lhs.shape[1]
        if y_rhs.shape[1] != nrhs or (x_lhs.shape[0] > 1 and x_lhs.stride(0) != 1) or (y_rhs.shape[0] > 1 and y_rhs.stride(0) != 1):
            raise B200SparseError("b200sparse: two-stage gauss_seidel_apply needs LayoutLeft multivectors with equal column counts")
        ldx, ldy = (x_lhs.stride(1), y_rhs.stride(1)) if nrhs > 1 else (ldx, ldy)
    elif x_lhs.stride(0) != 1 or y_rhs.stride(0) != 1:
        raise B200SparseError("b200sparse: rank-1 x and y must be contiguous")
    fn = _lib.sparse().b200sp_gs2_apply_f64_i32 if values.dtype == torch.float64 else _lib.sparse().b200sp_gs2_apply_f32_i32
    check(fn(gh._plan, _stream(), int(num_rows), int(num_cols), _idx(row_map), _idx(entries), _ptr(values), _ptr(x_lhs), ldx, _ptr(y_rhs), ldy,
             int(nrhs), int(bool(init_zero_x_vector)), omega, int(numIter), direction))


def _gs_apply(handle, num_rows, row_map, entries, values, x_lhs, y_rhs, init_zero_x_vector, omega, numIter, direction, num_cols=None):
    gh = _gs_handle(handle)
    if isinstance(gh, TwoStageGaussSeidelHandle):
        return _gs2_apply(gh, num_rows, num_rows if num_cols is None else num_cols, row_map, entries, values, x_lhs, y_rhs, init_zero_x_vector,
                          omega, numIter, direction)
    if values.dtype != x_lhs.dtype or x_lhs.dtype != y_rhs.dtype or x_lhs.dim() != 1 or y_rhs.dim() != 1:
        raise B200SparseError("b200sparse: gauss_seidel_apply needs rank-1 x, y of the matrix' scalar type")
    fn = _lib.sparse().b200sp_gs_apply_f64_i32 if values.dtype == torch.float64 else _lib.sparse().b200sp_gs_apply_f32_i32
    check(fn(gh._plan, _stream(), int(num_rows), _idx(row_map), _idx(entries), _ptr(values), _ptr(x_lhs), _ptr(y_rhs), int(bool(init_zero_x_vector)),
             omega, int(numIter), direction))


def symmetric_gauss_seidel_apply(handle, num_rows, num_cols, row_map, entries, values, x_lhs_output_vec, y_rhs_input_vec,
                                 init_zero_x_vector, update_y_vector, omega, numIter):
    """KokkosSparse::symmetric_gauss_seidel_apply (:363-470); update_y_vector is moot (y is never permuted or copied here)."""
    _gs_apply(handle, num_rows, row_map, entries, values, x_lhs_output_vec, y_rhs_input_vec, init_zero_x_vector, omega, numIter, 0, num_cols)


def forward_sweep_gauss_seidel_apply(handle, num_rows, num_cols, row_map, entries, values, x_lhs_output_vec, y_rhs_input_vec,
                                     init_zero_x_vector, update_y_vector, omega, numIter):
    _gs_apply(handle, num_rows, row_map, entries, values, x_lhs_output_vec, y_rhs_input_vec, init_zero_x_vector, omega, numIter, 1, num_cols)


def backward_sweep_gauss_seidel_apply(handle, num_rows, num_cols, row_map, entries, values, x_lhs_output_vec, y_rhs_input_vec,
                                      init_zero_x_vector, update_y_vector, omega, numIter):
    _gs_apply(handle, num_rows, row_map, entries, values, x_lhs_output_vec, y_rhs_input_vec, init_zero_x_vector, omega, numIter, 2, num_cols)


class CGSolveResult:
    """perf_test/sparse/KokkosSparse_pcg.hpp:38-45 (the fields this driver fills)."""

    def __init__(self, iteration, norm_res):
        self.iteration, self.norm_res = iteration, norm_res


def pcgsolve(handle, A, y_vector, x_vector, maximum_iteration=200, tolerance=2.220446049250313e-16, check_every=0, use_sgs=False,
             gs_handle=None):
    """KokkosKernels::Experimental::Example::pcgsolve(kh, crsMat, y_vector, x_vector, maximum_iteration, tolerance, &result,
    use_sgs) (perf_test/sparse/KokkosSparse_pcg.hpp:248-466): CG for a symmetric positive definite CrsMatrix, unpreconditioned or
    (use_sgs, the reference's default) preconditioned by one symmetric point Gauss-Seidel sweep; x_vector is the initial guess and
    receives the solution.  `handle` is the SPMVHandle of A (None: a throw-away one); gs_handle a GaussSeidelHandle whose symbolic /
    numeric already ran on A (None with use_sgs: created here, as the reference's driver does, :296-337), or a
    TwoStageGaussSeidelHandle / a KokkosKernelsHandle holding one: the preconditioner is then one symmetric two-stage sweep, as in the
    reference, whose symmetric_gauss_seidel_apply dispatches on the handle.  The loop runs on the
    device (b200sp_cg_solve_f64_i32 / b200sp_pcg_solve_f64_i32); double only, like the reference driver."""
    n = A.numRows()
    if A.numCols() != n or y_vector.shape[0] != n or x_vector.shape[0] != n or y_vector.dim() != 1 or x_vector.dim() != 1:
        raise B200SparseError("pcgsolve: A must be square and x, b rank-1 vectors of its size")
    if A.values.dtype != torch.float64 or x_vector.dtype != torch.float64 or y_vector.dtype != torch.float64:
        raise B200SparseError("pcgsolve: The PCG performance test only works with scalar = double.")  # pcg.hpp:258-259
    h = handle if handle is not None else SPMVHandle(SPMV_DEFAULT)
    it, nr = C.c_int(0), C.c_double(0.0)
    if use_sgs:
        gh = gs_handle
        if gh is None:
            gh = GaussSeidelHandle()
            gauss_seidel_symbolic(gh, n, n, A.row_map, A.entries, True)  # SPD: the pattern is symmetric
            gauss_seidel_numeric(gh, n, n, A.row_map, A.entries, A.values, True)
        gh = gh.get_gs_handle() if hasattr(gh, "get_gs_handle") else gh  # a KokkosKernelsHandle holding the GS handle, as the reference passes
        if isinstance(gh, TwoStageGaussSeidelHandle):
            if not gh.is_numeric_called():
                gauss_seidel_symbolic(gh, n, n, A.row_map, A.entries, True)
                gauss_seidel_numeric(gh, n, n, A.row_map, A.entries, A.values, True)
            solve = _lib.sparse().b200sp_pcg_solve_gs2_f64_i32
        else:
            solve = _lib.sparse().b200sp_pcg_solve_f64_i32
        check(solve(h._plan, gh._plan, _stream(), n, A.nnz(), _idx(A.row_map), _idx(A.entries), _ptr(A.values),
                                                     _ptr(y_vector), _ptr(x_vector), int(maximum_iteration), C.c_double(tolerance),
                                                     int(check_every), C.byref(it), C.byref(nr)))
        return CGSolveResult(it.value, nr.value)
    check(_lib.sparse().b200sp_cg_solve_f64_i32(h._plan, _stream(), n, A.nnz(), _idx(A.row_map), _idx(A.entries), _ptr(A.values),
                                                _ptr(y_vector), _ptr(x_vector), int(maximum_iteration), C.c_double(tolerance),
                                                int(check_every), C.byref(it), C.byref(nr)))
    return CGSolveResult(it.value, nr.value)


def spmv_scatter(handle, alpha, A, x, y, extra_ptrs):
    """Fused SpMV + all-gather: y (this rank's row block) is also stored to the raw device pointers in
    `extra_ptrs` (peer GPUs' next-x slots mapped into this process)."""
    arr = (C.c_void_p * max(len(extra_ptrs), 1))(*[C.c_void_p(int(q)) for q in extra_ptrs])
    check(_lib.sparse().b200sp_spmv_scatter_f64_i32(
        handle._plan, _stream(), A.numRows(), A.numCols(), A.nnz(), alpha, _idx(A.row_map), _idx(A.entries),
        _ptr(A.values), _ptr(x), _ptr(y), len(extra_ptrs), arr))
    return y


def spmv_forward(handle, alpha, A, x, y, forward_ptr):
    """Fused SpMV + all-gather through one destination (the NVSwitch multicast mapping): finished tiles of y are forwarded
    to the raw device pointer `forward_ptr` by the kernel's producer warp (b200sp_spmv_forward_f64_i32)."""
    check(_lib.sparse().b200sp_spmv_forward_f64_i32(
        handle._plan, _stream(), A.numRows(), A.numCols(), A.nnz(), alpha, _idx(A.row_map), _idx(A.entries),
        _ptr(A.values), _ptr(x), _ptr(y), C.c_void_p(int(forward_ptr))))
    return y


def spmv_hostvec(handle, mode, alpha, A, x_host, beta, y_host):
    """End-to-end entry: host x / y (pinned), device-resident matrix."""
    m, n = A.numRows(), A.numCols()
    check(_lib.sparse().b200sp_spmv_hostvec_f64_i32(
        handle._plan, _stream(), _mode_char(mode).encode(), m, n, A.nnz(), alpha, _idx(A.row_map),
        _idx(A.entries), _ptr(A.values), C.c_void_p(x_host.data_ptr()), beta, C.c_void_p(y_host.data_ptr())))
    return y_host


# --------------------------------------------------------------------------- SpGEMM
class SPGEMMHandle:
    """State flags and results of sparse/src/KokkosSparse_spgemm_handle.hpp:236-240,356-362,628-651."""

    def __init__(self, algo=SPGEMM_KK):
        self.algo = algo
        self._plan = C.c_void_p(0)
        check(_lib.sparse().b200sp_spgemm_plan_create(C.byref(self._plan)))
        self._symbolic = self._numeric = self._rowptrs = self._entries = False
        self._c_nnz = -1
        self._max_nnz = -1

    def is_symbolic_called(self): return self._symbolic
    def is_numeric_called(self): return self._numeric
    def are_rowptrs_computed(self): return self._rowptrs
    def are_entries_computed(self): return self._entries
    def get_c_nnz(self): return self._c_nnz
    def get_max_result_nnz(self): return self._max_nnz

    def set_window(self, max_entries):
        """64-bit offsets only: products and entries of A per 32-bit window of the next symbolic (default 2^31 - 65537;
        smaller values are for tests)."""
        check(_lib.sparse().b200sp_spgemm_plan_set_window(self._plan, int(max_entries)))

    def windows(self):
        """Windows of the last symbolic on 64-bit offsets (0 otherwise)."""
        return _lib.sparse().b200sp_spgemm_plan_windows(self._plan)

    def __del__(self):
        try:
            if self._plan:
                st = _stream() if torch.cuda.is_available() else C.c_void_p(0)
                _lib.sparse().b200sp_spgemm_plan_destroy(self._plan, st)
                self._plan = C.c_void_p(0)
        except Exception:
            pass


class SPADDHandle:
    """sparse/src/KokkosSparse_spadd_handle.hpp:24-137: input_sorted / input_merged flags, c_nnz, the
    called flags; a_pos / b_pos of the unsorted algorithm live in the C plan."""

    def __init__(self, input_is_sorted, input_is_merged=False):
        self.input_sorted, self.input_merged = bool(input_is_sorted), bool(input_is_merged)
        self._plan = C.c_void_p(0)
        check(_lib.sparse().b200sp_spadd_plan_create(C.byref(self._plan), int(self.input_sorted), int(self.input_merged)))
        self._symbolic = self._numeric = False
        self._c_nnz = 0

    def is_input_sorted(self): return self.input_sorted
    def is_input_merged(self): return self.input_merged
    def is_input_strict_crs(self): return self.input_sorted and self.input_merged
    def is_symbolic_called(self): return self._symbolic
    def is_numeric_called(self): return self._numeric
    def get_c_nnz(self): return self._c_nnz

    def __del__(self):
        try:
            if self._plan:
                st = _stream() if torch.cuda.is_available() else C.c_void_p(0)
                _lib.sparse().b200sp_spadd_plan_destroy(self._plan, st)
                self._plan = C.c_void_p(0)
        except Exception:
            pass


class KokkosKernelsHandle:
    def __init__(self):
        self._sh = None
        self._ah = None

    def create_spadd_handle(self, input_is_sorted=False, input_is_merged=False):
        self._ah = SPADDHandle(input_is_sorted, input_is_merged)

    def get_spadd_handle(self):
        return self._ah

    def destroy_spadd_handle(self):
        self._ah = None

    def create_gs_handle(self, gs_algorithm=GS_DEFAULT, *args, **kwargs):
        """KokkosKernelsHandle::create_gs_handle(GSAlgorithm, coloring algorithm) (sparse/src/KokkosKernels_Handle.hpp:624-630):
        GS_DEFAULT / GS_PERMUTED / GS_TEAM -> the point multicolour handle (colouring arguments are accepted and ignored),
        GS_TWOSTAGE -> the two-stage handle; GS_CLUSTER is not provided."""
        if gs_algorithm == GS_TWOSTAGE:
            self._gs = TwoStageGaussSeidelHandle()
        elif gs_algorithm in (GS_DEFAULT, GS_PERMUTED, GS_TEAM) or not isinstance(gs_algorithm, int):
            self._gs = GaussSeidelHandle()
        else:
            raise B200SparseError("b200sparse: cluster Gauss-Seidel is not provided (point and two-stage are)")

    def get_twostage_gs_handle(self):
        gh = getattr(self, "_gs", None)
        if not isinstance(gh, TwoStageGaussSeidelHandle):  # KokkosKernels_Handle.hpp:631-637
            raise B200SparseError("TwoStageGaussSeidelHandle has not been created, or is set to Default.")
        return gh

    def set_gs_set_num_outer_sweeps(self, n): self.get_twostage_gs_handle().setNumOuterSweeps(n)
    def set_gs_set_num_inner_sweeps(self, n): self.get_twostage_gs_handle().setNumInnerSweeps(n)
    def set_gs_set_inner_damp_factor(self, g): self.get_twostage_gs_handle().setInnerDampFactor(g)
    def set_gs_twostage(self, two_stage, nrows=0): self.get_twostage_gs_handle().setTwoStage(two_stage)
    def set_gs_twostage_compact_form(self, compact_form): self.get_twostage_gs_handle().setCompactForm(compact_form)

    def get_gs_handle(self):
        return getattr(self, "_gs", None)

    def get_point_gs_handle(self):
        return getattr(self, "_gs", None)

    def destroy_gs_handle(self):
        self._gs = None

    def create_gmres_handle(self, m=50, tol=1e-8, max_restart=50):  # KokkosKernels_Handle.hpp (create_gmres_handle)
        self._gmres = GMRESHandle(m, tol, max_restart)

    def get_gmres_handle(self):
        return self._gmres

    def destroy_gmres_handle(self):
        self._gmres = None

    def create_spgemm_handle(self, algo=SPGEMM_KK):
        self._sh = SPGEMMHandle(algo)

    def get_spgemm_handle(self):
        return self._sh

    def destroy_spgemm_handle(self):
        self._sh = None


def spgemm_symbolic_views(kh, m, n, k, row_mapA, entriesA, transposeA, row_mapB, entriesB, transposeB, row_mapC,
                          computeRowptrs=False):
    """View-level spgemm_symbolic (sparse/src/KokkosSparse_spgemm_symbolic.hpp:25-182).  The CUDA
    path always fills row_mapC (computeRowptrs is implied)."""
    if transposeA or transposeB:  # :61-65
        raise B200SparseError("KokkosSparse::spgemm_symbolic: transposing A or B is not supported")
    sh = kh.get_spgemm_handle()
    if sh is None:
        raise B200SparseInvalidArgument("spgemm_symbolic: create_spgemm_handle() was not called")
    if row_mapC.numel() != m + 1:
        raise B200SparseError("spgemm_symbolic: row_mapC must have m+1 entries")
    wide = _spgemm_wide((row_mapA, row_mapB, row_mapC), (entriesA, entriesB))
    c_nnz, c_max = C.c_int64(0), C.c_int(0)
    fn = _lib.sparse().b200sp_spgemm_symbolic_i64 if wide else _lib.sparse().b200sp_spgemm_symbolic_i32
    rp = _ptr if wide else _idx
    check(fn(sh._plan, _stream(), m, n, k, rp(row_mapA), _idx(entriesA), rp(row_mapB), _idx(entriesB),
             C.c_void_p(row_mapC.data_ptr()), C.byref(c_nnz), C.byref(c_max)))
    sh._c_nnz, sh._max_nnz = c_nnz.value, c_max.value
    sh._symbolic = True
    sh._rowptrs = True


def spgemm_numeric_views(kh, m, n, k, row_mapA, entriesA, valuesA, transposeA, row_mapB, entriesB, valuesB,
                         transposeB, row_mapC, entriesC, valuesC, block_dim=1):
    """View-level spgemm_numeric (sparse/src/KokkosSparse_spgemm_numeric.hpp:35-256).  block_dim > 1: m, n, k count
    blocks, the values hold bs*bs entries per block (row-major) and the product is the block SpGEMM
    (b200sp_bspgemm_numeric_*, bit-identical to the reference's bspgemm_debug_numeric); block_dim == 1 is the point
    product, as in the reference (:191)."""
    if transposeA or transposeB:
        raise B200SparseError("KokkosSparse::spgemm_numeric: transposing A or B is not supported")
    sh = kh.get_spgemm_handle()
    if sh is None or not sh.is_symbolic_called():  # numeric_spec.hpp:116-118
        raise B200SparseError("Call spgemm symbolic before spgemm numeric")
    if int(block_dim) > 1:
        _bspgemm_numeric(sh, m, n, k, int(block_dim), row_mapA, entriesA, valuesA, row_mapB, entriesB, valuesB, row_mapC,
                         entriesC, valuesC)
        return
    wide = _spgemm_wide((row_mapA, row_mapB, row_mapC), (entriesA, entriesB, entriesC))
    f64 = valuesA.dtype == torch.float64
    L = _lib.sparse()
    if wide:
        fn = L.b200sp_spgemm_numeric_f64_i64 if f64 else L.b200sp_spgemm_numeric_f32_i64
    else:
        fn = L.b200sp_spgemm_numeric_f64_i32 if f64 else L.b200sp_spgemm_numeric_f32_i32
    rp = _ptr if wide else _idx
    check(fn(sh._plan, _stream(), m, n, k, rp(row_mapA), _idx(entriesA), _ptr(valuesA), rp(row_mapB),
             _idx(entriesB), _ptr(valuesB), rp(row_mapC), _idx(entriesC), _ptr(valuesC)))
    sh._numeric = True
    sh._entries = True


def spgemm_symbolic(kh, A, Amode, B, Bmode, C_out=None):
    """Matrix-level wrapper (sparse/src/KokkosSparse_spgemm.hpp:40-61): allocates row_map(m+1)
    uninitialised, runs symbolic, sizes entries/values from get_c_nnz().  Returns C."""
    m, n, k = A.numRows(), A.numCols(), B.numCols()
    dev = A.row_map.device
    row_mapC = torch.empty(m + 1, dtype=A.row_map.dtype, device=dev)
    spgemm_symbolic_views(kh, m, n, k, A.row_map, A.entries, Amode, B.row_map, B.entries, Bmode, row_mapC)
    c_nnz = kh.get_spgemm_handle().get_c_nnz()
    entriesC = torch.empty(c_nnz, dtype=torch.int32, device=dev)
    valuesC = torch.empty(c_nnz, dtype=A.values.dtype, device=dev)
    return CrsMatrix(row_mapC, entriesC, valuesC, k)


def spgemm_numeric(kh, A, Amode, B, Bmode, Cm):
    spgemm_numeric_views(kh, A.numRows(), A.numCols(), B.numCols(), A.row_map, A.entries, A.values, Amode,
                         B.row_map, B.entries, B.values, Bmode, Cm.row_map, Cm.entries, Cm.values)
    return Cm


def spgemm_jacobi(kh, A, Amode, B, Bmode, Cm, omega, dinv):
    """KokkosSparse::Experimental::spgemm_jacobi (sparse/src/KokkosSparse_spgemm_jacobi.hpp:25-190):
    C = (I - omega * diag(dinv) * A) * B on the structure spgemm_symbolic(kh, A, B) produced; dinv has one entry
    per row (the reference passes an m x 1 view)."""
    if Amode or Bmode:
        raise B200SparseError("KokkosSparse::spgemm_jacobi: transposing A or B is not supported")
    if any(t.dtype == torch.int64 for t in (A.row_map, B.row_map, Cm.row_map)):
        raise B200SparseError("KokkosSparse::spgemm_jacobi: not provided on 64-bit offsets (int32 row maps only)")
    sh = kh.get_spgemm_handle()
    if sh is None or not sh.is_symbolic_called():
        raise B200SparseError("KokkosSparse::spgemm_jacobi: must first call spgemm_symbolic with the same handle.")
    dv = dinv.reshape(-1)
    if dv.numel() != A.numRows() or dv.dtype != A.values.dtype:
        raise B200SparseError("KokkosSparse::spgemm_jacobi: dinv must hold one value of the matrix scalar type per row")
    fn = getattr(_lib.sparse(), f"b200sp_spgemm_jacobi_{_sfx(A.values)}_i32")
    check(fn(sh._plan, _stream(), A.numRows(), A.numCols(), B.numCols(), _idx(A.row_map), _idx(A.entries), _ptr(A.values),
             _idx(B.row_map), _idx(B.entries), _ptr(B.values), _idx(Cm.row_map), _idx(Cm.entries), _ptr(Cm.values), omega,
             _ptr(dv.contiguous())))
    sh._numeric = True
    sh._entries = True
    return Cm


def _bspgemm_numeric(sh, mb, nb, kb, bs, row_mapA, entriesA, valuesA, row_mapB, entriesB, valuesB, row_mapC, entriesC, valuesC):
    if bs < 1:
        raise B200SparseError(f"KokkosSparse::block_spgemm_numeric: inappropriate block size {bs}")
    vals = (valuesA, valuesB, valuesC)
    if any(v.dtype != valuesA.dtype for v in vals):
        raise B200SparseError("KokkosSparse::block_spgemm_numeric: A, B and C must have the same scalar type "
                              f"(got {valuesA.dtype}, {valuesB.dtype}, {valuesC.dtype})")
    if any(t.dtype != torch.int32 for t in (row_mapA, entriesA, row_mapB, entriesB, row_mapC, entriesC)):
        raise B200SparseError("KokkosSparse::block_spgemm_numeric: 64-bit offsets or ordinals are not provided for block "
                              "SpGEMM (int32 row maps and entries only)")
    for v, nz, what in ((valuesA, entriesA.numel(), "A"), (valuesB, entriesB.numel(), "B"), (valuesC, entriesC.numel(), "C")):
        if v.numel() != nz * bs * bs:
            raise B200SparseError(f"KokkosSparse::block_spgemm_numeric: values of {what} must hold nnz*blockDim*blockDim entries")
    _sfx(valuesA)
    L = _lib.sparse()
    fn = L.b200sp_bspgemm_numeric_f64_i32 if valuesA.dtype == torch.float64 else L.b200sp_bspgemm_numeric_f32_i32
    check(fn(sh._plan, _stream(), mb, nb, kb, bs, _idx(row_mapA), _idx(entriesA), _ptr(valuesA), _idx(row_mapB), _idx(entriesB),
             _ptr(valuesB), _idx(row_mapC), _idx(entriesC), _ptr(valuesC)))
    sh._numeric = True
    sh._entries = True


def block_spgemm_symbolic(kh, A, transposeA, B, transposeB):
    """KokkosSparse::block_spgemm_symbolic (sparse/src/KokkosSparse_spgemm.hpp:77-103): the point symbolic on the block
    graphs.  Returns a BsrMatrix C whose entries hold nnz(C) blocks and whose values hold nnz(C)*bs*bs entries
    (uninitialised until block_spgemm_numeric)."""
    if not isinstance(A, BsrMatrix) or not isinstance(B, BsrMatrix):
        raise B200SparseError("KokkosSparse::block_spgemm_symbolic: A and B must be BsrMatrix")
    bs = A.blockDim()
    if bs != B.blockDim():
        raise B200SparseInvalidArgument("Block SpGEMM must be called for matrices with the same block size")
    if A.values.dtype != B.values.dtype:
        raise B200SparseError(f"KokkosSparse::block_spgemm_symbolic: A and B must have the same scalar type "
                              f"(got {A.values.dtype} and {B.values.dtype})")
    _sfx(A.values)
    m, n, k = A.numRows(), B.numRows(), B.numCols()
    dev = A.row_map.device
    row_mapC = torch.empty(m + 1, dtype=torch.int32, device=dev)
    spgemm_symbolic_views(kh, m, n, k, A.row_map, A.entries, transposeA, B.row_map, B.entries, transposeB, row_mapC)
    c_nnz = kh.get_spgemm_handle().get_c_nnz()
    entriesC = torch.empty(c_nnz, dtype=torch.int32, device=dev)
    valuesC = torch.empty(c_nnz * bs * bs, dtype=A.values.dtype, device=dev)
    return BsrMatrix(row_mapC, entriesC, valuesC, k, bs)


def block_spgemm_numeric(kh, A, transposeA, B, transposeB, Cm):
    """KokkosSparse::block_spgemm_numeric (sparse/src/KokkosSparse_spgemm.hpp:145-156): fills C's sorted block columns and
    values on the structure block_spgemm_symbolic produced with the same handle.  Re-runnable with new values."""
    if transposeA or transposeB:
        raise B200SparseError("KokkosSparse::spgemm_numeric: transposing A or B is not supported")
    bs = A.blockDim()
    if bs != B.blockDim() or bs != Cm.blockDim():
        raise B200SparseInvalidArgument("Block SpGEMM must be called for matrices with the same block size")
    spgemm_numeric_views(kh, A.numRows(), B.numRows(), B.numCols(), A.row_map, A.entries, A.values, transposeA, B.row_map,
                         B.entries, B.values, transposeB, Cm.row_map, Cm.entries, Cm.values, block_dim=bs)
    return Cm


def spgemm(A, Amode, B, Bmode):
    """No-reuse interface (sparse/src/KokkosSparse_spgemm.hpp:170-218)."""
    kh = KokkosKernelsHandle()
    kh.create_spgemm_handle()
    Cm = spgemm_symbolic(kh, A, Amode, B, Bmode)
    spgemm_numeric(kh, A, Amode, B, Bmode, Cm)
    kh.destroy_spgemm_handle()
    return Cm


# --------------------------------------------------------------------------- CrsMatrix utilities
def _sfx(t):
    if t.dtype == torch.float64:
        return "f64"
    if t.dtype == torch.float32:
        return "f32"
    raise B200SparseError("b200sparse: only double and float are instantiated")


def sort_crs_matrix(A_or_rowmap, entries=None, values=None):
    """sort_crs_matrix(A) / sort_crs_matrix(rowmap, entries, values): every row sorted by column,
    values permuted along, in place (SortCrs.hpp:43-146).  Stable, like the reference's host path."""
    if entries is None:
        rowmap, entries, values = A_or_rowmap.row_map, A_or_rowmap.entries, A_or_rowmap.values
    else:
        rowmap = A_or_rowmap
    if entries.numel() <= 1:  # :62-67
        return
    m = max(rowmap.numel() - 1, 0)
    fn = getattr(_lib.sparse(), f"b200sp_sort_crs_{_sfx(values)}_i32")
    check(fn(_stream(), m, _idx(rowmap), _idx(entries), _ptr(values)))


def sort_crs_graph(rowmap, entries):
    """SortCrs.hpp:209-300."""
    if entries.numel() <= 1:
        return
    check(_lib.sparse().b200sp_sort_crs_graph_i32(_stream(), max(rowmap.numel() - 1, 0), _idx(rowmap), _idx(entries)))


def sort_and_merge_matrix(A):
    """Returns the sorted, merged matrix; A itself is sorted in place on the way, and returned as is
    when it has no duplicate entries (SortCrs.hpp:303-400)."""
    m = A.numRows()
    dev = A.row_map.device
    if m == 0:
        return CrsMatrix(torch.zeros(A.row_map.numel(), dtype=torch.int32, device=dev), A.entries[:0], A.values[:0], A.numCols())
    sfx = _sfx(A.values)
    rowmap_out = torch.empty(m + 1, dtype=torch.int32, device=dev)
    merged = C.c_int64(0)
    check(getattr(_lib.sparse(), f"b200sp_sort_and_merge_count_{sfx}_i32")(
        _stream(), m, _idx(A.row_map), _idx(A.entries), _ptr(A.values), C.c_void_p(rowmap_out.data_ptr()), C.byref(merged)))
    if merged.value == A.nnz():
        return A
    entries_out = torch.empty(merged.value, dtype=torch.int32, device=dev)
    values_out = torch.empty(merged.value, dtype=A.values.dtype, device=dev)
    check(getattr(_lib.sparse(), f"b200sp_sort_and_merge_fill_{sfx}_i32")(
        _stream(), m, _idx(A.row_map), _idx(A.entries), _ptr(A.values), _idx(rowmap_out), _idx(entries_out), _ptr(values_out)))
    return CrsMatrix(rowmap_out, entries_out, values_out, A.numCols())


def sort_and_merge_graph(rowmap, entries):
    """Returns (rowmap_out, entries_out); the input is sorted in place (SortCrs.hpp:426-537)."""
    m = max(rowmap.numel() - 1, 0)
    dev = rowmap.device
    if m == 0:
        return torch.zeros(rowmap.numel(), dtype=torch.int32, device=dev), entries[:0]
    rowmap_out = torch.empty(m + 1, dtype=torch.int32, device=dev)
    merged = C.c_int64(0)
    lib = _lib.sparse()
    check(lib.b200sp_sort_and_merge_count_f32_i32(_stream(), m, _idx(rowmap), _idx(entries), C.c_void_p(0),
                                                  C.c_void_p(rowmap_out.data_ptr()), C.byref(merged)))
    if merged.value == entries.numel():
        return rowmap, entries
    entries_out = torch.empty(merged.value, dtype=torch.int32, device=dev)
    check(lib.b200sp_sort_and_merge_fill_f32_i32(_stream(), m, _idx(rowmap), _idx(entries), C.c_void_p(0), _idx(rowmap_out),
                                                 _idx(entries_out), C.c_void_p(0)))
    return rowmap_out, entries_out


def transpose_matrix(A):
    """KokkosSparse::Impl::transpose_matrix(A) (sparse/src/KokkosSparse_Utils.hpp:380-398); rows of the
    result list their entries in (row of A, position) order."""
    m, n = A.numRows(), A.numCols()
    dev = A.row_map.device
    t_rowmap = torch.empty(n + 1, dtype=torch.int32, device=dev)
    t_entries = torch.empty(A.nnz(), dtype=torch.int32, device=dev)
    t_values = torch.empty(A.nnz(), dtype=A.values.dtype, device=dev)
    check(getattr(_lib.sparse(), f"b200sp_transpose_{_sfx(A.values)}_i32")(
        _stream(), m, n, _idx(A.row_map), _idx(A.entries), _ptr(A.values), C.c_void_p(t_rowmap.data_ptr()), _idx(t_entries),
        _ptr(t_values)))
    return CrsMatrix(t_rowmap, t_entries, t_values, m)


def spadd_symbolic_views(kh, m, n, a_rowmap, a_entries, b_rowmap, b_entries, c_rowmap):
    """View-level spadd_symbolic (KokkosSparse_spadd.hpp:29-93): c_rowmap is allocated by the caller
    (not initialised) and fully written; nnz(C) is left in the handle."""
    ah = kh.get_spadd_handle()
    if ah is None:
        raise B200SparseInvalidArgument("spadd_symbolic: create_spadd_handle() was not called")
    c_nnz = C.c_int64(0)
    check(_lib.sparse().b200sp_spadd_symbolic_i32(ah._plan, _stream(), m, n, _idx(a_rowmap), _idx(a_entries), _idx(b_rowmap),
                                                  _idx(b_entries), _idx(c_rowmap), C.byref(c_nnz)))
    ah._c_nnz = c_nnz.value
    ah._symbolic, ah._numeric = True, False


def spadd_numeric_views(kh, m, n, a_rowmap, a_entries, a_values, alpha, b_rowmap, b_entries, b_values, beta, c_rowmap, c_entries,
                        c_values):
    ah = kh.get_spadd_handle()
    if ah is None or not ah.is_symbolic_called():
        raise B200SparseError("spadd_numeric: call spadd_symbolic first")
    fn = getattr(_lib.sparse(), f"b200sp_spadd_numeric_{_sfx(c_values)}_i32")
    check(fn(ah._plan, _stream(), m, n, _idx(a_rowmap), _idx(a_entries), _ptr(a_values), alpha, _idx(b_rowmap), _idx(b_entries),
             _ptr(b_values), beta, _idx(c_rowmap), _idx(c_entries), _ptr(c_values)))
    ah._numeric = True


def spadd_symbolic(kh, A, B):
    """Matrix-level spadd_symbolic (KokkosSparse_spadd.hpp:233-271): returns C with its row map filled,
    entries / values allocated from get_c_nnz(); C has A's dimensions even when trailing rows or
    columns are empty (test_spadd_known_columns)."""
    if A.numRows() != B.numRows() or A.numCols() != B.numCols():
        raise B200SparseError("KokkosSparse::spadd_symbolic: A and B must have the same dimensions")
    m, n = A.numRows(), A.numCols()
    dev = A.row_map.device
    c_rowmap = torch.empty(m + 1, dtype=torch.int32, device=dev)
    spadd_symbolic_views(kh, m, n, A.row_map, A.entries, B.row_map, B.entries, c_rowmap)
    c_nnz = kh.get_spadd_handle().get_c_nnz()
    return CrsMatrix(c_rowmap, torch.empty(c_nnz, dtype=torch.int32, device=dev),
                     torch.empty(c_nnz, dtype=A.values.dtype, device=dev), n)


def spadd_numeric(kh, alpha, A, beta, B, Cm):
    spadd_numeric_views(kh, A.numRows(), A.numCols(), A.row_map, A.entries, A.values, alpha, B.row_map, B.entries, B.values, beta,
                        Cm.row_map, Cm.entries, Cm.values)
    return Cm


# --------------------------------------------------------------------------- matrix files
def read_kokkos_crst_matrix(filename, dtype=torch.float64, device=None):
    """KokkosSparse::Impl::read_kokkos_crst_matrix (sparse/src/KokkosSparse_IOUtils.hpp:1237-1290): .mtx / .mm
    or .bin -> CrsMatrix (on `device`; host tensors when device is None)."""
    import numpy as np

    lib = _lib.sparse()
    m, n, nnz = C.c_int(0), C.c_int(0), C.c_int64(0)
    rp, ci, v = C.c_void_p(0), C.c_void_p(0), C.c_void_p(0)
    f64 = dtype == torch.float64
    if not f64 and dtype != torch.float32:
        raise B200SparseError("b200sparse: only double and float are instantiated")
    fn = lib.b200sp_read_crs_f64 if f64 else lib.b200sp_read_crs_f32
    check(fn(str(filename).encode(), C.byref(m), C.byref(n), C.byref(nnz), C.byref(rp), C.byref(ci), C.byref(v)))
    try:
        def take(ptr, count, ctype, npt):
            if count == 0:
                return torch.zeros(0, dtype=torch.from_numpy(np.zeros(0, npt)).dtype)
            arr = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ctype)), shape=(count,)).copy()
            return torch.from_numpy(arr)

        row_map = take(rp, m.value + 1, C.c_int, np.int32)
        entries = take(ci, nnz.value, C.c_int, np.int32)
        values = take(v, nnz.value, C.c_double if f64 else C.c_float, np.float64 if f64 else np.float32)
    finally:
        for q in (rp, ci, v):
            lib.b200sp_host_free(q)
    if device is not None:
        row_map, entries, values = row_map.to(device), entries.to(device), values.to(device)
    return CrsMatrix(row_map, entries, values, n.value)


def write_kokkos_crst_matrix(A, filename):
    """write_kokkos_crst_matrix (IOUtils.hpp:740-782): .mtx / .mm or .bin (square only)."""
    rp, ci, v = A.row_map.cpu().contiguous(), A.entries.cpu().contiguous(), A.values.cpu().contiguous()
    fn = getattr(_lib.sparse(), f"b200sp_write_crs_{_sfx(v)}_i32".replace("_i32", ""))
    check(fn(str(filename).encode(), A.numRows(), A.numCols(), A.nnz(), C.c_void_p(rp.data_ptr()), C.c_void_p(ci.data_ptr()),
             C.c_void_p(v.data_ptr())))
