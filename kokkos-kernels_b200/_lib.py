"""ctypes binding of libb200sparse.so (the C ABI in include/b200sparse.h) and
libb200matgen.so.  There is NO fallback: if the CUDA library is missing the
import fails loudly."""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIBDIR = os.path.join(HERE, "lib")
SPARSE_SO = os.path.join(LIBDIR, "libb200sparse.so")
MATGEN_SO = os.path.join(LIBDIR, "libb200matgen.so")

i32, i64, f32, f64, vp, cp = C.c_int, C.c_int64, C.c_float, C.c_double, C.c_void_p, C.c_char
u64 = C.c_uint64

# name -> (restype, argtypes); must list every symbol include/b200sparse.h declares
SPARSE_API = {
    "b200sp_last_error_string": (C.c_char_p, []),
    "b200sp_version": (i32, []),
    "b200sp_device_ok": (i32, []),
    "b200sp_spmv_plan_create": (i32, [C.POINTER(vp), i32]),
    "b200sp_spmv_plan_destroy": (i32, [vp, vp]),
    "b200sp_spmv_plan_set_option": (i32, [vp, i32, i32]),
    "b200sp_spmv_f64_i32": (i32, [vp, vp, cp, i32, i32, i64, f64, vp, vp, vp, vp, f64, vp]),
    "b200sp_spmv_f32_i32": (i32, [vp, vp, cp, i32, i32, i64, f32, vp, vp, vp, vp, f32, vp]),
    "b200sp_gs2_plan_create": (i32, [C.POINTER(vp)]),
    "b200sp_gs2_plan_destroy": (i32, [vp, vp]),
    "b200sp_gs2_plan_set": (i32, [vp, i32, f64]),
    "b200sp_gs2_symbolic_i32": (i32, [vp, vp, i32, i32, vp, vp]),
    "b200sp_gs2_numeric_f64_i32": (i32, [vp, vp, i32, i32, vp, vp, vp, vp]),
    "b200sp_gs2_numeric_f32_i32": (i32, [vp, vp, i32, i32, vp, vp, vp, vp]),
    "b200sp_gs2_apply_f64_i32": (i32, [vp, vp, i32, i32, vp, vp, vp, vp, i64, vp, i64, i32, i32, f64, i32, i32]),
    "b200sp_gs2_apply_f32_i32": (i32, [vp, vp, i32, i32, vp, vp, vp, vp, i64, vp, i64, i32, i32, f32, i32, i32]),
    "b200sp_sptrsv_plan_create": (i32, [C.POINTER(vp)]),
    "b200sp_sptrsv_plan_destroy": (i32, [vp, vp]),
    "b200sp_sptrsv_symbolic_i32": (i32, [vp, vp, i32, vp, vp, i32]),
    "b200sp_sptrsv_levels": (i32, [vp]),
    "b200sp_sptrsv_launches": (i32, [vp]),
    "b200sp_sptrsv_solve_f64_i32": (i32, [vp, vp, i32, vp, vp, vp, vp, vp]),
    "b200sp_sptrsv_solve_f32_i32": (i32, [vp, vp, i32, vp, vp, vp, vp, vp]),
    "b200sp_spmv_hostvec_flush": (i32, [vp, vp]),
    "b200sp_spmv64_plan_create": (i32, [C.POINTER(vp), i32]),
    "b200sp_spmv64_plan_destroy": (i32, [vp, vp]),
    "b200sp_spmv64_plan_set_window": (i32, [vp, i64]),
    "b200sp_spmv64_plan_windows": (i32, [vp]),
    "b200sp_spmv64_last_kernel": (C.c_char_p, [vp]),
    "b200sp_spmv_f64_i64": (i32, [vp, vp, cp, i64, i64, i64, f64, vp, vp, i32, vp, vp, f64, vp]),
    "b200sp_spmv_f32_i64": (i32, [vp, vp, cp, i64, i64, i64, f32, vp, vp, i32, vp, vp, f32, vp]),
    "b200sp_spmm_f64_i64": (i32, [vp, vp, cp, i64, i64, i64, i32, f64, vp, vp, i32, vp, vp, i64, i32, f64, vp, i64, i32]),
    "b200sp_spmm_f32_i64": (i32, [vp, vp, cp, i64, i64, i64, i32, f32, vp, vp, i32, vp, vp, i64, i32, f32, vp, i64, i32]),
    "b200sp_spmv_scatter_f64_i32": (i32, [vp, vp, i32, i32, i64, f64, vp, vp, vp, vp, vp, i32, C.POINTER(vp)]),
    "b200sp_spmv_forward_f64_i32": (i32, [vp, vp, i32, i32, i64, f64, vp, vp, vp, vp, vp, vp]),
    "b200sp_spmv_plan_invalidate": (i32, [vp, vp]),
    "b200sp_peer_push": (i32, [vp, vp, i64, i32, C.POINTER(vp)]),
    "b200sp_peer_push_async": (i32, [vp, C.POINTER(vp), i32, C.POINTER(vp), vp, i64]),
    "b200sp_peer_join": (i32, [vp, C.POINTER(vp), i32]),
    "b200sp_multicast_push": (i32, [vp, vp, vp, i64, i32]),
    "b200sp_peer_push_sm": (i32, [vp, vp, i64, i32, C.POINTER(vp), i32]),
    "b200sp_spmv_hostvec_f64_i32": (i32, [vp, vp, cp, i32, i32, i64, f64, vp, vp, vp, vp, f64, vp]),
    "b200sp_spmm_f64_i32": (i32, [vp, vp, cp, i32, i32, i64, i32, f64, vp, vp, vp, vp, i64, i32, f64, vp, i64, i32]),
    "b200sp_spmm_f32_i32": (i32, [vp, vp, cp, i32, i32, i64, i32, f32, vp, vp, vp, vp, i64, i32, f32, vp, i64, i32]),
    "b200sp_spmm_f16_i32": (i32, [vp, vp, cp, i32, i32, i64, i32, f32, vp, vp, vp, vp, i64, i32, f32, vp, i64, i32]),
    "b200sp_spgemm_plan_create": (i32, [C.POINTER(vp)]),
    "b200sp_spgemm_plan_destroy": (i32, [vp, vp]),
    "b200sp_spgemm_symbolic_i32": (i32, [vp, vp, i32, i32, i32, vp, vp, vp, vp, vp, C.POINTER(i64), C.POINTER(i32)]),
    "b200sp_spgemm_numeric_f64_i32": (i32, [vp, vp, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "b200sp_spgemm_numeric_f32_i32": (i32, [vp, vp, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "b200sp_spgemm_jacobi_f64_i32": (i32, [vp, vp, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, f64, vp]),
    "b200sp_spgemm_jacobi_f32_i32": (i32, [vp, vp, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, f32, vp]),
    "b200sp_spgemm_symbolic_i64": (i32, [vp, vp, i32, i32, i32, vp, vp, vp, vp, vp, C.POINTER(i64), C.POINTER(i32)]),
    "b200sp_spgemm_numeric_f64_i64": (i32, [vp, vp, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "b200sp_spgemm_numeric_f32_i64": (i32, [vp, vp, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "b200sp_spgemm_plan_set_window": (i32, [vp, i64]),
    "b200sp_spgemm_plan_windows": (i32, [vp]),
    "b200sp_spgemm_plan_paths": (i32, [vp, C.POINTER(i64), i32]),
    "b200sp_bspgemm_numeric_f64_i32": (i32, [vp, vp, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "b200sp_bspgemm_numeric_f32_i32": (i32, [vp, vp, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "b200sp_sort_crs_f64_i32": (i32, [vp, i32, vp, vp, vp]),
    "b200sp_sort_crs_f32_i32": (i32, [vp, i32, vp, vp, vp]),
    "b200sp_sort_crs_graph_i32": (i32, [vp, i32, vp, vp]),
    "b200sp_sort_and_merge_count_f64_i32": (i32, [vp, i32, vp, vp, vp, vp, C.POINTER(i64)]),
    "b200sp_sort_and_merge_count_f32_i32": (i32, [vp, i32, vp, vp, vp, vp, C.POINTER(i64)]),
    "b200sp_sort_and_merge_fill_f64_i32": (i32, [vp, i32, vp, vp, vp, vp, vp, vp]),
    "b200sp_sort_and_merge_fill_f32_i32": (i32, [vp, i32, vp, vp, vp, vp, vp, vp]),
    "b200sp_transpose_f64_i32": (i32, [vp, i32, i32, vp, vp, vp, vp, vp, vp]),
    "b200sp_transpose_f32_i32": (i32, [vp, i32, i32, vp, vp, vp, vp, vp, vp]),
    "b200sp_spadd_plan_create": (i32, [C.POINTER(vp), i32, i32]),
    "b200sp_spadd_plan_destroy": (i32, [vp, vp]),
    "b200sp_spadd_symbolic_i32": (i32, [vp, vp, i32, i32, vp, vp, vp, vp, vp, C.POINTER(i64)]),
    "b200sp_spadd_numeric_f64_i32": (i32, [vp, vp, i32, i32, vp, vp, vp, f64, vp, vp, vp, f64, vp, vp, vp]),
    "b200sp_spadd_numeric_f32_i32": (i32, [vp, vp, i32, i32, vp, vp, vp, f32, vp, vp, vp, f32, vp, vp, vp]),
    "b200sp_read_crs_f64": (i32, [C.c_char_p, C.POINTER(i32), C.POINTER(i32), C.POINTER(i64), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]),
    "b200sp_read_crs_f32": (i32, [C.c_char_p, C.POINTER(i32), C.POINTER(i32), C.POINTER(i64), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]),
    "b200sp_read_mtx_f64": (i32, [C.c_char_p, i32, i32, i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(i64), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]),
    "b200sp_read_mtx_f32": (i32, [C.c_char_p, i32, i32, i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(i64), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]),
    "b200sp_write_crs_f64": (i32, [C.c_char_p, i32, i32, i64, vp, vp, vp]),
    "b200sp_write_crs_f32": (i32, [C.c_char_p, i32, i32, i64, vp, vp, vp]),
    "b200sp_host_free": (None, [vp]),
    "b200sp_bsr_plan_create": (i32, [C.POINTER(vp)]),
    "b200sp_bsr_plan_destroy": (i32, [vp, vp]),
    "b200sp_bsr_spmv_f64_i32": (i32, [vp, vp, cp, i32, i32, i64, i32, f64, vp, vp, vp, vp, f64, vp]),
    "b200sp_bsr_spmv_f32_i32": (i32, [vp, vp, cp, i32, i32, i64, i32, f32, vp, vp, vp, vp, f32, vp]),
    "b200sp_bsr_spmm_f64_i32": (i32, [vp, vp, cp, i32, i32, i64, i32, i32, f64, vp, vp, vp, vp, i64, i32, f64, vp, i64, i32]),
    "b200sp_bsr_spmm_f32_i32": (i32, [vp, vp, cp, i32, i32, i64, i32, i32, f32, vp, vp, vp, vp, i64, i32, f32, vp, i64, i32]),
    "b200sp_bsr_last_kernel": (C.c_char_p, [vp]),
    "b200sp_bsr_plan_set_algorithm": (i32, [vp, i32]),
    "b200sp_gmres_f64_i32": (i32, [vp, vp, i32, i64, vp, vp, vp, vp, i64, vp, vp, vp, vp, vp, i32, f64, i32, i32, C.POINTER(i32), C.POINTER(f64), C.POINTER(i32)]),
    "b200sp_gmres_f32_i32": (i32, [vp, vp, i32, i64, vp, vp, vp, vp, i64, vp, vp, vp, vp, vp, i32, f32, i32, i32, C.POINTER(i32), C.POINTER(f32), C.POINTER(i32)]),
    "b200sp_gmres_bsr_f64_i32": (i32, [vp, vp, i32, i64, i32, vp, vp, vp, vp, i64, vp, vp, vp, vp, vp, i32, f64, i32, i32, C.POINTER(i32), C.POINTER(f64), C.POINTER(i32)]),
    "b200sp_gmres_bsr_f32_i32": (i32, [vp, vp, i32, i64, i32, vp, vp, vp, vp, i64, vp, vp, vp, vp, vp, i32, f32, i32, i32, C.POINTER(i32), C.POINTER(f32), C.POINTER(i32)]),
    "b200sp_gs_plan_create": (i32, [C.POINTER(vp)]),
    "b200sp_gs_plan_destroy": (i32, [vp, vp]),
    "b200sp_gs_symbolic_i32": (i32, [vp, vp, i32, vp, vp, i32]),
    "b200sp_gs_symbolic_nc_i32": (i32, [vp, vp, i32, i32, vp, vp, i32]),
    "b200sp_gs_numeric_f64_i32": (i32, [vp, vp, i32, vp, vp, vp]),
    "b200sp_gs_numeric_f32_i32": (i32, [vp, vp, i32, vp, vp, vp]),
    "b200sp_gs_apply_f64_i32": (i32, [vp, vp, i32, vp, vp, vp, vp, vp, i32, f64, i32, i32]),
    "b200sp_gs_apply_f32_i32": (i32, [vp, vp, i32, vp, vp, vp, vp, vp, i32, f32, i32, i32]),
    "b200sp_gs_copy_coloring": (i32, [vp, vp, vp, vp, vp]),
    "b200sp_gs_get_coloring": (i32, [vp, C.POINTER(i32), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]),
    "b200sp_gs_last_kernel": (C.c_char_p, [vp]),
    "b200sp_pcg_solve_f64_i32": (i32, [vp, vp, vp, i32, i64, vp, vp, vp, vp, vp, i32, f64, i32, C.POINTER(i32), C.POINTER(f64)]),
    "b200sp_pcg_solve_gs2_f64_i32": (i32, [vp, vp, vp, i32, i64, vp, vp, vp, vp, vp, i32, f64, i32, C.POINTER(i32), C.POINTER(f64)]),
    "b200sp_cg_solve_f64_i32": (i32, [vp, vp, i32, i64, vp, vp, vp, vp, vp, i32, f64, i32, C.POINTER(i32), C.POINTER(f64)]),
    "b200sp_launch_count": (i64, []),
    "b200sp_spmv_last_kernel": (C.c_char_p, [vp]),
    "b200sp_spmv_plan_tune": (i32, [vp, i32, i32, i32]),
}

MATGEN_API = {
    "b200gen_fill_f64": (None, [i64, vp, f64, f64, u64]),
    "b200gen_fill_f32": (None, [i64, vp, f32, f32, u64]),
    "b200gen_kk_rowptr": (i64, [i32, i32, i64, i32, vp]),
    "b200gen_kk_colidx": (None, [i32, i32, i64, i32, i32, vp, vp]),
    "b200gen_lap27_nnz": (i64, [i32, i32, i32, i32]),
    "b200gen_lap27_rows": (i64, [i32, i32, i32, i32, i64, i64, vp, vp, vp, f64, u64]),
    "b200gen_uniform": (None, [i32, i32, i32, u64, vp, vp]),
    "b200gen_rmat_build": (vp, [i32, i32, f64, f64, f64, u64, C.POINTER(i64)]),
    "b200gen_rmat_emit": (None, [vp, vp, vp]),
}


def _load(path, api, what):
    if not os.path.exists(path):
        raise ImportError(
            f"{what} not built: {path} is missing. Run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU or PyTorch fallback for the CUDA sparse kernels)."
        )
    lib = C.CDLL(path)
    for name, (res, args) in api.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export it
        fn.restype = res
        fn.argtypes = args
    return lib


_sparse = None
_matgen = None


def sparse():
    global _sparse
    if _sparse is None:
        _sparse = _load(SPARSE_SO, SPARSE_API, "libb200sparse")
    return _sparse


def matgen():
    global _matgen
    if _matgen is None:
        _matgen = _load(MATGEN_SO, MATGEN_API, "libb200matgen")
    return _matgen


class B200SparseError(RuntimeError):
    """std::runtime_error analogue (KokkosKernels::Impl::throw_runtime_exception)."""


class B200SparseInvalidArgument(ValueError):
    """std::invalid_argument analogue (handle misuse)."""


def check(rc):
    if rc == 0:
        return
    msg = sparse().b200sp_last_error_string().decode()
    if rc == 3:
        raise B200SparseInvalidArgument(msg)
    raise B200SparseError(f"b200sparse status {rc}: {msg}")
