"""kokkos-kernels_b200: H100-native (sm_90a) drop-in for Kokkos Kernels' sparse
hot path -- KokkosSparse::spmv on CrsMatrix (rank-1, rank-2) and
spgemm_symbolic / spgemm_numeric.  See DESIGN.md and include/b200sparse.h."""
from . import _lib, build  # noqa: F401
from ._lib import B200SparseError, B200SparseInvalidArgument  # noqa: F401

__all__ = ["_lib", "build", "sparse", "matgen"]


def __getattr__(name):
    # sparse needs torch; matgen needs numpy -- import lazily
    if name in ("sparse", "matgen"):
        import importlib

        return importlib.import_module(f"{__name__}.{name}")
    raise AttributeError(name)
