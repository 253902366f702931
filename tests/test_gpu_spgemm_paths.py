"""Every SpGEMM and spgemm_jacobi kernel path (csrc/spgemm.cu, csrc/spgemm_esc.cuh) on the GPU, on the cases of
spgemm_path_cases.py, in fp64 and fp32: the handle's path witness (SPGEMMHandle.paths()) equals the rows each case was
built for and is nonzero on every path the case targets; row_map and entries equal the exact structure (and the oracle's
where k is small); every value is within the per-entry rounding bound of the exact product (tests/exact_ref.py).  Each
case runs through sp.spgemm, through symbolic + numeric on one handle, through a second numeric with new values on the
same handle, and -- for the first cases -- through the 64-bit-offset entry points with a window limit that puts rows of
different paths in different windows."""
import numpy as np
import pytest
import torch

import exact_ref as R
import spgemm_path_cases as P
from spgemm_path_cases import check_addressing, check_paths, new_values

pytestmark = pytest.mark.gpu

DTYPES = [np.float64, np.float32]
SPGEMM = [c["name"] for c in P.spgemm_cases(np.float64)]
JACOBI = [c["name"] for c in P.jacobi_cases(np.float64)]


def dev(cuda, M, ncols, wide=False):
    from kokkos_kernels_b200 import sparse as sp

    rp = M[0].astype(np.int64) if wide else M[0]
    return sp.CrsMatrix(torch.from_numpy(rp).to(cuda), torch.from_numpy(M[1]).to(cuda), torch.from_numpy(M[2]).to(cuda), ncols)


def check_result(C, rp, ci, v, bound, what):
    torch.cuda.synchronize()
    assert np.array_equal(C.row_map.cpu().numpy().astype(np.int64), rp.astype(np.int64)), f"{what}: row_map"
    assert np.array_equal(C.entries.cpu().numpy(), ci), f"{what}: entries"
    R.assert_within(C.values.cpu().numpy(), v, bound, what)


def get_case(cases, name):
    return next(c for c in cases if c["name"] == name)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", SPGEMM)
def test_spgemm_paths(cuda, oracle, name, dtype):
    from kokkos_kernels_b200 import sparse as sp

    case = get_case(P.spgemm_cases(dtype), name)
    A, B, n, k = case["A"], case["B"], case["n"], case["k"]
    rp, ci, v, bound = R.spgemm_ref(A, B)
    if case["oracle"]:
        exp = oracle.spgemm(*A, *B, k)
        assert np.array_equal(exp[0], rp) and np.array_equal(exp[1], ci), f"{name}: exact structure != oracle's"
    check_addressing(case, rp, ci)
    what = f"{name} {dtype.__name__}"
    Ad, Bd = dev(cuda, A, n), dev(cuda, B, k)
    check_result(sp.spgemm(Ad, False, Bd, False), rp, ci, v, bound, what + " spgemm")
    kh = sp.KokkosKernelsHandle()
    kh.create_spgemm_handle()
    C = sp.spgemm_symbolic(kh, Ad, False, Bd, False)
    sp.spgemm_numeric(kh, Ad, False, Bd, False, C)
    check_result(C, rp, ci, v, bound, what + " symbolic+numeric")
    paths = kh.get_spgemm_handle().paths()
    check_paths(paths, case, rp, False, what)
    print(f"\n{what}: {dict((p, c) for p, c in paths.items() if c)}", end="")
    # reuse: new values, numeric only
    A2, B2 = new_values(case, dtype, 5)
    rp2, ci2, v2, bound2 = R.spgemm_ref(A2, B2)
    sp.spgemm_numeric(kh, dev(cuda, A2, n), False, dev(cuda, B2, k), False, C)
    check_result(C, rp2, ci2, v2, bound2, what + " reuse")
    check_paths(kh.get_spgemm_handle().paths(), case, rp, False, what + " reuse")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", JACOBI)
def test_jacobi_paths(cuda, oracle, name, dtype):
    from kokkos_kernels_b200 import sparse as sp

    case = get_case(P.jacobi_cases(dtype), name)
    A, B, n = case["A"], case["B"], case["n"]
    omega, dinv = P.jacobi_operands(case, dtype)
    rp, ci, v, bound = R.jacobi_ref(A, B, omega, dinv)
    if case["oracle"] and not case["no_diag"]:
        exp = oracle.spgemm_jacobi(*A, *B, case["k"], dtype(omega), dinv)
        assert np.array_equal(exp[0], rp) and np.array_equal(exp[1], ci), f"{name}: exact structure != oracle's"
    what = f"{name} {dtype.__name__} jacobi"
    Ad, Bd = dev(cuda, A, n), dev(cuda, B, n)
    kh = sp.KokkosKernelsHandle()
    kh.create_spgemm_handle()
    C = sp.spgemm_symbolic(kh, Ad, False, Bd, False)
    sp.spgemm_jacobi(kh, Ad, False, Bd, False, C, omega, torch.from_numpy(dinv).to(cuda))
    check_result(C, rp, ci, v, bound, what)
    paths = kh.get_spgemm_handle().paths()
    check_paths(paths, case, rp, True, what)
    print(f"\n{what}: {dict((p, c) for p, c in paths.items() if c)}", end="")


@pytest.mark.parametrize("dtype", DTYPES)
def test_i64_windows(cuda, dtype):
    """The _i64 entry points with a window limit at the longest row: rows of different paths in different windows."""
    from kokkos_kernels_b200 import sparse as sp

    for case in P.spgemm_cases(dtype)[:5]:
        A, B, n, k = case["A"], case["B"], case["n"], case["k"]
        rp, ci, v, bound = R.spgemm_ref(A, B)
        limit = max(int(R.product_rows(A, B).max()), int(np.diff(A[0]).max()), 8)
        Ad, Bd = dev(cuda, A, n, True), dev(cuda, B, k, True)
        kh = sp.KokkosKernelsHandle()
        kh.create_spgemm_handle()
        kh.get_spgemm_handle().set_window(limit)
        C = sp.spgemm_symbolic(kh, Ad, False, Bd, False)
        assert kh.get_spgemm_handle().windows() > 1, case["name"]
        sp.spgemm_numeric(kh, Ad, False, Bd, False, C)
        what = f"{case['name']} {dtype.__name__} i64"
        check_result(C, rp, ci, v, bound, what)
        check_paths(kh.get_spgemm_handle().paths(), case, rp, False, what)
