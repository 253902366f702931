"""GPU parity of SpGEMM on 64-bit offsets (kokkos-kernels_b200/csrc/spgemm64.cu: Kokkos' (int, size_t) instantiation)
through the mirror (kokkos_kernels_b200.sparse.spgemm on CrsMatrix objects whose row maps are int64): with the window limit
lowered the product is cut into many 32-bit windows and must equal the 32-bit path bit for bit -- row map, entries and the
values of every row the expand / sort / compress kernels compute (rows beyond their capacity go to hash kernels that add
with atomics, compared within the oracle's tolerance).  Then a product past 2^31 entries, which the 32-bit entry refuses.
The same cases run on the CPU in tests/test_emulated_spgemm64.py."""
import numpy as np
import pytest
import torch

from spgemm_cases import cases
from test_emulated_spgemm64 import limits_for, row_products

pytestmark = pytest.mark.gpu
INT32_MAX = 2 ** 31 - 1
ESC_CAP = 8192  # rows with more products (or 2 nnz(A_i)) go to the hash kernels


def dev_matrix(sp, dev, rp, ci, v, ncols, rp_dtype):
    return sp.CrsMatrix(torch.from_numpy(rp.astype(rp_dtype)).to(dev), torch.from_numpy(ci).to(dev), torch.from_numpy(v).to(dev),
                        ncols)


def product(sp, A, B, window=None):
    kh = sp.KokkosKernelsHandle()
    kh.create_spgemm_handle()
    if window is not None:
        kh.get_spgemm_handle().set_window(window)
    Cm = sp.spgemm_symbolic(kh, A, False, B, False)
    sp.spgemm_numeric(kh, A, False, B, False, Cm)
    torch.cuda.synchronize()
    return kh, Cm


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_windows_equal_the_32_bit_path(cuda, oracle, dtype):
    from kokkos_kernels_b200 import sparse as sp

    for name, A, B, m, n, k in cases(dtype):
        A32, B32 = dev_matrix(sp, cuda, *A, n, np.int32), dev_matrix(sp, cuda, *B, k, np.int32)
        A64, B64 = dev_matrix(sp, cuda, *A, n, np.int64), dev_matrix(sp, cuda, *B, k, np.int64)
        ref = sp.spgemm(A32, False, B32, False)
        rp = ref.row_map.cpu().numpy()
        esc = np.maximum(row_products(A, B), 2 * np.diff(A[0])) <= ESC_CAP
        exact = np.repeat(esc, np.diff(rp))
        for limit in limits_for(A, B):
            kh, Cm = product(sp, A64, B64, limit)
            what = (name, limit)
            assert Cm.row_map.dtype == torch.int64 and kh.get_spgemm_handle().windows() >= 1, what
            assert torch.equal(Cm.row_map, ref.row_map.long()), what
            assert torch.equal(Cm.entries, ref.entries), what
            got, want = Cm.values.cpu().numpy(), ref.values.cpu().numpy()
            assert np.array_equal(got[exact].view(np.uint8), want[exact].view(np.uint8)), what
            tol = 1e-12 if dtype == np.float64 else 1e-5
            assert oracle.rel_mismatch(got.astype(np.float64), want.astype(np.float64), tol) == 0, what


def test_numeric_rerun_and_oracle(cuda, oracle):
    from kokkos_kernels_b200 import sparse as sp

    for name, A, B, m, n, k in cases(np.float64)[:4]:
        A64, B64 = dev_matrix(sp, cuda, *A, n, np.int64), dev_matrix(sp, cuda, *B, k, np.int64)
        limit = limits_for(A, B)[1]
        kh, Cm = product(sp, A64, B64, limit)
        assert kh.get_spgemm_handle().windows() > 1
        for scale in (1.0, -3.0):
            vA, vB = A[2] * scale, B[2] - scale
            A64.values.copy_(torch.from_numpy(vA))
            B64.values.copy_(torch.from_numpy(vB))
            Cm.values.fill_(float("nan"))
            sp.spgemm_numeric(kh, A64, False, B64, False, Cm)
            exp = oracle.spgemm(A[0], A[1], vA, B[0], B[1], vB, k)
            assert np.array_equal(Cm.row_map.cpu().numpy(), exp[0].astype(np.int64)), name
            assert np.array_equal(Cm.entries.cpu().numpy(), exp[1]), name
            assert oracle.rel_mismatch(Cm.values.cpu().numpy(), exp[2], 1e-7) == 0, name


def test_mirror_errors(cuda):
    from kokkos_kernels_b200 import sparse as sp

    name, A, B, m, n, k = cases(np.float64)[2]
    A64, A32 = dev_matrix(sp, cuda, *A, n, np.int64), dev_matrix(sp, cuda, *A, n, np.int32)
    kh = sp.KokkosKernelsHandle()
    kh.create_spgemm_handle()
    with pytest.raises(sp.B200SparseError, match="share one dtype"):
        sp.spgemm_symbolic(kh, A64, False, A32, False)
    A64e = sp.CrsMatrix(A64.row_map, A64.entries.long(), A64.values, n)
    with pytest.raises(sp.B200SparseError, match="64-bit ordinals"):
        sp.spgemm_symbolic(kh, A64e, False, A64e, False)
    Cm = sp.spgemm_symbolic(kh, A64, False, A64, False)
    dinv = torch.ones(m, dtype=torch.float64, device=cuda)
    with pytest.raises(sp.B200SparseError, match="jacobi: not provided on 64-bit offsets"):
        sp.spgemm_jacobi(kh, A64, False, A64, False, Cm, 1.0, dinv)
    # a handle whose symbolic had 64-bit offsets refuses the 32-bit numeric (C ABI state error)
    C32 = sp.CrsMatrix(Cm.row_map.int(), Cm.entries, Cm.values, n)
    with pytest.raises(sp.B200SparseInvalidArgument, match="64-bit"):
        sp.spgemm_numeric(kh, A32, False, A32, False, C32)


def test_product_past_2_31(cuda, oracle):
    """A = uniform(2.2M x 2.2M, 32 per row), C = A*A in fp64: nnz(C) ~ 2.25e9 > INT32_MAX, two windows.  All of C is checked
    bit for bit against the 32-bit path on two row slices of A, sampled row blocks against the oracle."""
    from kokkos_kernels_b200 import matgen, sparse as sp

    n = 2_200_000
    rp, ci = matgen.uniform(n, n, 32, 4)
    va = matgen.fill(len(ci), 1.0, 50.0, 4)
    A32 = dev_matrix(sp, cuda, rp, ci, va, n, np.int32)
    # the 32-bit entry refuses the product
    kh32 = sp.KokkosKernelsHandle()
    kh32.create_spgemm_handle()
    with pytest.raises(sp.B200SparseError, match="exceeds int32"):
        sp.spgemm_symbolic(kh32, A32, False, A32, False)
    del kh32
    A64 = sp.CrsMatrix(A32.row_map.long(), A32.entries, A32.values, n)
    kh, Cm = product(sp, A64, A64)
    sh = kh.get_spgemm_handle()
    c_nnz = sh.get_c_nnz()
    assert c_nnz > INT32_MAX and int(Cm.row_map[-1]) == c_nnz
    assert sh.windows() == 2
    del kh
    # every row through the 32-bit path on two slices of A's rows, each below 2^31 entries of C
    half = n // 2
    for r0, r1 in ((0, half), (half, n)):
        a0, a1 = int(rp[r0]), int(rp[r1])
        As = sp.CrsMatrix(A32.row_map[r0:r1 + 1] - a0, A32.entries[a0:a1], A32.values[a0:a1], n)
        Cs = sp.spgemm(As, False, A32, False)
        c0, c1 = int(Cm.row_map[r0]), int(Cm.row_map[r1])
        assert torch.equal(torch.diff(Cm.row_map[r0:r1 + 1]), torch.diff(Cs.row_map).long()), (r0, r1)
        assert torch.equal(Cm.entries[c0:c1], Cs.entries), (r0, r1)
        assert torch.equal(Cm.values[c0:c1].view(torch.int64), Cs.values.view(torch.int64)), (r0, r1)
        del Cs, As
        torch.cuda.empty_cache()
    # sampled row blocks against the oracle: the first rows, both sides of the window boundary, the last rows
    rpC = Cm.row_map.cpu().numpy()
    bound = int(np.searchsorted(np.cumsum(np.full(n, 1024, np.int64)), 2 ** 31 - 1 - 65536, "right"))
    for r0 in (0, max(0, bound - 600), n - 1000):
        r1 = min(n, r0 + 1000)
        a0, a1 = int(rp[r0]), int(rp[r1])
        exp = oracle.spgemm((rp[r0:r1 + 1] - a0).astype(np.int32), ci[a0:a1].copy(), va[a0:a1].copy(), rp, ci, va, n)
        c0, c1 = int(rpC[r0]), int(rpC[r1])
        assert np.array_equal(rpC[r0:r1 + 1] - c0, exp[0].astype(np.int64)), r0
        assert np.array_equal(Cm.entries[c0:c1].cpu().numpy(), exp[1]), r0
        assert oracle.rel_mismatch(Cm.values[c0:c1].cpu().numpy(), exp[2], 1e-7) == 0, r0
