"""Sparse triangular solve (sptrsv.cu: level sets) and the classic (sptrsv) form of the two-stage Gauss-Seidel through the Python
mirror -- SPTRSVHandle / sptrsv_symbolic / sptrsv_solve (sparse/src/KokkosSparse_sptrsv.hpp) and create_gs_handle(GS_TWOSTAGE) +
set_gs_twostage(False, n) (sparse/impl/KokkosSparse_twostage_gauss_seidel_impl.hpp:880-925) -- against the oracle.  The triangular
solve computes every row as the oracle's serial substitution does: bit-exact.  Runs under the CPU emulation as well
(tests/test_emulated_sptrsv.py)."""
import os

import numpy as np
import pytest
import torch

import exact_ref as R
from test_oracle_gs2 import dd_matrix
from test_oracle_sptrsv import REFERENCE_FIXTURES, fixture_crs, triangle

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("lower", [True, False])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_sptrsv_bit_exact(cuda, oracle, lower, dtype):
    from kokkos_kernels_b200 import sparse as sp

    n = 4000
    rp, ci, v = dd_matrix(n, 21)
    T = triangle(rp, ci, v, lower)
    trp, tci, tv = T.indptr.astype(np.int32), T.indices.astype(np.int32), T.data.astype(dtype)
    # unsorted rows: the diagonal anywhere in its row, the sum in storage order
    rng = np.random.default_rng(5)
    for i in range(n):
        perm = rng.permutation(trp[i + 1] - trp[i]) + trp[i]
        tci[trp[i]:trp[i + 1]], tv[trp[i]:trp[i + 1]] = tci[perm], tv[perm]
    b = rng.uniform(-1, 1, n).astype(dtype)
    exp = oracle.sptrsv(trp, tci, tv, b, lower)
    t = lambda a: torch.from_numpy(a).to(cuda)
    h = sp.SPTRSVHandle(n, lower)
    rpd, cid, vd = t(trp), t(tci), t(tv)
    with pytest.raises(sp.B200SparseError):
        sp.sptrsv_solve(h, rpd, cid, vd, t(b), t(np.zeros(n, dtype)))  # solve before symbolic
    sp.sptrsv_symbolic(h, rpd, cid)
    assert 1 <= h.get_num_levels() <= n
    for _ in range(2):  # the handle is reusable
        xd = t(np.full(n, np.nan, dtype))
        sp.sptrsv_solve(h, rpd, cid, vd, t(b), xd)
        torch.cuda.synchronize()
        assert np.array_equal(xd.cpu().numpy(), exp)
    # a matrix with entries on the wrong side is refused by symbolic
    h2 = sp.SPTRSVHandle(n, lower)
    with pytest.raises(sp.B200SparseError):
        sp.sptrsv_symbolic(h2, t(rp), t(ci))


@pytest.mark.parametrize("name", sorted(REFERENCE_FIXTURES))
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_reference_fixtures(cuda, name, dtype):
    """the reference's own level-scheduling fixtures and check (sparse/unit_test/Test_Sparse_sptrsv.hpp:64-118, 140-157, 212-225):
    rhs = A * ones, the solution is ones and sums to nrows exactly"""
    from kokkos_kernels_b200 import sparse as sp

    lower, dense = REFERENCE_FIXTURES[name]
    rp, ci, v, rhs = fixture_crs(dense, dtype)
    n = len(dense)
    t = lambda a: torch.from_numpy(a).to(cuda)
    rpd, cid = t(rp), t(ci)
    h = sp.SPTRSVHandle(n, lower)
    sp.sptrsv_symbolic(h, rpd, cid)
    xd = t(np.zeros(n, dtype))
    sp.sptrsv_solve(h, rpd, cid, t(v), t(rhs), xd)
    torch.cuda.synchronize()
    x = xd.cpu().numpy()
    assert np.array_equal(x, np.ones(n, dtype)) and x.sum() == n


def test_sptrsv_chain_and_diagonal_only(cuda, oracle):
    """the two extremes of the level structure: a bidiagonal matrix (n levels) and a diagonal one (1 level); n = 0"""
    from kokkos_kernels_b200 import sparse as sp

    n = 300
    t = lambda a: torch.from_numpy(a).to(cuda)
    rp = np.concatenate([[0], np.cumsum([1] + [2] * (n - 1))]).astype(np.int32)
    ci = np.concatenate([[0]] + [[i - 1, i] for i in range(1, n)]).astype(np.int32)
    v = np.random.default_rng(1).uniform(1, 2, len(ci))
    b = np.random.default_rng(2).uniform(-1, 1, n)
    h = sp.SPTRSVHandle(n, True)
    rpt, cit = t(rp), t(ci)  # (the handle is tied to these arrays, like the reference's)
    sp.sptrsv_symbolic(h, rpt, cit)
    assert h.get_num_levels() == n
    xd = t(np.zeros(n))
    sp.sptrsv_solve(h, rpt, cit, t(v), t(b), xd)
    torch.cuda.synchronize()
    assert np.array_equal(xd.cpu().numpy(), oracle.sptrsv(rp, ci, v, b, True))
    rpd, cid = t(np.arange(n + 1, dtype=np.int32)), t(np.arange(n, dtype=np.int32))
    for lower in (True, False):
        h = sp.SPTRSVHandle(n, lower)
        sp.sptrsv_symbolic(h, rpd, cid)
        assert h.get_num_levels() == 1
        xd = t(np.zeros(n))
        sp.sptrsv_solve(h, rpd, cid, t(v[:n]), t(b), xd)
        torch.cuda.synchronize()
        assert np.array_equal(xd.cpu().numpy(), b / v[:n])
    h0 = sp.SPTRSVHandle(0, True)
    sp.sptrsv_symbolic(h0, t(np.zeros(1, np.int32)), t(np.zeros(0, np.int32)))
    assert h0.get_num_levels() == 0


def test_sptrsv_mixed_level_sizes(cuda, oracle, monkeypatch):
    """levels of more than 512 rows (one launch each) next to runs of small ones (one single-CTA launch per run, sptrsv.cu:
    tr_solve_chain_kernel) and a lone small level between two large ones; the same with the chaining switched off"""
    from kokkos_kernels_b200 import sparse as sp

    rng = np.random.default_rng(11)
    rows = []  # per row: list of dependency columns (all smaller than the row)
    def block(count, deps_of):
        base = len(rows)
        for q in range(count):
            rows.append(deps_of(base, q))
        return base
    block(2000, lambda base, q: [])                                  # level 0: large
    c1 = block(40, lambda base, q: [base + q - 1] if q else [5])     # 40 levels of one row
    last1 = c1 + 39
    block(1500, lambda base, q: [last1, int(rng.integers(0, 2000))])  # one large level
    big2 = len(rows) - 1
    block(3, lambda base, q: [big2])                                 # a lone small level (3 rows)
    lone = len(rows) - 1
    block(900, lambda base, q: [lone, big2 - q])                     # large again
    top = len(rows) - 1
    block(200, lambda base, q: [base + q - 1, int(rng.integers(0, base))] if q else [top])  # 200 small levels at the end
    n = len(rows)
    rp = np.zeros(n + 1, np.int32)
    ci, v = [], []
    for i, deps in enumerate(rows):
        cols = sorted(set(deps)) + [i]
        ci += cols
        v += list(rng.uniform(-0.4, 0.4, len(cols) - 1)) + [rng.uniform(1.5, 2.5)]
        rp[i + 1] = len(ci)
    ci, v = np.array(ci, np.int32), np.array(v)
    b = rng.uniform(-1, 1, n)
    exp = oracle.sptrsv(rp, ci, v, b, True)
    t = lambda a: torch.from_numpy(a).to(cuda)
    rpd, cid, vd, bd = t(rp), t(ci), t(v), t(b)
    for chain in ("1", "0"):
        monkeypatch.setenv("B200SP_SPTRSV_CHAIN", chain)
        h = sp.SPTRSVHandle(n, True)
        sp.sptrsv_symbolic(h, rpd, cid)
        assert h.get_num_levels() == 1 + 40 + 1 + 1 + 1 + 200
        # chained: large, run of 40, large, lone small, large, run of 200
        assert h.get_num_launches() == (6 if chain == "1" else h.get_num_levels())
        xd = t(np.full(n, np.nan))
        sp.sptrsv_solve(h, rpd, cid, vd, bd, xd)
        torch.cuda.synchronize()
        assert np.array_equal(xd.cpu().numpy(), exp)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("compact", [False, True])
def test_classic_two_stage_gauss_seidel(cuda, oracle, dtype, compact):
    from kokkos_kernels_b200 import sparse as sp

    # (under the CPU emulation every lane is a fiber and every shuffle a barrier between fibers: a smaller matrix there)
    n, ghosts = (6000, 80) if os.environ.get("B200SP_TEST_EMULATED") != "1" else (900, 30)
    rp, ci, v = dd_matrix(n, 13, extra_cols=ghosts)
    v = v.astype(dtype)
    ncols = n + ghosts
    rng = np.random.default_rng(4)
    b = rng.uniform(-1, 1, n).astype(dtype)
    x0 = rng.uniform(-1, 1, ncols).astype(dtype)
    diag = np.array([v[k] for i in range(n) for k in range(rp[i], rp[i + 1]) if ci[k] == i], dtype=np.float64)
    dinv = (1.0 / (diag * rng.uniform(1.0, 1.1, n))).astype(dtype)  # a caller-supplied inverse diagonal (close to the matrix' own)
    t = lambda a: torch.from_numpy(a).to(cuda)
    rpd, cid, vd, bd = t(rp), t(ci), t(v), t(b)
    tol = 1e-13 if dtype == np.float64 else 1e-5
    applies = (sp.symmetric_gauss_seidel_apply, sp.forward_sweep_gauss_seidel_apply, sp.backward_sweep_gauss_seidel_apply)
    if os.environ.get("B200SP_TEST_EMULATED") == "1":
        applies = applies[:1]  # the symmetric sweep runs both triangular solves
    for given in (None, dinv):
        kh = sp.KokkosKernelsHandle()
        kh.create_gs_handle(sp.GS_TWOSTAGE)
        kh.set_gs_twostage(False, n)
        kh.set_gs_twostage_compact_form(compact)
        kh.set_gs_set_num_outer_sweeps(2)
        sp.gauss_seidel_symbolic(kh, n, ncols, rpd, cid, False)
        if given is None:
            sp.gauss_seidel_numeric(kh, n, ncols, rpd, cid, vd, False)
        else:
            sp.gauss_seidel_numeric(kh, n, ncols, rpd, cid, vd, False, given_inverse_diagonal=t(given))
        for direction, fn in enumerate(applies):
            for init_zero, num_iter in ((False, 1), (True, 3)):
                xd = t(x0)
                fn(kh, n, ncols, rpd, cid, vd, xd, bd, init_zero, True, 1.0, num_iter)
                torch.cuda.synchronize()
                x = xd.cpu().numpy()
                xo = x0.copy()
                oracle.gs2_classic_apply(rp, ci, v, ncols, xo, b, init_zero, num_iter, direction, compact=compact, outer_sweeps=2,
                                         inverse_diagonal=given)
                err = np.max(np.abs(x.astype(np.float64) - xo.astype(np.float64)))
                assert err <= tol * 20 * max(1.0, np.max(np.abs(xo))), (given is not None, direction, init_zero, num_iter, err)
                ex, bnd = R.gs2_ref(rp, ci, v, ncols, x0, b, init_zero, 1.0, num_iter, direction, compact, 0, 2, 1.0, False, given)
                R.assert_within(x, ex, bnd, str((given is not None, direction, init_zero, num_iter)))
        # omega != 1 is refused, as the reference's apply throws (twostage_gauss_seidel_impl.hpp:886-893)
        with pytest.raises(sp.B200SparseError):
            sp.forward_sweep_gauss_seidel_apply(kh, n, ncols, rpd, cid, vd, t(x0), bd, False, True, 0.9, 1)
        kh.destroy_gs_handle()
