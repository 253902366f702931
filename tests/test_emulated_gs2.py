"""Two-stage Gauss-Seidel kernels (gs2.cu) executed on the CPU (tools/emu) against the oracle's restatement of the reference's
TwostageGaussSeidel::apply (oracle/kk_oracle_gs2.c): classic and compact recurrences, 0 .. 3 inner sweeps, inner damping, outer
sweeps, the three directions, ghost columns, several right-hand sides, a caller-supplied inverse diagonal -- and the reference
unit test's acceptance (sparse/unit_test/Test_Sparse_gauss_seidel.hpp:236-241).  The only difference to the oracle is the
summation order inside the SpMVs, so the tolerance is a few ulps of the iterate."""
import numpy as np
import pytest

import emu_lib as E
import exact_ref as R
from test_oracle_gs2 import dd_matrix


@pytest.fixture(scope="module")
def emu():
    return E.lib()


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("compact", [False, True])
def test_oracle_parity(emu, oracle, dtype, compact):
    n, ghosts = 3000, 60
    rp, ci, v = dd_matrix(n, 11, extra_cols=ghosts)
    v = v.astype(dtype)
    ncols = n + ghosts
    rng = np.random.default_rng(4)
    b = rng.uniform(-1, 1, n).astype(dtype)
    x0 = rng.uniform(-1, 1, ncols).astype(dtype)
    tol = 1e-13 if dtype == np.float64 else 1e-5
    for inner, gamma, outer in ((1, 1.0, 1), (0, 1.0, 1), (0, 0.7, 1), (3, 1.0, 1), (2, 0.9, 3)):
        plan = E.Gs2Plan(compact=compact, inner=inner, outer=outer, gamma=gamma)
        assert plan.numeric(n, ncols, rp, ci, v) == 3  # numeric before symbolic: refused (B200SP_ERR_STATE)
        assert plan.symbolic(n, ncols, rp, ci) == 0
        assert plan.apply(n, ncols, rp, ci, v, x0.copy(), b, False, 1.0, 1, 0) == 3  # apply before numeric
        assert plan.numeric(n, ncols, rp, ci, v) == 0
        for direction in (0, 1, 2):
            for omega, init_zero, num_iter in ((1.0, False, 1), (0.9, False, 2), (0.9, True, 2)):
                x = x0.copy()
                assert plan.apply(n, ncols, rp, ci, v, x, b, init_zero, omega, num_iter, direction) == 0
                xo = x0.copy()
                oracle.gs2_apply(rp, ci, v, ncols, xo, b, init_zero, dtype(omega), num_iter, direction, compact=compact, inner_sweeps=inner,
                                 outer_sweeps=outer, gamma=dtype(gamma))
                if init_zero:
                    assert np.all(x[n:] == 0)
                else:
                    assert np.array_equal(x[n:], x0[n:])  # ghosts untouched
                err = np.max(np.abs(x.astype(np.float64) - xo.astype(np.float64)))
                assert err <= tol * 20 * max(1.0, np.max(np.abs(xo))), (inner, gamma, outer, direction, omega, init_zero, err)
                ex, bnd = R.gs2_ref(rp, ci, v, ncols, x0, b, init_zero, omega, num_iter, direction, compact, inner, outer, gamma)
                R.assert_within(x, ex, bnd, str((inner, gamma, outer, direction, omega, init_zero)))
        plan.close()


def test_reference_unit_test_multiple_rhs_and_given_diagonal(emu, oracle):
    n = 4000
    rp, ci, v = dd_matrix(n, 245)
    rng = np.random.default_rng(3)
    k = 3
    xs = np.asfortranarray(rng.uniform(-1, 1, (n, k)))
    Y = np.zeros((n, k), order="F")
    for j in range(k):
        oracle.spmv_serial(rp, ci, v, np.ascontiguousarray(xs[:, j]), Y[:, j], 1.0, 0.0)
    plan = E.Gs2Plan()
    assert plan.symbolic(n, n, rp, ci) == 0 and plan.numeric(n, n, rp, ci, v) == 0
    init = np.linalg.norm(xs, axis=0)
    for direction in (0, 1, 2):
        X = np.asfortranarray(rng.uniform(-1, 1, (n, k)))  # overwritten: init_zero_x_vector
        assert plan.apply(n, n, rp, ci, v, X, Y, True, 0.9, 2, direction) == 0
        assert np.all(np.linalg.norm(X - xs, axis=0) < init)  # EXPECT_LT(result_norm_res, initial_norm_res)
        for j in range(k):
            xo = np.zeros(n)
            oracle.gs2_apply(rp, ci, v, n, xo, np.ascontiguousarray(Y[:, j]), True, 0.9, 2, direction)
            assert np.allclose(X[:, j], xo, rtol=0, atol=1e-13)
    # more sweeps keep converging
    X = np.zeros((n, 1), order="F")
    assert plan.apply(n, n, rp, ci, v, X, Y[:, :1], True, 1.0, 12, 0) == 0
    assert np.linalg.norm(X[:, 0] - xs[:, 0]) < 1e-3 * init[0]
    # a caller-supplied inverse diagonal replaces 1 / a_ii
    rows = np.repeat(np.arange(n), np.diff(rp))
    dinv = 0.8 / v[rows == ci]
    assert plan.numeric(n, n, rp, ci, v, dinv) == 0
    x = np.zeros(n)
    assert plan.apply(n, n, rp, ci, v, x, np.ascontiguousarray(Y[:, 0]), True, 1.0, 1, 1) == 0
    xo = np.zeros(n)
    oracle.gs2_apply(rp, ci, v, n, xo, np.ascontiguousarray(Y[:, 0]), True, 1.0, 1, 1, inverse_diagonal=dinv)
    assert np.allclose(x, xo, rtol=0, atol=1e-13)
    plan.close()


def test_corner_cases_and_errors(emu):
    plan = E.Gs2Plan()
    rp0, ci0 = np.zeros(1, np.int32), np.zeros(1, np.int32)[:0]
    assert plan.symbolic(0, 0, rp0, ci0) == 0  # empty matrix
    assert plan.numeric(0, 0, rp0, ci0, np.zeros(0)) == 0
    assert plan.apply(0, 0, rp0, ci0, np.zeros(0), np.zeros(0), np.zeros(0), True, 1.0, 1, 0) == 0
    # identity: one sweep solves
    n = 10
    rp, ci, v = np.arange(n + 1, dtype=np.int32), np.arange(n, dtype=np.int32), np.full(n, 2.0)
    assert plan.symbolic(n, n, rp, ci) == 0 and plan.numeric(n, n, rp, ci, v) == 0
    x, b = np.full(n, 7.0), np.arange(n, dtype=np.float64)
    assert plan.apply(n, n, rp, ci, v, x, b, False, 1.0, 1, 1) == 0
    assert np.allclose(x, b / 2)
    assert plan.apply(n, n, rp, ci, v, x, b, False, 1.0, 1, 5) == 1  # bad direction
    assert plan.numeric(n, n, rp, ci, v.astype(np.float32)) == 0       # another scalar type: buffers rebuilt
    assert plan.apply(n, n, rp, ci, v, x, b, False, 1.0, 1, 1) == 3    # ... and the f64 apply is refused
    rp2 = rp.copy()
    assert plan.apply(n, n, rp2, ci, v.astype(np.float32), x.astype(np.float32), b.astype(np.float32), False, 1.0, 1, 1) == 3  # another matrix
    # a row without a diagonal entry
    rpb, cib = np.array([0, 1, 2, 3], np.int32), np.array([0, 0, 2], np.int32)
    assert plan.symbolic(3, 3, rpb, cib) == 1 and b"row 1 has no diagonal" in emu.b200sp_last_error_string()
    assert plan.symbolic(3, 2, rpb, cib) == 1  # fewer columns than rows
    assert plan.set(9, 1.0) == 1 and plan.set(2, -1.0) == 1
    # the compact flag changes what symbolic builds: a new symbolic is required
    assert plan.symbolic(n, n, rp, ci) == 0 and plan.numeric(n, n, rp, ci, v) == 0
    assert plan.set(1, 1.0) == 0
    assert plan.numeric(n, n, rp, ci, v) == 3
    plan.close()


@pytest.mark.parametrize("inner,compact", [(1, False), (3, False), (4, True)])
def test_pcg_with_two_stage_preconditioner(emu, oracle, inner, compact):
    """pcgsolve with a GS_TWOSTAGE handle (perf_test/sparse/KokkosSparse_pcg.hpp:321-335: symmetric_gauss_seidel_apply dispatches on
    the handle): the device-resident loop with one symmetric two-stage sweep as preconditioner follows the oracle iteration for
    iteration and beats plain CG."""
    from test_oracle_cg import spd_lap27

    rp, ci, v = spd_lap27(12, shift=0.5)
    n = len(rp) - 1
    xs = np.random.default_rng(0).uniform(-1, 1, n)
    b = np.zeros(n)
    oracle.spmv_serial(rp, ci, v, xs, b, 1.0, 0.0)
    xo = np.zeros(n)
    it_o, nr_o = oracle.pcg_gs2(rp, ci, v, b, xo, 500, 1e-9, inner_sweeps=inner, compact=compact)
    it_c, _ = oracle.cg(rp, ci, v, b, np.zeros(n), 500, 1e-9)
    g2, p = E.Gs2Plan(compact=compact, inner=inner), E.SpmvPlan()
    assert g2.symbolic(n, n, rp, ci) == 0 and g2.numeric(n, n, rp, ci, v) == 0
    x = np.zeros(n)
    it, nr = E.pcg_solve_gs2(p, g2, rp, ci, v, b, x, 500, 1e-9, check_every=3)
    assert abs(it - it_o) <= 1 and it < it_c, (it, it_o, it_c)
    assert nr <= 1e-9 and np.linalg.norm(x - xs) / np.linalg.norm(xs) < 1e-8
    if it == it_o:
        assert np.max(np.abs(x - xo)) <= 1e-10 * max(1.0, np.max(np.abs(xo)))
    g2.close()
    p.close()


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("compact", [False, True])
def test_several_right_hand_sides_use_the_multivector_products(emu, oracle, dtype, compact):
    """k > 1: every product is one SpMM over all columns (the matrix is read once), x and b with padded leading dimensions and ghost
    rows; each column must equal the oracle's single-vector run."""
    n, ghosts, k = 2500, 30, 4
    rp, ci, v = dd_matrix(n, 21, extra_cols=ghosts)
    v = v.astype(dtype)
    ncols = n + ghosts
    rng = np.random.default_rng(6)
    Xfull = np.asfortranarray(rng.uniform(-1, 1, (ncols + 5, k)).astype(dtype))
    Bfull = np.asfortranarray(rng.uniform(-1, 1, (n + 3, k)).astype(dtype))
    X0, B = Xfull[:ncols], Bfull[:n]  # views: leading dimensions ncols + 5 and n + 3
    tol = 1e-13 if dtype == np.float64 else 1e-5
    plan = E.Gs2Plan(compact=compact, inner=2, gamma=0.9)
    assert plan.symbolic(n, ncols, rp, ci) == 0 and plan.numeric(n, ncols, rp, ci, v) == 0
    for direction, omega, init_zero in ((0, 0.9, False), (1, 1.0, True), (2, 1.1, False)):
        Xw = Xfull.copy(order="F")
        X = Xw[:ncols]
        assert plan.apply(n, ncols, rp, ci, v, X, B, init_zero, omega, 2, direction) == 0
        assert np.array_equal(Xw[ncols:], Xfull[ncols:])  # the padding rows are not touched
        for j in range(k):
            xo = np.ascontiguousarray(X0[:, j]).copy()
            oracle.gs2_apply(rp, ci, v, ncols, xo, np.ascontiguousarray(B[:, j]), init_zero, dtype(omega), 2, direction, compact=compact,
                             inner_sweeps=2, gamma=dtype(0.9))
            err = np.max(np.abs(X[:, j].astype(np.float64) - xo.astype(np.float64)))
            assert err <= tol * 20 * max(1.0, np.max(np.abs(xo))), (direction, j, err)
    # one column afterwards on the same plan (rank-1 products again), then more columns than before (work vectors regrown)
    x1 = np.ascontiguousarray(X0[:, 0]).copy()
    assert plan.apply(n, ncols, rp, ci, v, x1, np.ascontiguousarray(B[:, 0]), False, 1.0, 1, 0) == 0
    X6 = np.asfortranarray(rng.uniform(-1, 1, (ncols, 6)).astype(dtype))
    B6 = np.asfortranarray(rng.uniform(-1, 1, (n, 6)).astype(dtype))
    assert plan.apply(n, ncols, rp, ci, v, X6, B6, True, 1.0, 1, 0) == 0
    assert np.all(np.isfinite(X6))
    plan.close()
