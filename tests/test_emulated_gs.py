"""Point (multicolour) Gauss-Seidel kernels executed on the CPU (tools/emu) against the oracle: the colouring symbolic produces is
a proper distance-1 colouring of pattern(A) + pattern(A^T) whose sets partition the rows; the sweeps equal the oracle's
restatement of the reference's PSGS functor over the same sets; and the reference's unit test passes
(sparse/unit_test/Test_Sparse_gauss_seidel.hpp:180-216: diagonally dominant matrix, x = 0, two sweeps with omega = 0.9,
symmetric / forward / backward: the error norm drops below the norm of the solution)."""
import numpy as np
import pytest
import scipy.sparse as sps

import emu_lib as E
import exact_ref as R
from gmres_cases import gmres_matrix


@pytest.fixture(scope="module")
def emu():
    return E.lib()


def symmetrize(rp, ci, v, n):
    import scipy.sparse as sps

    A = sps.csr_matrix((v, ci, rp), shape=(n, n))
    S = ((A + A.T) * 0.5).tocsr()
    S.sort_indices()
    return S.indptr.astype(np.int32), S.indices.astype(np.int32), S.data.copy()


def check_coloring(n, rp, ci, nc, colors, color_ptr, color_rows):
    assert nc >= 1 and colors.min() >= 0 and colors.max() == nc - 1
    rows = np.repeat(np.arange(n), np.diff(rp))
    off = rows != ci
    assert not np.any(colors[rows[off]] == colors[ci[off]]), "two adjacent rows share a colour"
    assert color_ptr[0] == 0 and color_ptr[-1] == n and np.all(np.diff(color_ptr) >= 0)
    assert np.array_equal(np.sort(color_rows), np.arange(n))
    for c in range(nc):
        seg = color_rows[color_ptr[c]:color_ptr[c + 1]]
        assert np.all(colors[seg] == c) and np.all(np.diff(seg) > 0)  # the set of colour c, rows ascending


@pytest.mark.parametrize("symmetric", [True, False])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_reference_unit_test_and_oracle_parity(emu, oracle, symmetric, dtype):
    n = 3000
    rp, ci, v = gmres_matrix(n, 1.0, seed=245)  # kk_generate_diagonally_dominant_sparse_matrix family (IOUtils.hpp:112-177)
    if symmetric:
        rp, ci, v = symmetrize(rp, ci, v, n)
    v = v.astype(dtype)
    rng = np.random.default_rng(3)
    xs = rng.uniform(-1, 1, n).astype(dtype)
    y = np.zeros(n, dtype=dtype)
    oracle.spmv_serial(rp, ci, v, xs, y, 1.0, 0.0)
    plan = E.GsPlan()
    with pytest.raises(Exception):
        assert plan.numeric(n, rp, ci, v) == 0  # numeric before symbolic: refused
        raise RuntimeError
    plan.symbolic(n, rp, ci, symmetric)
    nc, colors, cptr, crows = plan.coloring(n)
    check_coloring(n, rp, ci, nc, colors, cptr, crows)
    assert plan.apply(n, rp, ci, v, np.zeros(n, dtype), y, True, 0.9, 1, 0) != 0  # apply before numeric: refused
    assert plan.numeric(n, rp, ci, v) == 0
    rows = np.repeat(np.arange(n), np.diff(rp))
    dinv = (1.0 / np.bincount(rows[rows == ci], weights=v[rows == ci].astype(np.float64), minlength=n)).astype(dtype)
    init = np.linalg.norm(xs.astype(np.float64))
    for direction in (0, 1, 2):  # symmetric, forward, backward (apply_type of the reference's test)
        x = rng.uniform(-1, 1, n).astype(dtype)  # overwritten: init_zero_x
        assert plan.apply(n, rp, ci, v, x, y, True, 0.9, 2, direction) == 0
        xo = oracle.gs_apply(rp, ci, v, cptr, crows, dinv, y, np.ones(n, dtype), True, dtype(0.9), 2, direction)
        tol = 1e-12 if dtype == np.float64 else 2e-5
        assert np.max(np.abs(x.astype(np.float64) - xo.astype(np.float64))) <= tol * max(1.0, np.max(np.abs(xo)))
        assert np.linalg.norm(x.astype(np.float64) - xs.astype(np.float64)) < init  # EXPECT_LT(result_norm_res, initial_norm_res)
        if direction:  # one more sweep from here, each row within its local bound
            x2 = x.copy()
            assert plan.apply(n, rp, ci, v, x2, y, False, 0.9, 1, direction) == 0
            R.assert_within(x2, R.gs_sweep_exact(rp, ci, v, colors, x, x2, y, 0.9, direction),
                            R.gs_sweep_bound(rp, ci, v, colors, x, x2, y, 0.9, direction), plan.kernel())
    # more sweeps from the current x (init_zero_x = false) keep converging
    before = np.linalg.norm(x.astype(np.float64) - xs.astype(np.float64))
    assert plan.apply(n, rp, ci, v, x, y, False, 0.9, 3, 0) == 0
    assert np.linalg.norm(x.astype(np.float64) - xs.astype(np.float64)) < 0.5 * before
    plan.close()


@pytest.mark.parametrize("symmetric", [True, False])
def test_iterated_greedy_recolouring_never_adds_colours(emu, monkeypatch, symmetric):
    """gs.cu re-colours class by class (Culberson) after Jones-Plassmann: valid, deterministic, never more colours."""
    n = 2500
    rp, ci, v = gmres_matrix(n, 1.0, seed=99)
    if symmetric:
        rp, ci, v = symmetrize(rp, ci, v, n)
    counts = {}
    for passes in ("0", "1", "2", "5"):
        monkeypatch.setenv("B200SP_GS_RECOLOR", passes)
        got = []
        for _ in range(2):
            plan = E.GsPlan()
            plan.symbolic(n, rp, ci, symmetric)
            nc, colors, cptr, crows = plan.coloring(n)
            if not symmetric:  # the colouring is of the symmetrised graph
                S = sps.csr_matrix((np.ones(len(ci)), ci, rp), shape=(n, n))
                S = (S + S.T).tocsr()
                check_coloring(n, S.indptr, S.indices, nc, colors, cptr, crows)
            else:
                check_coloring(n, rp, ci, nc, colors, cptr, crows)
            got.append(colors.copy())
            plan.close()
        assert np.array_equal(got[0], got[1])  # same input, same colouring
        counts[passes] = nc
    assert counts["0"] >= counts["1"] >= counts["2"] >= counts["5"]


def test_structure_corner_cases(emu, oracle):
    plan = E.GsPlan()
    plan.symbolic(0, np.zeros(1, np.int32), np.zeros(0, np.int32), True)  # empty matrix
    assert plan.numeric(0, np.zeros(1, np.int32), np.zeros(0, np.int32), np.zeros(0)) == 0
    assert plan.apply(0, np.zeros(1, np.int32), np.zeros(0, np.int32), np.zeros(0), np.zeros(0), np.zeros(0), True, 1.0, 1, 0) == 0
    # diagonal matrix: one colour, one sweep with omega = 1 solves it
    n = 50
    rp, ci, v = np.arange(n + 1, dtype=np.int32), np.arange(n, dtype=np.int32), np.linspace(1, 5, n)
    plan.symbolic(n, rp, ci, True)
    nc, colors, cptr, crows = plan.coloring(n)
    assert nc == 1
    assert plan.numeric(n, rp, ci, v) == 0
    y = np.linspace(-1, 1, n)
    x = np.zeros(n)
    assert plan.apply(n, rp, ci, v, x, y, True, 1.0, 1, 1) == 0
    assert np.allclose(x, y / v, rtol=1e-15)
    # a dense 40 x 40 block: 40 colours (a clique), and a row without a diagonal is refused by numeric
    m = 40
    rp = (np.arange(m + 1) * m).astype(np.int32)
    ci = np.tile(np.arange(m), m).astype(np.int32)
    v = np.random.default_rng(1).uniform(0.1, 1, m * m) + np.tile(np.eye(m), 1).ravel() * m
    plan.symbolic(m, rp, ci, True)
    nc, colors, cptr, crows = plan.coloring(m)
    check_coloring(m, rp, ci, nc, colors, cptr, crows)
    assert nc == m
    rp2, ci2 = np.array([0, 1, 2], np.int32), np.array([1, 0], np.int32)  # 2 x 2 without diagonal
    plan.symbolic(2, rp2, ci2, True)
    assert plan.numeric(2, rp2, ci2, np.ones(2)) != 0 and b"diagonal" in emu.b200sp_last_error_string()
    plan.close()


def test_long_rows_and_many_colors(emu, oracle):
    """Skewed pattern: a few rows adjacent to most others (long rows, several 64-colour windows are not needed but the JP
    rounds are many); unsymmetric pattern coloured on A + A^T."""
    rng = np.random.default_rng(9)
    n = 1500
    lens = rng.integers(2, 7, n)
    lens[[3, 700]] = [900, 1200]
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    cols = []
    for i, l in enumerate(lens):
        c = set(rng.choice(n, int(l) - 1, replace=False).tolist()) - {i}
        cols.append(np.sort(np.array(sorted(c | {i}))))
    rp = np.concatenate([[0], np.cumsum([len(c) for c in cols])]).astype(np.int32)
    ci = np.concatenate(cols).astype(np.int32)
    rows = np.repeat(np.arange(n), np.diff(rp))
    v = rng.uniform(-1, 1, len(ci))
    v[rows == ci] = 3000.0  # strongly dominant diagonal
    plan = E.GsPlan()
    plan.symbolic(n, rp, ci, False)
    nc, colors, cptr, crows = plan.coloring(n)
    # proper on the symmetrised pattern: check both directions
    assert not np.any((colors[rows] == colors[ci]) & (rows != ci))
    assert plan.numeric(n, rp, ci, v) == 0
    xs = rng.uniform(-1, 1, n)
    y = np.zeros(n)
    oracle.spmv_serial(rp, ci, v, xs, y, 1.0, 0.0)
    x = np.zeros(n)
    assert plan.apply(n, rp, ci, v, x, y, True, 1.0, 2, 0) == 0
    dinv = 1.0 / np.full(n, 3000.0)
    xo = oracle.gs_apply(rp, ci, v, cptr, crows, dinv, y, np.zeros(n), True, 1.0, 2, 0)
    assert np.max(np.abs(x - xo)) <= 1e-12 and np.linalg.norm(x - xs) < 1e-3 * np.linalg.norm(xs)
    plan.close()


def test_pcg_with_symmetric_gauss_seidel(emu, oracle):
    """b200sp_pcg_solve (the reference's pcgsolve with its default use_sgs = true, perf_test/sparse/KokkosSparse_pcg.hpp:248-466)
    against the oracle's restatement run over the SAME colour sets: same iteration count, same solution; and fewer
    iterations than the unpreconditioned solve."""
    from test_oracle_cg import spd_lap27

    rp, ci, v = spd_lap27(14, shift=0.5)
    n = len(rp) - 1
    rng = np.random.default_rng(0)
    xs = rng.uniform(-1, 1, n)
    b = np.zeros(n)
    oracle.spmv_serial(rp, ci, v, xs, b, 1.0, 0.0)
    gs = E.GsPlan()
    gs.symbolic(n, rp, ci, True)
    assert gs.numeric(n, rp, ci, v) == 0
    nc, colors, cptr, crows = gs.coloring(n)
    rows = np.repeat(np.arange(n), np.diff(rp))
    dinv = 1.0 / v[rows == ci]
    xo = np.zeros(n)
    it_o, nr_o = oracle.pcg(rp, ci, v, b, xo, 100000, 1e-7, cptr, crows, dinv)
    xc = np.zeros(n)
    it_plain, _ = oracle.cg(rp, ci, v, b, xc, 100000, 1e-7)
    assert 0 < it_o < it_plain  # the preconditioner pays
    plan = E.SpmvPlan()
    for check_every in (1, 8):
        x = np.zeros(n)
        it, nr = E.pcg_solve(plan, gs, rp, ci, v, b, x, 100000, 1e-7, check_every)
        assert abs(it - it_o) <= 1 and nr <= 1e-7, (it, it_o, nr)
        assert np.linalg.norm(x - xo) / np.linalg.norm(xo) < 1e-8
    plan.close()
    gs.close()


@pytest.mark.parametrize("symmetric", [True, False])
def test_ghost_columns(emu, oracle, symmetric):
    """num_cols > num_rows -- the local matrix of a distributed one (what Ifpack2 / MueLu pass): columns >= num_rows are ghost entries
    of x, read by the sweeps, never written, outside the colouring; init_zero_x zeroes all of x as the reference does."""
    from test_oracle_gs2 import dd_matrix

    n, ghosts = 2500, 70
    rp, ci, v = dd_matrix(n, 31, extra_cols=ghosts)
    ncols = n + ghosts
    if symmetric:  # symmetrise the square part, keep the ghost columns
        A = sps.csr_matrix((v, ci, rp), shape=(n, ncols)).tocsc()
        S = ((A[:, :n] + A[:, :n].T) * 0.5)
        A = sps.hstack([S, A[:, n:]]).tocsr()
        A.sort_indices()
        rp, ci, v = A.indptr.astype(np.int32), A.indices.astype(np.int32), A.data.copy()
    plan = E.GsPlan()
    plan.symbolic(n, rp, ci, symmetric, ncols=ncols)
    nc, colors, cptr, crows = plan.coloring(n)
    sq = ci < n  # the colouring is of the square part (symmetrised when the graph is not symmetric)
    rows = np.repeat(np.arange(n), np.diff(rp))
    G = sps.csr_matrix((np.ones(sq.sum()), (rows[sq], ci[sq])), shape=(n, n))
    G = (G + G.T).tocsr()
    check_coloring(n, G.indptr, G.indices, nc, colors, cptr, crows)
    assert plan.numeric(n, rp, ci, v) == 0
    dinv = 1.0 / np.bincount(rows[rows == ci], weights=v[rows == ci], minlength=n)
    rng = np.random.default_rng(5)
    b = rng.uniform(-1, 1, n)
    x0 = rng.uniform(-1, 1, ncols)
    for direction in (0, 1, 2):
        x = x0.copy()
        assert plan.apply(n, rp, ci, v, x, b, False, 0.9, 2, direction) == 0
        xo = oracle.gs_apply(rp, ci, v, cptr, crows, dinv, b, x0.copy(), False, 0.9, 2, direction)
        assert np.array_equal(x[n:], x0[n:]) and np.max(np.abs(x - xo)) <= 1e-12
    x = x0.copy()
    assert plan.apply(n, rp, ci, v, x, b, True, 1.0, 1, 0) == 0
    xo = oracle.gs_apply(rp, ci, v, cptr, crows, dinv, b, np.zeros(ncols), False, 1.0, 1, 0)
    assert np.all(x[n:] == 0) and np.max(np.abs(x - xo)) <= 1e-12
    assert E.lib().b200sp_gs_symbolic_nc_i32(plan.h, None, n, n - 1, E.ptr(rp), E.ptr(ci), 1) == 1  # fewer columns than rows
    plan.close()
