"""Cases for the Gauss-Seidel path tests (test_gpu_gs_paths.py, test_emulated_gs_paths.py): matrices built to reach every
point-sweep kernel (lanes per row 2 .. 32, chosen from the average row length or forced), colour sets that wrap the sweep
kernel's grid-stride loop, more than 64 colours, nonsymmetric and unsorted patterns, rows that hold only their diagonal,
duplicate diagonal entries, ghost columns, n = 1; and the option grid of the two-stage and classic forms.

Every matrix is diagonally dominant with mixed-sign values over several binades, so that repeated sweeps stay bounded.
`scale` shrinks the sizes for the CPU emulation; the structure of each case is the same at every scale."""
import numpy as np

from spmm_cases import _values

LPRS = (2, 4, 8, 16, 32)


def _finish(rows, n, ncols, rng, dtype=np.float64, dup_diag=None, shuffle=False):
    """CSR from per-row column lists (each holding its diagonal), values mixed-sign, the diagonal dominant and of random
    sign.  dup_diag: rows whose diagonal is split into two pieces of one sign.  shuffle: entries of every row in random order."""
    rp = np.zeros(n + 1, dtype=np.int64)
    np.cumsum([len(r) for r in rows], out=rp[1:])
    ci = np.concatenate([np.asarray(r, dtype=np.int64) for r in rows]) if n else np.zeros(0, np.int64)
    v = _values(rng, len(ci), np.float64)
    row = np.repeat(np.arange(n), np.diff(rp))
    diag = ci == row
    off = np.bincount(row[~diag], weights=np.abs(v[~diag]), minlength=n)
    dval = (off + rng.uniform(0.5, 1.5, n) * np.maximum(off, 1.0)) * rng.choice([-1.0, 1.0], n)
    v[diag] = dval[row[diag]]
    if dup_diag is not None:  # a second piece on the chosen rows: the pieces keep the sign and add up to the same diagonal
        keep = np.zeros(n, dtype=bool)
        keep[dup_diag] = True
        new_rows = []
        new_vals = []
        for i in range(n):
            c, w = ci[rp[i]:rp[i + 1]], v[rp[i]:rp[i + 1]]
            if keep[i]:
                k = int(np.flatnonzero(c == i)[0])
                f = rng.uniform(0.25, 0.75)
                c = np.insert(c, len(c), i)
                w = np.insert(w, len(w), w[k] * (1 - f))
                w[k] *= f
            new_rows.append(c)
            new_vals.append(w)
        rp = np.zeros(n + 1, dtype=np.int64)
        np.cumsum([len(r) for r in new_rows], out=rp[1:])
        ci, v = np.concatenate(new_rows), np.concatenate(new_vals)
    if shuffle:
        perm = np.concatenate([rp[i] + rng.permutation(rp[i + 1] - rp[i]) for i in range(n)]) if n else np.zeros(0, np.int64)
        ci, v = ci[perm], v[perm]
    assert rp[-1] < 2**31
    return dict(n=n, ncols=ncols, rp=rp.astype(np.int32), ci=ci.astype(np.int32), v=v.astype(dtype))


def _band_plus_ghosts(lens, n, ghosts, rng, band=2):
    """Row i: its diagonal, neighbours i-band .. i+band inside [0, n), then distinct ghost columns up to lens[i] entries.
    The band keeps the colouring to a few colours whatever the row length."""
    rows = []
    for i in range(n):
        near = [j for j in range(max(0, i - band), min(n, i + band + 1))]
        L = int(lens[i])
        if L <= len(near):  # short row: the diagonal first, then neighbours
            near = [i] + [j for j in near if j != i]
            rows.append(np.asarray(near[:L]))
        else:
            extra = rng.choice(ghosts, L - len(near), replace=False) + n
            rows.append(np.concatenate([near, np.sort(extra)]))
    return rows


def threshold_case(avg_num, avg_den, n, rng):
    """Average row length exactly avg_num / avg_den (rows of floor and floor + 1), around an LPR threshold of symbolic."""
    nnz = n * avg_num // avg_den
    assert nnz * avg_den == n * avg_num, "pick n so the average is exact"
    base = nnz // n
    lens = np.full(n, base)
    lens[rng.choice(n, nnz - base * n, replace=False)] += 1
    ghosts = int(lens.max()) + 8
    c = _finish(_band_plus_ghosts(lens, n, ghosts, rng), n, n + ghosts, rng)
    c["name"] = f"avg{avg_num / avg_den:g}"
    c["symmetric"] = True  # the square part (the band) is symmetric
    return c


def expected_lpr(rp, n):
    avg = float(rp[-1]) / n
    return 2 if avg <= 8.0 else 4 if avg <= 96.0 else 8 if avg <= 384.0 else 16 if avg <= 1536.0 else 32


def threshold_cases(scale=1.0):
    """(case, expected LPR) on both sides of each threshold: 8 / 8.01, 96 / 97, 384 / 385, 1536 / 1537."""
    rng = np.random.default_rng(11)
    out = []
    n_small = max(100, int(2000 * scale) // 100 * 100)
    n_large = max(40, int(400 * scale))
    for num, den, n in ((8, 1, n_small), (801, 100, n_small), (96, 1, n_small), (97, 1, n_small), (384, 1, n_large),
                        (385, 1, n_large), (1536, 1, n_large // 2), (1537, 1, n_large // 2)):
        c = threshold_case(num, den, n, rng)
        out.append((c, expected_lpr(c["rp"], c["n"])))
    return out


def lpr_edge_case(scale=1.0):
    """Rows of length 1 (the diagonal alone), LPR - 1, LPR, LPR + 1 for every LPR, and a few of about 5000 entries; run with
    every forced LPR.  Rows unsorted, the diagonal anywhere in them."""
    rng = np.random.default_rng(12)
    lens_cycle = sorted({1} | {l + d for l in LPRS for d in (-1, 0, 1)})
    n = max(len(lens_cycle) * 6, int(1200 * scale))
    lens = np.array([lens_cycle[i % len(lens_cycle)] for i in range(n)])
    lens[rng.choice(n, 3, replace=False)] = [4999, 5000, 5003]
    ghosts = 5100
    c = _finish(_band_plus_ghosts(lens, n, ghosts, rng), n, n + ghosts, rng, shuffle=True)
    c.update(name="lpr_edges", symmetric=False)  # short rows cut the band on one side: not symmetric
    return c


def wrap_case(rows):
    """Tridiagonal: two or three colour sets of about rows / 2 each -- more rows than one grid-stride pass of the sweep
    kernel covers, at LPR 2 (average length < 3)."""
    rng = np.random.default_rng(13)
    n = int(rows)
    cols = np.stack([np.arange(n) - 1, np.arange(n), np.arange(n) + 1], axis=1)
    ok = (cols >= 0) & (cols < n)
    rp = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(ok.sum(axis=1), out=rp[1:])
    ci = cols[ok]
    v = _values(rng, len(ci), np.float64)
    row = np.repeat(np.arange(n), np.diff(rp))
    diag = ci == row
    off = np.bincount(row[~diag], weights=np.abs(v[~diag]), minlength=n)
    v[diag] = (off + rng.uniform(0.5, 1.5, n)) * rng.choice([-1.0, 1.0], n)
    return dict(n=n, ncols=n, rp=rp.astype(np.int32), ci=ci.astype(np.int32), v=v, name=f"wrap{n}", symmetric=True)


def clique_case(scale=1.0):
    """A 130-row clique (130 colours: three 64-colour windows of the colouring) inside a sparse banded matrix."""
    rng = np.random.default_rng(14)
    n = max(400, int(3000 * scale))
    q0, q = 37, 130
    rows = []
    for i in range(n):
        near = set(range(max(0, i - 2), min(n, i + 3)))
        if q0 <= i < q0 + q:
            near |= set(range(q0, q0 + q))
        rows.append(np.array(sorted(near)))
    c = _finish(rows, n, n, rng)
    c.update(name="clique130", symmetric=True)
    return c


def nonsymmetric_case(scale=1.0, ghosts=0):
    """Random one-sided pattern (entry (i, j) without (j, i)), coloured on A + A^T (is_graph_symmetric = False); rows that
    hold only their diagonal, two same-sign diagonal pieces in some rows, unsorted rows; ghost columns on request."""
    rng = np.random.default_rng(15 + ghosts)
    n = max(300, int(4000 * scale))
    rows = []
    for i in range(n):
        if i % 17 == 0:
            rows.append(np.array([i]))
            continue
        k = int(rng.integers(1, 12))
        cols = set(rng.integers(0, n, k).tolist())
        if ghosts:
            cols |= set((n + rng.integers(0, ghosts, int(rng.integers(0, 4)))).tolist())
        cols.discard(i)
        rows.append(np.array(sorted(cols | {i})))
    dup = np.arange(5, n, 23)
    c = _finish(rows, n, n + ghosts, rng, dup_diag=dup, shuffle=True)
    c.update(name="nonsym" + ("_ghost" if ghosts else ""), symmetric=False)
    return c


def single_row_case():
    c = _finish([np.array([0])], 1, 1, np.random.default_rng(16))
    c.update(name="n1", symmetric=True)
    return c


def point_cases(scale=1.0):
    """The cases every LPR runs on: (case) list; LPR threshold cases come from threshold_cases."""
    return [lpr_edge_case(scale), clique_case(scale), nonsymmetric_case(scale), nonsymmetric_case(scale, ghosts=97), single_row_case()]


def vectors(c, dtype, seed):
    """y (n) and x0 (ncols), mixed signs over several binades."""
    rng = np.random.default_rng(seed)
    return _values(rng, c["n"], dtype), _values(rng, c["ncols"], dtype)


# ---- two-stage and classic ---------------------------------------------------------------------------------------------
def gs2_case(scale=1.0):
    """Nonsymmetric, unsorted rows with the diagonal anywhere, ghost columns; one diagonal entry per row (numeric keeps
    one)."""
    rng = np.random.default_rng(21)
    n = max(300, int(3000 * scale))
    ghosts = 41
    rows = []
    for i in range(n):
        if i % 29 == 0:
            rows.append(np.array([i]))
            continue
        cols = set(rng.integers(max(0, i - 60), min(n, i + 60), int(rng.integers(1, 10))).tolist())
        cols |= set((n + rng.integers(0, ghosts, int(rng.integers(0, 3)))).tolist())
        cols.discard(i)
        rows.append(np.array(sorted(cols | {i})))
    c = _finish(rows, n, n + ghosts, rng, shuffle=True)
    c.update(name="gs2")
    return c


def gs2_grid():
    """(inner, gamma, outer, compact) for every combination, each with omega 1 and 0.9 and the inverse diagonal given or not;
    the direction and init_zero cycle so that each combination sees several."""
    out = []
    k = 0
    for compact in (False, True):
        for inner in (0, 1, 2, 3):
            for gamma in (1.0, 0.7):
                for outer in (1, 3):
                    for omega in (1.0, 0.9):
                        for given in (False, True):
                            out.append(dict(compact=compact, inner=inner, gamma=gamma, outer=outer, omega=omega, given=given,
                                            direction=k % 3, init_zero=(k // 3) % 2 == 1, num_iter=1 + (k % 2)))
                            k += 1
    return out


def classic_grid():
    out = []
    for compact in (False, True):
        for given in (False, True):
            for direction in (0, 1, 2):
                for init_zero in (False, True):
                    out.append(dict(compact=compact, given=given, direction=direction, init_zero=init_zero, outer=1 + 2 * (direction == 1),
                                    num_iter=1))
    return out


def given_dinv(c, dtype, seed=3):
    """A caller-supplied inverse diagonal close to the matrix' own."""
    rng = np.random.default_rng(seed)
    rp, ci, v, n = c["rp"], c["ci"], c["v"], c["n"]
    row = np.repeat(np.arange(n), np.diff(rp))
    d = np.zeros(n)
    d[row[ci == row]] = v[ci == row]
    return (1.0 / (d * rng.uniform(1.0, 1.1, n))).astype(dtype)


# ---- checks shared by the GPU and the emulated test files -------------------------------------------------------------
# A point runner has symbolic(c), numeric(c, v), apply(c, v, x, y, init_zero, omega, sweeps, direction) -> x (numpy, ncols),
# coloring() -> (num_colors, colors, color_ptr, color_rows) and kernel() -> the plan's last_kernel label.
def _pattern(c):
    """Square part of the pattern as a 0/1 scipy CSR."""
    import scipy.sparse as sps

    n, rp, ci = c["n"], c["rp"], c["ci"]
    row = np.repeat(np.arange(n), np.diff(rp))
    sq = ci < n
    return sps.csr_matrix((np.ones(int(sq.sum())), (row[sq], ci[sq])), shape=(n, n))


def check_coloring(n, P, nc, colors, color_ptr, color_rows):
    """A proper distance-1 colouring of the pattern P (scipy CSR) whose sets partition the rows, ascending inside a set."""
    assert nc >= 1 and colors.min() >= 0 and colors.max() == nc - 1
    P = P.tocoo()
    off = P.row != P.col
    assert not np.any(colors[P.row[off]] == colors[P.col[off]]), "two adjacent rows share a colour"
    assert color_ptr[0] == 0 and color_ptr[-1] == n and np.all(np.diff(color_ptr) >= 0)
    assert np.array_equal(np.sort(color_rows), np.arange(n))
    assert np.array_equal(colors[color_rows], np.repeat(np.arange(nc), np.diff(color_ptr)))
    starts = np.asarray(color_ptr[1:-1])
    inner = np.ones(n - 1, dtype=bool) if n > 1 else np.zeros(0, dtype=bool)
    inner[starts[(starts > 0) & (starts < n)] - 1] = False
    assert np.all(np.diff(color_rows)[inner] > 0), "rows of a colour set must be ascending"


def check_coloring_both(c, coloring):
    """On A and on A^T (the colouring is of A + A^T when the pattern is not symmetric)."""
    P = _pattern(c)
    check_coloring(c["n"], P, *coloring)
    check_coloring(c["n"], P.T.tocsr(), *coloring)


def check_sweeps(run, c, dtype, lpr, seed=1):
    """One forward and one backward sweep, each row within gs_sweep_bound of its local reference; ghosts unchanged.  Returns
    the labels the plan reported."""
    import exact_ref as R

    n = c["n"]
    v = c["v"].astype(dtype)
    y, x0 = vectors(c, dtype, seed)
    tag = "f64" if np.dtype(dtype) == np.float64 else "f32"
    labels = set()
    _, colors, _, _ = run.coloring()
    for direction in (1, 2):
        x = run.apply(c, v, x0, y, False, 0.9, 1, direction)
        label = run.kernel()
        assert label.startswith(f"gs_set<{tag},LPR={lpr}>x"), (c["name"], label)
        labels.add(label.split(">x")[0] + ">")
        assert _same(x[n:], x0[n:]), "ghost entries written"
        ex = R.gs_sweep_exact(c["rp"], c["ci"], v, colors, x0, x, y, 0.9, direction)
        bd = R.gs_sweep_bound(c["rp"], c["ci"], v, colors, x0, x, y, 0.9, direction)
        R.assert_within(x[:n], ex, bd, f"{c['name']} {label} direction {direction}")
    return labels


def _same(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


def check_laws(run, c, dtype, seed=2):
    """Bit-for-bit laws of a fixed colouring and LPR: symmetric = forward then backward; sweeps = s equals s single sweeps;
    init_zero equals a zeroed x (ghosts included); two runs agree."""
    v = c["v"].astype(dtype)
    y, x0 = vectors(c, dtype, seed)
    sym = run.apply(c, v, x0, y, False, 0.9, 1, 0)
    fb = run.apply(c, v, run.apply(c, v, x0, y, False, 0.9, 1, 1), y, False, 0.9, 1, 2)
    assert _same(sym, fb), "symmetric != forward then backward"
    three = run.apply(c, v, x0, y, False, 0.9, 3, 0)
    seq = x0
    for _ in range(3):
        seq = run.apply(c, v, seq, y, False, 0.9, 1, 0)
    assert _same(three, seq), "sweeps = 3 != three single sweeps"
    assert _same(three, run.apply(c, v, x0, y, False, 0.9, 3, 0)), "two runs differ"
    for direction in (1, 2):
        garbage = np.full(c["ncols"], 7.5, dtype=dtype)
        z = run.apply(c, v, garbage, y, True, 0.9, 2, direction)
        z0 = run.apply(c, v, np.zeros(c["ncols"], dtype), y, False, 0.9, 2, direction)
        assert _same(z, z0) and np.all(z[c["n"]:] == 0), "init_zero differs from a zeroed x"


# A two-stage runner has setup(c, v, compact, inner, outer, gamma, two_stage, dinv) and apply(X, B, init_zero, omega, num_iter,
# direction) -> X, with X (ncols rows) and B (n rows) 1-D or 2-D column-major views into padded buffers.
def padded(rows, k, pad, dtype, fill):
    """A (rows, k) column-major view with leading dimension rows + pad into a buffer whose padding holds NaN."""
    buf = np.full((k, rows + pad), np.nan, dtype=dtype)
    buf[:, :rows] = fill.T if fill.ndim == 2 else fill[None, :]
    return buf.T[:rows], buf


def check_gs2(run, c, dtype, g, nrhs=1, pad=0, seed=5, two_stage=True):
    """One apply with the options g (a gs2_grid / classic_grid entry) on nrhs right-hand sides: each column within gs2_bound
    of its own single-column reference, ghosts and padding bitwise unchanged (ghosts zeroed under init_zero)."""
    import exact_ref as R

    n, ncols = c["n"], c["ncols"]
    v = c["v"].astype(dtype)
    dinv = given_dinv(c, dtype) if g["given"] else None
    rng = np.random.default_rng(seed)
    X0 = np.stack([_values(rng, ncols, dtype) for _ in range(nrhs)], axis=1)
    B0 = np.stack([_values(rng, n, dtype) for _ in range(nrhs)], axis=1)
    omega = g.get("omega", 1.0)
    inner, gamma = g.get("inner", 0), g.get("gamma", 1.0)
    run.setup(c, v, g["compact"], inner, g["outer"], gamma, two_stage, dinv)
    if nrhs == 1 and pad == 0:
        X = run.apply(X0[:, 0].copy(), B0[:, 0].copy(), g["init_zero"], omega, g["num_iter"], g["direction"])[:, None]
        Xbuf = None
    else:
        Xv, Xbuf = padded(ncols, nrhs, pad, dtype, X0)
        Xbuf0 = Xbuf.copy()
        Bv, _ = padded(n, nrhs, pad + 3, dtype, B0)
        Xbuf = run.apply(Xv, Bv, g["init_zero"], omega, g["num_iter"], g["direction"], buffers=True)
        assert _same(Xbuf[:, ncols:], Xbuf0[:, ncols:]), "padding written"
        X = Xbuf[:, :ncols].T
    what = f"{'two-stage' if two_stage else 'classic'} {g} k={nrhs}"
    for j in range(nrhs):
        ex, bd = R.gs2_ref(c["rp"], c["ci"], v, ncols, X0[:, j], B0[:, j], g["init_zero"], omega, g["num_iter"], g["direction"], g["compact"],
                           inner, g["outer"], gamma, two_stage, dinv)
        if g["init_zero"]:
            assert np.all(X[n:, j] == 0), what + ": ghosts not zeroed"
        else:
            assert _same(X[n:, j], X0[n:, j]), what + ": ghosts written"
        R.assert_within(X[:, j], ex, bd, f"{what} column {j}")


def check_classic_local(run, c, dtype, given, compact):
    """Classic form, init_zero, one forward or backward sweep: x = Z exactly, so each row of the triangular solve is checked
    locally against the kernel's own Z."""
    import exact_ref as R

    n, ncols = c["n"], c["ncols"]
    v = c["v"].astype(dtype)
    dinv = given_dinv(c, dtype) if given else None
    b, x0 = vectors(c, dtype, 9)
    run.setup(c, v, compact, 0, 1, 1.0, False, dinv)
    for direction in (1, 2):
        z = run.apply(x0.copy(), b.copy(), True, 1.0, 1, direction)
        ex, bd = R.trsv_row_bound(c["rp"], c["ci"], v, b, z[:n], direction == 1, dinv)
        R.assert_within(z[:n], ex, bd, f"classic local direction {direction} given={given} compact={compact}")
