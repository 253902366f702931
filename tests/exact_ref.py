"""Exact reference and per-entry rounding-error bound of SpMV, y = beta*y0 + alpha*op(A)*x, rank 1 and rank 2, on
CrsMatrix and (through bsr_to_point_crs) BsrMatrix.

The oracle (oracle_lib.Oracle.spmv_mv) computes in the kernel's own precision, so its rounding error is about as large as
the error it is meant to detect.  spmm_exact computes the same product in a wider format (float64 for fp32 data,
np.longdouble for fp64 data), and spmm_bound gives, for every entry of Y, how far a correctly implemented kernel may be
from it.  assert_within checks a kernel's output entry by entry against that bound.  All three take 1-D x and y (rank 1)
as well as 2-D X and Y."""
import numpy as np

assert np.finfo(np.longdouble).nmant >= 63, "the fp64 reference needs an x87-extended or quad np.longdouble"

_CHUNK = 1 << 23  # products held at once (entries x columns): keeps the wide temporaries to a few hundred MB


def wide(dtype):
    """The reference's working format: fp32 products are exact in float64, fp64 products nearly so in long double."""
    return np.float64 if np.dtype(dtype) == np.float32 else np.longdouble


def unit_roundoff(dtype):
    return float(np.finfo(dtype).eps) / 2


def gamma(n, u):
    """Higham's gamma_n = n*u / (1 - n*u): bound on |prod (1 + d_i)^(+-1) - 1| over n roundings with |d_i| <= u."""
    n = np.asarray(n, dtype=np.float64)
    return n * u / (1.0 - n * u)


def _op_rows(rp, ci, ncols, trans):
    """Rows of op(A) as (start offsets, row of A of each entry, column of X of each entry, permutation of the entries).
    For T/H the entries are stably sorted by column, so row c of op(A) is column c of A in storage order."""
    rp = np.asarray(rp, dtype=np.int64)
    ci = np.asarray(ci, dtype=np.int64)
    m = len(rp) - 1
    arow = np.repeat(np.arange(m, dtype=np.int64), np.diff(rp))
    if not trans:
        return rp, arow, ci, None
    order = np.argsort(ci, kind="stable")
    starts = np.zeros(ncols + 1, dtype=np.int64)
    np.cumsum(np.bincount(ci, minlength=ncols), out=starts[1:])
    return starts, ci[order], arow[order], order


def _segment_sums(starts, xrow, w, X, dt):
    """out[r, :] = sum over entries e of row r of w[e] * X[xrow[e], :], in dt; rows without entries give 0.
    np.add.reduceat over the non-empty rows only (it returns the element itself, not 0, for an empty segment)."""
    nrows = len(starts) - 1
    k = X.shape[1]
    out = np.zeros((nrows, k), dtype=dt)
    lens = np.diff(starts)
    nz = np.flatnonzero(lens > 0)
    if len(nz) == 0 or k == 0:
        return out
    step = max(1, _CHUNK // max(k, 1))
    i = 0
    while i < len(nz):
        # a block of non-empty rows whose entries fit in one chunk (at least one row, however long)
        e0 = starts[nz[i]]
        j = int(np.searchsorted(starts[nz + 1], e0 + step, side="right"))
        j = max(j, i + 1)
        rows = nz[i:j]
        e1 = starts[rows[-1] + 1]
        prod = w[e0:e1, None].astype(dt) * X[xrow[e0:e1]].astype(dt)
        out[rows] = np.add.reduceat(prod, starts[rows] - e0, axis=0)
        i = j
    return out


def _check_args(rp, ci, v, X, Y0):
    X = np.asarray(X)
    Y0 = np.asarray(Y0)
    if X.ndim == 1:
        X = X[:, None]
    if Y0.ndim == 1:
        Y0 = Y0[:, None]
    assert X.shape[1] == Y0.shape[1], (X.shape, Y0.shape)
    assert len(ci) == len(v) == int(rp[-1]) - int(rp[0]) and int(rp[0]) == 0
    return X, Y0


def spmm_exact(rp, ci, v, X, Y0, alpha, beta, trans=False):
    """beta*Y0 + alpha*op(A)*X in the wide format of v's dtype (float64 for fp32, np.longdouble for fp64).

    A is (rp, ci, v) with as many columns as op(A)'s shape needs: rows of Y0 are the rows of op(A), rows of X its columns.
    alpha and beta are first rounded to v's dtype, as the library receives them.  beta == 0 ignores Y0 (NaN included);
    alpha == 0 gives beta*Y0 without reading X (KokkosSparse_spmv.hpp:145-154).  The product of two fp32 numbers is exact in
    float64 and of two fp64 numbers nearly so in long double, and the sums carry about len*2^-53 resp. len*2^-64 relative
    error -- spmm_bound adds that in as well."""
    X, Y0 = _check_args(rp, ci, v, X, Y0)
    dt = wide(v.dtype)
    a = dt(np.asarray(alpha, dtype=v.dtype))
    b = dt(np.asarray(beta, dtype=v.dtype))
    out = np.zeros(Y0.shape, dtype=dt)
    if b != 0:
        out += b * Y0.astype(dt)
    if a == 0:
        return out
    starts, _, xrow, order = _op_rows(rp, ci, Y0.shape[0] if trans else None, trans)
    w = v if order is None else v[order]
    with np.errstate(invalid="ignore"):  # an Inf in X times a zero of A is NaN, as on the device
        out += a * _segment_sums(starts, xrow, w, X, dt)
    return out


def op_row_lengths(rp, ci, nrows_out, trans=False):
    """Entries in each row of op(A), duplicates counted."""
    if not trans:
        return np.diff(np.asarray(rp, dtype=np.int64))
    return np.bincount(np.asarray(ci, dtype=np.int64), minlength=nrows_out)


def spmm_bound(rp, ci, v, X, Y0, alpha, beta, trans=False):
    """Per entry of Y: gamma(len_i + 4) * (|alpha| * sum_j |a_ij||x_jc| + |beta||y0_ic|) + the reference's own error.

    gamma(n) = n*u / (1 - n*u), u = eps/2 of v's dtype, len_i the length of row i of op(A) (not the matrix maximum).

    Derivation (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., sections 3.1 and 3.3).  The computed entry
    is a sum of len_i + 1 terms: beta*y0 and the len_i products alpha*a_ij*x_jc.  Whatever the order or tree of the
    additions, an addition tree over len_i + 1 leaves has at most len_i levels, so each term passes through at most len_i
    rounded additions -- a split of the row into pieces or segments, a shuffle or shared-memory reduce, an atomicAdd onto a
    pre-scaled beta*y0 are all such trees.  A product a_ij*x_jc is rounded at most once (not at all when it is fused into
    an FMA).  alpha is applied with at most two roundings: once to a partial sum (or to a_ij, or to the product) and once
    more when a kernel folds it into a partial before the final multiply-add.  beta*y0 is rounded once, and the final
    multiply-add beta*y0 + alpha*s adds at most one rounding that the addition count above already includes.  So every
    term carries a factor (1 + theta) with |theta| <= gamma(len_i + 3) (Higham lemma 3.1, which also covers FMA: a fused
    multiply-add is one rounding of the exact a*b + c), and the error is at most gamma(len_i + 3) times the sum of the
    terms' magnitudes.  The bound uses len_i + 4, one spare rounding; it still fails any kernel that drops a term larger
    than about (len_i + 4)*u of the row's scale.  Underflow is not modelled: the test data keep products far from the
    subnormal range.

    The reference itself is off from the exact value by at most gamma_w(len_i + 2) times the same scale, with u_w the
    unit roundoff of its wide format (2^-53 for fp32 data, 2^-64 for fp64 data); that is added so the bound holds against
    the reference, not only against the exact product."""
    scale = spmm_scale(rp, ci, v, X, Y0, alpha, beta, trans)
    lens = op_row_lengths(rp, ci, scale.shape[0], trans).astype(np.float64)
    u = unit_roundoff(v.dtype)
    uw = unit_roundoff(wide(v.dtype))
    factor = gamma(lens + 4, u) + gamma(lens + 2, uw)
    # the scale is summed in float64: at most (len + 1)*2^-53 relative error, far below the spare rounding above
    return factor[:, None] * scale


def spmm_scale(rp, ci, v, X, Y0, alpha, beta, trans=False):
    """|alpha| * sum_j |a_ij||x_jc| + |beta||y0_ic| in float64 (the Y0 term only for beta != 0, the A term only for
    alpha != 0, as the product reads them)."""
    X, Y0 = _check_args(rp, ci, v, X, Y0)
    a = abs(float(np.asarray(alpha, dtype=v.dtype)))
    b = abs(float(np.asarray(beta, dtype=v.dtype)))
    scale = np.zeros(Y0.shape, dtype=np.float64)
    if b != 0:
        scale += b * np.abs(Y0.astype(np.float64))
    if a != 0:
        starts, _, xrow, order = _op_rows(rp, ci, Y0.shape[0] if trans else None, trans)
        w = np.abs(v if order is None else v[order]).astype(np.float64)
        with np.errstate(invalid="ignore"):  # 0 * Inf where X holds an Inf: that entry's exact value is not finite either
            scale += a * _segment_sums(starts, xrow, w, np.abs(X.astype(np.float64)), np.float64)
    return scale


def bsr_to_point_crs(bs, rp, ci, v):
    """A BsrMatrix (block row map rp, block columns ci, values of nnzb blocks of bs x bs, each row-major as the library
    stores them) as point CSR (rp, ci, v).  Point row br*bs + i holds, block by block in storage order, the bs entries of
    row i of each block of block row br at columns ci[k]*bs + j.  Its length is bs * (block degree), the len_i the bound
    of a block kernel's row needs: every point entry of a block is one term, explicit zeros included."""
    bs = int(bs)
    rp = np.asarray(rp, dtype=np.int64)
    ci = np.asarray(ci, dtype=np.int64)
    v = np.asarray(v)
    mb = len(rp) - 1
    nnzb = int(rp[-1])
    assert len(ci) == nnzb and v.size == nnzb * bs * bs
    deg = np.diff(rp)
    prp = np.zeros(mb * bs + 1, dtype=np.int64)
    np.cumsum(np.repeat(deg * bs, bs), out=prp[1:])
    assert prp[-1] < 2**31
    # entry (i, j) of block k (the q-th of its block row br) goes to bs*bs*rp[br] + bs*(i*deg[br] + q) + j: block row, then
    # point row inside the block, then block of the row, then column inside the block
    br = np.repeat(np.arange(mb, dtype=np.int64), deg)
    q = np.arange(nnzb, dtype=np.int64) - rp[br]
    i = np.arange(bs, dtype=np.int64)[None, :, None]
    j = np.arange(bs, dtype=np.int64)[None, None, :]
    pos = bs * bs * rp[br][:, None, None] + bs * (i * deg[br][:, None, None] + q[:, None, None]) + j
    pci = np.empty(nnzb * bs * bs, dtype=np.int32)
    pv = np.empty(nnzb * bs * bs, dtype=v.dtype)
    pci[pos.reshape(-1)] = np.broadcast_to(ci[:, None, None] * bs + j, pos.shape).reshape(-1)
    pv[pos.reshape(-1)] = v.reshape(-1)
    return prp.astype(np.int32), pci, pv


def assert_within(got, exact, bound, what):
    """Fail on the first entry (row-major order) of `got` that is further than `bound` from `exact`, or that is NaN/Inf
    where `exact` is finite.  Where `exact` is NaN, `got` must be NaN; where it is +-Inf, `got` must be the same Inf.
    `what` names the call (the tests put the handle's last_kernel() in it)."""
    got = np.asarray(got)
    exact = np.asarray(exact)
    if got.ndim == 1:
        got = got[:, None]
    if exact.ndim == 1:
        exact = exact[:, None]
    bound = np.broadcast_to(np.asarray(bound, dtype=np.float64).reshape(exact.shape[0], -1), exact.shape)
    assert got.shape == exact.shape, f"{what}: shape {got.shape} != {exact.shape}"
    gw = got.astype(exact.dtype)
    fin = np.isfinite(exact)
    with np.errstate(invalid="ignore", over="ignore"):
        err = np.abs(gw - exact)
        bad = np.where(fin, ~(err <= bound), ~((np.isnan(exact) & np.isnan(gw)) | (gw == exact)))
    if bad.any():
        r, c = (int(t) for t in np.argwhere(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} entries off; first at row {r}, column {c}: got {got[r, c]!r}, "
                             f"exact {exact[r, c]!r}, error {float(err[r, c]):.3e}, bound {float(bound[r, c]):.3e}")


# ---- SpGEMM: C = A*B and spgemm_jacobi's C = B - omega*diag(dinv)*A*B ----------------------------------------------------
def product_rows(A, B):
    """Products per row of A*B (int64)."""
    rpA, ciA = np.asarray(A[0], dtype=np.int64), np.asarray(A[1], dtype=np.int64)
    lenB = np.diff(np.asarray(B[0], dtype=np.int64))
    per_entry = lenB[ciA]
    cum = np.concatenate([[0], np.cumsum(per_entry)])
    return cum[rpA[1:]] - cum[rpA[:-1]]


def _spgemm_parts(A, B, omega=None, dinv=None):
    """Structure of A*B with, per entry, the wide sum, the number n_ij of products that land on it and the sum of their
    magnitudes (float64).  With omega / dinv: the sums are of -omega*dinv_i*a_ik*b_kj plus b_ij where (i, j) is in the
    pattern of A*B, and the magnitudes include |b_ij|.  Rows are expanded in blocks of at most _CHUNK products, each block
    sorted by (row, column); nothing of size k is allocated."""
    rpA, ciA, vA = (np.asarray(x) for x in A)
    rpB, ciB, vB = (np.asarray(x) for x in B)
    dtype = vA.dtype
    dt = wide(dtype)
    m = len(rpA) - 1
    rpA64, rpB64 = rpA.astype(np.int64), rpB.astype(np.int64)
    lenB = np.diff(rpB64)
    per_entry = lenB[ciA.astype(np.int64)]
    cumE = np.concatenate([[0], np.cumsum(per_entry)])  # products before entry e of A
    prow = cumE[rpA64]  # products before row i
    ncol = int(ciB.max()) + 1 if len(ciB) else 1
    jac = omega is not None
    if jac:
        wrow = -(dt(np.asarray(omega, dtype=dtype)) * np.asarray(dinv, dtype=dtype).astype(dt))  # -omega*dinv_i, wide
    out_len = np.zeros(m, dtype=np.int64)
    cols, vals, cnts, scales = [], [], [], []
    r0 = 0
    while r0 < m:
        r1 = int(np.searchsorted(prow, prow[r0] + _CHUNK, side="right")) - 1
        r1 = min(max(r1, r0 + 1), m)
        e0, e1 = int(rpA64[r0]), int(rpA64[r1])
        cnt = per_entry[e0:e1]
        P = int(cnt.sum())
        ent = np.repeat(np.arange(e0, e1, dtype=np.int64), cnt)  # entry of A of each product
        within = np.arange(P, dtype=np.int64) - np.repeat(cumE[e0:e1] - cumE[e0], cnt)
        bidx = rpB64[ciA[ent].astype(np.int64)] + within
        arow = np.repeat(np.arange(r0, r1, dtype=np.int64), np.diff(rpA64[r0:r1 + 1]))
        row = np.repeat(arow - r0, cnt)
        col = ciB[bidx].astype(np.int64)
        a = vA[ent].astype(dt)
        if jac:
            a = wrow[row + r0] * a
        term = a * vB[bidx].astype(dt)
        mag = np.abs(term.astype(np.float64))
        key = row * ncol + col
        order = np.argsort(key, kind="stable")
        key, term, mag = key[order], term[order], mag[order]
        first = np.flatnonzero(np.concatenate([[True], key[1:] != key[:-1]])) if P else np.zeros(0, np.int64)
        ukey = key[first]
        s = np.add.reduceat(term, first) if P else np.zeros(0, dt)
        sc = np.add.reduceat(mag, first) if P else np.zeros(0)
        n = np.diff(np.concatenate([first, [P]]))
        urow, ucol = ukey // ncol, ukey % ncol
        if jac:  # row i of B, weight 1, where its column is in the pattern
            b0, b1 = int(rpB64[min(r0, len(rpB64) - 1)]), int(rpB64[min(r1, len(rpB64) - 1)])
            brow = np.repeat(np.arange(r0, min(r1, len(rpB64) - 1), dtype=np.int64), lenB[r0:r1]) - r0
            bkey = brow * ncol + ciB[b0:b1].astype(np.int64)
            pos = np.searchsorted(ukey, bkey)
            hit = pos < len(ukey)
            hit[hit] = ukey[pos[hit]] == bkey[hit]
            s[pos[hit]] += vB[b0:b1][hit].astype(dt)  # columns are distinct within a row of B
            sc[pos[hit]] += np.abs(vB[b0:b1][hit].astype(np.float64))
        out_len[r0:r1] = np.bincount(urow, minlength=r1 - r0)
        cols.append(ucol.astype(np.int32))
        vals.append(s.astype(dt))
        cnts.append(n)
        scales.append(sc)
        r0 = r1
    rp = np.concatenate([[0], np.cumsum(out_len)])
    assert rp[-1] < 2**31
    cat = lambda xs, t: np.concatenate(xs) if xs else np.zeros(0, t)
    return rp.astype(np.int32), cat(cols, np.int32), cat(vals, dt), cat(cnts, np.int64), cat(scales, np.float64)


def spgemm_exact(A, B):
    """C = A*B for A = (row_map, entries, values), B likewise: (row_map, entries, values) with sorted rows, the values in the
    wide format of A's dtype.  Every product (i, c, a*b) is expanded, sorted by (row, column) and reduced; an entry whose
    products cancel to 0 stays in the structure, as in the library's symbolic phase."""
    rp, ci, v, _, _ = _spgemm_parts(A, B)
    return rp, ci, v


def spgemm_bound(A, B):
    """Per entry of spgemm_exact: gamma(n_ij + 2, u) * S_ij + gamma(n_ij + 1, u_w) * S_ij, S_ij = sum |a_ik b_kj| over the
    n_ij products that land on (i, j) (not the row's maximum), u the unit roundoff of the data and u_w that of the wide
    format.

    Derivation (as spmm_bound's).  Each product b_kj*a_ik is rounded once.  However the kernel groups the additions -- a
    sorted run added left to right, a shared-memory atomicAdd per product onto a zero slot, a global hash slot -- they form
    a tree over the n_ij products, plus at most one addition onto the initial +0 (exact, but counted), so each product
    passes through at most n_ij rounded additions: n_ij + 1 roundings in all, a factor (1 + theta), |theta| <=
    gamma(n_ij + 1).  One spare rounding gives n_ij + 2.  The wide reference rounds each product at most once (fp64 data in
    long double) and its sorted sum has n_ij - 1 additions: gamma_w(n_ij + 1) covers it, so the bound holds against the
    reference and not only against the exact product.  Underflow is not modelled."""
    _, _, _, n, S = _spgemm_parts(A, B)
    return _spgemm_factor(A[2].dtype, n, 2, 1) * S


def _spgemm_factor(dtype, n, extra, extra_w):
    n = n.astype(np.float64)
    return gamma(n + extra, unit_roundoff(dtype)) + gamma(n + extra_w, unit_roundoff(wide(dtype)))


def spgemm_ref(A, B):
    """(row_map, entries, exact values, bound) in one expansion."""
    rp, ci, v, n, S = _spgemm_parts(A, B)
    return rp, ci, v, _spgemm_factor(A[2].dtype, n, 2, 1) * S


def jacobi_exact(A, B, omega, dinv):
    """spgemm_jacobi's C = B - omega*diag(dinv)*A*B on the pattern of A*B (the library's symbolic structure): entry (i, j)
    is b_ij (0 where B has no entry) - omega*dinv_i*sum_k a_ik b_kj.  omega and dinv are rounded to the data type first, as
    the library receives them.  Where A lacks its diagonal, entries of row i of B outside the pattern are dropped."""
    rp, ci, v, _, _ = _spgemm_parts(A, B, omega, dinv)
    return rp, ci, v


def jacobi_bound(A, B, omega, dinv):
    """Per entry of jacobi_exact: gamma(n_ij + 4, u) * S_ij + gamma(n_ij + 4, u_w) * S_ij, S_ij = |b_ij| + sum |omega dinv_i
    a_ik b_kj| over the n_ij products of A*B on (i, j).

    Each product carries three roundings -- mult = -omega*dinv[i], a*mult, b*(a*mult) -- and b_ij none (weight 1); the
    n_ij + 1 terms meet in a tree of at most n_ij rounded additions (plus the exact one onto +0), so every term is within
    gamma(n_ij + 3) relatively; one spare rounding gives n_ij + 4.  The wide reference rounds each product at most three
    times and adds n_ij times: gamma_w(n_ij + 4) covers it."""
    _, _, _, n, S = _spgemm_parts(A, B, omega, dinv)
    return _spgemm_factor(A[2].dtype, n, 4, 4) * S


def jacobi_ref(A, B, omega, dinv):
    """(row_map, entries, exact values, bound) in one expansion."""
    rp, ci, v, n, S = _spgemm_parts(A, B, omega, dinv)
    return rp, ci, v, _spgemm_factor(A[2].dtype, n, 4, 4) * S


# ---- Gauss-Seidel: one point sweep (gs.cu), and the two-stage / classic forms (gs2.cu, sptrsv.cu) --------------------------
def _rows_of(rp):
    rp = np.asarray(rp, dtype=np.int64)
    return np.repeat(np.arange(len(rp) - 1, dtype=np.int64), np.diff(rp))


def _segment_max(starts, vals, empty):
    """out[r] = max of vals over the entries of row r (int64); `empty` for rows without entries."""
    nrows = len(starts) - 1
    out = np.full(nrows, empty, dtype=np.int64)
    nz = np.flatnonzero(np.diff(starts) > 0)
    if len(nz):
        out[nz] = np.maximum.reduceat(np.asarray(vals, dtype=np.int64), np.asarray(starts, dtype=np.int64)[nz])
    return out


def _row_sums(starts, w, xe, dt):
    """sum over the entries e of row r of w[e] * xe[e] in dt (xe already gathered per entry)."""
    return _segment_sums(np.asarray(starts, dtype=np.int64), np.arange(len(w), dtype=np.int64), w, np.asarray(xe)[:, None], dt)[:, 0]


def _gs_sweep_parts(rp, ci, v, colors, x_old, x_new, y, omega, direction):
    dtype = v.dtype
    dt = wide(dtype)
    rp = np.asarray(rp, dtype=np.int64)
    ci = np.asarray(ci, dtype=np.int64)
    n = len(rp) - 1
    row = _rows_of(rp)
    colors = np.asarray(colors, dtype=np.int64)
    assert direction in (1, 2), "one forward (1) or one backward (2) sweep"
    sq = ci < n
    cc = np.full(len(ci), -1, dtype=np.int64)
    cc[sq] = colors[ci[sq]]
    diag = ci == row
    # forward: columns of an earlier colour were swept before row i and hold their new value; backward: the mirror image.
    # The diagonal and the ghost columns read x_old.
    newer = (cc < colors[row]) if direction == 1 else (cc > colors[row])
    newer &= sq & ~diag
    x_old = np.asarray(x_old)
    xe = np.where(newer, np.asarray(x_new)[ci], x_old[ci])
    dpiece = np.where(diag, v, 0).astype(dtype)
    same_sign = np.ones(n, dtype=bool)
    if diag.any():
        pos = np.bincount(row[diag & (v > 0)], minlength=n)
        neg = np.bincount(row[diag & (v < 0)], minlength=n)
        same_sign = (pos == 0) | (neg == 0)
    assert same_sign.all(), "a row's diagonal pieces must share a sign (their sum then has a relative error bound)"
    ndiag = np.bincount(row[diag], minlength=n)
    assert (ndiag > 0).all(), "every row needs a diagonal entry"
    d = _row_sums(rp, dpiece, np.ones(len(ci)), dt)
    s = _row_sums(rp, v, xe, dt)
    om = dt(np.asarray(omega, dtype=dtype))
    exact = x_old[:n].astype(dt) + om * (np.asarray(y).astype(dt) - s) / d
    mag = _row_sums(rp, np.abs(v).astype(np.float64), np.abs(xe.astype(np.float64)), np.float64)
    scale = np.abs(x_old[:n].astype(np.float64)) + abs(float(om)) / np.abs(d.astype(np.float64)) * (np.abs(np.asarray(y, np.float64)) + mag)
    steps = np.diff(rp).astype(np.float64) + 4 + ndiag
    bound = (gamma(steps, unit_roundoff(dtype)) + gamma(steps, unit_roundoff(dt))) * scale
    return exact, bound


def gs_sweep_exact(rp, ci, v, colors, x_old, x_new, y, omega, direction):
    """Rows 0 .. n-1 of one point Gauss-Seidel sweep, each computed from the kernel's own neighbour values: row i of colour
    c reads x_new_j where colour(j) < c (forward, direction 1) or colour(j) > c (backward, direction 2), x_old_j otherwise,
    and x_old on its diagonal and ghost columns (j >= n).  Value x_old_i + omega * (y_i - sum_j a_ij x*_j) / d_i with d_i
    the exact sum of the row's diagonal entries, in the wide format; omega is first rounded to v's dtype.  A local check:
    the error of one row does not travel along the colour chain into the next one's reference."""
    return _gs_sweep_parts(rp, ci, v, colors, x_old, x_new, y, omega, direction)[0]


def gs_sweep_bound(rp, ci, v, colors, x_old, x_new, y, omega, direction):
    """Per row of gs_sweep_exact: gamma(len_i + 4 + ndiag_i) * (|x_old_i| + |omega| / |d_i| * (|y_i| + sum_j |a_ij x*_j|)),
    plus the same with the wide format's unit roundoff.

    The kernel rounds each product a_ij x*_j once (or fuses it) and adds the len_i products in some tree (at most len_i
    levels with the subtraction from y_i), multiplies by omega and by its inverse diagonal, and adds x_old_i: every term
    passes through at most len_i + 3 roundings there.  The inverse diagonal is 1/d̂_i with d̂_i the rounded sum of ndiag_i
    pieces of one sign: ndiag_i - 1 roundings, and one more for the division, counted as a rounding rather than reproduced,
    so the bound holds whether or not the division is IEEE and with or without FMA contraction.  Total len_i + 4 + ndiag_i
    - 1, one spare.  The wide reference does the same operations in its own format."""
    return _gs_sweep_parts(rp, ci, v, colors, x_old, x_new, y, omega, direction)[1]


_gamma_n = gamma  # the two-stage functions take a parameter named gamma


class _Tracked:
    """A vector of the two-stage evaluator: its value in the wide format (or the data's own, for a plain run), its magnitude
    -- the same expression evaluated on |inputs| with every subtraction an addition -- and per entry the depth, the most
    rounding steps on any path from an input to it.  For a straight-line program of additions, multiplications and
    divisions by inputs, the computed value differs from the exact one by at most gamma(depth) * magnitude (Higham, lemma
    3.1 and the bookkeeping of section 3.4, applied per monomial)."""

    def __init__(self, val, mag, dep):
        self.val, self.mag, self.dep = val, mag, np.asarray(dep, dtype=np.int64)

    def copy(self):
        return _Tracked(self.val.copy(), self.mag.copy(), self.dep.copy())


class _Gs2Program:
    def __init__(self, rp, ci, v, dinv, dt):
        self.dtype = v.dtype
        self.dt = dt
        self.rp = np.asarray(rp, dtype=np.int64)
        self.ci = np.asarray(ci, dtype=np.int64)
        self.v = v
        self.n = n = len(self.rp) - 1
        row = self.row = _rows_of(self.rp)
        diag = self.ci == row
        idx = np.flatnonzero(diag)
        r = row[idx]
        assert len(np.unique(r)) == n, "every row needs a diagonal entry"
        last = np.r_[r[1:] != r[:-1], True]  # numeric keeps the last diagonal entry of a row
        a_d = np.zeros(n, dtype=self.dtype)
        a_d[r[last]] = v[idx[last]]
        self.Da = a_d
        if dinv is None:  # D = 1/a_ii: one rounding
            self.D = (dt(1) / a_d.astype(dt)), np.abs(1.0 / a_d.astype(np.float64)), 1
        else:
            dinv = np.asarray(dinv, dtype=self.dtype)
            self.D = dinv.astype(dt), np.abs(dinv.astype(np.float64)), 0
        self.given = dinv is not None
        lower, upper, ghost = self.ci < row, (self.ci > row) & (self.ci < n), self.ci >= n
        self.parts = {"A": np.ones(len(self.ci), dtype=bool), "L": lower, "U": upper, "La": lower | ghost, "Ua": upper | ghost}

    def _sub(self, mask):
        starts = np.zeros(self.n + 1, dtype=np.int64)
        np.cumsum(np.bincount(self.row[mask], minlength=self.n), out=starts[1:])
        return starts, self.ci[mask], self.v[mask], self.row[mask]

    def matvec(self, part, alpha, x, y0, scaled=False):
        """y0 + alpha * M x, M the part of A (scaled: rows times D, the values numeric stores for L and U)."""
        starts, c, w, r = self._sub(self.parts[part])
        dt = self.dt
        ww, wm, wdep = w.astype(dt), np.abs(w.astype(np.float64)), 0
        if scaled:
            Dv, Dm, Dd = self.D
            ww, wm, wdep = ww * Dv[r], wm * Dm[r], Dd + 1
        al = dt(np.asarray(alpha, dtype=self.dtype))
        with np.errstate(invalid="ignore"):
            val = y0.val + al * _row_sums(starts, ww, x.val[c], dt)
        mag = y0.mag + abs(float(al)) * _row_sums(starts, wm, x.mag[c], np.float64)
        dep = np.maximum(y0.dep, _segment_max(starts, x.dep[c] + wdep, 0)) + np.diff(starts) + 4
        return _Tracked(val, mag, dep)

    def dscale(self, r):  # D .* r
        Dv, Dm, Dd = self.D
        return _Tracked(Dv * r.val, Dm * r.mag, r.dep + Dd + 1)

    def scal(self, g, x):
        gw = self.dt(np.asarray(g, dtype=self.dtype))
        return _Tracked(gw * x.val, abs(float(gw)) * x.mag, x.dep + 1)

    def damp(self, g, z, r):  # g z + (1 - g) r, with 1 - g rounded once
        gw = self.dt(np.asarray(g, dtype=self.dtype))
        hw = self.dt(1) - gw
        return _Tracked(gw * z.val + hw * r.val, abs(float(gw)) * z.mag + abs(float(hw)) * r.mag,
                        np.maximum(z.dep + 2, r.dep + 3))

    def diag_term(self, om2, x, r):  # r + om2 * (Da .* x)
        ow = self.dt(om2)
        return _Tracked(r.val + ow * self.Da.astype(self.dt) * x.val[:self.n],
                        r.mag + abs(float(ow)) * np.abs(self.Da.astype(np.float64)) * x.mag[:self.n],
                        np.maximum(r.dep, x.dep[:self.n] + 2) + 1)

    def update(self, x, z, omega, overwrite):
        ow = self.dt(np.asarray(omega, dtype=self.dtype))
        y = x.copy()
        n = self.n
        if overwrite:
            y.val[:n], y.mag[:n], y.dep[:n] = ow * z.val, abs(float(ow)) * z.mag, z.dep + 1
        else:
            y.val[:n] = x.val[:n] + ow * z.val
            y.mag[:n] = x.mag[:n] + abs(float(ow)) * z.mag
            y.dep[:n] = np.maximum(x.dep[:n], z.dep + 1) + 1
        return y

    def trsv(self, r, forward):
        """(L + D)^{-1} r (forward) or (U + D)^{-1} r, D the diagonal entry or 1/dinv; rows in dependency levels."""
        dt, n = self.dt, self.n
        starts, c, w, rr = self._sub(self.parts["L" if forward else "U"])
        lvl = np.zeros(n, dtype=np.int64)
        while True:  # longest chain below each row
            nl = _segment_max(starts, lvl[c] + 1, 0)
            if np.array_equal(nl, lvl):
                break
            lvl = nl
        if self.given:
            inv, invm = self.D[0], self.D[1]
        else:
            inv, invm = dt(1) / self.Da.astype(dt), np.abs(1.0 / self.Da.astype(np.float64))
        z = _Tracked(np.zeros(n, dtype=dt), np.zeros(n), np.zeros(n, dtype=np.int64))
        for L in range(int(lvl.max()) + 1 if n else 0):
            rows = np.flatnonzero(lvl == L)
            lens = starts[rows + 1] - starts[rows]
            sub = np.zeros(len(rows) + 1, dtype=np.int64)
            np.cumsum(lens, out=sub[1:])
            e = np.repeat(starts[rows] - sub[:-1], lens) + np.arange(int(sub[-1]), dtype=np.int64)
            s = _segment_sums(sub, c[e], w[e], z.val[:, None], dt)[:, 0] if len(e) else np.zeros(len(rows), dt)
            sm = _segment_sums(sub, c[e], np.abs(w[e]).astype(np.float64), z.mag[:, None], np.float64)[:, 0] if len(e) else 0.0
            z.val[rows] = (r.val[rows] - s) * inv[rows]
            z.mag[rows] = (r.mag[rows] + sm) * invm[rows]
            z.dep[rows] = np.maximum(r.dep[rows], _segment_max(sub, z.dep[c[e]] + 1, 0) if len(e) else 0) + lens + 1 + int(self.given)
        return z


def _gs2_run(rp, ci, v, ncols, x0, b, init_zero, omega, num_iter, direction, compact, inner, outer, gamma_, two_stage, dinv, dt,
             variant=None):
    dtype = v.dtype
    P = _Gs2Program(rp, ci, v, dinv, dt)
    n = P.n
    one = dtype.type(1)
    om = dtype.type(omega)
    g = dtype.type(gamma_)
    inp = lambda a: _Tracked(np.asarray(a).astype(dt), np.abs(np.asarray(a).astype(np.float64)), np.zeros(len(a), dtype=np.int64))
    x = inp(np.zeros(ncols, dtype) if init_zero else np.asarray(x0)[:ncols])  # init_zero: all ncols entries, ghosts included
    bt = inp(b)
    sweeps = max(outer, num_iter) * (2 if direction == 0 else 1)
    for sweep in range(sweeps):
        forward = direction == 1 or (direction == 0 and sweep % 2 == 0)
        R = bt.copy()
        if sweep > 0 or not init_zero:
            if compact:
                R = P.matvec("Ua" if forward else "La", -1.0, x, R)
                if om != one:
                    with np.errstate(divide="ignore"):
                        R = P.diag_term(one / om - one, x, R)  # the scalar as the host computes it in the data's type
            else:
                R = P.matvec("A", -1.0, x, R)
        if not two_stage:
            Z = P.trsv(R, forward)
            x = P.update(x, Z, 1.0, compact)
            continue
        if inner == 0:
            Z = P.dscale(R)
            if g != one:
                Z = P.scal(g, Z)
        else:
            T = P.dscale(R)
            R = T.copy()
            if g != one:
                R = P.scal(g, R)
            for ii in range(inner):
                Z = P.matvec("L" if forward else "U", -om, R, T, scaled=True)
                if g != one:
                    Z = P.damp(g, Z, Z if variant == "damp_z" else R)
                if ii + 1 < inner:
                    R = Z
        x = P.update(x, Z, om, compact and variant != "accumulate")
    return x


def gs2_exact(rp, ci, v, ncols, x0, b, init_zero, omega, num_iter, direction, compact=False, inner_sweeps=1, outer_sweeps=1, gamma=1.0,
              two_stage=True, inverse_diagonal=None):
    """x (ncols entries) after b200sp_gs2_apply, in the wide format, for one right-hand side.

    The algorithm as the reference's TwostageGaussSeidel::apply states it (sparse/impl/KokkosSparse_twostage_gauss_seidel_impl.hpp
    :778-1035): NumSweeps = max(outer, numIter), doubled for symmetric (forward, backward, ...); init_zero zeroes all ncols
    entries of x, ghosts included.  Per sweep R = b - A x (compact: b - Ua x or b - La x, plus (1/omega - 1) Da.*x when
    omega != 1; skipped on the first sweep after init_zero).  Two-stage: Z = gamma D.*R without inner sweeps; otherwise T = D.*R,
    R = gamma T, and per inner sweep Z = T - omega (DL or DU) R, Z = gamma Z + (1 - gamma) R when gamma != 1, R = Z before the
    next; then x += omega Z (compact: x = omega Z).  Classic (two_stage = False, omega = 1): Z = (L + D)^{-1} R or (U + D)^{-1}
    R, then x += Z (compact: x = Z).  D = 1 / a_ii, or the caller's inverse diagonal; a_ii is the row's (last) diagonal entry.
    omega, gamma and the inverse diagonal are first rounded to v's dtype, and 1/omega - 1 is the data-type scalar the host
    computes, as the library receives them."""
    return _gs2_run(rp, ci, v, ncols, x0, b, init_zero, omega, num_iter, direction, compact, inner_sweeps, outer_sweeps, gamma, two_stage,
                    inverse_diagonal, wide(v.dtype)).val


def gs2_bound(rp, ci, v, ncols, x0, b, init_zero, omega, num_iter, direction, compact=False, inner_sweeps=1, outer_sweeps=1, gamma=1.0,
              two_stage=True, inverse_diagonal=None):
    """Per entry of gs2_exact: (gamma(depth_i, u) + gamma(depth_i, u_w)) * magnitude_i.

    The evaluator carries, with every vector, the magnitude (the program on |A|, |x|, |b|, |D|, |omega|, |gamma|, |1 - gamma|
    with subtraction replaced by addition) and per entry the rounding depth: a product with a row of len_i entries adds len_i
    + 4 to the deepest input of that row, as spmm_bound counts it (entries of DL and DU carry the rounding of a_ij * d_i, and
    of d_i = 1/a_ii); a diagonal scaling, a scaling by gamma or omega, and an update add one or two; a row of the triangular
    substitution adds its off-diagonal count, the division, and the rounding of 1/dinv when the caller supplied dinv.  The
    bound is rigorous for any evaluation order the kernels choose; the wide reference's own error is added over the same
    depth.  Ghost entries keep their input (depth 0, bound 0): they must come back unchanged."""
    x = _gs2_run(rp, ci, v, ncols, x0, b, init_zero, omega, num_iter, direction, compact, inner_sweeps, outer_sweeps, gamma, two_stage,
                 inverse_diagonal, wide(v.dtype))
    d = x.dep.astype(np.float64)
    return (_gamma_n(d, unit_roundoff(v.dtype)) + _gamma_n(d, unit_roundoff(wide(v.dtype)))) * x.mag


def gs2_ref(rp, ci, v, ncols, x0, b, init_zero, omega, num_iter, direction, compact=False, inner_sweeps=1, outer_sweeps=1, gamma=1.0,
            two_stage=True, inverse_diagonal=None):
    """(gs2_exact, gs2_bound) in one evaluation."""
    x = _gs2_run(rp, ci, v, ncols, x0, b, init_zero, omega, num_iter, direction, compact, inner_sweeps, outer_sweeps, gamma, two_stage,
                 inverse_diagonal, wide(v.dtype))
    d = x.dep.astype(np.float64)
    return x.val, (_gamma_n(d, unit_roundoff(v.dtype)) + _gamma_n(d, unit_roundoff(wide(v.dtype)))) * x.mag



def trsv_row_bound(rp, ci, v, b, z, forward, inverse_diagonal=None):
    """Local check of one triangular substitution from the kernel's own solution z: per row, the exact (b_i - sum_j a_ij z_j) / d_i
    over the lower (forward) or upper off-diagonal entries (ghost columns skipped) and the bound gamma(len_i + 2) *
    (|b_i| + sum_j |a_ij z_j|) / |d_i|, len_i the row's full length: at most len_i - 1 products and subtractions, the
    division, and the rounding of 1/dinv.  Returns (exact, bound) for rows 0 .. n-1."""
    dtype = v.dtype
    dt = wide(dtype)
    rp = np.asarray(rp, dtype=np.int64)
    ci = np.asarray(ci, dtype=np.int64)
    n = len(rp) - 1
    row = _rows_of(rp)
    take = (ci < row) if forward else ((ci > row) & (ci < n))
    w = np.where(take, v, 0).astype(dtype)
    zz = np.asarray(z)
    ze = np.where(take, zz[np.minimum(ci, n - 1)], 0).astype(dtype)
    s = _row_sums(rp, w, ze, dt)
    sm = _row_sums(rp, np.abs(w).astype(np.float64), np.abs(ze.astype(np.float64)), np.float64)
    P = _Gs2Program(rp, ci, v, inverse_diagonal, dt)
    if inverse_diagonal is not None:
        inv, invm = P.D[0], P.D[1]
    else:
        inv, invm = dt(1) / P.Da.astype(dt), np.abs(1.0 / P.Da.astype(np.float64))
    bb = np.asarray(b)
    exact = (bb.astype(dt) - s) * inv
    steps = np.diff(rp).astype(np.float64) + 2
    bound = (gamma(steps, unit_roundoff(dtype)) + gamma(steps, unit_roundoff(dt))) * (np.abs(bb.astype(np.float64)) + sm) * invm
    return exact, bound
