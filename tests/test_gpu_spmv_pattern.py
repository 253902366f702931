"""GPU checks of the tiled SpMV kernel's pattern form (one 16-bit pattern start per row into a dictionary of in-row column
offsets, plus one anchor column per row, DESIGN.md section 3.6): which matrices take it, and that it returns the same bits
as the 32-bit columns, the delta form and the row-vector kernel.  The form is known once the plan's verdict has reached the
host, so every handle is called once and synchronised before the call that is checked."""
import os

import numpy as np
import pytest
import torch

import exact_ref as R
import pattern_cases as K
from helpers import rowwise_scale

pytestmark = pytest.mark.gpu


class setenv:
    def __init__(self, **kv):
        self.kv = kv

    def __enter__(self):
        self.old = {k: os.environ.get(k) for k in self.kv}
        os.environ.update(self.kv)

    def __exit__(self, *a):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def dev(cuda, A, dtype=np.float64):
    from kokkos_kernels_b200 import sparse as sp

    rp, ci, v, ncols = A
    return sp.CrsMatrix(torch.from_numpy(rp).to(cuda), torch.from_numpy(ci).to(cuda),
                        torch.from_numpy(v.astype(dtype)).to(cuda), ncols)


def handle(cfg=-1, lpr=-1, algo=None):
    from kokkos_kernels_b200 import sparse as sp

    h = sp.SPMVHandle(sp.SPMV_DEFAULT if algo is None else algo)
    h.tune(cfg, lpr, -1)
    return h


def call(h, Ad, x, y0, alpha, beta):
    from kokkos_kernels_b200 import sparse as sp

    y = y0.clone()
    sp.spmv(h, "N", alpha, Ad, x, beta, y)
    torch.cuda.synchronize()
    return y.cpu().numpy(), h.last_kernel()


def settled(h, Ad, x, y0, alpha, beta):
    call(h, Ad, x, y0, alpha, beta)  # builds the streams; the verdict is on the host after the synchronise
    return call(h, Ad, x, y0, alpha, beta)


def inputs(cuda, A, beta, seed=0, dtype=np.float64):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-1, 1, A[3]).astype(dtype)
    y0 = rng.uniform(-1, 1, len(A[0]) - 1).astype(dtype)
    if beta == 0.0:
        y0[::7] = np.nan
    return x, y0, torch.from_numpy(x).to(cuda), torch.from_numpy(y0).to(cuda)


def check_oracle(oracle, A, x, y0, alpha, beta, y):
    rp, ci, v, _ = A
    v = v.astype(x.dtype)
    exp = oracle.spmv_serial(rp, ci, v, x, y0.copy(), alpha, beta)
    scale = rowwise_scale(rp, ci, v, x, y0, alpha, beta)
    tol = 1e-10 if x.dtype == np.float64 else 1e-4
    assert not np.isnan(y).any()
    assert np.all(np.abs(y - exp) <= tol * scale + 1e-300)
    R.assert_within(y, R.spmm_exact(rp, ci, v, x, y0, alpha, beta), R.spmm_bound(rp, ci, v, x, y0, alpha, beta), f"a={alpha} b={beta}")


def three_forms(cfg, lpr, Ad, xd, y0d, alpha, beta):
    """pattern handle, the same handle on the 32-bit columns, and a handle built under B200SP_SPMV_PATTERN=0"""
    h = handle(cfg, lpr)
    y, k = settled(h, Ad, xd, y0d, alpha, beta)
    with setenv(B200SP_SPMV_IDX16="0"):
        y32, k32 = call(h, Ad, xd, y0d, alpha, beta)
    assert "IDX=i32" in k32, k32
    with setenv(B200SP_SPMV_PATTERN="0"):
        yd, kd = settled(handle(cfg, lpr), Ad, xd, y0d, alpha, beta)
    return y, k, y32, yd, kd


@pytest.mark.parametrize("case", ["dof1", "dof2", "dof3", "flat2", "flat3", "shard"])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_lap27_pattern_same_bits(cuda, oracle, case, dtype):
    from kokkos_kernels_b200 import sparse as sp

    A = K.lap_case(case)
    Ad = dev(cuda, A, dtype)
    for alpha, beta in K.AB:
        x, y0, xd, y0d = inputs(cuda, A, beta, dtype=dtype)
        yv, kv = call(handle(lpr=4, algo=sp.SPMV_FAST_SETUP), Ad, xd, y0d, alpha, beta)
        assert kv.startswith("vector"), kv
        y, k, y32, yd, kd = three_forms(8, 4, Ad, xd, y0d, alpha, beta)
        assert "IDX=u16,COLS=pat" in k and "IDX=u16,COLS=delta" in kd, (k, kd)
        check_oracle(oracle, A, x, y0, alpha, beta, y)
        assert np.array_equal(y, y32) and np.array_equal(y, yd) and np.array_equal(y, yv), (alpha, beta)


@pytest.fixture(scope="module")
def big(cuda):
    """96^3 x 2 dof: many waves of every ring configuration"""
    A = K.lap27(96, 96, 96)
    return A, dev(cuda, A)


@pytest.mark.parametrize("lpr", [2, 4, 8, 16, 32])
def test_big_lap27_every_lpr_and_ring(cuda, big, lpr):
    A, Ad = big
    _, _, xd, y0d = inputs(cuda, A, 1.3)
    ref = None
    for cfg in (0, 1, 2, 3, 4, 8):
        y, k, y32, yd, kd = three_forms(cfg, lpr, Ad, xd, y0d, -0.7, 1.3)
        assert "COLS=pat" in k and f"LPR={lpr}," in k and "COLS=delta" in kd, (k, kd)
        assert np.array_equal(y, y32) and np.array_equal(y, yd), cfg
        ref = y if ref is None else ref
        assert np.array_equal(y, ref), cfg


def test_big_lap27_default_handle(cuda, oracle, big):
    """untuned handle (self-tuning between the tiled and the row-vector kernel): every call returns the same bits"""
    A, Ad = big
    x, y0, xd, y0d = inputs(cuda, A, 0.0)
    h = handle()
    outs = [call(h, Ad, xd, y0d, 1.0, 0.0) for _ in range(6)]
    assert any("COLS=pat" in k for _, k in outs), [k for _, k in outs]
    for y, _ in outs[1:]:
        assert np.array_equal(y, outs[0][0])


@pytest.mark.parametrize("total,form", [(K.DCAP, "pat"), (K.DCAP + 1, "delta")])
def test_dictionary_boundary(cuda, oracle, total, form):
    A = K.dict_matrix(total)
    Ad = dev(cuda, A)
    x, y0, xd, y0d = inputs(cuda, A, 0.0)
    y, k, y32, yd, _ = three_forms(8, -1, Ad, xd, y0d, 1.0, 0.0)
    assert f"COLS={form}" in k, k
    check_oracle(oracle, A, x, y0, 1.0, 0.0, y)
    assert np.array_equal(y, y32) and np.array_equal(y, yd)


@pytest.mark.parametrize("name", ["near_patterns_matrix", "diagonal_matrix", "long_rows_matrix", "empty_rows_matrix"])
@pytest.mark.parametrize("cfg", [3, 8])
def test_special_matrices(cuda, oracle, name, cfg):
    A = getattr(K, name)()
    Ad = dev(cuda, A)
    for lpr in (2, 8):
        for alpha, beta in K.AB:
            x, y0, xd, y0d = inputs(cuda, A, beta, seed=1)
            y, k, y32, yd, _ = three_forms(cfg, lpr, Ad, xd, y0d, alpha, beta)
            assert "COLS=pat" in k, k
            check_oracle(oracle, A, x, y0, alpha, beta, y)
            assert np.array_equal(y, y32) and np.array_equal(y, yd), (lpr, alpha, beta)


def test_new_col_idx_same_row_ptr(cuda, oracle):
    from kokkos_kernels_b200 import sparse as sp

    rp, ci, v, n = A1 = K.lap27(20, 18, 16)
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    ci2 = ((ci.astype(np.int64) + 2 * rows) % n).astype(np.int32)
    for r in range(len(rp) - 1):
        ci2[rp[r]:rp[r + 1]].sort()
    ci3 = K.random_rows(rp, n)
    A1d = dev(cuda, A1)
    x, y0, xd, y0d = inputs(cuda, A1, 0.0)
    h = handle(8)
    for cols in (ci, ci2, ci3, ci):
        A = (rp, cols, v, n)
        Ad = sp.CrsMatrix(A1d.row_map, torch.from_numpy(cols).to(cuda), A1d.values, n)  # the same row_ptr tensor
        y, k = settled(h, Ad, xd, y0d, 1.0, 0.0)
        assert f"IDX=u16,COLS={K.expected_cols(A, 512)}" in k, k
        check_oracle(oracle, A, x, y0, 1.0, 0.0, y)


def test_forward_and_hostvec_entries(cuda, big):
    """the fused all-gather entry and the pipelined host-vector entry take the pattern form, with the 32-bit form's bits"""
    from kokkos_kernels_b200 import sparse as sp

    A, Ad = big
    x, y0, xd, _ = inputs(cuda, A, 1.3)
    n = len(y0)
    outs = {}
    for form in ("pat", "i32"):
        with setenv(B200SP_SPMV_IDX16="0" if form == "i32" else "1"):
            h = handle(8, 4)
            for _ in range(2):
                loc = torch.full((n,), float("nan"), dtype=torch.float64, device=cuda)
                fwd = torch.full((n,), float("nan"), dtype=torch.float64, device=cuda)
                sp.spmv_forward(h, 1.0, Ad, xd, loc, fwd.data_ptr())
                torch.cuda.synchronize()
            kf = h.last_kernel()
            xh = torch.from_numpy(x).pin_memory()
            for _ in range(2):
                yh = torch.from_numpy(y0.copy()).pin_memory()
                sp.spmv_hostvec(h, "N", -0.7, Ad, xh, 1.3, yh)
                torch.cuda.synchronize()
            kh = h.last_kernel()
        want = "IDX=u16,COLS=pat" if form == "pat" else "IDX=i32"
        assert want in kf and want in kh, (kf, kh)
        assert torch.equal(loc, fwd)
        outs[form] = (loc.cpu().numpy(), yh.numpy().copy())
    assert np.array_equal(outs["pat"][0], outs["i32"][0]) and np.array_equal(outs["pat"][1], outs["i32"][1])
