"""GPU checks of the tiled SpMV kernel's 16-bit column form (in-row column deltas + one anchor per row, DESIGN.md section
3.5): the bench family takes it and returns the same bits as the 32-bit columns and the row-vector kernel; the qualification
boundary; rows the tiled kernel does not read; empty rows; a new col_idx under the same row_ptr.  The form is known once the
plan's flag has reached the host, so every handle is called once and synchronised before the call that is checked."""
import os

import numpy as np
import pytest
import torch

import idx16_cases as K
from helpers import rowwise_scale

pytestmark = pytest.mark.gpu


class idx16_off:
    def __enter__(self):
        self.old = os.environ.get("B200SP_SPMV_IDX16")
        os.environ["B200SP_SPMV_IDX16"] = "0"

    def __exit__(self, *a):
        if self.old is None:
            os.environ.pop("B200SP_SPMV_IDX16", None)
        else:
            os.environ["B200SP_SPMV_IDX16"] = self.old


def dev(cuda, A):
    from kokkos_kernels_b200 import sparse as sp

    rp, ci, v, ncols = A
    return sp.CrsMatrix(torch.from_numpy(rp).to(cuda), torch.from_numpy(ci).to(cuda), torch.from_numpy(v).to(cuda), ncols)


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


def inputs(cuda, A, beta, seed=0):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-1, 1, A[3])
    y0 = rng.uniform(-1, 1, len(A[0]) - 1)
    if beta == 0.0:
        y0[::7] = np.nan
    return x, y0, torch.from_numpy(x).to(cuda), torch.from_numpy(y0).to(cuda)


def check_oracle(oracle, A, x, y0, alpha, beta, y):
    rp, ci, v, _ = A
    exp = oracle.spmv_serial(rp, ci, v, x, y0.copy(), alpha, beta)
    scale = rowwise_scale(rp, ci, v, x, y0, alpha, beta)
    assert not np.isnan(y).any()
    assert np.all(np.abs(y - exp) <= 1e-10 * scale + 1e-300)


@pytest.fixture(scope="module")
def lap(cuda):
    A = K.lap27(48, 40, 32)
    return A, dev(cuda, A)


@pytest.mark.parametrize("lpr", [2, 4, 8, 16, 32])
def test_lap27_u16_same_bits_as_i32_and_vector(cuda, oracle, lap, lpr):
    from kokkos_kernels_b200 import sparse as sp

    A, Ad = lap
    for alpha, beta in K.AB:
        x, y0, xd, y0d = inputs(cuda, A, beta)
        yv, kv = call(handle(lpr=lpr, algo=sp.SPMV_FAST_SETUP), Ad, xd, y0d, alpha, beta)
        assert kv.startswith("vector"), kv
        if lpr == 4:
            check_oracle(oracle, A, x, y0, alpha, beta, yv)
        for cfg in range(5):
            h = handle(cfg, lpr)
            call(h, Ad, xd, y0d, alpha, beta)  # builds the stream; its verdict is on the host after the synchronise
            y16, k16 = call(h, Ad, xd, y0d, alpha, beta)
            assert "IDX=u16" in k16 and f"LPR={lpr}," in k16, k16
            with idx16_off():
                y32, k32 = call(h, Ad, xd, y0d, alpha, beta)
            assert "IDX=i32" in k32, k32
            assert np.array_equal(y16, y32) and np.array_equal(y16, yv), (cfg, alpha, beta)


def test_default_handle_takes_u16(cuda, oracle, lap):
    """untuned handle (self-tuning between the tiled and the row-vector kernel): every call returns the same bits"""
    A, Ad = lap
    x, y0, xd, y0d = inputs(cuda, A, 0.0)
    h = handle()
    outs = [call(h, Ad, xd, y0d, 1.0, 0.0) for _ in range(6)]
    assert any("IDX=u16" in k for _, k in outs), [k for _, k in outs]
    for y, _ in outs[1:]:
        assert np.array_equal(y, outs[0][0])
    check_oracle(oracle, A, x, y0, 1.0, 0.0, outs[0][0])


@pytest.mark.parametrize("gap,form", [(65535, "u16"), (65536, "i32")])
def test_gap_boundary(cuda, oracle, gap, form):
    A = K.gap_matrix(gap)
    Ad = dev(cuda, A)
    x, y0, xd, y0d = inputs(cuda, A, 0.0)
    h = handle(8)
    call(h, Ad, xd, y0d, 1.0, 0.0)
    y, k = call(h, Ad, xd, y0d, 1.0, 0.0)
    assert f"IDX={form}" in k, k
    check_oracle(oracle, A, x, y0, 1.0, 0.0, y)
    with idx16_off():
        y32, _ = call(h, Ad, xd, y0d, 1.0, 0.0)
    assert np.array_equal(y, y32)


def test_unsorted_row_keeps_i32(cuda, oracle):
    A = K.unsorted_matrix()
    Ad = dev(cuda, A)
    x, y0, xd, y0d = inputs(cuda, A, 0.5)
    h = handle(8)
    for _ in range(2):
        y, k = call(h, Ad, xd, y0d, -1.0, 0.5)
        assert "IDX=i32" in k, k
        check_oracle(oracle, A, x, y0, -1.0, 0.5, y)


@pytest.mark.parametrize("cfg", [0, 1, 3, 8])
def test_long_rows_with_wide_gaps_still_qualify(cuda, oracle, cfg):
    A = K.long_wide_matrix()
    Ad = dev(cuda, A)
    x, y0, xd, y0d = inputs(cuda, A, 0.0)
    h = handle(cfg)
    call(h, Ad, xd, y0d, 2.0, 0.0)
    y, k = call(h, Ad, xd, y0d, 2.0, 0.0)
    assert "IDX=u16" in k, k
    check_oracle(oracle, A, x, y0, 2.0, 0.0, y)
    with idx16_off():
        y32, k32 = call(h, Ad, xd, y0d, 2.0, 0.0)
    assert "IDX=i32" in k32 and np.array_equal(y, y32)


@pytest.mark.parametrize("lpr", [2, 8, 32])
def test_empty_rows_and_ragged_nnz(cuda, oracle, lpr):
    A = K.empty_rows_matrix()
    assert len(A[1]) % 8 != 0
    Ad = dev(cuda, A)
    for alpha, beta in K.AB:
        x, y0, xd, y0d = inputs(cuda, A, beta, seed=1)
        h = handle(8, lpr)
        call(h, Ad, xd, y0d, alpha, beta)
        y, k = call(h, Ad, xd, y0d, alpha, beta)
        assert "IDX=u16" in k, k
        check_oracle(oracle, A, x, y0, alpha, beta, y)
        with idx16_off():
            y32, _ = call(h, Ad, xd, y0d, alpha, beta)
        assert np.array_equal(y, y32)


def test_new_col_idx_same_row_ptr(cuda, oracle):
    from kokkos_kernels_b200 import sparse as sp

    rp, ci, v, n = A1 = K.lap27(20, 18, 16)
    rows = np.repeat(np.arange(len(rp) - 1), np.diff(rp))
    ci2 = ((ci.astype(np.int64) + 2 * rows) % n).astype(np.int32)
    for r in range(len(rp) - 1):
        ci2[rp[r]:rp[r + 1]].sort()
    A1d = dev(cuda, A1)
    A2d = sp.CrsMatrix(A1d.row_map, torch.from_numpy(ci2).to(cuda), A1d.values, n)  # the same row_ptr tensor
    x, y0, xd, y0d = inputs(cuda, A1, 0.0)
    h = handle(8)
    for A, Ad in ((A1, A1d), ((rp, ci2, v, n), A2d), (A1, A1d)):
        call(h, Ad, xd, y0d, 1.0, 0.0)
        y, k = call(h, Ad, xd, y0d, 1.0, 0.0)
        assert "IDX=u16" in k, k
        check_oracle(oracle, A, x, y0, 1.0, 0.0, y)
