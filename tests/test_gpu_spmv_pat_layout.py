"""GPU checks of the pattern form's own stage layout (DESIGN.md section 3.6: stages of PAT_CAP values and PAT_RCAP row slots,
on a tile table of its own cut with the cfg's LMAX), against the 32-bit columns on the cfg's tiles: the same bits on every
matrix, entry point and switch between the two."""
import numpy as np
import pytest
import torch

import pattern_cases as K
import test_gpu_spmv_pattern as P

pytestmark = pytest.mark.gpu

PAT_CAP, PAT_TILE_CAP, PAT_RCAP = 4096, 4040, 256
LAYOUT = f"pat<STAGES=3,CAP={PAT_CAP},RCAP={PAT_RCAP}>"


def pat_tiles(A, lmax=512):
    return len(A[1]) // (PAT_TILE_CAP - lmax - 8) + 1


def same_as_i32(cuda, A, dtype=np.float64, cfg=8, lpr=4, alpha=-0.7, beta=1.3):
    x, y0, xd, y0d = P.inputs(cuda, A, beta, dtype=dtype)
    Ad = P.dev(cuda, A, dtype)
    h = P.handle(cfg, lpr)
    y, k = P.settled(h, Ad, xd, y0d, alpha, beta)
    with P.setenv(B200SP_SPMV_IDX16="0"):
        y32, k32 = P.call(h, Ad, xd, y0d, alpha, beta)
    assert "IDX=u16,COLS=pat>" + LAYOUT in k, k
    assert "IDX=i32>grid" in k32, k32
    assert np.array_equal(y, y32), (k, k32)
    return x, y0, y


@pytest.mark.parametrize("ndof", [1, 2, 3])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_lap27_dof(cuda, oracle, ndof, dtype):
    A = K.lap27(40, 36, 32, ndof)
    for alpha, beta in K.AB:
        x, y0, y = same_as_i32(cuda, A, dtype, alpha=alpha, beta=beta)
        P.check_oracle(oracle, A, x, y0, alpha, beta, y)


@pytest.mark.parametrize("lpr", [2, 4, 8, 16, 32])
@pytest.mark.parametrize("cfg", [0, 1, 3, 8, 10])
def test_every_ring_and_lpr(cuda, cfg, lpr):
    same_as_i32(cuda, K.lap27(48, 40, 36, 2), cfg=cfg, lpr=lpr)


@pytest.mark.parametrize("name", ["diagonal_matrix", "near_patterns_matrix", "empty_rows_matrix"])
def test_rows_past_the_row_slots(cuda, oracle, name):
    """short rows: a tile holds more rows than a stage has row slots, and the rest read row_ptr, anchor and pattern start
    from global memory"""
    A = getattr(K, name)(m=200000)
    first = np.searchsorted(A[0], np.arange(pat_tiles(A)) * (PAT_TILE_CAP - 512 - 8), side="right") - 1
    assert np.max(np.diff(first)) > PAT_RCAP
    for lpr in (2, 8):
        x, y0, y = same_as_i32(cuda, A, lpr=lpr)
        P.check_oracle(oracle, A, x, y0, -0.7, 1.3, y)


def test_rows_of_lmax_and_lmax_plus_one(cuda, oracle):
    from test_emulated_spmv_pat_layout import lmax_rows_matrix

    A = lmax_rows_matrix(m=40000)
    assert K.expected_cols(A, 512) == "pat"
    for cfg in (0, 8):
        x, y0, y = same_as_i32(cuda, A, cfg=cfg)
        P.check_oracle(oracle, A, x, y0, -0.7, 1.3, y)


def test_first_call_and_switches(cuda):
    """the first calls (the verdict may still be on its way: the cfg's tiles), then the pattern tiles, the 32-bit columns
    and the pattern tiles again on one handle: every call the same bits"""
    from kokkos_kernels_b200 import sparse as sp

    A = K.lap27(64, 64, 64, 2)
    x, y0, xd, y0d = P.inputs(cuda, A, 1.3)
    Ad = P.dev(cuda, A)
    h = P.handle(8, 4)
    ys, ks = [], []
    for i, i32 in enumerate((False, False, False, True, False)):
        with P.setenv(B200SP_SPMV_IDX16="0" if i32 else "1"):
            y = y0d.clone()
            sp.spmv(h, "N", -0.7, Ad, xd, 1.3, y)
            ys.append(y)
            ks.append(h.last_kernel())
        if i == 1:
            torch.cuda.synchronize()  # the verdict is on the host: the next calls run the pattern tiles
    torch.cuda.synchronize()
    assert LAYOUT in ks[2], ks
    assert LAYOUT in ks[-1] and "IDX=i32" in ks[3], ks
    assert all(torch.equal(ys[0], y) for y in ys[1:]), ks


def test_forward_and_hostvec_over_64_rows(cuda):
    """the fused all-gather form on pattern tiles of more than 64 rows (1 dof: about 170), and the pipelined host-vector
    entry after the switch to the pattern tiles"""
    from kokkos_kernels_b200 import sparse as sp

    A = K.lap27(96, 96, 96, 1)
    first = np.searchsorted(A[0], np.arange(pat_tiles(A)) * (PAT_TILE_CAP - 512 - 8), side="right") - 1
    assert np.min(np.diff(first)) > 64 and len(A[1]) >= 1 << 22
    Ad = P.dev(cuda, A)
    x, y0, xd, _ = P.inputs(cuda, A, 1.3)
    n = len(y0)
    outs = {}
    for form in ("pat", "i32"):
        with P.setenv(B200SP_SPMV_IDX16="0" if form == "i32" else "1"):
            h = P.handle(8, 4)
            for _ in range(3):
                loc = torch.full((n,), float("nan"), dtype=torch.float64, device=cuda)
                fwd = torch.full((n,), float("nan"), dtype=torch.float64, device=cuda)
                sp.spmv_forward(h, 1.0, Ad, xd, loc, fwd.data_ptr())
                torch.cuda.synchronize()
            kf = h.last_kernel()
            xh = torch.from_numpy(x).pin_memory()
            for _ in range(3):
                yh = torch.from_numpy(y0.copy()).pin_memory()
                sp.spmv_hostvec(h, "N", -0.7, Ad, xh, 1.3, yh)
                torch.cuda.synchronize()
            kh = h.last_kernel()
        assert (LAYOUT in kf) == (LAYOUT in kh) == (form == "pat"), (kf, kh)
        assert torch.equal(loc, fwd)
        outs[form] = (loc.cpu().numpy(), yh.numpy().copy())
    assert np.array_equal(outs["pat"][0], outs["i32"][0]) and np.array_equal(outs["pat"][1], outs["i32"][1])

