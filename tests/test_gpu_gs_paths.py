"""Point, two-stage and classic Gauss-Seidel on the GPU through the Python mirror, on the cases of gs_cases.py: the colouring
(recolour passes 0, 1, 2), one forward and one backward sweep of every case at every lanes-per-row kernel (the plan's
last_kernel() names the one that ran) with every row within gs_sweep_bound of its local exact reference (tests/exact_ref.py),
the bit-for-bit sweep laws, colour sets that wrap the sweep kernel's grid-stride loop, numeric re-run on changed values and
across scalar types, and every two-stage / classic option, several right-hand sides included, within gs2_bound.
tests/test_emulated_gs_paths.py runs the same checks on the CPU at reduced sizes."""
import numpy as np
import pytest
import torch

import gs_cases as G

pytestmark = pytest.mark.gpu

DTYPES = [np.float64, np.float32]


def _t(cuda, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(cuda)


class PointRun:
    def __init__(self, cuda):
        from kokkos_kernels_b200 import sparse as sp

        self.sp, self.cuda = sp, cuda
        self.h = sp.GaussSeidelHandle()
        self.vd = None

    def symbolic(self, c):
        self.c = c
        self.rpd, self.cid = _t(self.cuda, c["rp"]), _t(self.cuda, c["ci"])
        self.sp.gauss_seidel_symbolic(self.h, c["n"], c["ncols"], self.rpd, self.cid, c["symmetric"])

    def numeric(self, c, v):
        if self.vd is not None and self.vd.dtype == torch.from_numpy(v[:1]).dtype and self.vd.numel() == len(v):
            self.vd.copy_(torch.from_numpy(v))  # in place: the same device array, new values
        else:
            self.vd = _t(self.cuda, v)
        self.sp.gauss_seidel_numeric(self.h, c["n"], c["ncols"], self.rpd, self.cid, self.vd, c["symmetric"])

    def apply(self, c, v, x, y, init_zero, omega, sweeps, direction):
        fn = (self.sp.symmetric_gauss_seidel_apply, self.sp.forward_sweep_gauss_seidel_apply, self.sp.backward_sweep_gauss_seidel_apply)[direction]
        xd = _t(self.cuda, np.asarray(x, dtype=v.dtype))
        fn(self.h, c["n"], c["ncols"], self.rpd, self.cid, self.vd, xd, _t(self.cuda, np.asarray(y, dtype=v.dtype)), init_zero, True, omega, sweeps)
        torch.cuda.synchronize()
        return xd.cpu().numpy()

    def coloring(self):
        colors, cptr, crows = self.h.get_coloring(self.c["n"])
        return len(cptr) - 1, colors, cptr, crows

    def kernel(self):
        return self.h.last_kernel()


class Gs2Run:
    def __init__(self, cuda):
        from kokkos_kernels_b200 import sparse as sp

        self.sp, self.cuda = sp, cuda

    def setup(self, c, v, compact, inner, outer, gamma, two_stage, dinv):
        sp = self.sp
        self.c = c
        kh = self.kh = sp.KokkosKernelsHandle()
        kh.create_gs_handle(sp.GS_TWOSTAGE)
        kh.set_gs_twostage(two_stage, c["n"])
        kh.set_gs_twostage_compact_form(compact)
        kh.set_gs_set_num_inner_sweeps(inner)
        kh.set_gs_set_num_outer_sweeps(outer)
        kh.set_gs_set_inner_damp_factor(gamma)
        self.rpd, self.cid, self.vd = _t(self.cuda, c["rp"]), _t(self.cuda, c["ci"]), _t(self.cuda, v)
        sp.gauss_seidel_symbolic(kh, c["n"], c["ncols"], self.rpd, self.cid, False)
        sp.gauss_seidel_numeric(kh, c["n"], c["ncols"], self.rpd, self.cid, self.vd, False,
                                given_inverse_diagonal=None if dinv is None else _t(self.cuda, dinv))

    def apply(self, X, B, init_zero, omega, num_iter, direction, buffers=False):
        sp, c = self.sp, self.c
        fn = (sp.symmetric_gauss_seidel_apply, sp.forward_sweep_gauss_seidel_apply, sp.backward_sweep_gauss_seidel_apply)[direction]
        if X.ndim == 1:
            Xd, Bd = _t(self.cuda, X), _t(self.cuda, B)
            fn(self.kh, c["n"], c["ncols"], self.rpd, self.cid, self.vd, Xd, Bd, init_zero, True, omega, num_iter)
            torch.cuda.synchronize()
            return Xd.cpu().numpy()
        Xbuf, Bbuf = _t(self.cuda, X.base), _t(self.cuda, B.base)  # (k, ld) row-major buffers: column-major views with ld > rows
        Xd, Bd = Xbuf.t()[:X.shape[0]], Bbuf.t()[:B.shape[0]]
        fn(self.kh, c["n"], c["ncols"], self.rpd, self.cid, self.vd, Xd, Bd, init_zero, True, omega, num_iter)
        torch.cuda.synchronize()
        out = Xbuf.cpu().numpy()
        return out if buffers else out.T[:X.shape[0]]


def _coloring_passes(monkeypatch, run, c):
    counts = []
    for passes in ("0", "1", "2"):
        monkeypatch.setenv("B200SP_GS_RECOLOR", passes)
        run.symbolic(c)
        col = run.coloring()
        G.check_coloring_both(c, col)
        counts.append(col[0])
    monkeypatch.delenv("B200SP_GS_RECOLOR")
    assert counts[0] >= counts[1] >= counts[2], counts


@pytest.mark.parametrize("case", G.point_cases(1.0), ids=lambda c: c["name"])
def test_point_every_lpr(cuda, monkeypatch, case):
    run = PointRun(cuda)
    _coloring_passes(monkeypatch, run, case)
    if case["name"] == "clique130":
        assert run.coloring()[0] >= 130
    labels = set()
    for lpr in G.LPRS:
        monkeypatch.setenv("B200SP_GS_LPR", str(lpr))
        run.symbolic(case)
        for dtype in DTYPES:
            run.numeric(case, case["v"].astype(dtype))
            labels |= G.check_sweeps(run, case, dtype, lpr)
            G.check_laws(run, case, dtype)
    assert labels == {f"gs_set<{t},LPR={l}>" for t in ("f64", "f32") for l in G.LPRS}


@pytest.mark.parametrize("dtype", DTYPES)
def test_point_lpr_thresholds(cuda, dtype):
    run = PointRun(cuda)
    for case, lpr in G.threshold_cases(1.0):
        run.symbolic(case)
        G.check_coloring_both(case, run.coloring())
        run.numeric(case, case["v"].astype(dtype))
        G.check_sweeps(run, case, dtype, lpr)


@pytest.mark.parametrize("dtype", DTYPES)
def test_point_grid_stride_wrap(cuda, dtype):
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    per_pass = sms * 16 * 256 // 2  # rows one pass of the LPR-2 sweep kernel covers
    case = G.wrap_case(max(1_000_000, 2.5 * per_pass))
    run = PointRun(cuda)
    run.symbolic(case)
    col = run.coloring()
    G.check_coloring_both(case, col)
    assert np.diff(col[2]).max() > per_pass
    run.numeric(case, case["v"].astype(dtype))
    G.check_sweeps(run, case, dtype, 2)
    G.check_laws(run, case, dtype)


def test_point_numeric_rerun_and_scalar_switch(cuda):
    case = G.nonsymmetric_case(1.0, ghosts=97)
    lpr = G.expected_lpr(case["rp"], case["n"])
    run = PointRun(cuda)
    run.symbolic(case)
    v = case["v"].copy()
    run.numeric(case, v)
    G.check_sweeps(run, case, np.float64, lpr)
    v *= np.random.default_rng(3).uniform(0.5, 2.0, len(v))
    run.numeric(case, v)  # new values into the same device array, same symbolic
    c2 = dict(case, v=v)
    G.check_sweeps(run, c2, np.float64, lpr)
    run.numeric(c2, v.astype(np.float32))
    G.check_sweeps(run, c2, np.float32, lpr)
    run.numeric(c2, v)
    G.check_sweeps(run, c2, np.float64, lpr)


GS2_CASE = G.gs2_case(1.0)


@pytest.mark.parametrize("dtype", DTYPES)
def test_two_stage_grid(cuda, dtype):
    run = Gs2Run(cuda)
    for g in G.gs2_grid():
        G.check_gs2(run, GS2_CASE, dtype, g)


@pytest.mark.parametrize("dtype", DTYPES)
def test_classic_grid(cuda, dtype):
    run = Gs2Run(cuda)
    for g in G.classic_grid():
        G.check_gs2(run, GS2_CASE, dtype, g, two_stage=False)
    for given in (False, True):
        for compact in (False, True):
            G.check_classic_local(run, GS2_CASE, dtype, given, compact)


@pytest.mark.parametrize("nrhs", [1, 2, 7])
def test_several_right_hand_sides(cuda, nrhs):
    run = Gs2Run(cuda)
    for dtype in DTYPES:
        for g in (dict(compact=False, inner=2, gamma=0.7, outer=1, omega=0.9, given=False, direction=0, init_zero=False, num_iter=1),
                  dict(compact=True, inner=3, gamma=1.0, outer=1, omega=0.9, given=True, direction=2, init_zero=True, num_iter=2)):
            G.check_gs2(run, GS2_CASE, dtype, g, nrhs=nrhs, pad=5)
        G.check_gs2(run, GS2_CASE, dtype, dict(compact=True, given=False, direction=0, init_zero=False, outer=1, num_iter=1), nrhs=nrhs, pad=5,
                    two_stage=False)
