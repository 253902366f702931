"""Point, two-stage and classic Gauss-Seidel EXECUTED on the CPU (tools/emu) on the cases of gs_cases.py, with the checks of
tests/test_gpu_gs_paths.py at reduced sizes: the colouring (recolour passes 0, 1, 2), one forward and one backward sweep of
every case at every lanes-per-row kernel within gs_sweep_bound (tests/exact_ref.py), the bit-for-bit sweep laws, numeric
re-run on changed values and across scalar types, and every two-stage / classic option within gs2_bound."""
import numpy as np
import pytest

import emu_lib as E
import gs_cases as G

DTYPES = [np.float64, np.float32]
SCALE = 0.1


@pytest.fixture(scope="module")
def emu():
    return E.lib()


class PointRun:
    def __init__(self):
        self.plan = E.GsPlan()

    def close(self):
        self.plan.close()

    def symbolic(self, c):
        self.c = c
        self.plan.symbolic(c["n"], c["rp"], c["ci"], c["symmetric"], ncols=c["ncols"])

    def numeric(self, c, v):
        E.ok(self.plan.numeric(c["n"], c["rp"], c["ci"], v))

    def apply(self, c, v, x, y, init_zero, omega, sweeps, direction):
        x = np.array(x, dtype=v.dtype, copy=True)
        E.ok(self.plan.apply(c["n"], c["rp"], c["ci"], v, x, np.ascontiguousarray(y, dtype=v.dtype), init_zero, omega, sweeps, direction))
        return x

    def coloring(self):
        return self.plan.coloring(self.c["n"])

    def kernel(self):
        return self.plan.kernel()


class Gs2Run:
    def __init__(self):
        self.plan = None

    def close(self):
        if self.plan:
            self.plan.close()

    def setup(self, c, v, compact, inner, outer, gamma, two_stage, dinv):
        self.close()
        self.c, self.v = c, v
        self.plan = E.Gs2Plan(compact=compact, inner=inner, outer=outer, gamma=gamma)
        E.ok(self.plan.set(5, float(two_stage)))
        E.ok(self.plan.symbolic(c["n"], c["ncols"], c["rp"], c["ci"]))
        E.ok(self.plan.numeric(c["n"], c["ncols"], c["rp"], c["ci"], v, dinv))

    def apply(self, X, B, init_zero, omega, num_iter, direction, buffers=False):
        c = self.c
        E.ok(self.plan.apply(c["n"], c["ncols"], c["rp"], c["ci"], self.v, X, B, init_zero, omega, num_iter, direction))
        return X.base if buffers else X


@pytest.fixture
def point():
    r = PointRun()
    yield r
    r.close()


@pytest.fixture
def gs2():
    r = Gs2Run()
    yield r
    r.close()


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


@pytest.mark.parametrize("case", G.point_cases(SCALE), ids=lambda c: c["name"])
def test_point_every_lpr(emu, monkeypatch, point, case):
    _coloring_passes(monkeypatch, point, case)
    if case["name"] == "clique130":
        assert point.coloring()[0] >= 130
    labels = set()
    for lpr in G.LPRS:
        monkeypatch.setenv("B200SP_GS_LPR", str(lpr))
        point.symbolic(case)
        for dtype in DTYPES:
            point.numeric(case, case["v"].astype(dtype))
            labels |= G.check_sweeps(point, case, dtype, lpr)
            if lpr in (2, 32):
                G.check_laws(point, case, dtype)
    assert labels == {f"gs_set<{t},LPR={l}>" for t in ("f64", "f32") for l in G.LPRS}


@pytest.mark.parametrize("dtype", DTYPES)
def test_point_lpr_thresholds(emu, point, dtype):
    for case, lpr in G.threshold_cases(SCALE):
        point.symbolic(case)
        G.check_coloring_both(case, point.coloring())
        point.numeric(case, case["v"].astype(dtype))
        G.check_sweeps(point, case, dtype, lpr)


def test_point_grid_stride_wrap(emu, point):
    case = G.wrap_case(4 * 16 * 256 // 2 * 2.5)  # the emulated device has 4 SMs: 8192 rows per pass at LPR 2
    point.symbolic(case)
    col = point.coloring()
    G.check_coloring_both(case, col)
    assert np.diff(col[2]).max() > 4 * 16 * 256 // 2
    point.numeric(case, case["v"])
    G.check_sweeps(point, case, np.float64, 2)
    G.check_laws(point, case, np.float64)


def test_point_numeric_rerun_and_scalar_switch(emu, point):
    case = G.nonsymmetric_case(SCALE, ghosts=97)
    point.symbolic(case)
    v = case["v"].copy()
    point.numeric(case, v)
    G.check_sweeps(point, case, np.float64, G.expected_lpr(case["rp"], case["n"]))
    v *= np.random.default_rng(3).uniform(0.5, 2.0, len(v))  # in place, same symbolic
    point.numeric(case, v)
    c2 = dict(case, v=v)
    G.check_sweeps(point, c2, np.float64, G.expected_lpr(case["rp"], case["n"]))
    point.numeric(c2, v.astype(np.float32))
    G.check_sweeps(point, c2, np.float32, G.expected_lpr(case["rp"], case["n"]))
    point.numeric(c2, v)
    G.check_sweeps(point, c2, np.float64, G.expected_lpr(case["rp"], case["n"]))


GS2_CASE = G.gs2_case(SCALE)


@pytest.mark.parametrize("dtype", DTYPES)
def test_two_stage_grid(emu, gs2, dtype):
    for g in G.gs2_grid():
        G.check_gs2(gs2, GS2_CASE, dtype, g)


@pytest.mark.parametrize("dtype", DTYPES)
def test_classic_grid(emu, gs2, dtype):
    for g in G.classic_grid():
        G.check_gs2(gs2, GS2_CASE, dtype, g, two_stage=False)
    for given in (False, True):
        for compact in (False, True):
            G.check_classic_local(gs2, GS2_CASE, dtype, given, compact)


@pytest.mark.parametrize("nrhs", [1, 2, 7])
def test_several_right_hand_sides(emu, gs2, nrhs):
    for dtype in DTYPES:
        for g in (dict(compact=False, inner=2, gamma=0.7, outer=1, omega=0.9, given=False, direction=0, init_zero=False, num_iter=1),
                  dict(compact=True, inner=3, gamma=1.0, outer=1, omega=0.9, given=True, direction=2, init_zero=True, num_iter=2)):
            G.check_gs2(gs2, GS2_CASE, dtype, g, nrhs=nrhs, pad=5)
        G.check_gs2(gs2, GS2_CASE, dtype, dict(compact=True, given=False, direction=0, init_zero=False, outer=1, num_iter=1), nrhs=nrhs, pad=5,
                    two_stage=False)
