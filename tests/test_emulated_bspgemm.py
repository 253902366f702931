"""The block SpGEMM kernels (kokkos-kernels_b200/csrc/bspgemm.cu) under the CUDA-on-CPU emulation (tools/emu, TEST
INFRASTRUCTURE), with every device allocation between inaccessible pages (B200EMU_GUARD=1) and threads of a block run in
random order (B200EMU_ORDER=random): structure equal to, and values bit-identical with, the restatement of the reference's
bspgemm_debug_numeric.  Every path: the 1024- and 4096-product shared-memory bins, the long-row kernel on global scratch,
bs = 1 forwarding, fp64 and fp32, and destroying the plan gives back every allocation.

The emulator reads B200EMU_* once per process, so the cases run in a child process (this file run as a script)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


def _run_cases(group):
    import emu_lib as E
    import bspgemm_cases as BC

    L = E.lib()
    L.b200emu_live_allocations.restype = C.c_longlong
    L.b200emu_live_allocations.argtypes = [C.POINTER(C.c_longlong)]
    orc = BC.BlockOracle()

    def run(name, bs, A, B, m, n, k, reruns=1):
        dt = A[2].dtype
        Ag = tuple(E.guarded(x) for x in A)
        Bg = tuple(E.guarded(x) for x in B)
        live0 = L.b200emu_live_allocations(None)
        h = C.c_void_p()
        E.ok(L.b200sp_spgemm_plan_create(C.byref(h)))
        rpC = E.guarded(np.full(m + 1, 123, dtype=np.int32))
        nnz, mx = C.c_int64(), C.c_int()
        E.ok(L.b200sp_spgemm_symbolic_i32(h, None, m, n, k, E.ptr(Ag[0]), E.ptr(Ag[1]), E.ptr(Bg[0]), E.ptr(Bg[1]), E.ptr(rpC),
                                          C.byref(nnz), C.byref(mx)))
        fn = getattr(L, "b200sp_bspgemm_numeric_%s_i32" % E.sfx(dt))
        for rerun in range(reruns):
            vA = Ag[2] if rerun == 0 else E.guarded(A[2] * -1.5)
            ciC = E.guarded(np.full(nnz.value, -1, dtype=np.int32))
            vC = E.guarded(np.full(nnz.value * bs * bs, np.nan, dtype=dt))
            E.ok(fn(h, None, m, n, k, bs, E.ptr(Ag[0]), E.ptr(Ag[1]), E.ptr(vA), E.ptr(Bg[0]), E.ptr(Bg[1]), E.ptr(Bg[2]), E.ptr(rpC),
                    E.ptr(ciC), E.ptr(vC)))
            exp = orc.bspgemm(bs, (A[0], A[1], np.array(vA)), B, m, n, k)
            assert np.array_equal(rpC, exp[0]), name
            assert np.array_equal(ciC, exp[1]), name
            assert BC.same_bits(np.array(vC), exp[2]), (name, rerun)
        E.ok(L.b200sp_spgemm_plan_destroy(h, None))
        assert L.b200emu_live_allocations(None) == live0, name  # the plan (and its block-row grouping) is gone
        E.guarded_release()
        print("ok", name, bs, np.dtype(dt).name, flush=True)

    for dt in (np.float64, np.float32):
        if group == "sweep":
            for bs in (2, 3):
                for c in BC.ref_sweep_cases(bs, dt):
                    if c[4] <= 50:
                        run(*c)
            for c in BC.ref_sweep_cases(1, dt)[:2]:  # bs = 1: the point numeric, bit-identical by construction
                run(*c)
        elif group == "special":
            for bs in (2, 4):
                for c in BC.special_cases(bs, dt):
                    run(*c)
            run(*BC.special_cases(17, dt)[0])
        elif group == "long":
            run(*BC.long_row_case(2, dt, products=2000), reruns=2)  # a row in the 4096-product bin
            run(*BC.long_row_case(2, dt, products=6000), reruns=2)  # a row beyond it: global scratch
            run(*BC.long_row_case(8, dt, products=5000))            # A's blocks of the long row do not fit the staging area


@pytest.mark.parametrize("group", ["sweep", "special", "long"])
def test_emulated_bspgemm(group):
    env = dict(os.environ, B200EMU_GUARD="1", B200EMU_ORDER="random:7")
    out = subprocess.run([sys.executable, os.path.abspath(__file__), group], env=env, cwd=HERE, capture_output=True, text=True,
                         timeout=1500)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert "ok" in out.stdout


if __name__ == "__main__":
    sys.path.insert(0, HERE)
    sys.path.insert(0, os.path.dirname(HERE))
    _run_cases(sys.argv[1])
