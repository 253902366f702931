"""The half_t SPMV_MV specialisations of the Kokkos shim (kokkos_shim/KokkosSparse_spmv_b200_tpl_spec_*.hpp under
KOKKOS_HALF_T_IS_FLOAT == 0), compiled by build() into shim_half_driver against the View mock: its static_asserts check
that spmv_mv_tpl_spec_avail is true for half_t in every layout pair and both memory spaces; on a GPU it runs
KokkosSparse::spmv's dispatch on half LayoutLeft / LayoutRight views, compares with the C ABI bit for bit and checks
that the native SPMV_MV stand-in was never called."""
import os
import subprocess

import pytest

import kokkos_kernels_b200 as kk

DRV = os.path.join(kk._lib.LIBDIR, "shim_half_driver")


def test_shim_half_compiles_and_links():
    assert os.path.exists(DRV), "build() did not produce the half shim driver"
    out = subprocess.run([DRV], capture_output=True, text=True, timeout=300)
    assert out.returncode in (0, 77), out.stdout + out.stderr


@pytest.mark.gpu
def test_shim_runs_on_gpu(cuda):
    out = subprocess.run([DRV], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "SHIM HALF DRIVER OK" in out.stdout and "native SPMV_MV calls: 0" in out.stdout, out.stdout
    for pair in ("LL", "RL", "LR", "RR"):
        assert f"half spmv_mv {pair} through SPMV_MV<...,false,true>::spmv_mv : ok" in out.stdout, out.stdout
