"""The block SpGEMM path of the Kokkos shim (kokkos_shim/KokkosSparse_bspgemm_b200_tpl_spec_*.hpp), compiled by build() into
shim_bspgemm_driver against the View mock plus Kokkos_Mock_Bspgemm.hpp: its static_asserts check that
bspgemm_numeric_tpl_spec_avail is true for double and float; on a GPU, Kokkos' block_spgemm_symbolic / block_spgemm_numeric
sequence (the point SPGEMM_SYMBOLIC slot on the block graphs, then BSPGEMM_NUMERIC with its defaulted tpl argument) must give
the C ABI's bits, throw when numeric comes before symbolic, and never call the native struct."""
import os
import subprocess

import pytest

import kokkos_kernels_b200 as kk

DRV = os.path.join(kk._lib.LIBDIR, "shim_bspgemm_driver")


def test_shim_bspgemm_compiles_and_links():
    assert os.path.exists(DRV), "build() did not produce the block SpGEMM shim driver"
    out = subprocess.run([DRV], capture_output=True, text=True, timeout=300)
    assert out.returncode in (0, 77), out.stdout + out.stderr


@pytest.mark.gpu
def test_shim_bspgemm_runs_on_gpu(cuda):
    out = subprocess.run([DRV], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "SHIM BSPGEMM DRIVER OK" in out.stdout and "native BSPGEMM_NUMERIC calls: 0" in out.stdout, out.stdout
    for name in ("f64", "f32"):
        assert f"{name} numeric before symbolic throws: ok" in out.stdout, out.stdout
        assert "C ABI bits identical" in out.stdout, out.stdout
