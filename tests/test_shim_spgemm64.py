"""The (int, size_t) SPGEMM_SYMBOLIC / SPGEMM_NUMERIC specialisations of the Kokkos shim
(kokkos_shim/KokkosSparse_spgemm_b200_tpl_spec_*.hpp: 64-bit offsets, 32-bit ordinals), compiled by build() into
shim_spgemm64_driver against the View mock: its static_asserts check that spgemm_{symbolic,numeric}_tpl_spec_avail is true for
double and float in CudaSpace and CudaUVMSpace (and false for 64-bit ordinals); on a GPU it runs the slots as Kokkos dispatches
them, compares C bit for bit with direct b200sp_spgemm_*_i64 calls and checks that the native stand-ins were never called."""
import os
import subprocess

import pytest

import kokkos_kernels_b200 as kk

DRV = os.path.join(kk._lib.LIBDIR, "shim_spgemm64_driver")


def test_shim_spgemm64_compiles_and_links():
    assert os.path.exists(DRV), "build() did not produce the (int, size_t) SpGEMM shim driver"
    out = subprocess.run([DRV], capture_output=True, text=True, timeout=300)
    assert out.returncode in (0, 77), out.stdout + out.stderr


@pytest.mark.gpu
def test_shim_spgemm64_runs_on_gpu(cuda):
    out = subprocess.run([DRV], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "SHIM SPGEMM64 DRIVER OK" in out.stdout and "native SPGEMM_SYMBOLIC/NUMERIC calls: 0" in out.stdout, out.stdout
    for name in ("f64", "f32"):
        assert f"{name} (int, size_t) spgemm through SPGEMM_SYMBOLIC/NUMERIC<...,true,true> : " in out.stdout, out.stdout
        assert "C ABI bits identical" in out.stdout, out.stdout
