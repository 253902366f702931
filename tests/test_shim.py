"""The Kokkos Kernels TPL specialisations (kokkos-kernels_b200/kokkos_shim/*.hpp) compile against a
minimal mock of the Kokkos declarations they specialise (tests/shim_mock/Kokkos_Mock.hpp) and, on a
GPU, run end to end: SPMV<...,true>::spmv, SPMV_MV<...,false,true>::spmv_mv,
SPGEMM_SYMBOLIC/NUMERIC<...,true,true> -> C ABI -> CUDA kernels, checked on the host."""
import os
import subprocess

import pytest

import kokkos_kernels_b200 as kk

DRV = os.path.join(kk._lib.LIBDIR, "shim_driver")


def test_shim_compiles_and_links():
    assert os.path.exists(DRV), "build() did not produce the shim driver"
    out = subprocess.run([DRV], capture_output=True, text=True)
    # without a device the driver stops right after its static_asserts were compiled in
    assert out.returncode in (0, 77), out.stdout + out.stderr


@pytest.mark.gpu
def test_shim_runs_on_gpu(cuda):
    out = subprocess.run([DRV], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "SHIM DRIVER OK" in out.stdout


@pytest.mark.gpu
def test_shim_bsr_runs_on_gpu(cuda):
    """SPMV_BSRMATRIX / SPMV_MV_BSRMATRIX / SPGEMM_JACOBI specialisations (run on the GPU by tests/test_gpu_bsr.py)."""
    out = subprocess.run([DRV, "--bsr", "--jacobi", "--gs", "--gmres", "--spmv64", "--sptrsv"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "SHIM DRIVER OK" in out.stdout and "BsrMatrix spmv through" in out.stdout and "spgemm_jacobi through" in out.stdout and \
        "Gauss-Seidel through" in out.stdout and "gmres through" in out.stdout and "sptrsv through" in out.stdout
