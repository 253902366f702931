import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with -m gpu)")
    config.addinivalue_line("markers", "gpu_next: GPU tests of code that has not had its first run on an H100 yet "
                                       "(validated with tools/gpu_check first, then promoted to `gpu`)")


# GPU tests that need the real CUDA runtime (pinned host memory, torch streams, the nvcc-built shim driver)
_NEEDS_REAL_CUDA = {"test_hostvec_entry", "test_interfaces_and_errors", "test_hostvec_pipeline", "test_shim_runs_on_gpu",
                    "test_shim_bsr_runs_on_gpu", "test_hostvec_deferred_completion",
                    # BASELINE-size workloads: hours under the emulation
                    "test_config4_full_size", "test_config3_full_size"}


def pytest_collection_modifyitems(config, items):
    if os.environ.get("B200SP_TEST_EMULATED") != "1":
        return
    skip = pytest.mark.skip(reason="needs the real CUDA runtime (B200SP_TEST_EMULATED=1 runs the kernels under the CPU emulation)")
    for it in items:
        if it.originalname in _NEEDS_REAL_CUDA or it.name in _NEEDS_REAL_CUDA:
            it.add_marker(skip)


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Build the native libraries once (no-op when up to date)."""
    import __graft_entry__ as g

    g.build(verbose=False)


@pytest.fixture(scope="session")
def oracle():
    import oracle_lib

    return oracle_lib.Oracle()


def _emulated_device():
    """B200SP_TEST_EMULATED=1: run the GPU test files on the CPU -- the Python mirror (kokkos_kernels_b200.sparse) is
    pointed at the CUDA-on-CPU emulation of the library (tools/emu, tests/emu_lib.py) and torch CPU tensors stand in for
    device memory.  Checks the tests themselves and the mirror's Python code before they reach a GPU; says nothing
    about the GPU.  Usage:  B200SP_TEST_EMULATED=1 python -m pytest tests/test_gpu_bsr.py -m "gpu or gpu_next" """
    import ctypes
    import torch

    import emu_lib
    import kokkos_kernels_b200 as kk
    from kokkos_kernels_b200 import sparse

    lib = emu_lib.lib()
    kk._lib.sparse = lambda: lib
    sparse._stream = lambda: ctypes.c_void_p(0)
    torch.cuda.synchronize = lambda *a, **k: None
    # .to("cpu") of a CPU tensor is the tensor itself: give "device" tensors their own storage, as a real upload does
    orig_from_numpy = torch.from_numpy
    torch.from_numpy = lambda a: orig_from_numpy(a.copy())
    return torch.device("cpu")


@pytest.fixture(scope="session")
def cuda():
    import torch

    if os.environ.get("B200SP_TEST_EMULATED") == "1":
        return _emulated_device()
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import kokkos_kernels_b200 as kk

    assert kk._lib.sparse().b200sp_device_ok() == 1, "libb200sparse needs a compute-capability 9.0 (H100) device"
    return torch.device("cuda:0")
