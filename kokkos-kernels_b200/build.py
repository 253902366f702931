"""In-tree build of the native libraries (no JIT cache: the .so files travel
with the repo snapshot to the GPU box).

  lib/libb200sparse.so   CUDA kernels + C ABI (include/b200sparse.h), sm_90a (H100)
  lib/libb200matgen.so   host-side synthetic matrix generators (C + OpenMP)
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "lib")
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
]
CU_SOURCES = ["spmv.cu", "spmv64.cu", "spmm.cu", "spgemm.cu", "spgemm64.cu", "bspgemm.cu", "crs_utils.cu", "bsr.cu", "cg.cu", "gmres.cu", "gs.cu", "gs2.cu", "sptrsv.cu", "crs_io.cpp"]


def _newer(target, sources):
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(s) <= t for s in sources)


def _nvcc():
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def build(force=False, verbose=True):
    """Serialised across processes by a lock file (pytest-xdist workers all call this at session start)."""
    os.makedirs(LIB, exist_ok=True)
    import fcntl

    with open(os.path.join(LIB, ".build.lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            return _build_locked(force, verbose)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)


def _build_locked(force, verbose):
    out = os.path.join(LIB, "libb200sparse.so")
    srcs = [os.path.join(CSRC, s) for s in CU_SOURCES if os.path.exists(os.path.join(CSRC, s))]
    deps = srcs + [os.path.join(CSRC, "common.cuh"), os.path.join(CSRC, "scan.cuh"), os.path.join(CSRC, "tile_ring.cuh"), os.path.join(CSRC, "spgemm_esc.cuh"), os.path.join(CSRC, "bspgemm.cuh"), os.path.join(CSRC, "spmm_items.h"), os.path.join(HERE, "..", "include", "b200sparse.h")]
    if force or not _newer(out, deps):
        objs = []
        procs = []
        for s in srcs:
            o = os.path.join(LIB, os.path.basename(s) + ".o")
            objs.append(o)
            cmd = [_nvcc()] + NVCC_FLAGS + ["-c", s, "-o", o]
            if verbose:
                print("[build]", " ".join(cmd), flush=True)
            procs.append((subprocess.Popen(cmd), cmd))
        for p, cmd in procs:
            if p.wait() != 0:
                raise RuntimeError("nvcc failed: " + " ".join(cmd))
        cmd = [_nvcc(), "-shared", "-o", out] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
        if verbose:
            print("[build]", " ".join(cmd), flush=True)
        subprocess.check_call(cmd)
    gen = os.path.join(LIB, "libb200matgen.so")
    gsrc = os.path.join(CSRC, "matgen.c")
    if force or not _newer(gen, [gsrc]):
        cmd = ["gcc", "-O2", "-fPIC", "-shared", "-fopenmp", "-fvisibility=hidden", "-std=gnu11", "-o", gen, gsrc, "-lm"]
        if verbose:
            print("[build]", " ".join(cmd), flush=True)
        subprocess.check_call(cmd)
    # C++ drop-in check: the Kokkos TPL specialisations (kokkos_shim/) compiled against the View mock
    drv = os.path.join(LIB, "shim_driver")
    root = os.path.join(HERE, "..")
    dsrc = os.path.join(root, "tests", "shim_mock", "shim_driver.cpp")
    shim = [os.path.join(HERE, "kokkos_shim", f) for f in sorted(os.listdir(os.path.join(HERE, "kokkos_shim")))]
    if os.path.exists(dsrc) and (force or not _newer(drv, [dsrc, out, os.path.join(root, "tests", "shim_mock", "Kokkos_Mock.hpp")] + shim)):
        cmd = [_nvcc(), "-std=c++17", "-O1", "-Wno-deprecated-gpu-targets", "-I", os.path.join(root, "tests", "shim_mock"),
               "-I", os.path.join(HERE, "kokkos_shim"), "-I", os.path.join(root, "include"), dsrc, "-o", drv,
               "-L", LIB, "-lb200sparse", "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN"]
        if verbose:
            print("[build]", " ".join(cmd), flush=True)
        subprocess.check_call(cmd)
    # the same for the half_t SPMV_MV specialisations (half_t stand-in: Kokkos_Mock_Half.hpp, under KOKKOS_HALF_T_IS_FLOAT == 0)
    hdrv = os.path.join(LIB, "shim_half_driver")
    hsrc = os.path.join(root, "tests", "shim_mock", "shim_half_driver.cpp")
    hdeps = [os.path.join(root, "tests", "shim_mock", f) for f in ("Kokkos_Mock.hpp", "Kokkos_Mock_Half.hpp")]
    if os.path.exists(hsrc) and (force or not _newer(hdrv, [hsrc, out] + hdeps + shim)):
        cmd = [_nvcc(), "-std=c++17", "-O1", "-Wno-deprecated-gpu-targets", "-I", os.path.join(root, "tests", "shim_mock"),
               "-I", os.path.join(HERE, "kokkos_shim"), "-I", os.path.join(root, "include"), hsrc, "-o", hdrv,
               "-L", LIB, "-lb200sparse", "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN"]
        if verbose:
            print("[build]", " ".join(cmd), flush=True)
        subprocess.check_call(cmd)
    # the same for the block SpGEMM path: SPGEMM_SYMBOLIC on the block graphs + BSPGEMM_NUMERIC (Kokkos_Mock_Bspgemm.hpp)
    bdrv = os.path.join(LIB, "shim_bspgemm_driver")
    bsrc = os.path.join(root, "tests", "shim_mock", "shim_bspgemm_driver.cpp")
    bdeps = [os.path.join(root, "tests", "shim_mock", f) for f in ("Kokkos_Mock.hpp", "Kokkos_Mock_Bspgemm.hpp")]
    if os.path.exists(bsrc) and (force or not _newer(bdrv, [bsrc, out] + bdeps + shim)):
        cmd = [_nvcc(), "-std=c++17", "-O1", "-Wno-deprecated-gpu-targets", "-I", os.path.join(root, "tests", "shim_mock"),
               "-I", os.path.join(HERE, "kokkos_shim"), "-I", os.path.join(root, "include"), bsrc, "-o", bdrv,
               "-L", LIB, "-lb200sparse", "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN"]
        if verbose:
            print("[build]", " ".join(cmd), flush=True)
        subprocess.check_call(cmd)
    # the same for the (int, size_t) SPGEMM_SYMBOLIC / SPGEMM_NUMERIC specialisations (64-bit offsets)
    sdrv = os.path.join(LIB, "shim_spgemm64_driver")
    ssrc = os.path.join(root, "tests", "shim_mock", "shim_spgemm64_driver.cpp")
    sdeps = [os.path.join(root, "tests", "shim_mock", "Kokkos_Mock.hpp")]
    if os.path.exists(ssrc) and (force or not _newer(sdrv, [ssrc, out] + sdeps + shim)):
        cmd = [_nvcc(), "-std=c++17", "-O1", "-Wno-deprecated-gpu-targets", "-I", os.path.join(root, "tests", "shim_mock"),
               "-I", os.path.join(HERE, "kokkos_shim"), "-I", os.path.join(root, "include"), ssrc, "-o", sdrv,
               "-L", LIB, "-lb200sparse", "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN"]
        if verbose:
            print("[build]", " ".join(cmd), flush=True)
        subprocess.check_call(cmd)
    # torch-free GPU validation harness (tools/gpu_check.cpp; links the oracle as the CHECKER -- test infrastructure)
    chk = os.path.join(LIB, "gpu_check")
    csrc = os.path.join(root, "tools", "gpu_check.cpp")
    orc = os.path.join(root, "oracle", "libkkoracle.so")
    if os.path.exists(csrc) and os.path.exists(orc) and (force or not _newer(chk, [csrc, out, gen, orc])):
        cmd = [_nvcc(), "-std=c++17", "-O2", "-Wno-deprecated-gpu-targets", "-I", os.path.join(root, "include"), csrc, "-o", chk,
               "-L", LIB, "-lb200sparse", "-lb200matgen", "-L", os.path.join(root, "oracle"), "-lkkoracle",
               "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN", "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN/../../oracle"]
        if verbose:
            print("[build]", " ".join(cmd), flush=True)
        subprocess.check_call(cmd)
    return out, gen


if __name__ == "__main__":
    build(force="--force" in sys.argv)
