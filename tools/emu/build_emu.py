#!/usr/bin/env python
"""Build the CUDA-on-CPU emulation of libb200sparse (TEST INFRASTRUCTURE; see tools/emu/cuda_emu.h).

  python tools/emu/build_emu.py            -> tools/emu/_build/libb200sparse_emu.so, tools/emu/_build/gpu_check_emu

The library's .cu sources are compiled by g++ after two mechanical source transformations:
  kern<<<grid, block, smem, stream>>>(args);   ->  B200_EMU_LAUNCH((kern), grid, block, smem, args);
  extern __shared__ [__align__(n)] T name[];   ->  T* name = reinterpret_cast<T*>(b200emu::dyn_smem());
everything else (qualifiers, intrinsics, the runtime API, the PTX wrappers of common.cuh) is handled by
tools/emu/cuda_emu.h and the B200SP_EMU branch of common.cuh.  The C ABI of the result is the product's, so
tools/gpu_check.cpp runs unchanged against it (gpu_check_emu): every harness suite then EXECUTES the kernels on the
host and checks them against the oracle.  Nothing here is linked into or shipped with the product library."""
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "kokkos-kernels_b200", "csrc")
OUT = os.path.join(HERE, "_build")
SOURCES = ["spmv.cu", "spmv64.cu", "spmm.cu", "spgemm.cu", "spgemm64.cu", "bspgemm.cu", "crs_utils.cu", "bsr.cu", "cg.cu", "gmres.cu", "gs.cu", "gs2.cu", "sptrsv.cu", "crs_io.cpp"]
HEADERS = ["common.cuh", "scan.cuh", "tile_ring.cuh", "spgemm_esc.cuh", "bspgemm.cuh", "spmm_items.h"]


def _match_back_angle(text, end):
    """text[end-1] == '>': index of the matching '<' (template argument list of the kernel expression)."""
    depth = 0
    i = end - 1
    while i >= 0:
        c = text[i]
        if c == ">":
            depth += 1
        elif c == "<":
            depth -= 1
            if depth == 0:
                return i
        i -= 1
    raise ValueError("unbalanced template argument list before <<<")


def _match_paren(text, start):
    """text[start] == '(': index just past the matching ')'."""
    depth = 0
    i = start
    while i < len(text):
        c = text[i]
        if c == "(":
            depth += 1
        elif c == ")":
            depth -= 1
            if depth == 0:
                return i + 1
        i += 1
    raise ValueError("unbalanced parentheses after >>>")


def _split_top(s):
    parts, depth, cur = [], 0, ""
    for c in s:
        if c in "([{":
            depth += 1
        elif c in ")]}":
            depth -= 1
        if c == "," and depth == 0:
            parts.append(cur.strip())
            cur = ""
        else:
            cur += c
    parts.append(cur.strip())
    return parts


def transform(text):
    # extern __shared__ declarations -> pointer into the emulator's dynamic shared memory
    text = re.sub(r"extern\s+__shared__\s+(?:__align__\(\d+\)\s+)?([A-Za-z_][\w ]*?)\s+(\w+)\[\];",
                  lambda m: f"{m.group(1)}* {m.group(2)} = reinterpret_cast<{m.group(1)}*>(b200emu::dyn_smem());", text)
    out, pos = "", 0
    while True:
        k = text.find("<<<", pos)
        if k < 0:
            out += text[pos:]
            break
        # kernel expression: identifier (possibly qualified) with an optional template argument list, right before <<<
        j = k
        while j > 0 and text[j - 1].isspace():
            j -= 1
        if text[j - 1] == ">":
            j = _match_back_angle(text, j)
        while j > 0 and (text[j - 1].isalnum() or text[j - 1] in "_:"):
            j -= 1
        kern = text[j:k].strip()
        e = text.find(">>>", k)
        cfg = _split_top(text[k + 3:e])
        while len(cfg) < 3:
            cfg.append("0")
        a0 = e + 3
        while text[a0].isspace():
            a0 += 1
        assert text[a0] == "(", "launch without argument list"
        a1 = _match_paren(text, a0)
        args = text[a0 + 1:a1 - 1].strip()
        out += text[pos:j] + f"B200_EMU_LAUNCH(({kern}), {cfg[0]}, {cfg[1]}, {cfg[2]}" + (", " + args if args else "") + ")"
        pos = a1
    return out


def up_to_date():
    """True when the emulated library is newer than every file it is built from."""
    lib = os.path.join(OUT, "libb200sparse_emu.so")
    chk = os.path.join(OUT, "gpu_check_emu")
    if not (os.path.exists(lib) and os.path.exists(chk) and os.path.exists(os.path.join(OUT, "shim_driver_emu"))):
        return False
    deps = [os.path.join(CSRC, n) for n in SOURCES + HEADERS]
    deps += [os.path.join(HERE, n) for n in ("cuda_emu.h", "emu_runtime.cpp", "build_emu.py", "cuda_runtime.h")]
    deps += [os.path.join(ROOT, "include", "b200sparse.h"), os.path.join(ROOT, "tools", "gpu_check.cpp")]
    shim = os.path.join(ROOT, "kokkos-kernels_b200", "kokkos_shim")
    deps += [os.path.join(shim, f) for f in os.listdir(shim)]
    deps += [os.path.join(ROOT, "tests", "shim_mock", f) for f in ("shim_driver.cpp", "Kokkos_Mock.hpp")]
    newest = max(os.path.getmtime(d) for d in deps)
    return min(os.path.getmtime(lib), os.path.getmtime(chk)) >= newest


def build(verbose=True):
    os.makedirs(OUT, exist_ok=True)
    srcdir = os.path.join(OUT, "src", "csrc")
    os.makedirs(srcdir, exist_ok=True)
    # the sources include "../../include/b200sparse.h": keep that relative layout
    incdir = os.path.join(OUT, "include")
    os.makedirs(incdir, exist_ok=True)
    with open(os.path.join(ROOT, "include", "b200sparse.h")) as f, open(os.path.join(incdir, "b200sparse.h"), "w") as g:
        g.write(f.read())
    objs = []
    for name in SOURCES + HEADERS:
        with open(os.path.join(CSRC, name)) as f:
            text = transform(f.read())
        dst = os.path.join(srcdir, name if not name.endswith(".cu") else name[:-3] + "_emu.cpp")
        with open(dst, "w") as g:
            g.write(text)
    flags = ["-std=c++17", "-O1", "-g", "-fPIC", "-ffp-contract=off", "-DB200SP_EMU", "-I", HERE, "-I", srcdir,
             "-Wno-unused-function", "-Wno-unused-variable", "-Wno-unknown-pragmas"]
    procs = []
    for name in SOURCES:
        src = os.path.join(srcdir, name if not name.endswith(".cu") else name[:-3] + "_emu.cpp")
        obj = os.path.join(OUT, os.path.basename(src) + ".o")
        objs.append(obj)
        cmd = ["g++"] + flags + ["-c", src, "-o", obj]
        if verbose:
            print("[emu]", " ".join(cmd), flush=True)
        procs.append((subprocess.Popen(cmd), cmd))
    rt = os.path.join(OUT, "emu_runtime.o")
    cmd = ["g++"] + flags + ["-c", os.path.join(HERE, "emu_runtime.cpp"), "-o", rt]
    procs.append((subprocess.Popen(cmd), cmd))
    for p, cmd in procs:
        if p.wait() != 0:
            raise RuntimeError("emulation build failed: " + " ".join(cmd))
    lib = os.path.join(OUT, "libb200sparse_emu.so")
    subprocess.check_call(["g++", "-shared", "-Wl,-Bsymbolic", "-o", lib] + objs + [rt])
    # the harness against the emulated library (its <cuda_runtime.h> is tools/emu/cuda_runtime.h)
    libdir = os.path.join(ROOT, "kokkos-kernels_b200", "lib")
    chk = os.path.join(OUT, "gpu_check_emu")
    cmd = ["g++", "-std=c++17", "-O1", "-g", "-DB200SP_EMU", "-I", HERE, "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tools", "gpu_check.cpp"), "-o", chk, "-L", OUT, "-lb200sparse_emu", "-L", libdir, "-lb200matgen",
           "-L", os.path.join(ROOT, "oracle"), "-lkkoracle", "-Wl,-rpath," + OUT, "-Wl,-rpath," + libdir,
           "-Wl,-rpath," + os.path.join(ROOT, "oracle")]
    if verbose:
        print("[emu]", " ".join(cmd), flush=True)
    subprocess.check_call(cmd)
    # the Kokkos TPL shim driver (tests/shim_mock) against the emulated library: the specialisations run on the host
    drv = os.path.join(OUT, "shim_driver_emu")
    cmd = ["g++", "-std=c++17", "-O1", "-g", "-DB200SP_EMU", "-I", HERE, "-I", os.path.join(ROOT, "tests", "shim_mock"),
           "-I", os.path.join(ROOT, "kokkos-kernels_b200", "kokkos_shim"), "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "shim_mock", "shim_driver.cpp"), "-o", drv, "-L", OUT, "-lb200sparse_emu", "-Wl,-rpath," + OUT]
    if verbose:
        print("[emu]", " ".join(cmd), flush=True)
    subprocess.check_call(cmd)
    return lib, chk


if __name__ == "__main__":
    build()
    print("built", OUT)
