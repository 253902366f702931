"""SpGEMM on 64-bit offsets against the 32-bit entry points (needs a GPU).  fp64, C = A*A, A with exactly 32 distinct
uniform-random columns per row and values U(1, 50) (bench.py:secondary_spgemm's generator).
  (a) bench.py's config 4 (2M x 2M, seed 4) through the 32-bit and the 64-bit entries, alternating for --rounds rounds after a
      warm-up: symbolic and numeric ms of each (CUDA events), the window count, and whether C is bit-identical;
  (b) the 2.2M x 2.2M product, whose nnz(C) passes 2^31 (only the 64-bit entries take it): symbolic and numeric ms, windows,
      nnz(C), and whether C equals the 32-bit path run on two row slices of A, bit for bit (with the 32-bit entries' own
      symbolic and numeric ms on those slices, for comparison).
Algorithmic bytes follow BASELINE.md section 3's SpGEMM model (A*A: the matrix counted once; S = 8 B values, I = 4 B
indices, O = 4 or 8 B offsets).  The card's name, power limit and maximum SM clock are read in the same run.  One JSON line,
also written to --out when given."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from kokkos_kernels_b200 import matgen, sparse as sp  # noqa: E402


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:  # report what could not be read instead of a guess
        return {"error": str(e)}


def bytes_model(m, nnz_a, nnz_c, off):
    S, I = 8, 4
    return {"symbolic": I * nnz_a + off * (m + 1) + off * (m + 1),
            "numeric": (S + I) * nnz_a + off * (m + 1) + off * (m + 1) + (S + I) * nnz_c}


def matrix(n, dev):
    rp, ci = matgen.uniform(n, n, 32, 4)
    va = matgen.fill(len(ci), 1.0, 50.0, 4)
    return rp, sp.CrsMatrix(torch.from_numpy(rp).to(dev), torch.from_numpy(ci).to(dev), torch.from_numpy(va).to(dev), n)


def timed_product(A, B):
    """symbolic and numeric of C = A*B on a new handle, each between CUDA events.  As in the reference's driver
    (perf_test/sparse/KokkosSparse_spgemm.cpp:395-417) row_mapC exists before the symbolic timer starts, and entriesC /
    valuesC are allocated between the two timers, so neither time includes a device allocation of C."""
    kh = sp.KokkosKernelsHandle()
    kh.create_spgemm_handle()
    m, n, k = A.numRows(), A.numCols(), B.numCols()
    row_mapC = torch.empty(m + 1, dtype=A.row_map.dtype, device=A.row_map.device)
    e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    torch.cuda.synchronize()
    e[0].record()
    sp.spgemm_symbolic_views(kh, m, n, k, A.row_map, A.entries, False, B.row_map, B.entries, False, row_mapC)
    e[1].record()
    sh = kh.get_spgemm_handle()
    c_nnz = sh.get_c_nnz()
    Cm = sp.CrsMatrix(row_mapC, torch.empty(c_nnz, dtype=torch.int32, device=A.row_map.device),
                      torch.empty(c_nnz, dtype=A.values.dtype, device=A.row_map.device), k)
    e[2].record()
    sp.spgemm_numeric(kh, A, False, B, False, Cm)
    e[3].record()
    torch.cuda.synchronize()
    return Cm, e[0].elapsed_time(e[1]), e[2].elapsed_time(e[3]), sh.windows()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=2_000_000, help="rows of (a), bench.py's config 4")
    ap.add_argument("--n-big", type=int, default=2_200_000, help="rows of (b), past 2^31 entries of C")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the result to this JSON file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    res = {"card": card(), "scalar": "fp64", "product": "C = A*A, 32 uniform-random columns per row, seed 4"}

    # (a) config 4 through both entries
    n = args.n
    rp, A32 = matrix(n, dev)
    A64 = sp.CrsMatrix(A32.row_map.long(), A32.entries, A32.values, n)
    t = {"i32": ([], []), "i64": ([], [])}
    same, wins, nnz_c = True, 0, 0
    for r in range(args.rounds + 1):  # round 0 warms up both paths
        C32, s32, n32, _ = timed_product(A32, A32)
        nnz_c = int(C32.row_map[-1])
        C32 = (C32.row_map.long(), C32.entries, C32.values)
        C64, s64, n64, wins = timed_product(A64, A64)
        if r > 0:
            t["i32"][0].append(s32), t["i32"][1].append(n32)
            t["i64"][0].append(s64), t["i64"][1].append(n64)
        same = same and torch.equal(C64.row_map, C32[0]) and torch.equal(C64.entries, C32[1]) and \
            torch.equal(C64.values.view(torch.int64), C32[2].view(torch.int64))
        del C32, C64
    res["a_config4"] = {
        "rows": n, "nnz_A": int(rp[-1]), "nnz_C": nnz_c, "windows": wins, "rounds": args.rounds, "bit_identical": bool(same),
        "ms": {p: {"symbolic": round(float(np.mean(t[p][0])), 3), "numeric": round(float(np.mean(t[p][1])), 3),
                   "symbolic_rounds": [round(x, 3) for x in t[p][0]], "numeric_rounds": [round(x, 3) for x in t[p][1]]}
               for p in t},
        "bytes": {p: bytes_model(n, int(rp[-1]), nnz_c, 4 if p == "i32" else 8) for p in t}}
    del A32, A64
    torch.cuda.empty_cache()

    # (b) past 2^31
    n = args.n_big
    rp, A32 = matrix(n, dev)
    A64 = sp.CrsMatrix(A32.row_map.long(), A32.entries, A32.values, n)
    for _ in range(2):  # the first repetition warms the allocator up; the second one's C is kept for the check
        C64 = None
        C64, s64, n64, wins = timed_product(A64, A64)
    nnz_c = int(C64.row_map[-1])
    same, slice_ms = True, []
    half = n // 2
    for r0, r1 in ((0, half), (half, n)):
        a0, a1 = int(rp[r0]), int(rp[r1])
        As = sp.CrsMatrix(A32.row_map[r0:r1 + 1] - a0, A32.entries[a0:a1], A32.values[a0:a1], n)
        timed_product(As, A32)  # warm-up of the slice's shape
        Cs, ss, ns, _ = timed_product(As, A32)
        slice_ms.append({"rows": r1 - r0, "symbolic": round(ss, 3), "numeric": round(ns, 3)})
        c0, c1 = int(C64.row_map[r0]), int(C64.row_map[r1])
        same = same and torch.equal(torch.diff(C64.row_map[r0:r1 + 1]), torch.diff(Cs.row_map).long()) and \
            torch.equal(C64.entries[c0:c1], Cs.entries) and torch.equal(C64.values[c0:c1].view(torch.int64), Cs.values.view(torch.int64))
        del Cs, As
        torch.cuda.empty_cache()
    b = bytes_model(n, int(rp[-1]), nnz_c, 8)
    res["b_past_2_31"] = {"rows": n, "nnz_A": int(rp[-1]), "nnz_C": nnz_c, "windows": wins, "bit_identical": bool(same),
                          "ms": {"symbolic": round(s64, 3), "numeric": round(n64, 3)}, "bytes": b,
                          "i32_on_row_slices_ms": slice_ms,
                          "numeric_GBps": round(b["numeric"] / n64 / 1e6, 1)}
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)
    print(json.dumps(res))
    assert res["a_config4"]["bit_identical"] and res["b_past_2_31"]["bit_identical"], "64-bit and 32-bit products differ"


if __name__ == "__main__":
    main()
