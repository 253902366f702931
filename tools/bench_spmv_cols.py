"""A/B of the tiled SpMV kernel's three column forms on the bench matrix (needs a GPU): 32-bit columns (B200SP_SPMV_IDX16=0),
16-bit deltas + anchors (a handle built under B200SP_SPMV_PATTERN=0) and pattern starts + anchors + dictionary (default).
Alternates rounds of launches of each form, timed with CUDA events after warm-up, checks that the three y are bit-identical,
and prints per form the ms per launch, the bytes a launch moves (DESIGN.md sections 3.5 and 3.6) and the rate, with the
card's name, power limit and SM clock read in the same run, as one JSON line (also written to --out when given)."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from kokkos_kernels_b200 import matgen, sparse as sp  # noqa: E402


def real_bytes(form, m, nnz, val=8):
    """what a launch reads and writes: values, row_ptr, x and y, plus the form's column data"""
    base = val * nnz + 4 * (m + 1) + 2 * val * m
    cols = {"i32": 4 * nnz, "delta": 2 * nnz + 4 * m, "pat": 4 * m + 2 * m}[form]
    return base + cols


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:  # report what could not be read instead of a guess
        return {"error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=171)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--out", default=None, help="also write the result to this JSON file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    rp, ci, va, n, _, _ = bench.build_shard(1, 0, args.grid)
    m, nnz = len(rp) - 1, len(ci)
    A = sp.CrsMatrix(torch.from_numpy(rp).to(dev), torch.from_numpy(ci).to(dev), torch.from_numpy(va).to(dev), n)
    x = torch.from_numpy(matgen.fill(n, -1, 1, 1)).to(dev)
    forms = ("i32", "delta", "pat")
    env = {"i32": ("B200SP_SPMV_IDX16", "0"), "delta": ("B200SP_SPMV_PATTERN", "0"), "pat": (None, None)}
    handles, ys = {}, {}

    def run(form, k):
        key, val = env[form]
        if key:
            os.environ[key] = val
        try:
            for _ in range(k):
                sp.spmv(handles[form], "N", 1.0, A, x, 0.0, ys[form])
        finally:
            if key:
                os.environ.pop(key)

    for f in forms:
        handles[f] = sp.SPMVHandle(sp.SPMV_DEFAULT)
        handles[f].tune(8, -1, -1)  # the default ring, no self-tuning between the tiled and the row-vector kernel
        ys[f] = torch.empty(n, dtype=torch.float64, device=dev)
        run(f, 3)
        torch.cuda.synchronize()  # the verdicts are on the host
        run(f, 5)
        torch.cuda.synchronize()
    labels = {f: handles[f].last_kernel() for f in forms}
    times = {f: [] for f in forms}
    for _ in range(args.rounds):
        for f in forms:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run(f, args.launches)
            e1.record()
            torch.cuda.synchronize()
            times[f].append(e0.elapsed_time(e1) / args.launches)
    same = all(torch.equal(ys["pat"], ys[f]) for f in forms)
    res = {"card": card(), "rows": m, "nnz": nnz, "bit_identical": same, "forms": {}}
    for f in forms:
        ms = float(np.mean(times[f]))
        b = real_bytes(f, m, nnz)
        res["forms"][f] = {"kernel": labels[f], "ms_per_launch": round(ms, 4), "ms_rounds": [round(t, 4) for t in times[f]],
                           "real_bytes": b, "real_GBs": round(b / ms / 1e6, 1), "GFLOPs": round(2 * nnz / ms / 1e6, 1)}
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)
    print(json.dumps(res))
    assert same, "the three forms disagree"


if __name__ == "__main__":
    main()
