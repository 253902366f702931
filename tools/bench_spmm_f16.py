"""Half-precision rank-2 SpMV against fp32 on bench.py's config 3 (needs a GPU): R-MAT scale 23 with bench.py's seeds, values
and X rounded to fp16, k = 16, alpha = 1, beta = 0.  The fp32 call runs on the widened fp16 inputs, so both compute the same
product: the script checks Y16 == round_fp16(Y32) bit for bit.  fp32 and fp16 rounds alternate, for LayoutRight and
LayoutLeft, timed with CUDA events after warm-up; one JSON line reports per variant the ms per call, GFLOP/s, the kernel
label, and the algorithmic bytes of the fp16 call
    nnz*(2+4) + 16*items + 4*(m+1) + n*k*2 + m*k*2
and its gather model (n*k*2 replaced by nnz*k*2: every entry fetches its X row), with the card's name, power limit and
maximum SM clock read in the same run.  Also written to --out when given."""
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


def n_items(rp, lmax=64):
    """work items of the item kernels (csrc/spmm.cu): one per row of up to LMAX entries, ceil(len / LMAX) per longer row"""
    lens = np.diff(rp.astype(np.int64))
    return int(np.where(lens <= lmax, 1, (lens + lmax - 1) // lmax).sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=23)
    ap.add_argument("--k", type=int, default=16)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--calls", type=int, default=20, help="timed calls per round")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the result to this JSON file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    k = args.k
    rp, ci = matgen.rmat(args.scale, 16)  # as bench.py:secondary_spmm
    n, nnz = len(rp) - 1, len(ci)
    va16 = matgen.fill(nnz, 0.0, 1.0, 23, dtype=np.float32).astype(np.float16)
    X16 = matgen.fill(n * k, -1.0, 1.0, 5, dtype=np.float32).reshape(n, k).astype(np.float16)
    rpd, cid = torch.from_numpy(rp).to(dev), torch.from_numpy(ci).to(dev)
    A = {"f16": sp.CrsMatrix(rpd, cid, torch.from_numpy(va16).to(dev), n),
         "f32": sp.CrsMatrix(rpd, cid, torch.from_numpy(va16.astype(np.float32)).to(dev), n)}
    Xr = {"f16": torch.from_numpy(X16).to(dev)}
    Xr["f32"] = Xr["f16"].float()
    variants = [(p, lay) for lay in ("right", "left") for p in ("f32", "f16")]
    X, Y, h = {}, {}, {}
    for p, lay in variants:
        dt = torch.float16 if p == "f16" else torch.float32
        X[p, lay] = Xr[p] if lay == "right" else Xr[p].t().contiguous().t()
        Y[p, lay] = torch.full((n, k) if lay == "right" else (k, n), float("nan"), dtype=dt, device=dev)
        if lay == "left":
            Y[p, lay] = Y[p, lay].t()
        h[p, lay] = sp.SPMVHandle()
        for _ in range(args.warmup):
            sp.spmv(h[p, lay], "N", 1.0, A[p], X[p, lay], 0.0, Y[p, lay])
    torch.cuda.synchronize()
    times = {v: [] for v in variants}
    for _ in range(args.rounds):
        for v in variants:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.calls):
                sp.spmv(h[v], "N", 1.0, A[v[0]], X[v], 0.0, Y[v])
            e1.record()
            torch.cuda.synchronize()
            times[v].append(e0.elapsed_time(e1) / args.calls)
    ident = {lay: bool(torch.equal(Y["f16", lay].contiguous().view(torch.int16), Y["f32", lay].half().contiguous().view(torch.int16)))
             for lay in ("right", "left")}
    items = n_items(rp)
    alg16 = nnz * (2 + 4) + 16 * items + 4 * (n + 1) + n * k * 2 + n * k * 2
    gather16 = alg16 - n * k * 2 + nnz * k * 2
    res = {"card": card(), "config": f"R-MAT scale {args.scale}, k = {k}, alpha = 1, beta = 0", "rows": n, "nnz": nnz, "items": items,
           "bytes_f16": {"algorithmic": alg16, "gather_model": gather16}, "bit_identical": ident,
           "calls_per_round": args.calls, "rounds": args.rounds, "variants": {}}
    for p, lay in variants:
        ms = float(np.mean(times[p, lay]))
        res["variants"][f"{p}_{lay}"] = {"kernel": h[p, lay].last_kernel(), "ms_per_call": round(ms, 4),
                                         "ms_rounds": [round(t, 4) for t in times[p, lay]], "GFLOPs": round(2 * nnz * k / ms / 1e6, 1)}
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)
    print(json.dumps(res))
    assert all(ident.values()), "fp16 and fp32 disagree"


if __name__ == "__main__":
    main()
