"""Block SpGEMM (BsrMatrix C = A*A) against the point SpGEMM on the same operator.

Workloads (inputs generated from seeds):
  lap27   matgen.lap27(64, 64, 64, ndof=3): with node-major rows it is exactly a BsrMatrix of dense 3x3 blocks (262,144 block
          rows, 27 blocks per interior row).  Block: symbolic on the block graph + block numeric.  Point: the same operator as
          CSR through point symbolic + numeric -- what a user has without block SpGEMM.  Rounds alternate block and point.
  rand4 / rand8   a random block matrix at bs = 4 and bs = 8 (block graph from matgen.kk_generate).
For each: symbolic ms (host wall clock: symbolic returns nnz(C) to the host), numeric ms (CUDA events; the first numeric on a
plan also groups the block rows and is reported apart), block GFLOP/s = 2*bs^3*products/t, algorithmic bytes (A, B and C
once) and gather-model bytes (a B block and its column per product), and their fraction of 3.35 TB/s.  Bits of sampled block
rows are checked against the restatement of the reference's bspgemm_debug_numeric.  Prints the card's name and power limit
and one JSON line (stdout; --out FILE also writes it there)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from kokkos_kernels_b200 import matgen, sparse as sp  # noqa: E402
import bspgemm_cases as BC  # noqa: E402

HBM_BPS = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable ({e})"
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q}


def point_to_bsr(rp, ci, va, bs):
    """node-major point CSR whose bs x bs node blocks are all dense -> (block row map, block columns, row-major values)"""
    n = len(rp) - 1
    rows = np.repeat(np.arange(n, dtype=np.int64), np.diff(rp))
    br, bc = rows // bs, ci.astype(np.int64) // bs
    nbc = (int(ci.max()) // bs + 1) if len(ci) else 0
    key = br * nbc + bc
    uk, inv = np.unique(key, return_inverse=True)
    assert len(ci) == len(uk) * bs * bs, "not a BsrMatrix of dense blocks"
    vals = np.empty(len(uk) * bs * bs, dtype=va.dtype)
    vals[inv * bs * bs + (rows % bs) * bs + (ci % bs)] = va
    mb = n // bs
    brp = np.zeros(mb + 1, dtype=np.int32)
    np.add.at(brp, (uk // nbc) + 1, 1)
    return np.cumsum(brp).astype(np.int32), (uk % nbc).astype(np.int32), vals


def timed_numeric(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def run_block(A, bs, reps):
    """symbolic + numeric on a fresh handle; then `reps` timed numeric re-runs on the same structure"""
    kh = sp.KokkosKernelsHandle()
    kh.create_spgemm_handle()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    C = sp.block_spgemm_symbolic(kh, A, False, A, False)
    t_sym = (time.perf_counter() - t0) * 1e3
    t_first = timed_numeric(lambda: sp.block_spgemm_numeric(kh, A, False, A, False, C))
    ts = [timed_numeric(lambda: sp.block_spgemm_numeric(kh, A, False, A, False, C)) for _ in range(reps)]
    return C, t_sym, t_first, ts


def run_point(P, reps):
    kh = sp.KokkosKernelsHandle()
    kh.create_spgemm_handle()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    C = sp.spgemm_symbolic(kh, P, False, P, False)
    t_sym = (time.perf_counter() - t0) * 1e3
    t_first = timed_numeric(lambda: sp.spgemm_numeric(kh, P, False, P, False, C))
    ts = [timed_numeric(lambda: sp.spgemm_numeric(kh, P, False, P, False, C)) for _ in range(reps)]
    return C, t_sym, t_first, ts


def model(bs, rp, ci, nnzC, products, itemsize, t_ms):
    bb = bs * bs
    mb = len(rp) - 1
    alg = (len(ci) * (4 + bb * itemsize)) * 2 + 4 * 3 * (mb + 1) + nnzC * (4 + bb * itemsize)
    gather = alg + products * (4 + bb * itemsize)
    t = t_ms * 1e-3
    flops = 2.0 * bs ** 3 * products
    return {"gflops": flops / t / 1e9, "alg_bytes": alg, "gather_bytes": gather, "alg_frac_hbm": alg / t / HBM_BPS,
            "gather_frac_hbm": gather / t / HBM_BPS}


def check_rows(orc, bs, rp, ci, va, C, nrows=64, seed=0):
    """bits of sampled block rows against the restatement (A restricted to those rows, all of B)"""
    mb = len(rp) - 1
    rows = np.unique(np.random.default_rng(seed).integers(0, mb, nrows))
    rows = np.union1d(rows, [0, mb - 1])
    lens = rp[rows + 1] - rp[rows]
    srp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    sci = np.concatenate([ci[rp[r]:rp[r + 1]] for r in rows]).astype(np.int32)
    bb = bs * bs
    sva = np.concatenate([va[rp[r] * bb:rp[r + 1] * bb] for r in rows])
    ncols = int(ci.max()) + 1
    exp = orc.bspgemm(bs, (srp, sci, sva), (rp, ci, va), len(rows), mb, ncols)
    rpC = C.row_map.cpu().numpy()
    bad = 0
    for t, r in enumerate(rows):
        s, e = int(rpC[r]), int(rpC[r + 1])
        gc = C.entries[s:e].cpu().numpy()
        gv = C.values[s * bb:e * bb].cpu().numpy()
        ec = exp[1][exp[0][t]:exp[0][t + 1]]
        ev = exp[2][exp[0][t] * bb:exp[0][t + 1] * bb]
        if not (np.array_equal(gc, ec) and BC.same_bits(gv, ev)):
            bad += 1
    return int(len(rows)), bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    info = card()
    print("card:", info, flush=True)
    orc = BC.BlockOracle()
    res = {"card": info, "workloads": []}

    # ---- lap27 x 3 dof: block vs point, alternating
    g = args.grid
    t = time.time()
    prp, pci, pva = matgen.lap27(g, g, g, ndof=3, noise=0.5)
    brp, bci, bva = point_to_bsr(prp, pci, pva, 3)
    print(f"lap27 {g}^3 x 3: point n={len(prp) - 1} nnz={len(pci)}; block mb={len(brp) - 1} nnzb={len(bci)} ({time.time() - t:.1f}s)",
          flush=True)
    td = lambda x: torch.from_numpy(x).to(dev)
    Ab = sp.BsrMatrix(td(brp), td(bci), td(bva), len(brp) - 1, 3)
    Ap = sp.CrsMatrix(td(prp), td(pci), td(pva), len(prp) - 1)
    products = int(np.sum(np.diff(brp)[bci].astype(np.int64)))
    pproducts = int(np.sum(np.diff(prp)[pci].astype(np.int64)))
    w = {"name": f"lap27({g},{g},{g}) ndof=3, C = A*A, fp64", "bs": 3, "block_rows": len(brp) - 1, "nnzb": len(bci),
         "block_products": products, "point_products": pproducts, "rounds": []}
    for rnd in range(args.rounds + 1):
        Cb, bs_sym, bs_first, bs_num = run_block(Ab, 3, args.reps)
        Cp, p_sym, p_first, p_num = run_point(Ap, args.reps)
        r = {"block_symbolic_ms": bs_sym, "block_first_numeric_ms": bs_first, "block_numeric_ms": min(bs_num),
             "point_symbolic_ms": p_sym, "point_first_numeric_ms": p_first, "point_numeric_ms": min(p_num)}
        print(("warm-up " if rnd == 0 else "") + json.dumps(r), flush=True)
        if rnd > 0:
            w["rounds"].append(r)
        if rnd < args.rounds:
            del Cb, Cp
    best = {k: min(r[k] for r in w["rounds"]) for k in w["rounds"][0]}
    w["best"] = best
    w["nnzC_blocks"] = Cb.nnz()
    w["block_model"] = model(3, brp, bci, Cb.nnz(), products, 8, best["block_numeric_ms"])
    w["point_numeric_gflops"] = 2.0 * pproducts / (best["point_numeric_ms"] * 1e-3) / 1e9
    w["block_total_ms"] = best["block_symbolic_ms"] + best["block_numeric_ms"]
    w["point_total_ms"] = best["point_symbolic_ms"] + best["point_numeric_ms"]
    w["checked_rows"], w["bad_rows"] = check_rows(orc, 3, brp, bci, bva, Cb)
    # the point result is the same operator: its values equal the block values up to association (not bit-compared)
    print(json.dumps({k: w[k] for k in ("best", "block_model", "block_total_ms", "point_total_ms", "checked_rows", "bad_rows")}),
          flush=True)
    res["workloads"].append(w)
    del Cb, Cp, Ab, Ap
    torch.cuda.empty_cache()

    # ---- random block matrices
    for bs, mb, per in ((4, 200_000, 12), (8, 100_000, 10)):
        rp, ci, va = BC.random_bsr(mb, mb, mb * per, mb, per // 2, bs, seed=17 + bs)
        A = sp.BsrMatrix(td(rp), td(ci), td(va), mb, bs)
        products = int(np.sum(np.diff(rp)[ci].astype(np.int64)))
        rounds = []
        for rnd in range(args.rounds + 1):
            C, t_sym, t_first, ts = run_block(A, bs, args.reps)
            if rnd > 0:
                rounds.append({"block_symbolic_ms": t_sym, "block_first_numeric_ms": t_first, "block_numeric_ms": min(ts)})
            if rnd < args.rounds:
                del C
        best = {k: min(r[k] for r in rounds) for k in rounds[0]}
        ww = {"name": f"random bs={bs} mb={mb} ~{per} blocks/row, C = A*A, fp64", "bs": bs, "block_products": products,
              "nnzC_blocks": C.nnz(), "rounds": rounds, "best": best,
              "block_model": model(bs, rp, ci, C.nnz(), products, 8, best["block_numeric_ms"])}
        ww["checked_rows"], ww["bad_rows"] = check_rows(orc, bs, rp, ci, va, C)
        print(json.dumps({k: ww[k] for k in ("name", "best", "block_model", "checked_rows", "bad_rows")}), flush=True)
        res["workloads"].append(ww)
        del C, A
        torch.cuda.empty_cache()

    line = json.dumps(res)
    print(line, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    assert all(w["bad_rows"] == 0 for w in res["workloads"])


if __name__ == "__main__":
    main()
