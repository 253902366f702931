"""The achievable HBM read rate of the card (needs a GPU): compiles tools/hbm_read.cu into a temporary directory, runs it, and
prints one JSON line with every case it timed, the best bulk-copy rate, and the card's name, power limit and SM clock (median
of samples taken while it runs).  This is the ceiling the tiled SpMV's bytes per launch are set against (DESIGN.md section 7).

  python tools/bench_hbm_read.py [--gb 4.3] [--reps 20] [--out FILE]
"""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import threading

HERE = os.path.dirname(os.path.abspath(__file__))


def nvcc():
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def smi(q):
    out = subprocess.run(["nvidia-smi", "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0], f"--query-gpu={q}",
                          "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout.strip()
    return [s.strip() for s in out.splitlines()[0].split(",")] if out else []


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gb", type=float, default=4.3, help="bytes streamed per launch, in GB (the SpMV moves 4.5)")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the result to this JSON file")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "hbm_read")
        subprocess.check_call([nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-o", exe,
                               os.path.join(HERE, "hbm_read.cu")])
        card = dict(zip(("name", "power_limit_w", "clocks_max_sm_mhz"), smi("name,power.limit,clocks.max.sm")))
        clocks, done = [], threading.Event()

        def sample():
            while not done.wait(0.25):
                try:
                    clocks.append(int(smi("clocks.sm")[0]))
                except Exception:
                    pass

        th = threading.Thread(target=sample, daemon=True)
        th.start()
        try:
            out = subprocess.run([exe, str(args.gb), str(args.reps)], capture_output=True, text=True, check=True).stdout
        finally:
            done.set()
            th.join()
    cases = [json.loads(line) for line in out.splitlines() if line.startswith("{")]
    bulk = [c for c in cases if c["kind"] == "bulk"]
    res = {"card": card, "sm_clock_mhz_median": statistics.median(clocks) if clocks else None,
           "device": next(c for c in cases if c["kind"] == "device"),
           "hbm_read_gbs_bulk_best": max(c["gbs"] for c in bulk),
           "hbm_read_gbs_ld128_best": max(c["gbs"] for c in cases if c["kind"] == "ld128"),
           "cases": [c for c in cases if c["kind"] != "device"]}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
