"""tools/gpu_check (the torch-free GPU validation harness) must build and its host side -- generators, oracle calls,
comparison code of every suite -- must run to completion without a GPU (`--dry`: device buffers live in host memory,
C-ABI calls are skipped, so every comparison fails by construction but nothing may crash)."""
import collections
import json
import os
import subprocess

import kokkos_kernels_b200 as kk

CHK = os.path.join(kk._lib.LIBDIR, "gpu_check")


def test_harness_host_side_runs(tmp_path):
    assert os.path.exists(CHK), "build() did not produce tools/gpu_check"
    out = tmp_path / "dry.jsonl"
    suites = ["crs", "jacobi", "spmv_t", "spmm_sweep"]
    cmd = [CHK, "--dry", "--out", str(out)]
    for s in suites:
        cmd += ["--suite", s]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    recs = [json.loads(l) for l in open(out)]
    summary = {r["check"]: r["detail"] for r in recs if r["suite"] == "summary"}
    assert set(summary) == set(suites), res.stderr[-2000:]
    for s in suites:
        assert "signal=0" in summary[s] and "exit=1" in summary[s], (s, summary[s])  # ran to the end, comparisons failed as they must
    assert res.returncode == len(suites)
    # every case of every suite is recorded; spmm_sweep: 4 matrices, each with a plan and without one
    per_suite = collections.Counter(r["suite"] for r in recs if r["suite"] != "summary")
    assert per_suite == {"crs": 24, "jacobi": 4, "spmv_t": 4, "spmm_sweep": 8}, per_suite
