"""bench.py --dump-outputs on the host (no GPU needed): file names, float64, the per-result size cap, whole results when they
fit, and a sample of positions that is the same run after run and holds the values found at those positions."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# bench.py sets OpenMP variables when imported: run it in a process of its own
SCRIPT = """
import json, sys, torch
sys.path.insert(0, sys.argv[1])
import bench
out = sys.argv[2]
bench.dump_outputs(out, "y", {"y": torch.arange(10_000_000, dtype=torch.float64) * 0.5})
bench.dump_outputs(out, "spgemm_row_map", {"spgemm_row_map": torch.arange(1001, dtype=torch.int32)})
n = 3_000_000
bench.dump_outputs(out, "spgemm_C", {"spgemm_entries": torch.arange(n, dtype=torch.int32),
                                     "spgemm_values": torch.arange(n, dtype=torch.float64) * -2.0})
print(json.dumps(bench.DUMP_BYTES))
"""


def _dump(out):
    r = subprocess.run([sys.executable, "-c", SCRIPT, ROOT, str(out)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_dump_outputs(tmp_path):
    caps = _dump(tmp_path / "a")
    _dump(tmp_path / "b")
    assert sum(caps.values()) <= 64_000_000
    a = tmp_path / "a"
    names = sorted(os.listdir(a))
    assert names == sorted(os.listdir(tmp_path / "b")) == ["spgemm_C_rows.npy", "spgemm_entries.npy", "spgemm_row_map.npy",
                                                           "spgemm_values.npy", "y.npy", "y_rows.npy"]
    for name in names:  # same positions and values in both runs
        assert (a / name).read_bytes() == (tmp_path / "b" / name).read_bytes(), name
    arrays = {name: np.load(a / name) for name in names}
    assert all(v.dtype == np.float64 and v.ndim == 1 for v in arrays.values())
    # y (80 MB) is sampled within its cap
    rows = arrays["y_rows.npy"]
    assert (a / "y.npy").stat().st_size + (a / "y_rows.npy").stat().st_size <= caps["y"] + 256
    assert len(rows) > 1_000_000 and np.all(np.diff(rows) > 0) and rows[0] >= 0 and rows[-1] < 10_000_000
    assert np.array_equal(arrays["y.npy"], rows * 0.5)
    # a small result is written whole, without positions
    assert np.array_equal(arrays["spgemm_row_map.npy"], np.arange(1001, dtype=np.float64))
    # two arrays of one result share the positions
    rows = arrays["spgemm_C_rows.npy"]
    assert sum((a / f).stat().st_size for f in ("spgemm_C_rows.npy", "spgemm_entries.npy", "spgemm_values.npy")) <= caps["spgemm_C"] + 384
    assert np.array_equal(arrays["spgemm_entries.npy"], rows) and np.array_equal(arrays["spgemm_values.npy"], rows * -2.0)
