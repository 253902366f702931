"""A short campaign of tools/emu/fuzz_guard.py: random shapes / scalar types / modes / kernel variants of every C-ABI
operation, run under the CPU emulation with EVERY array (inputs, outputs, the library's temporaries) fenced by
inaccessible pages, results compared with the oracle.  A kernel that reads or writes one element outside an array
faults (the seed is printed before each case); on a GPU the same access is usually silent.  Longer campaigns:
`python tools/emu/fuzz_guard.py --seeds 0:3000`."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("order,seeds", [("forward", "0:25"), ("random:3", "25:50")])
def test_guarded_fuzz(order, seeds):
    env = dict(os.environ, B200EMU_ORDER=order, B200EMU_GUARD="1")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "emu", "fuzz_guard.py"), "--seeds", seeds], capture_output=True,
                         text=True, timeout=1200, env=env, cwd=ROOT)
    tail = (out.stdout + out.stderr)[-2500:]
    assert out.returncode == 0, tail
    assert "0 mismatches" in out.stdout, tail
