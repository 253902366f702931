#!/usr/bin/env python
"""Static SASS instructions per source line of one kernel (no GPU needed): which source constructs a kernel's
instruction count comes from.  Uses the object files of the in-tree build (compiled with -lineinfo).

  python tools/sass_lines.py spgemm num_hash_kernel 'double, (int)128, (int)4096'
  python tools/sass_lines.py spmm spmm_item_coop_kernel 'float, (int)4, (int)4'

Prints `line  #instructions  source text` for the kernel whose demangled name contains every given substring
(first match), plus totals per opcode class.  Weigh the lines with the trip counts of the case at hand."""
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "kokkos-kernels_b200", "lib")
CSRC = os.path.join(ROOT, "kokkos-kernels_b200", "csrc")


def main():
    if len(sys.argv) < 3:
        print(__doc__)
        return 2
    unit, needles = sys.argv[1], sys.argv[2:]
    obj = os.path.join(LIB, unit + ".cu.o")
    with tempfile.TemporaryDirectory() as tmp:
        subprocess.run(["cuobjdump", "-xelf", "all", obj], cwd=tmp, check=True, capture_output=True)
        cubin = [f for f in os.listdir(tmp) if f.endswith(".cubin")][0]
        lst = subprocess.run(["nvdisasm", "--print-line-info", cubin], cwd=tmp, capture_output=True, text=True).stdout.split("\n")
    names = sorted({m.group(1) for l in lst for m in [re.match(r"\s*\.section\s+\.text\.(\S+?),", l)] if m})
    dem = dict(zip(names, subprocess.run(["c++filt"] + names, capture_output=True, text=True).stdout.split("\n")))
    pick = [n for n in names if all(s in dem[n] for s in needles)]
    if not pick:
        print("no kernel matches; candidates:\n  " + "\n  ".join(sorted(set(re.sub(r"\(.*", "", d) for d in dem.values()))))
        return 1
    name = pick[0]
    print("kernel:", dem[name][:200])
    start = next(i for i, l in enumerate(lst) if re.match(r"\s*\.section\s+\.text\." + re.escape(name) + ",", l))
    cur, per_line, per_op, total = None, collections.Counter(), collections.Counter(), 0
    for l in lst[start + 1:]:
        if l.strip().startswith(".section"):
            break
        m = re.search(r'//## File "([^"]+)", line (\d+)', l)
        if m:
            cur = (os.path.basename(m.group(1)), int(m.group(2)))
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", l)
        if m:
            per_line[cur] += 1
            per_op[m.group(1).split(".")[0]] += 1
            total += 1
    src_cache = {}
    print(f"total SASS instructions: {total}")
    for (f, ln), c in sorted(per_line.items(), key=lambda kv: (kv[0] or ("", 0))):
        if f not in src_cache:
            p = os.path.join(CSRC, f)
            src_cache[f] = open(p).read().split("\n") if os.path.exists(p) else []
        text = src_cache[f][ln - 1].strip()[:100] if 0 < ln <= len(src_cache[f]) else ""
        print(f"{f}:{ln:5d} {c:5d}  {text}")
    print("by opcode:", ", ".join(f"{k} {v}" for k, v in per_op.most_common(14)))
    return 0


if __name__ == "__main__":
    sys.exit(main())
