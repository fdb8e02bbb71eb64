"""Static resource usage of every kernel instantiation in the in-tree library (runs without a GPU):
registers / thread, stack bytes (local-memory frame: spills or indexed locals), static shared memory, from
`cuobjdump --dump-resource-usage`.   python scripts/resource_summary.py > resource_usage.txt"""
import re
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
LIB = ROOT / "mimo_b200" / "libmimo_b200.so"


def main():
    out = subprocess.run(["cuobjdump", "--dump-resource-usage", str(LIB)], capture_output=True, text=True, check=True).stdout
    rows, name = [], None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            d = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
            name = re.sub(r"\(.*", "", d).replace("void ", "").replace("mimo::", "")
            continue
        m = re.match(r"\s*REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", line)
        if m and name:
            rows.append((name, *map(int, m.groups())))
            name = None
    print(f"Resource usage of {LIB.name}: {len(rows)} kernel instantiations (sm_90a)\n"
          "dynamic shared memory is set at launch and not listed; STACK > 0 marks a local-memory frame\n")
    print(f"{'kernel':72s} {'regs':>5s} {'stack':>6s} {'smem':>6s} {'local':>6s}")
    for r in sorted(rows):
        print(f"{r[0][:72]:72s} {r[1]:5d} {r[2]:6d} {r[3]:6d} {r[4]:6d}")
    print(f"\nmax registers: {max(r[1] for r in rows)}; kernels with a stack frame: "
          f"{sum(1 for r in rows if r[2] > 0)} of {len(rows)}")


if __name__ == "__main__":
    sys.exit(main())
