"""Writes tests/golden/context_sweep.json from the reference's OWN src/pipelines/context.py (pure numpy, importable as it
is): a sweep of (step, num_frames, context_size, context_stride, context_overlap, closed_loop) with, per case, the number
of windows and a CRC-32 of their JSON text (keeps the fixture small), the full lists of a few cases, bit-reversal
fractions of `ordered_halving`, and `get_total_steps` values.   python oracle/gen_context_golden.py
Test infrastructure: needs a checkout of the original project, named by MIMO_REFERENCE."""
import importlib.util
import json
import os
import sys
import zlib
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
REF = Path(os.environ.get("MIMO_REFERENCE") or sys.exit(__doc__)) / "src" / "pipelines" / "context.py"


def sweep_cases():
    for frames in (1, 7, 24, 25, 26, 31, 47, 48, 49, 64, 100, 150, 257):
        for size, overlap in ((24, 4), (16, 4), (24, 0), (12, 6), (8, 2)):
            for stride in (1, 2, 3, 4):
                for step in (0, 1, 2, 3, 19):
                    for closed in (True, False):
                        yield step, frames, size, stride, overlap, closed


def crc(windows) -> int:
    return zlib.crc32(json.dumps(windows, separators=(",", ":")).encode())


def main():
    spec = importlib.util.spec_from_file_location("ref_context", REF)
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    cases, full = [], {}
    for c in sweep_cases():
        step, frames, size, stride, overlap, closed = c
        w = list(ref.uniform(step, 20, frames, size, stride, overlap, closed))
        cases.append([*c[:5], int(closed), len(w), crc(w)])
        if (frames, size, overlap, stride) in ((48, 24, 4, 1), (64, 24, 4, 1), (150, 24, 4, 3), (31, 16, 4, 2)) and step in (0, 3):
            full[",".join(map(str, [*c[:5], int(closed)]))] = w
    halving = {str(v): ref.ordered_halving(v) for v in (0, 1, 2, 3, 4, 7, 19, 24, 1000, 12345, 2 ** 32, 2 ** 63, 2 ** 64 - 1)}
    sched = ref.get_context_scheduler("uniform")
    totals = [[n, frames, size, stride, overlap,
               ref.get_total_steps(sched, list(range(n)), 20, frames, size, stride, overlap)]
              for n in (1, 2, 20, 25) for frames, size, stride, overlap in ((24, 24, 1, 4), (48, 24, 1, 4), (150, 24, 3, 4), (64, 16, 2, 4))]
    out = {"generator": "oracle/gen_context_golden.py over the original project's src/pipelines/context.py",
           "case_fields": ["step", "num_frames", "context_size", "context_stride", "context_overlap", "closed_loop",
                           "n_windows", "crc32_of_json"],
           "cases": cases, "full": full, "ordered_halving": halving,
           "total_steps_fields": ["n_timesteps", "num_frames", "context_size", "context_stride", "context_overlap", "total"],
           "total_steps": totals}
    p = ROOT / "tests" / "golden" / "context_sweep.json"
    p.write_text(json.dumps(out, separators=(",", ":")))
    print(f"{len(cases)} cases, {len(full)} full lists, {len(totals)} totals -> {p} ({p.stat().st_size >> 10} KiB)")


if __name__ == "__main__":
    main()
