"""Cost of rescaled classifier-free guidance (guidance_rescale).

Prints, in one run on one GPU, as one JSON document:
  * the card's name and power limit;
  * the CUDA-event time of one mimo_cfg_rescale call (statistics pass + apply pass) on 2 x [1, 4, 24, 64, 64] fp16
    without a counter, and on 2 x [1, 4, 64, 64, 64] with one (64 frames, as 4 context windows leave them), with the
    bytes the algorithm moves (read both halves, write one output; the apply pass's second read of the halves is not
    counted: at these sizes it is served from L2) and the rate that makes;
  * for the 512 x 512 x 24-frame, 20-step DDIM clip at CFG 3.5 (fp16, inputs resident on the device, as bench.py's
    value): seconds per clip at guidance_rescale 0 and 0.7, timed in alternation round after round so that clock drift
    falls on both alike; median and min-max over the rounds.
Usage: python scripts/guidance_rescale_bench.py [--rounds K] [--json FILE]
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

import bench  # noqa: E402  (pipeline construction and inputs of the benchmark)
from mimo_b200 import ops  # noqa: E402
from mimo_b200.host import scheduler as S  # noqa: E402
from scripts.any_size_bench import card  # noqa: E402

FRAMES, GUIDANCE, SIZE, STEPS, PHI = 24, 3.5, 512, 20, 0.7


def kernel_times(device, iters: int = 200):
    """{case: (ms per call, algorithmic bytes per call)} of ops.cfg_rescale on the clip's latent shape."""
    out = {}
    for name, frames, windows in (("24 frames, no counter", 24, 1), ("64 frames, counter", 64, 4)):
        shape = (1, 4, frames, SIZE // 8, SIZE // 8)
        g = torch.Generator(device=device).manual_seed(0)
        pred = torch.randn((2,) + shape[1:], device=device, generator=g).half()
        pu, pc = pred[0].contiguous(), pred[1].contiguous()
        counter = torch.full((frames,), 2.0, device=device).half() if windows > 1 else None
        dst = torch.empty_like(pu)
        fn = lambda: ops.cfg_rescale(pu, pc, GUIDANCE, PHI, out=dst, counter=counter, frame_stride=shape[3] * shape[4])
        for _ in range(10):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        n = pu.numel()
        out[name] = (e0.elapsed_time(e1) / iters, 3 * n * pu.element_size() + (frames * 2 if counter is not None else 0))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3, help="timed rounds (each times both variants once)")
    ap.add_argument("--json", default=None, help="also write the result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("guidance_rescale_bench.py: no CUDA device (the engine has no CPU fallback)")
    device = torch.device("cuda", 0)
    res = {"card": card(), "workload": f"{SIZE}x{SIZE} x {FRAMES} frames, DDIM {STEPS} steps, CFG {GUIDANCE}, fp16"}
    res["kernel"] = [{"case": k, "us": round(1e3 * ms, 2), "bytes": b, "GB_per_s": round(b / (ms * 1e-3) / 1e9, 1)}
                     for k, (ms, b) in kernel_times(device).items()]
    pipe = bench.build_pipeline(device)
    pipe.scheduler = S.DDIMScheduler(**bench.SCHED_KW)
    ref_img, poses, bks = bench.synthetic_inputs(FRAMES, SIZE)
    host = pipe.preprocess(ref_img, poses, bks, SIZE, SIZE, FRAMES, torch.Generator().manual_seed(42), torch.float16,
                           STEPS)
    dev_in = {k: v.to(device) for k, v in host.items()}
    run = lambda phi: pipe.sample_tensors(dev_in, STEPS, GUIDANCE, guidance_rescale=phi)
    variants = (0.0, PHI)
    for phi in variants:  # warm-up: the first forward of a shape runs eager, the second captures its graph
        run(phi)
        run(phi)
    torch.cuda.synchronize()
    times = {phi: [] for phi in variants}
    for _ in range(args.rounds):
        for phi in variants:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = run(phi)
            e1.record()
            torch.cuda.synchronize()
            times[phi].append(e0.elapsed_time(e1) / 1e3)
            assert bool(torch.isfinite(out["videos"]).all()), phi
    res["clip"] = [{"guidance_rescale": phi, "clip_s_median": round(statistics.median(t), 4),
                    "clip_s_min": round(min(t), 4), "clip_s_max": round(max(t), 4), "clip_s_all": [round(x, 4) for x in t]}
                   for phi, t in times.items()]
    print(json.dumps(res, indent=1))
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
