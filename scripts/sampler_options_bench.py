"""Cost of the sampler options eta > 0 (stochastic DDIM) and interpolation_factor = 2 (latent frame interpolation).

Prints, in one run on one GPU:
  * the card's name and power limit;
  * for a 512 x 512 x 24-frame clip, 20 DDIM steps, CFG 3.5, fp16, inputs resident on the device
    (pipeline.sample_tensors, as bench.py's value): seconds per clip and output frames/s of four variants -
    default, eta = 1, interpolation_factor = 2 (slerp; 47 output frames), and both - timed in alternation, round after
    round, so that clock drift falls on all four alike; the median over the rounds is reported.
Usage: python scripts/sampler_options_bench.py [--rounds K] [--json FILE]
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
from mimo_b200.host import interpolation as I  # noqa: E402
from scripts.any_size_bench import card  # noqa: E402

FRAMES, STEPS, GUIDANCE, SIZE = 24, 20, 3.5, 512
VARIANTS = {"default": dict(eta=0.0, interpolation_factor=1), "eta=1": dict(eta=1.0, interpolation_factor=1),
            "k=2": dict(eta=0.0, interpolation_factor=2), "eta=1,k=2": dict(eta=1.0, interpolation_factor=2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3, help="timed rounds (each times every variant once)")
    ap.add_argument("--json", default=None, help="also write the result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sampler_options_bench.py: no CUDA device (the engine has no CPU fallback)")
    device = torch.device("cuda", 0)
    res = {"card": card(), "workload": f"{SIZE}x{SIZE} x {FRAMES} frames, {STEPS} DDIM steps, CFG {GUIDANCE}, fp16, "
                                       "inputs resident; interpolation: slerp"}
    pipe = bench.build_pipeline(device)
    I.set_tensor_interpolation_method(True)
    ref_img, poses, bks = bench.synthetic_inputs(FRAMES, SIZE)
    # eta > 0 reads its per-step noise from preprocess(), drawn from the generator right after the initial latents
    host = pipe.preprocess(ref_img, poses, bks, SIZE, SIZE, FRAMES, torch.Generator().manual_seed(42), torch.float16,
                           STEPS, 1.0)
    dev_in = {k: v.to(device) for k, v in host.items()}

    def run(kw):
        return pipe.sample_tensors(dev_in, STEPS, GUIDANCE, **kw)

    for kw in VARIANTS.values():  # warm-up: the first forward of a shape runs eager, the second captures its graph
        run(kw)
        run(kw)
    torch.cuda.synchronize()
    times = {name: [] for name in VARIANTS}
    frames_out = {}
    for _ in range(args.rounds):
        for name, kw in VARIANTS.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = run(kw)
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / 1e3)
            frames_out[name] = out["videos"].shape[2]
            assert bool(torch.isfinite(out["videos"]).all()), name
    base = statistics.median(times["default"])
    res["variants"] = []
    for name in VARIANTS:
        s = statistics.median(times[name])
        res["variants"].append({"variant": name, "clip_s": round(s, 4), "clip_s_all": [round(t, 4) for t in times[name]],
                                "output_frames": frames_out[name], "output_frames_per_s": round(frames_out[name] / s, 3),
                                "time_vs_default": round(s / base, 4)})
    print(json.dumps(res, indent=1))
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
