"""Cost of window-mode GroupNorm (use_inflated_groupnorm=False) against per-frame GroupNorm, on one GPU.

Times one captured UNet3D forward (full SD1.5 width, 2 CFG branches x 24 frames, 512 x 512 -> 64 x 64 latents, fp16)
with each mode, alternating, with CUDA events; prints the medians and the difference as one JSON line.

    python scripts/window_gn_bench.py [--reps 20] [--frames 24] [--size 512]
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--frames", type=int, default=24)
    ap.add_argument("--size", type=int, default=512)
    args = ap.parse_args()
    from mimo_b200 import engine as E
    from oracle import torch_oracle as O
    dev = torch.device("cuda")
    f, hw = args.frames, args.size // 8
    cfg = O.UNetConfig()
    sd_den, sd_ref = O.make_denoising_unet_sd(cfg, 1), O.make_reference_unet_sd(cfg, 2)
    g = torch.Generator().manual_seed(3)
    ref_lat = torch.randn(1, 4, hw, hw, generator=g).half().to(dev)
    emb = torch.randn(1, 1, 768, generator=g)
    ehs = torch.cat([torch.zeros_like(emb), emb]).half().to(dev)
    x = torch.randn(2, 8, f, hw, hw, generator=g).half().to(dev)
    pose = (torch.randn(2 * f * hw * hw, 320, generator=g) * 0.1).half().to(dev)
    ref = E.UNetEngine(sd_ref, E.UNetSpec(in_channels=4, motion=False, out_head=False), dev)
    engines = {}
    for name, inflated in (("per_frame", True), ("window", False)):
        den = E.UNetEngine(sd_den, E.UNetSpec(inflated_groupnorm=inflated), dev)
        den.begin_clip(ehs, ref.write_banks(ref_lat, ehs, den), cfg=True, frames=f)
        for _ in range(3):  # eager, capture, replay
            den.forward(x, 499, pose)
        engines[name] = den
    torch.cuda.synchronize()
    times = {k: [] for k in engines}
    for _ in range(args.reps):
        for name, den in engines.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            den.forward(x, 499, pose)
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1))
    med = {k: statistics.median(v) for k, v in times.items()}
    spread = {k: [min(v), max(v)] for k, v in times.items()}
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "frames": f, "latent": hw, "median_ms": med,
                      "min_max_ms": spread, "window_minus_per_frame_ms": med["window"] - med["per_frame"],
                      "window_over_per_frame": med["window"] / med["per_frame"]}))


if __name__ == "__main__":
    main()
