"""Cost of the motion-module layouts: inference_v2.yaml's against the AnimateDiff-v1-style and v3-style layouts (no
mid-block module; v1 also runs its ResBlock GroupNorms over the window), on one GPU.

Times one captured UNet3D forward (full SD1.5 width, 2 CFG branches x 24 frames, 512 x 512 -> 64 x 64 latents, fp16)
per layout, alternating, with CUDA events; prints the GPU, its power limit, the medians and their spread as one JSON
line. The weights are seeded random ones; the spatial weights are the same for every layout.

    python scripts/motion_layout_bench.py [--reps 20] [--frames 24] [--size 512]
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

# name -> (use_inflated_groupnorm, motion_module_mid_block, temporal_position_encoding_max_len)
LAYOUTS = {"v2": (True, True, 32), "v1": (False, False, 24), "v3": (True, False, 32)}


def _power_limit() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--frames", type=int, default=24)
    ap.add_argument("--size", type=int, default=512)
    args = ap.parse_args()
    from mimo_b200 import engine as E
    from mimo_b200.host.schema import MotionLayout
    from oracle import motion_layout_oracle as ML
    from oracle import torch_oracle as O
    dev = torch.device("cuda")
    f, hw = args.frames, args.size // 8
    cfg = O.UNetConfig()
    sd_ref = O.make_reference_unet_sd(cfg, 2)
    g = torch.Generator().manual_seed(3)
    ref_lat = torch.randn(1, 4, hw, hw, generator=g).half().to(dev)
    emb = torch.randn(1, 1, 768, generator=g)
    ehs = torch.cat([torch.zeros_like(emb), emb]).half().to(dev)
    x = torch.randn(2, 8, f, hw, hw, generator=g).half().to(dev)
    pose = (torch.randn(2 * f * hw * hw, 320, generator=g) * 0.1).half().to(dev)
    ref = E.UNetEngine(sd_ref, E.UNetSpec(in_channels=4, motion=False, out_head=False), dev)
    engines = {}
    for name, (inflated, mid, max_len) in LAYOUTS.items():
        spec = E.UNetSpec(inflated_groupnorm=inflated, motion_layout=MotionLayout(mid_block=mid, max_len=max_len))
        lay = ML.Layout(mid_block=mid, max_len=max_len)
        den = E.UNetEngine(ML.make_denoising_unet_sd(cfg, lay, 1), spec, dev)
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
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "power_limit": _power_limit(), "frames": f, "latent": hw,
                      "median_ms": med, "min_max_ms": spread,
                      "v1_minus_v2_ms": med["v1"] - med["v2"], "v3_minus_v2_ms": med["v3"] - med["v2"]}))


if __name__ == "__main__":
    main()
