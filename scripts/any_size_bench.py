"""Throughput at the reference's default image size, 784 x 784 (98 x 98 latents), where the two coarsest UNet up steps
are not exact doublings (13 -> 25, 25 -> 49) and run as a nearest resize + 3x3 conv instead of the fused mimo_conv_up2x.

Prints, in one run on one GPU:
  * the card's name and power limit;
  * clip frames/s at 784 x 784 and, for scale, 768 x 768 (every level on the fused path): 24 frames, 20 DDIM steps,
    CFG 3.5, fp16, inputs resident on the device (pipeline.sample_tensors, as bench.py's value);
  * per up step of the 784 x 784 denoising UNet (48 frame-samples = 24 frames x 2 CFG branches): CUDA-event times of
    resize + conv3x3 and of conv_up2x on the same input (which computes the 2h x 2w image, the fused path's cost), and the
    difference as the cost of the general path;
  * the M-tile fill of the 3x3 convolutions at w = 98 (a count from the tile rule, not a measurement).
Usage: python scripts/any_size_bench.py [--clips K] [--json FILE]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

import bench  # noqa: E402  (pipeline construction and inputs of the benchmark)
from mimo_b200 import engine as E  # noqa: E402
from mimo_b200 import ops  # noqa: E402

FRAMES, STEPS, GUIDANCE = 24, 20, 3.5


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return {"name": name, "power_limit": power, "sm_clock_max": clock}
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        return {"name": torch.cuda.get_device_name(0), "power_limit": "unknown", "sm_clock_max": "unknown"}


def clip_rate(pipe, size: int, clips: int, device) -> dict:
    ref_img, poses, bks = bench.synthetic_inputs(FRAMES, size)
    host = pipe.preprocess(ref_img, poses, bks, size, size, FRAMES, torch.Generator().manual_seed(42), torch.float16)
    dev_in = {k: v.to(device) for k, v in host.items()}
    pipe.sample_tensors(dev_in, STEPS, GUIDANCE)  # first forward of a shape eager, second captures its graph
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(clips):
        out = pipe.sample_tensors(dev_in, STEPS, GUIDANCE)
    e1.record()
    torch.cuda.synchronize()
    s = e0.elapsed_time(e1) / 1e3 / clips
    assert out["videos"].shape == (1, 3, FRAMES, size, size) and bool(torch.isfinite(out["videos"]).all())
    return {"size": size, "clip_s": round(s, 3), "frames_per_s": round(FRAMES / s, 3)}


def time_ms(fn, iters: int = 20) -> float:
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def up_steps(eng, size: int) -> list:
    lv = eng.levels(size // 8, size // 8)
    nb = len(lv)
    n = 2 * FRAMES
    rows = []
    for i in range(nb - 1):
        (h, w), (th, tw) = lv[nb - 1 - i], lv[nb - 2 - i]
        p = f"up_blocks.{i}.up"
        w4, b = eng.w[p]
        w9, _ = eng.w[p + "_conv"]
        c = w9.shape[1] // 9
        x = torch.randn(n * h * w, c, device=eng.device, dtype=eng.dtype)
        fused_ms = time_ms(lambda: ops.conv_up2x(x, w4, n, h, w, bias=b))
        row = {"level": i, "from": [h, w], "to": [th, tw], "channels": c, "fused_conv_up2x_ms": round(fused_ms, 4),
               "path": "fused" if (th, tw) == (2 * h, 2 * w) else "resize+conv3x3"}
        if row["path"] != "fused":
            r = ops.upsample_nearest(x, n, h, w, th, tw)
            resize_ms = time_ms(lambda: ops.upsample_nearest(x, n, h, w, th, tw, out=r))
            conv_ms = time_ms(lambda: ops.conv3x3(r, w9, n, th, tw, bias=b))
            general_ms = time_ms(lambda: eng._up(p, x, n, h, w, th, tw))
            row.update(resize_ms=round(resize_ms, 4), conv3x3_ms=round(conv_ms, 4), general_ms=round(general_ms, 4),
                       general_minus_fused_ms=round(general_ms - fused_ms, 4))
        rows.append(row)
    return rows


def conv_tile_fill(h: int, w: int, bm: int = 128) -> dict:
    """Rows of a 128-row conv M-tile that hold output pixels, from the tile rule of conv_launch (csrc/gemm_wgmma.cu):
    TW = min(w, 128), TH = min(128 // TW, h), TN images only when a tile spans whole images."""
    tw = min(w, bm)
    th = max(1, min(bm // tw, h))
    tn = max(1, bm // (tw * th)) if th == h else 1
    return {"w": w, "TW": tw, "TH": th, "TN": tn, "rows_used": tw * th * tn, "rows": bm}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=2, help="timed clips per size (after one untimed clip)")
    ap.add_argument("--json", default=None, help="also write the result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("any_size_bench.py: no CUDA device (the engine has no CPU fallback)")
    torch.backends.cuda.matmul.allow_tf32 = False
    device = torch.device("cuda", 0)
    res = {"card": card(), "workload": f"{FRAMES} frames, {STEPS} DDIM steps, CFG {GUIDANCE}, fp16, inputs resident"}
    pipe = bench.build_pipeline(device)
    res["clips"] = [clip_rate(pipe, s, args.clips, device) for s in (784, 768)]
    res["up_steps_784"] = up_steps(pipe.denoising_unet.engine(), 784)
    res["conv_tile_fill"] = [conv_tile_fill(h, w) for h, w in E.latent_levels(98, 98, 4)]
    print(json.dumps(res, indent=1))
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
