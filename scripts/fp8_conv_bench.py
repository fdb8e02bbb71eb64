"""FP8 ResBlock convolutions against fp16 and against the projections-only FP8 path, on the benchmark workload (512 x 512,
24 frames, CFG 3.5, DDIM 20). One call prints one JSON document with:
  * the card's name and power limit;
  * per call, every ResnetBlock3D conv1 / conv2 shape of one UNet forward (48 images of the CFG window at each level),
    fp16 (mimo_conv3x3) against e4m3 (mimo_conv3x3_e4m3, with conv2's residual), and e4m3 at C = 1280 with both tile
    widths (BN 160 and 256);
  * GroupNorm + SiLU against GroupNorm + SiLU -> e4m3 at each (resolution, width);
  * the captured UNet forward and the whole clip with fp16, FP8 projections, and FP8 projections + convs, alternated over
    --rounds rounds (medians and min / max; after each switch, untimed runs re-capture the graphs, so the timed ones
    replay);
  * the device bytes of the e4m3 conv weight copies, and the clip's rel-L2 difference to the fp16 clip.
Usage:  python scripts/fp8_conv_bench.py [--rounds 3] [--json out.json]"""
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
from mimo_b200 import lib as L  # noqa: E402
from mimo_b200 import ops  # noqa: E402
from scripts.any_size_bench import card  # noqa: E402
from scripts.fp8_bench import _time  # noqa: E402

FRAMES, GUIDANCE, SIZE, STEPS = 24, 3.5, 512, 20
PEAK_F16, PEAK_F8 = 989e12, 1979e12  # H100 SXM data sheet, dense


def conv_shapes(eng):
    """(side, cin, cout, residual, count) of every ResBlock conv in one forward at 512 x 512 (64 x 64 latents)"""
    nb = len(eng.spec.block_out_channels)
    shapes = {}
    for p in eng.resnets:
        part, i = p.split(".")[0], int(p.split(".")[1]) if p.startswith(("down", "up")) else 0
        side = {"down_blocks": 64 >> i, "mid_block": 64 >> (nb - 1), "up_blocks": 64 >> (nb - 1 - i)}[part]
        for key, res in (("c1", False), ("c2", True)):
            cout, k = eng.w[p][key][0].shape
            sk = (side, k // 9, cout, res)
            shapes[sk] = shapes.get(sk, 0) + 1
    return [(*k, v) for k, v in sorted(shapes.items())]


def kernel_times(eng, device):
    g = torch.Generator(device=device).manual_seed(0)
    n = 2 * FRAMES
    convs, gns, seen_gn = [], [], set()
    for side, cin, cout, res, count in conv_shapes(eng):
        M = n * side * side
        x = torch.randn(M, cin, device=device, generator=g).half()
        gm = (torch.randn(cin, device=device, generator=g) * 0.2 + 1).half()
        bt = (torch.randn(cin, device=device, generator=g) * 0.2).half()
        q, sx = ops.groupnorm_e4m3(x, gm, bt, n, side * side)
        t = ops.groupnorm(x, gm, bt, n, side * side, silu=True)
        w = (torch.randn(cout, 9 * cin, device=device, generator=g) * 0.02).half()
        b = torch.randn(cout, device=device, generator=g).half()
        w8, sw = ops.pack_e4m3_weight(w)
        r = torch.randn(M, cout, device=device, generator=g).half() if res else None
        iters = max(10, int(4e4 / side / side * 64 / cin))
        f16 = _time(lambda: ops.conv3x3(t, w, n, side, side, bias=b, residual=r), iters)
        f8 = _time(lambda: ops.conv3x3_e4m3(q, sx, w8, sw, n, side, side, torch.float16, bias=b, residual=r), iters)
        flop = 2.0 * M * cout * 9 * cin
        row = {"side": side, "cin": cin, "cout": cout, "residual": res, "per_forward": count,
               "fp16_us": round(1e3 * f16, 2), "e4m3_us": round(1e3 * f8, 2),
               "fp16_TFLOP_s": round(flop / f16 / 1e9, 1), "e4m3_TFLOP_s": round(flop / f8 / 1e9, 1),
               "fp16_of_989": round(flop / f16 / 1e-3 / PEAK_F16, 3), "e4m3_of_1979": round(flop / f8 / 1e-3 / PEAK_F8, 3),
               "speedup": round(f16 / f8, 3)}
        if cout == 1280:  # both e4m3 tile widths that divide 1280
            for bn in (160, 256):
                L.load().mimo_debug_force_bn(bn)
                try:
                    row[f"e4m3_bn{bn}_us"] = round(1e3 * _time(
                        lambda: ops.conv3x3_e4m3(q, sx, w8, sw, n, side, side, torch.float16, bias=b, residual=r), iters), 2)
                finally:
                    L.load().mimo_debug_force_bn(0)
        convs.append(row)
        if (side, cin) not in seen_gn:
            seen_gn.add((side, cin))
            g16 = _time(lambda: ops.groupnorm(x, gm, bt, n, side * side, silu=True), iters)
            g8 = _time(lambda: ops.groupnorm_e4m3(x, gm, bt, n, side * side), iters)
            gns.append({"side": side, "C": cin, "gn_silu_us": round(1e3 * g16, 2), "gn_silu_e4m3_us": round(1e3 * g8, 2),
                        "gn_TB_s": round(4 * M * cin / g16 / 1e9, 3), "gn_e4m3_TB_s": round(3 * M * cin / g8 / 1e9, 3)})
    return convs, gns


def spread(v):
    return {"median": round(statistics.median(v), 4), "min": round(min(v), 4), "max": round(max(v), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3, help="timed rounds; each times fp16, FP8 projections, FP8 + convs")
    ap.add_argument("--json", default=None, help="also write the result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_conv_bench.py: no CUDA device (the engine has no CPU fallback)")
    device = torch.device("cuda", 0)
    res = {"card": card(), "workload": f"{SIZE}x{SIZE} x {FRAMES} frames, CFG {GUIDANCE}, DDIM {STEPS}, fp16 model"}
    pipe = bench.build_pipeline(device)
    den = pipe.denoising_unet
    eng = den.engine()
    res["conv_per_call"], res["groupnorm_per_call"] = kernel_times(eng, device)

    ref_img, poses, bks = bench.synthetic_inputs(FRAMES, SIZE)
    host = pipe.preprocess(ref_img, poses, bks, SIZE, SIZE, FRAMES, torch.Generator().manual_seed(42), torch.float16,
                           STEPS)
    dev_in = {k: v.to(device) for k, v in host.items()}
    modes = {"fp16": den.disable_fp8, "fp8": den.enable_fp8, "fp8_convs": lambda: den.enable_fp8(convs=True)}
    videos = {}
    for name, on in modes.items():  # warm-up: first forward of a shape eager, the second captures
        on()
        for _ in range(2):
            videos[name] = pipe.sample_tensors(dev_in, STEPS, GUIDANCE)["videos"].float()
    g = torch.Generator(device=device).manual_seed(1)
    ehs = torch.randn(2, 1, 768, device=device, generator=g).half()
    lat = torch.randn(2, 4, SIZE // 8, SIZE // 8, device=device, generator=g).half()
    eng.begin_clip(ehs, pipe.reference_unet.engine().write_banks(lat, ehs, eng), cfg=True, frames=FRAMES)
    sample = torch.randn(2, 8, FRAMES, SIZE // 8, SIZE // 8, device=device, generator=g).half()
    fwd = {k: [] for k in modes}
    clip = {k: [] for k in modes}
    for _ in range(args.rounds):
        for name, on in modes.items():
            on()
            fwd[name].append(_time(lambda: eng.forward(sample, 499, None), 5))
    for _ in range(args.rounds):
        for name, on in modes.items():
            on()
            pipe.sample_tensors(dev_in, STEPS, GUIDANCE)  # re-captures after the switch
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = pipe.sample_tensors(dev_in, STEPS, GUIDANCE)
            e1.record()
            torch.cuda.synchronize()
            clip[name].append(e0.elapsed_time(e1) / 1e3)
            assert bool(torch.isfinite(out["videos"]).all()), name
    res["unet_forward_ms"] = {k: spread(v) for k, v in fwd.items()}
    res["clip_s"] = {k: spread(v) for k, v in clip.items()}
    med = lambda d, k: d[k]["median"]
    res["forward_speedup_vs_fp16"] = {k: round(med(res["unet_forward_ms"], "fp16") / med(res["unet_forward_ms"], k), 4)
                                      for k in ("fp8", "fp8_convs")}
    res["clip_speedup_vs_fp16"] = {k: round(med(res["clip_s"], "fp16") / med(res["clip_s"], k), 4)
                                   for k in ("fp8", "fp8_convs")}
    b16 = videos["fp16"]
    res["video_rel_l2_vs_fp16"] = {k: float((videos[k] - b16).norm() / b16.norm()) for k in ("fp8", "fp8_convs")}
    res["e4m3_conv_weight_bytes"] = sum(wq.numel() + ws.numel() * 4 for m in eng.w8c.values() for wq, ws in m.values())
    res["e4m3_weight_bytes_total"] = eng.fp8_bytes()
    den.disable_fp8()
    print(json.dumps(res, indent=1))
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
