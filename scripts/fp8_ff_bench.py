"""FP8 feed-forward output projections against the FP8 path without them and against fp16, on the benchmark workload
(512 x 512, 24 frames, CFG 3.5, DDIM 20). One call prints one JSON document with:
  * the card's name and power limit;
  * per call, at the feed-forward shapes of one UNet forward (the 48 images of the CFG window at each level, C = 320 /
    640 / 1280): the e4m3 GEGLU with a 16-bit output (mimo_gemm_e4m3) against the one with the e4m3 block output
    (mimo_gemm_e4m3_geglu_e4m3), and the 16-bit FF-out (mimo_gemm with the residual) against the block-scaled e4m3 one
    (mimo_gemm_e4m3_blockscaled, with both tile widths), each variant alternated over --rounds rounds, with TFLOP/s and
    the bytes each call must move, counted from the shapes;
  * the captured UNet forward and the whole clip with fp16, enable_fp8(convs=True) and enable_fp8(convs=True,
    ff_out=True), alternated over --rounds rounds (medians and min / max; after each switch, untimed runs re-capture the
    graphs, so the timed ones replay);
  * the device bytes of the e4m3 ff.net.2 copies, and the decoded clip's rel-L2 difference to the fp16 clip.
Usage:  python scripts/fp8_ff_bench.py [--rounds 3] [--json out.json]"""
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
# (latent side, C, feed-forward calls per forward: spatial transformers + motion blocks)
FF_SHAPES = [(64, 320, 10), (32, 640, 10), (16, 1280, 10), (8, 1280, 7)]


def spread(v):
    return {"median": round(statistics.median(v), 4), "min": round(min(v), 4), "max": round(max(v), 4)}


def kernel_times(device, rounds):
    g = torch.Generator(device=device).manual_seed(0)
    rows = []
    for side, C, count in FF_SHAPES:
        M, inner = 2 * FRAMES * side * side, 4 * C
        x = torch.randn(M, C, device=device, generator=g).half()
        q, sc = ops.quantize_e4m3_rows(torch.randn(M, C, device=device, generator=g))
        wp, bp = ops.pack_geglu_weight((torch.randn(2 * inner, C, device=device, generator=g) / C ** 0.5).half(),
                                       (torch.randn(2 * inner, device=device, generator=g) * 0.1).half())
        w8, sw = ops.pack_e4m3_weight(wp)
        w2 = (torch.randn(C, inner, device=device, generator=g) / inner ** 0.5).half()
        b2 = (torch.randn(C, device=device, generator=g) * 0.1).half()
        w28, sw2 = ops.pack_e4m3_weight(w2)
        gg = ops.gemm_e4m3(q, sc, w8, sw, torch.float16, bias=bp, act=L.ACT_GEGLU)
        g8, gs = ops.gemm_e4m3_geglu_e4m3(q, sc, w8, sw, torch.float16, bias=bp)
        iters = max(10, int(2e4 * 64 * 64 / (side * side) / C * 320 / 64))

        def blockscaled(bn):
            def run():
                L.load().mimo_debug_force_bn(bn)
                try:
                    ops.gemm_e4m3_blockscaled(g8, gs, w28, sw2, torch.float16, bias=b2, residual=x)
                finally:
                    L.load().mimo_debug_force_bn(0)
            return run

        variants = {
            "geglu_16bit_out": lambda: ops.gemm_e4m3(q, sc, w8, sw, torch.float16, bias=bp, act=L.ACT_GEGLU),
            "geglu_e4m3_out": lambda: ops.gemm_e4m3_geglu_e4m3(q, sc, w8, sw, torch.float16, bias=bp),
            "ff_out_fp16": lambda: ops.gemm(gg, w2, bias=b2, residual=x),
            "ff_out_e4m3": lambda: ops.gemm_e4m3_blockscaled(g8, gs, w28, sw2, torch.float16, bias=b2, residual=x),
            "ff_out_e4m3_bn64": blockscaled(64),
            "ff_out_e4m3_bn128": blockscaled(128),
        }
        t = {k: [] for k in variants}
        for _ in range(rounds):
            for k, fn in variants.items():
                t[k].append(1e3 * _time(fn, iters))
        fl_geglu, fl_ffo = 2.0 * M * 2 * inner * C, 2.0 * M * C * inner
        nblk = inner // 128
        by = {  # bytes each call must move, from the shapes
            "geglu_16bit_out": M * C + 2 * inner * C + 4 * (M + 2 * inner) + 2 * M * inner,
            "geglu_e4m3_out": M * C + 2 * inner * C + 4 * (M + 2 * inner) + M * inner + 4 * M * nblk,
            "ff_out_fp16": 2 * M * inner + 2 * C * inner + 2 * M * C * 2,
            "ff_out_e4m3": M * inner + 4 * M * nblk + C * inner + 4 * C + 2 * M * C * 2,
        }
        by["ff_out_e4m3_bn64"] = by["ff_out_e4m3_bn128"] = by["ff_out_e4m3"]
        row = {"side": side, "C": C, "M": M, "per_forward": count}
        for k in variants:
            med = statistics.median(t[k])
            fl = fl_geglu if k.startswith("geglu") else fl_ffo
            row[k] = {"us": spread(t[k]), "TFLOP_s": round(fl / med / 1e6, 1), "MB": round(by[k] / 1e6, 2),
                      "TB_s": round(by[k] / med / 1e6, 3)}
        row["geglu_speedup"] = round(statistics.median(t["geglu_16bit_out"]) / statistics.median(t["geglu_e4m3_out"]), 3)
        row["ff_out_speedup"] = round(statistics.median(t["ff_out_fp16"]) / statistics.median(t["ff_out_e4m3"]), 3)
        rows.append(row)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3, help="timed rounds; each alternates every variant")
    ap.add_argument("--json", default=None, help="also write the result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_ff_bench.py: no CUDA device (the engine has no CPU fallback)")
    device = torch.device("cuda", 0)
    res = {"card": card(), "workload": f"{SIZE}x{SIZE} x {FRAMES} frames, CFG {GUIDANCE}, DDIM {STEPS}, fp16 model"}
    res["ff_per_call"] = kernel_times(device, args.rounds)
    pipe = bench.build_pipeline(device)
    den = pipe.denoising_unet
    eng = den.engine()

    ref_img, poses, bks = bench.synthetic_inputs(FRAMES, SIZE)
    host = pipe.preprocess(ref_img, poses, bks, SIZE, SIZE, FRAMES, torch.Generator().manual_seed(42), torch.float16,
                           STEPS)
    dev_in = {k: v.to(device) for k, v in host.items()}
    modes = {"fp16": den.disable_fp8, "fp8_convs": lambda: den.enable_fp8(convs=True),
             "fp8_convs_ff_out": lambda: den.enable_fp8(convs=True, ff_out=True)}
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
                                      for k in ("fp8_convs", "fp8_convs_ff_out")}
    res["clip_speedup_vs_fp16"] = {k: round(med(res["clip_s"], "fp16") / med(res["clip_s"], k), 4)
                                   for k in ("fp8_convs", "fp8_convs_ff_out")}
    b16 = videos["fp16"]
    res["video_rel_l2_vs_fp16"] = {k: float((videos[k] - b16).norm() / b16.norm()) for k in ("fp8_convs", "fp8_convs_ff_out")}
    res["e4m3_ff_out_weight_bytes"] = sum(wq.numel() + ws.numel() * 4 for wq, ws in eng.w8f.values())
    res["e4m3_weight_bytes_total"] = eng.fp8_bytes()
    den.disable_fp8()
    print(json.dumps(res, indent=1))
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
