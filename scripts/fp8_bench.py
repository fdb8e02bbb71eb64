"""FP8 (e4m3) against fp16 for the denoising UNet's LN-fed projections, on the benchmark workload (512 x 512, 24 frames,
CFG 3.5, DDIM 20). One call prints one JSON document with:
  * the card's name and power limit;
  * per call, every LN-fed GEMM shape of one UNet forward (q|k|v N = 3C and GEGLU N = 8C, M = 2 x 24 x h x w tokens),
    fp16 (mimo_gemm) against e4m3 (mimo_gemm_e4m3), with TFLOP/s against the data sheet's 989 (fp16) / 1 979 (fp8);
  * LayerNorm against LayerNorm -> e4m3 at each width, with bytes/s;
  * the captured UNet forward and the whole clip, fp16 and FP8 alternated over --rounds rounds (medians; after each
    switch, untimed runs re-capture the graphs, so the timed ones replay);
  * the device bytes of the e4m3 weight copies.
Usage:  python scripts/fp8_bench.py [--rounds 5] [--json out.json]"""
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

FRAMES, GUIDANCE, SIZE, STEPS = 24, 3.5, 512, 20
PEAK_F16, PEAK_F8 = 989e12, 1979e12  # H100 SXM data sheet, dense
# (tokens h x w, C) of the levels that hold LN-fed projections at 512 x 512: spatial transformers at 64 / 32 / 16 and the
# mid block (8 x 8); motion modules at every level
LEVELS = [(64 * 64, 320), (32 * 32, 640), (16 * 16, 1280), (8 * 8, 1280)]


def _time(fn, iters):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters  # ms


def kernel_times(device):
    g = torch.Generator(device=device).manual_seed(0)
    gemms, lns = [], []
    for hw, C in LEVELS:
        M = 2 * FRAMES * hw
        x = torch.randn(M, C, device=device, generator=g).half()
        gm, bt = torch.randn(C, device=device, generator=g).half(), torch.randn(C, device=device, generator=g).half()
        q, sa = ops.layernorm_e4m3(x, gm, bt)
        nh = ops.layernorm(x, gm, bt)
        iters = max(20, int(2e5 / hw))
        t16 = _time(lambda: ops.layernorm(x, gm, bt), iters)
        t8 = _time(lambda: ops.layernorm_e4m3(x, gm, bt), iters)
        lns.append({"M": M, "C": C, "ln_us": round(1e3 * t16, 2), "ln_TB_s": round(4 * M * C / t16 / 1e9, 3),
                    "ln_e4m3_us": round(1e3 * t8, 2), "ln_e4m3_TB_s": round((3 * M * C + 4 * M) / t8 / 1e9, 3)})
        for name, N, act in (("qkv", 3 * C, L.ACT_NONE), ("geglu", 8 * C, L.ACT_GEGLU)):
            w = (torch.randn(N, C, device=device, generator=g) * 0.05).half()
            b = torch.randn(N, device=device, generator=g).half() if act == L.ACT_GEGLU else None
            w8, sw = ops.pack_e4m3_weight(w)
            f16 = _time(lambda: ops.gemm(nh, w, bias=b, act=act), iters)
            f8 = _time(lambda: ops.gemm_e4m3(q, sa, w8, sw, torch.float16, bias=b, act=act), iters)
            flop = 2.0 * M * N * C
            gemms.append({"gemm": name, "M": M, "N": N, "K": C, "fp16_us": round(1e3 * f16, 2),
                          "e4m3_us": round(1e3 * f8, 2), "fp16_TFLOP_s": round(flop / f16 / 1e9, 1),
                          "e4m3_TFLOP_s": round(flop / f8 / 1e9, 1), "fp16_of_989": round(flop / f16 / 1e-3 / PEAK_F16, 3),
                          "e4m3_of_1979": round(flop / f8 / 1e-3 / PEAK_F8, 3), "speedup": round(f16 / f8, 3)})
    return gemms, lns


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5, help="timed rounds; each times fp16 then FP8")
    ap.add_argument("--json", default=None, help="also write the result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_bench.py: no CUDA device (the engine has no CPU fallback)")
    device = torch.device("cuda", 0)
    res = {"card": card(), "workload": f"{SIZE}x{SIZE} x {FRAMES} frames, CFG {GUIDANCE}, DDIM {STEPS}, fp16 model"}
    gemms, lns = kernel_times(device)
    res["gemm_per_call"], res["layernorm_per_call"] = gemms, lns

    pipe = bench.build_pipeline(device)
    ref_img, poses, bks = bench.synthetic_inputs(FRAMES, SIZE)
    host = pipe.preprocess(ref_img, poses, bks, SIZE, SIZE, FRAMES, torch.Generator().manual_seed(42), torch.float16,
                           STEPS)
    dev_in = {k: v.to(device) for k, v in host.items()}
    den = pipe.denoising_unet
    modes = {"fp16": den.disable_fp8, "fp8": den.enable_fp8}
    videos = {}
    for name, on in modes.items():  # warm-up: first forward of a shape eager, the second captures
        on()
        for _ in range(2):
            videos[name] = pipe.sample_tensors(dev_in, STEPS, GUIDANCE)["videos"].float()
    # the forward alone: one CFG window with reference banks, as inside the clip
    eng = den.engine()
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
            # switching drops the captured graphs: one untimed clip re-captures them, so the timed clip only replays
            pipe.sample_tensors(dev_in, STEPS, GUIDANCE)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = pipe.sample_tensors(dev_in, STEPS, GUIDANCE)
            e1.record()
            torch.cuda.synchronize()
            clip[name].append(e0.elapsed_time(e1) / 1e3)
            assert bool(torch.isfinite(out["videos"]).all()), name
    res["unet_forward_ms"] = {k: round(statistics.median(v), 2) for k, v in fwd.items()}
    res["unet_forward_ms_all"] = {k: [round(t, 2) for t in v] for k, v in fwd.items()}
    res["clip_s"] = {k: round(statistics.median(v), 4) for k, v in clip.items()}
    res["clip_s_all"] = {k: [round(t, 4) for t in v] for k, v in clip.items()}
    res["forward_speedup"] = round(res["unet_forward_ms"]["fp16"] / res["unet_forward_ms"]["fp8"], 4)
    res["clip_speedup"] = round(res["clip_s"]["fp16"] / res["clip_s"]["fp8"], 4)
    a, b = videos["fp8"], videos["fp16"]
    res["video_rel_l2_fp8_vs_fp16"] = float((a - b).norm() / b.norm())
    res["e4m3_weight_bytes"] = eng.fp8_bytes()
    den.disable_fp8()
    print(json.dumps(res, indent=1))
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
