"""Cost of the schedulers: DDIM against DPM-Solver++ 2M and Euler-ancestral, and of the fused step kernels.

Prints, in one run on one GPU:
  * the card's name and power limit;
  * for a 512 x 512 x 24-frame clip, CFG 3.5, fp16, inputs resident on the device (pipeline.sample_tensors, as
    bench.py's value): seconds per clip, per step and clips/s of four variants - DDIM 20 steps, DPM-Solver++ 2M 20 and
    10 steps, Euler-ancestral 20 steps - timed in alternation, round after round, so that clock drift falls on all
    variants alike; the median over the rounds is reported;
  * the CUDA-event time of one mimo_cfg_multistep call (third-order form: both history tensors, plus noise) and of one
    mimo_cfg_ddim_step call on that clip's latents, with the bytes each moves, the bandwidth that makes, its share of
    the 3.35 TB/s data-sheet bound, and the kernel's share of one DDIM step.
Usage: python scripts/scheduler_bench.py [--rounds K] [--json FILE]
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

FRAMES, GUIDANCE, SIZE = 24, 3.5, 512
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
VARIANTS = {"DDIM 20": (S.DDIMScheduler, {}, 20),
            "DPM-Solver++ 2M 20": (S.DPMSolverMultistepScheduler, dict(solver_order=2), 20),
            "DPM-Solver++ 2M 10": (S.DPMSolverMultistepScheduler, dict(solver_order=2), 10),
            "Euler-ancestral 20": (S.EulerAncestralDiscreteScheduler, {}, 20)}


def kernel_times(device, iters: int = 200):
    """(ms per call, bytes per call) of mimo_cfg_multistep (h1, h2, noise) and mimo_cfg_ddim_step on [1, 4, 24, 64, 64]."""
    shape = (1, 4, FRAMES, SIZE // 8, SIZE // 8)
    g = torch.Generator(device=device).manual_seed(0)
    pred = torch.randn((2,) + shape[1:], device=device, generator=g).half()
    pu, pc = pred[0].contiguous(), pred[1].contiguous()
    lat = torch.randn(shape, device=device, generator=g).half()
    noise = torch.randn(shape, device=device, generator=g).half()
    ring = torch.randn((2,) + shape, device=device, generator=g).half()
    dpm = S.DPMSolverMultistepScheduler(solver_order=3, **bench.SCHED_KW)
    dpm.set_timesteps(20)
    co = dpm.multistep_coefficients(7)[:6] + (0.1,)
    ddim = S.DDIMScheduler(**bench.SCHED_KW)
    ddim.set_timesteps(20)
    dco = ddim.step_coefficients(int(ddim.timesteps[7]))
    n, esz = lat.numel(), lat.element_size()
    calls = {"cfg_multistep": (lambda: ops.cfg_multistep(pu, pc, lat, GUIDANCE, co, ring[0], h1=ring[1], h2=ring[0],
                                                         noise=noise), 8 * n * esz),
             "cfg_ddim": (lambda: ops.cfg_ddim_step(pu, pc, lat, GUIDANCE, *dco), 4 * n * esz)}
    out = {}
    for name, (fn, nbytes) in calls.items():
        for _ in range(10):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out[name] = (e0.elapsed_time(e1) / iters, nbytes)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3, help="timed rounds (each times every variant once)")
    ap.add_argument("--json", default=None, help="also write the result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scheduler_bench.py: no CUDA device (the engine has no CPU fallback)")
    device = torch.device("cuda", 0)
    res = {"card": card(), "workload": f"{SIZE}x{SIZE} x {FRAMES} frames, CFG {GUIDANCE}, fp16, inputs resident"}
    pipe = bench.build_pipeline(device)
    ref_img, poses, bks = bench.synthetic_inputs(FRAMES, SIZE)
    inputs = {}
    for name, (cls, kw, steps) in VARIANTS.items():
        # each scheduler's initial latents (init_noise_sigma) and, for Euler-ancestral, its per-step draws
        pipe.scheduler = cls(**bench.SCHED_KW, **kw)
        host = pipe.preprocess(ref_img, poses, bks, SIZE, SIZE, FRAMES, torch.Generator().manual_seed(42),
                               torch.float16, steps)
        inputs[name] = (pipe.scheduler, {k: v.to(device) for k, v in host.items()}, steps)

    def run(name):
        sched, dev_in, steps = inputs[name]
        pipe.scheduler = sched
        return pipe.sample_tensors(dev_in, steps, GUIDANCE)

    for name in VARIANTS:  # warm-up: the first forward of a shape runs eager, the second captures its graph
        run(name)
        run(name)
    torch.cuda.synchronize()
    times = {name: [] for name in VARIANTS}
    for _ in range(args.rounds):
        for name in VARIANTS:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = run(name)
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / 1e3)
            assert bool(torch.isfinite(out["videos"]).all()), name
    base = statistics.median(times["DDIM 20"])
    res["variants"] = []
    for name, (_, _, steps) in VARIANTS.items():
        s = statistics.median(times[name])
        res["variants"].append({"variant": name, "steps": steps, "clip_s": round(s, 4),
                                "clip_s_all": [round(t, 4) for t in times[name]],
                                "step_s": round(s / steps, 5), "clips_per_s": round(1.0 / s, 4),
                                "clip_rate_vs_ddim20": round(base / s, 4)})
    step_ms = 1e3 * base / 20
    res["kernels"] = []
    for name, (ms, nbytes) in kernel_times(device).items():
        bw = nbytes / (ms * 1e-3)
        res["kernels"].append({"kernel": name, "us_per_call": round(1e3 * ms, 2), "bytes_per_call": nbytes,
                               "TB_per_s": round(bw / 1e12, 3), "of_3.35TB_s": round(bw / HBM_BYTES_PER_S, 3),
                               "share_of_ddim_step": round(ms / step_ms, 6)})
    print(json.dumps(res, indent=1))
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
