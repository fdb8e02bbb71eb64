"""Spatial-attention kernel rates at the calls the engine issues for the benchmark clip (bench.py: 512 x 512, 24 frames,
CFG, so n = 48 frame-samples, of which the 24 unconditional ones skip the reference bank) and for CLIP's vision tower.

Prints one JSON object: the card's name and power limit, then per call shape and dtype the CUDA-event time per launch
(median of 5 windows of >= 20 launches and >= 20 ms each, after warm-up), the algorithmic TFLOP/s
(4 C lq (n lq + n_bank lb), the count ops.attn_spatial reports) and the fraction of the MUFU bound: one ex2 per score at
16 per clock per SM, over every SM at the card's maximum SM clock.
  python scripts/attn_bench.py [--json FILE]
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

from any_size_bench import card  # noqa: E402
from mimo_b200 import ops  # noqa: E402

N, HEADS = 48, 8
# (lq = lb, d): the four latent levels of the denoising UNet at 512 x 512 (64 x 64 down to 8 x 8 tokens)
UNET = [(4096, 40), (1024, 80), (256, 160), (64, 160)]
CLIP = (1, 257, 16, 64)  # n, tokens, heads, d (clip_engine.py)


def time_ms(fn, windows: int = 5) -> float:
    """Median time per launch over `windows` event-timed windows of >= 20 launches and >= 20 ms each."""
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    iters, res = 20, []
    while len(res) < windows:
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        if ms < 20.0:  # a short window measures launch jitter: lengthen it and start over
            iters = int(iters * 25.0 / max(ms, 1e-3)) + 1
            res = []
            continue
        res.append(ms / iters)
    return statistics.median(res)


def call(n, lq, heads, d, lb, dtype, sm_clock_hz, device) -> dict:
    g = torch.Generator().manual_seed(0)
    C = heads * d
    qkv = torch.randn(n * lq, 3 * C, generator=g).to(dtype).to(device)
    out = torch.empty(n * lq, C, dtype=dtype, device=device)
    kw, n_bank = {}, 0
    if lb:
        bkv = torch.randn(2, lb, 2 * C, generator=g).to(dtype).to(device)
        bidx = [-1] * (n // 2) + [1] * (n - n // 2)
        n_bank = sum(i >= 0 for i in bidx)
        kw = dict(bank_k=bkv[:, :, :C], bank_v=bkv[:, :, C:], bank_index=torch.tensor(bidx, dtype=torch.int32,
                                                                                        device=device))
    fn = lambda: ops.attn_spatial(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], n, lq, heads, out=out, **kw)
    ms = time_ms(fn)
    scores = heads * lq * (n * lq + n_bank * lb)
    mufu_ms = scores / (16 * torch.cuda.get_device_properties(device).multi_processor_count * sm_clock_hz) * 1e3
    return {"n": n, "lq": lq, "lb": lb, "heads": heads, "d": d, "dtype": str(dtype).split(".")[-1],
            "ms": round(ms, 4), "tflops": round(4.0 * C * lq * (n * lq + n_bank * lb) / ms / 1e9, 1),
            "frac_mufu_bound": round(mufu_ms / ms, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None, help="also write the result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attn_bench.py: no CUDA device (the engine has no CPU fallback)")
    device = torch.device("cuda", 0)
    res = {"card": card()}
    try:
        mhz = float(res["card"]["sm_clock_max"].split()[0])
    except (ValueError, IndexError):
        mhz = 1980.0  # H100 SXM maximum SM clock
    res["mufu_bound_clock_mhz"] = mhz
    res["calls"] = []
    for dtype in (torch.float16, torch.bfloat16):
        for lq, d in UNET:
            res["calls"].append(call(N, lq, HEADS, d, lq, dtype, mhz * 1e6, device))
        n, tok, heads, d = CLIP
        res["calls"].append(call(n, tok, heads, d, 0, dtype, mhz * 1e6, device))
    print(json.dumps(res, indent=1))
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
