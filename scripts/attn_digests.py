"""Bit-exact fingerprints of mimo_attn_spatial (csrc/attn_spatial.cu): the SHA-256 of the output bytes for a fixed list of
cases, so that a rework of the kernel's schedule can be checked to compute exactly what it computed before.

Inputs come from a seeded CPU torch.Generator and are then moved to the device, so they do not depend on the GPU's RNG.
The cases cover the attention calls of the benchmark clip (n reduced, with its mix of unconditional rows that skip the
bank and conditional rows that read it), CLIP's call, every head-dim instantiation (DP = d rounded up to 16) once in fp16
and bf16, and the edges of the per-tile pipeline: one key tile, two key tiles, one self tile with several bank tiles,
every row without bank, ragged self and bank tails, and a single query row.

  python scripts/attn_digests.py [--out tests/golden/attn_spatial_digests.json]
tests/test_attn_spatial_exact_gpu.py recomputes every case and requires the stored digest.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

GOLDEN = ROOT / "tests" / "golden" / "attn_spatial_digests.json"
DTYPES = {"f16": torch.float16, "bf16": torch.bfloat16}


def _case(name, n, lq, heads, d, lb=0, nb=0, bidx=None, sharp=False):
    return {"name": name, "n": n, "lq": lq, "heads": heads, "d": d, "lb": lb, "nb": nb, "bidx": bidx, "sharp": sharp}


def cases() -> list:
    out = []
    for dn in DTYPES:
        # the benchmark clip's calls (n = 48 there: 24 unconditional rows without bank, 24 reading bank 1)
        for lq, d in ((4096, 40), (1024, 80), (256, 160), (64, 160)):
            out.append(_case(f"bench_lq{lq}_d{d}_{dn}", 4, lq, 8, d, lb=lq, nb=2, bidx=[-1, -1, 1, 1]))
        out.append(_case(f"clip_257_h16_d64_{dn}", 1, 257, 16, 64))
        # one case per instantiation; sharp logits (std ~ 12) make the running max move between tiles
        for dp in range(16, 193, 16):
            d = dp - 8 if dp % 32 == 0 else dp
            out.append(_case(f"dp{dp}_d{d}_{dn}", 2, 200, 2, d, lb=150, nb=2, bidx=[1, -1], sharp=True))
        # pipeline edges, on a lookahead instantiation (d = 40), the largest two-warpgroup one (d = 144) and the
        # one-warpgroup path (d = 160)
        for d in (40, 144, 160):
            out += [
                _case(f"one_tile_d{d}_{dn}", 2, 100, 2, d, sharp=True),
                _case(f"two_tiles_d{d}_{dn}", 2, 256, 2, d, sharp=True),
                _case(f"self1_bank4_d{d}_{dn}", 2, 100, 2, d, lb=500, nb=2, bidx=[0, 1], sharp=True),
                _case(f"all_rows_no_bank_d{d}_{dn}", 3, 300, 2, d, lb=200, nb=2, bidx=[-1, -1, -1], sharp=True),
                _case(f"ragged_tails_d{d}_{dn}", 3, 300, 2, d, lb=200, nb=2, bidx=[1, 0, -1], sharp=True),
                _case(f"lq1_d{d}_{dn}", 2, 1, 2, d, lb=100, nb=2, bidx=[1, 0], sharp=True),
            ]
    for i, c in enumerate(out):
        c["seed"] = 1000 + i
    return out


def inputs(c: dict):
    """(qkv [n lq, 3C], bank [nb, lb, 2C] or None) on the CPU in fp32."""
    g = torch.Generator().manual_seed(c["seed"])
    C = c["heads"] * c["d"]
    s, mu = (3.0, 3.0) if c["sharp"] else (1.0, 0.0)
    qkv = torch.randn(c["n"] * c["lq"], 3 * C, generator=g)
    qkv[:, :C] = qkv[:, :C] * s + mu
    qkv[:, C:2 * C] *= s
    bkv = None
    if c["lb"]:
        bkv = torch.randn(c["nb"], c["lb"], 2 * C, generator=g)
        bkv[..., :C] *= s
    return qkv, bkv


def run(ops, c: dict, device) -> str:
    dtype = DTYPES[c["name"].rsplit("_", 1)[1]]
    qkv, bkv = inputs(c)
    qkv = qkv.to(dtype).to(device)
    C = c["heads"] * c["d"]
    bank = {}
    if bkv is not None:
        bkv = bkv.to(dtype).to(device)
        bank = dict(bank_k=bkv[:, :, :C], bank_v=bkv[:, :, C:],
                    bank_index=torch.tensor(c["bidx"], dtype=torch.int32, device=device))
    out = ops.attn_spatial(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], c["n"], c["lq"], c["heads"], **bank)
    torch.cuda.synchronize()
    return hashlib.sha256(out.contiguous().view(torch.int16).cpu().numpy().tobytes()).hexdigest()


def digests(device) -> dict:
    from mimo_b200 import ops
    return {c["name"]: run(ops, c, device) for c in cases()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=str(GOLDEN))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attn_digests.py: no CUDA device (the engine has no CPU fallback)")
    res = {"card": torch.cuda.get_device_name(0), "digests": digests(torch.device("cuda", 0))}
    Path(args.out).parent.mkdir(parents=True, exist_ok=True)
    Path(args.out).write_text(json.dumps(res, indent=1) + "\n")
    print(f"{len(res['digests'])} digests -> {args.out}")


if __name__ == "__main__":
    main()
