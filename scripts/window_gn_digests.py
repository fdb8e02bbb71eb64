"""SHA-256 digests of what the engine computes with use_inflated_groupnorm=True (per-frame GroupNorm), on an H100.

Window-mode GroupNorm must leave the per-frame network untouched: this script runs a seeded Pose2VideoPipeline.__call__
(128 x 128, 26 frames = two context windows, 2 DDIM steps, CFG 3.5) and one UNet3D forward of the engine with a default
UNetSpec, and prints the digests of their output bytes. Run from a build of the previous version with --out, it writes
tests/golden/inflated_groupnorm_digests.json, which tests/test_window_groupnorm_gpu.py requires of every later build.

    python scripts/window_gn_digests.py [--tree <checkout>] [--out digests.json]
"""
from __future__ import annotations

import argparse
import hashlib
import json
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]


def _sha(t: torch.Tensor) -> str:
    return hashlib.sha256(t.detach().contiguous().cpu().view(torch.uint8).numpy().tobytes()).hexdigest()


def digests() -> dict:
    import PIL.Image
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection

    from mimo_b200 import engine as E
    from mimo_b200.host import modules as M
    from mimo_b200.host.pipeline import Pose2VideoPipeline
    from mimo_b200.host.scheduler import DDIMScheduler
    from oracle import torch_oracle as O
    dev = torch.device("cuda")
    widths, seed = (128, 256, 512, 512), 930
    cfg, vcfg = O.UNetConfig(block_out_channels=widths), O.VAEConfig()
    mk = dict(num_attention_heads=8, num_transformer_block=1, attention_block_types=["Temporal_Self", "Temporal_Self"],
              temporal_position_encoding=True, temporal_position_encoding_max_len=32, temporal_attention_dim_div=1)
    den = M.UNet3DConditionModel(block_out_channels=widths, cross_attention_dim=768, use_inflated_groupnorm=True,
                                 use_motion_module=True, motion_module_mid_block=True, motion_module_type="Vanilla",
                                 motion_module_kwargs=mk)
    ref = M.UNet2DConditionModel(block_out_channels=widths, cross_attention_dim=768)
    pg = M.PoseGuider(widths[0], 3, (16, 32, 96, 256))
    vae = M.AutoencoderKL()
    sds = dict(den=O.make_denoising_unet_sd(cfg, seed), ref=O.make_reference_unet_sd(cfg, seed + 1),
               pg=O.make_pose_guider_sd(seed + 2, widths[0]), vae=O.make_vae_sd(vcfg, seed + 3))
    for m, k in ((den, "den"), (ref, "ref"), (pg, "pg"), (vae, "vae")):
        m.load_state_dict(sds[k], strict=True)
    torch.manual_seed(seed + 4)
    clip = CLIPVisionModelWithProjection(CLIPVisionConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=2,
                                                          num_attention_heads=4, image_size=224, patch_size=32,
                                                          projection_dim=768)).eval()
    sched = DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
                          steps_offset=1, prediction_type="v_prediction", rescale_betas_zero_snr=True,
                          timestep_spacing="trailing")
    pipe = Pose2VideoPipeline(vae=vae, image_encoder=clip, reference_unet=ref, denoising_unet=den, pose_guider=pg,
                              scheduler=sched).to(dev, dtype=torch.float16)
    F_, size = 26, 128
    rng = np.random.RandomState(seed)
    ref_img = PIL.Image.fromarray(rng.randint(0, 256, (size, size, 3), dtype=np.uint8))
    poses, bks = [], []
    for i in range(F_):
        a = np.zeros((size, size, 3), np.uint8)
        a[size // 4: size // 2 + i % 8, size // 3: size // 3 + 20] = rng.randint(11, 256, 3)
        poses.append(PIL.Image.fromarray(a))
        bks.append(PIL.Image.fromarray(rng.randint(0, 256, (size, size, 3), dtype=np.uint8)))
    out = pipe(ref_img, poses, bks, size, size, F_, 2, 3.5, generator=torch.manual_seed(42))
    res = {"call_latents": _sha(pipe.last_latents), "call_videos": _sha(out.videos)}

    # the engine directly, default UNetSpec: eager, capture, replay
    f, hw = 6, 16
    g = torch.Generator().manual_seed(seed + 10)
    ref_lat = torch.randn(1, 4, hw, hw, generator=g).repeat(2, 1, 1, 1).half().to(dev)
    emb = torch.randn(1, 1, 768, generator=g)
    ehs = torch.cat([torch.zeros_like(emb), emb]).half().to(dev)
    x = torch.randn(1, 8, f, hw, hw, generator=g).repeat(2, 1, 1, 1, 1).half().to(dev)
    pose = (torch.randn(2 * f * hw * hw, widths[0], generator=g) * 0.1).half().to(dev)
    eng = E.UNetEngine(sds["den"], E.UNetSpec(block_out_channels=widths), dev)
    reng = E.UNetEngine(sds["ref"], E.UNetSpec(block_out_channels=widths, in_channels=4, motion=False, out_head=False),
                        dev)
    eng.begin_clip(ehs, reng.write_banks(ref_lat, ehs, eng), cfg=True, frames=f)
    outs = [_sha(eng.forward(x, 499, pose)) for _ in range(3)]
    torch.cuda.synchronize()
    res["engine_forward"] = outs[0] if len(set(outs)) == 1 else "eager/replay differ: " + ",".join(outs)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", default=str(ROOT), help="checkout whose mimo_b200 / oracle to run")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    sys.path.insert(0, str(Path(args.tree).resolve()))
    torch.backends.cuda.matmul.allow_tf32 = False
    res = digests()
    print(json.dumps(res, indent=1))
    if args.out:
        Path(args.out).write_text(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
