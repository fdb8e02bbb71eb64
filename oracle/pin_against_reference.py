"""Pin the functional oracle (oracle/torch_oracle.py) against the reference's OWN code, and write golden fixtures.

Needs a checkout of the original project, named by MIMO_REFERENCE (read-only). It imports its src/** verbatim
on top of oracle/diffusers_shim, loads the same seeded state dicts into the reference's modules (strict=True: this
also pins the state-dict key schema) and checks, in fp32 on CPU:

  1. reference_unet "write" pass + ReferenceAttentionControl.update + denoising_unet "read" pass  == oracle
  2. PoseGuider                                                                                     == oracle
  3. Pose2VideoPipeline.__call__ end to end (config 1 of BASELINE.json: 1 frame 256x256, 2 DDIM steps, and a
     multi-window case F=26 > 24 frames at low resolution)                                          == oracle
  4. context windows and DDIM timestep tables                                                       == oracle (bit-exact)

then stores inputs-by-seed + expected outputs under tests/golden/ for the GPU parity tests (which run without the
original project). Usage:  MIMO_REFERENCE=<checkout> python oracle/pin_against_reference.py [--write]
"""
from __future__ import annotations

import argparse
import os
import json
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
REF = Path(os.environ.get("MIMO_REFERENCE") or sys.exit(__doc__))
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "oracle" / "diffusers_shim"))
sys.path.insert(0, str(REF))

from oracle import torch_oracle as O  # noqa: E402

MOTION_KW = dict(num_attention_heads=8, num_transformer_block=1, attention_block_types=["Temporal_Self", "Temporal_Self"],
                 temporal_position_encoding=True, temporal_position_encoding_max_len=32, temporal_attention_dim_div=1)
UNET_EXTRA = dict(use_inflated_groupnorm=True, unet_use_cross_frame_attention=False, unet_use_temporal_attention=False,
                  use_motion_module=True, motion_module_resolutions=[1, 2, 4, 8], motion_module_mid_block=True,
                  motion_module_decoder_only=False, motion_module_type="Vanilla", motion_module_kwargs=MOTION_KW)


def build_reference_models(cfg: O.UNetConfig):
    from src.models.pose_guider import PoseGuider
    from src.models.unet_2d_condition import UNet2DConditionModel
    from src.models.unet_3d_edit_bkfill import UNet3DConditionModel
    common = dict(sample_size=64, in_channels=4, out_channels=4, block_out_channels=tuple(cfg.block_out_channels),
                  layers_per_block=cfg.layers_per_block, cross_attention_dim=cfg.cross_attention_dim,
                  attention_head_dim=cfg.heads, norm_num_groups=cfg.norm_num_groups, norm_eps=cfg.norm_eps,
                  flip_sin_to_cos=True, freq_shift=0)
    den = UNet3DConditionModel(**common, **UNET_EXTRA)
    ref = UNet2DConditionModel(**common,
                               down_block_types=("CrossAttnDownBlock2D",) * 3 + ("DownBlock2D",),
                               up_block_types=("UpBlock2D",) + ("CrossAttnUpBlock2D",) * 3)
    pg = PoseGuider(cfg.block_out_channels[0], conditioning_channels=3, block_out_channels=O.POSE_CHANNELS)
    return den.eval(), ref.eval(), pg.eval()


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def check(name, got, want, tol):
    e = rel(got, want)
    status = "ok" if e <= tol else "FAIL"
    print(f"[{status}] {name}: rel_l2 = {e:.3e} (tol {tol:.0e})")
    if e > tol:
        raise SystemExit(f"oracle disagrees with the reference on {name}")
    return e


def unet_case(cfg: O.UNetConfig, f: int, hw: int, seed: int):
    """reference_unet(write) -> update -> denoising_unet(read) on one CFG window."""
    from src.models.mutual_self_attention import ReferenceAttentionControl
    den, ref, pg = build_reference_models(cfg)
    sd_den = O.make_denoising_unet_sd(cfg, seed=seed)
    sd_ref = O.make_reference_unet_sd(cfg, seed=seed + 1)
    sd_pg = O.make_pose_guider_sd(seed=seed + 2, out_channels=cfg.block_out_channels[0])
    den.load_state_dict(sd_den, strict=True)
    ref.load_state_dict(sd_ref, strict=True)
    pg.load_state_dict(sd_pg, strict=True)

    g = torch.Generator().manual_seed(seed + 10)
    ref_lat = torch.randn(1, 4, hw, hw, generator=g)
    emb = torch.randn(1, 1, cfg.cross_attention_dim, generator=g)
    ehs = torch.cat([torch.zeros_like(emb), emb])
    x = torch.randn(1, 8, f, hw, hw, generator=g).repeat(2, 1, 1, 1, 1)
    pose_img = torch.rand(1, 3, f, hw * 8, hw * 8, generator=g)
    t = torch.tensor(499)

    with torch.no_grad():
        writer = ReferenceAttentionControl(ref, do_classifier_free_guidance=True, mode="write", batch_size=1,
                                           fusion_blocks="full")
        reader = ReferenceAttentionControl(den, do_classifier_free_guidance=True, mode="read", batch_size=1,
                                           fusion_blocks="full")
        ref(ref_lat.repeat(2, 1, 1, 1), torch.zeros_like(t), encoder_hidden_states=ehs, return_dict=False)
        reader.update(writer)
        pose_ref = pg(pose_img)
        want = den(x, t, encoder_hidden_states=ehs, pose_cond_fea=pose_ref.repeat(2, 1, 1, 1, 1), return_dict=False)[0]
        reader.clear()
        writer.clear()

        banks = O.reference_unet_banks(sd_ref, ref_lat.repeat(2, 1, 1, 1), ehs, cfg)
        pose_or = O.pose_guider(sd_pg, pose_img)
        got = O.denoising_unet(sd_den, x, 499, ehs, pose_or.repeat(2, 1, 1, 1, 1), banks, cfg, cfg=True)
    check(f"pose_guider (F={f}, {hw*8}px)", pose_or, pose_ref, 1e-5)
    check(f"denoising_unet read-mode, widths {cfg.block_out_channels}, f={f}, latent {hw}x{hw}", got, want, 2e-5)
    return dict(seed=seed, f=f, hw=hw, out=got)


def pipeline_case(cfg: O.UNetConfig, vae_cfg: O.VAEConfig, F: int, size: int, steps: int, seed: int):
    """Pose2VideoPipeline.__call__ verbatim vs oracle.sample_clip on the same PIL inputs."""
    import PIL.Image
    from diffusers import AutoencoderKL, DDIMScheduler
    from src.pipelines.pipeline_pose2vid_long_edit_bkfill_roiclip import Pose2VideoPipeline
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection

    den, ref, pg = build_reference_models(cfg)
    sds = dict(den=O.make_denoising_unet_sd(cfg, seed), ref=O.make_reference_unet_sd(cfg, seed + 1),
               pg=O.make_pose_guider_sd(seed + 2, cfg.block_out_channels[0]), vae=O.make_vae_sd(vae_cfg, seed + 3))
    den.load_state_dict(sds["den"], strict=True)
    ref.load_state_dict(sds["ref"], strict=True)
    pg.load_state_dict(sds["pg"], strict=True)
    vae = AutoencoderKL(sds["vae"], vae_cfg)
    torch.manual_seed(seed + 4)
    clip = CLIPVisionModelWithProjection(CLIPVisionConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=2,
                                                          num_attention_heads=4, image_size=224, patch_size=32,
                                                          projection_dim=cfg.cross_attention_dim)).eval()
    sched = DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
                          steps_offset=1, prediction_type="v_prediction", rescale_betas_zero_snr=True,
                          timestep_spacing="trailing")
    pipe = Pose2VideoPipeline(vae=vae, image_encoder=clip, reference_unet=ref, denoising_unet=den, pose_guider=pg,
                              scheduler=sched)
    rng = np.random.RandomState(seed)
    ref_img = PIL.Image.fromarray(rng.randint(0, 256, (size, size, 3), dtype=np.uint8))
    poses, bks = [], []
    for i in range(F):
        a = np.zeros((size, size, 3), np.uint8)
        a[size // 4: size // 2 + i % 8, size // 3: size // 3 + 40] = rng.randint(11, 256, 3)
        poses.append(PIL.Image.fromarray(a))
        bks.append(PIL.Image.fromarray(rng.randint(0, 256, (size, size, 3), dtype=np.uint8)))
    gen = torch.manual_seed(42)
    with torch.no_grad():
        want = pipe(ref_img, poses, bks, size, size, F, steps, 3.5, generator=gen).videos

    # oracle on the same pre-processed tensors
    from diffusers.image_processor import VaeImageProcessor
    from transformers import CLIPImageProcessor
    vp, cp = VaeImageProcessor(vae_scale_factor=8, do_convert_rgb=True), VaeImageProcessor(vae_scale_factor=8, do_convert_rgb=True, do_normalize=False)
    with torch.no_grad():
        clip_in = CLIPImageProcessor().preprocess(ref_img.resize((224, 224)), return_tensors="pt").pixel_values
        emb = clip(clip_in).image_embeds
        gen = torch.manual_seed(42)
        lat0 = torch.randn((1, 4, F, size // 8, size // 8), generator=gen, dtype=emb.dtype)
        W = O.Weights(sds["den"], sds["ref"], sds["pg"], sds["vae"], cfg, vae_cfg)
        got = O.sample_clip(W, vp.preprocess(ref_img, height=size, width=size),
                            torch.stack([cp.preprocess(p, height=size, width=size)[0] for p in poses], dim=1).unsqueeze(0),
                            torch.cat([vp.preprocess(b, height=size, width=size) for b in bks]), emb, lat0, steps, 3.5)
    check(f"Pose2VideoPipeline end-to-end F={F} {size}px steps={steps}", got["videos"], want, 5e-5)
    return got


def integer_tables():
    from src.pipelines.context import uniform
    out = {"windows": {}, "timesteps": {}}
    for F in (1, 24, 25, 48, 64, 150):
        want = list(uniform(0, 20, F, 24, 1, 4))
        got = O.uniform_windows(0, F, 24, 1, 4)
        assert got == want, f"window mismatch F={F}"
        out["windows"][str(F)] = got
    print("[ok] context windows bit-exact for F in {1,24,25,48,64,150}")
    from diffusers import DDIMScheduler
    for N in (2, 20, 25, 30):
        s = DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
                          steps_offset=1, prediction_type="v_prediction", rescale_betas_zero_snr=True,
                          timestep_spacing="trailing")
        s.set_timesteps(N)
        out["timesteps"][str(N)] = [int(v) for v in s.timesteps]
    d = O.DDIM()
    out["alphas_cumprod_probe"] = {str(i): float(d.alphas_cumprod[i]) for i in (0, 49, 499, 949, 999)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--write", action="store_true", help="write tests/golden/*")
    ap.add_argument("--full", action="store_true", help="also pin the full-width UNet (slow, ~6 GB)")
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    torch.manual_seed(0)
    gold = ROOT / "tests" / "golden"
    gold.mkdir(parents=True, exist_ok=True)

    tables = integer_tables()
    small = O.UNetConfig(block_out_channels=(128, 256, 512, 512))
    r1 = unet_case(small, f=4, hw=16, seed=100)
    small_vae = O.VAEConfig(block_out_channels=(32, 64, 128, 128))
    # BASELINE config 1 shape; the VAE at full sd-vae-ft-mse width so that the engine (GroupNorm needs >= 4 channels
    # per group) can consume the fixture in tests/test_parity_gpu.py
    p1 = pipeline_case(small, O.VAEConfig(), F=1, size=256, steps=2, seed=200)
    p2 = pipeline_case(small, small_vae, F=26, size=64, steps=2, seed=300)       # > 24 frames: 2 windows
    if args.full:
        rfull = unet_case(O.UNetConfig(), f=2, hw=16, seed=400)
    if args.write:
        (gold / "integer_tables.json").write_text(json.dumps(tables, indent=1))
        torch.save({"cfg": list(small.block_out_channels), "seed": 100, "f": 4, "hw": 16,
                    "out": r1["out"].half()}, gold / "unet_small_read.pt")
        torch.save({"seed": 200, "F": 1, "size": 256, "steps": 2, "vae_widths": list(O.VAEConfig().block_out_channels),
                    "latents": p1["latents"].half(),
                    "videos_mean": float(p1["videos"].mean()), "videos": p1["videos"][:, :, :, ::8, ::8].half()},
                   gold / "pipeline_cfg1.pt")
        if args.full:
            torch.save({"seed": 400, "f": 2, "hw": 16, "out": rfull["out"].half()}, gold / "unet_full_read.pt")
        print("golden fixtures written to", gold)


if __name__ == "__main__":
    main()
