"""Golden clips for the schedulers DPM-Solver++ (multistep), Euler and Euler-ancestral, made by the reference's OWN
Pose2VideoPipeline.__call__ (pipeline_pose2vid_long_edit_bkfill_roiclip.py:338-578) on the CPU in fp32 with reduced
widths, over oracle/diffusers_shim, whose scheduler names are bound here to the restatements of
oracle/schedulers_oracle.py. The reference's file decides where scale_model_input is applied (:519-521), how
init_noise_sigma scales the initial latents (:182) and which schedulers receive the caller's generator (:128-147).
Cases, 5 frames each, CFG 3.5, 64 x 64 pixels, generator seeded for the initial latents (and the ancestral draws):

  DPM-Solver++ 2M, 4 steps   (first-order warm-up, lower_order_final: the last step is first order)
  DPM-Solver++ 3M, 5 steps   (orders 1, 2, 3, 2, 1)
  Euler-ancestral, 3 steps   (one draw per step from the generator)
  Euler, 3 steps

The same clips are recomputed with oracle/schedulers_oracle.sample_clip (fed the same draws) as a check, then the
denoised latents and the decoded videos (fp16, every 4th pixel) go to tests/golden/pipeline_schedulers.pt.
Usage:  MIMO_REFERENCE=<checkout of the original project> python oracle/gen_scheduler_golden.py [--write]
"""
from __future__ import annotations

import argparse
import os
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
REF = Path(os.environ.get("MIMO_REFERENCE") or sys.exit(__doc__))
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "oracle" / "diffusers_shim"))
sys.path.insert(0, str(REF))

from oracle import schedulers_oracle as SC  # noqa: E402
from oracle import torch_oracle as O  # noqa: E402

CASES = [dict(name="dpmpp_2m", scheduler="DPMSolverMultistepScheduler", solver_order=2, steps=4),
         dict(name="dpmpp_3m", scheduler="DPMSolverMultistepScheduler", solver_order=3, steps=5),
         dict(name="euler_a", scheduler="EulerAncestralDiscreteScheduler", steps=3),
         dict(name="euler", scheduler="EulerDiscreteScheduler", steps=3)]
F, SIZE, GUIDANCE, SEED, GEN_SEED = 5, 64, 3.5, 600, 43
WIDTHS, VAE_WIDTHS = (128, 256, 512, 512), (32, 64, 128, 128)


def bind_schedulers():
    """The shim's scheduler names -> the oracle's restatements (the reference's pipeline imports them, :11-18)."""
    import diffusers
    import diffusers.schedulers as S
    for name, cls in (("DPMSolverMultistepScheduler", SC.DPMSolverPP), ("EulerDiscreteScheduler", SC.Euler),
                      ("EulerAncestralDiscreteScheduler", SC.EulerAncestral)):
        setattr(S, name, cls)
        setattr(diffusers, name, cls)


def make_scheduler(case):
    import diffusers.schedulers as S
    cls = getattr(S, case["scheduler"])
    return cls(solver_order=case["solver_order"]) if "solver_order" in case else cls()


def inputs(seed: int, size: int, frames: int):
    """The synthetic PIL clip of pin_against_reference.pipeline_case."""
    import PIL.Image
    rng = np.random.RandomState(seed)
    ref_img = PIL.Image.fromarray(rng.randint(0, 256, (size, size, 3), dtype=np.uint8))
    poses, bks = [], []
    for i in range(frames):
        a = np.zeros((size, size, 3), np.uint8)
        a[size // 4: size // 2 + i % 8, size // 3: size // 3 + 40] = rng.randint(11, 256, 3)
        poses.append(PIL.Image.fromarray(a))
        bks.append(PIL.Image.fromarray(rng.randint(0, 256, (size, size, 3), dtype=np.uint8)))
    return ref_img, poses, bks


def run_case(case):
    from diffusers import AutoencoderKL
    from diffusers.image_processor import VaeImageProcessor
    from src.pipelines.pipeline_pose2vid_long_edit_bkfill_roiclip import Pose2VideoPipeline
    from transformers import CLIPImageProcessor, CLIPVisionConfig, CLIPVisionModelWithProjection

    from oracle.pin_against_reference import build_reference_models, check
    cfg, vae_cfg = O.UNetConfig(block_out_channels=WIDTHS), O.VAEConfig(block_out_channels=VAE_WIDTHS)
    den, ref, pg = build_reference_models(cfg)
    sds = dict(den=O.make_denoising_unet_sd(cfg, SEED), ref=O.make_reference_unet_sd(cfg, SEED + 1),
               pg=O.make_pose_guider_sd(SEED + 2, cfg.block_out_channels[0]), vae=O.make_vae_sd(vae_cfg, SEED + 3))
    den.load_state_dict(sds["den"], strict=True)
    ref.load_state_dict(sds["ref"], strict=True)
    pg.load_state_dict(sds["pg"], strict=True)
    vae = AutoencoderKL(sds["vae"], vae_cfg)
    torch.manual_seed(SEED + 4)
    clip = CLIPVisionModelWithProjection(CLIPVisionConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=2,
                                                          num_attention_heads=4, image_size=224, patch_size=32,
                                                          projection_dim=cfg.cross_attention_dim)).eval()
    pipe = Pose2VideoPipeline(vae=vae, image_encoder=clip, reference_unet=ref, denoising_unet=den, pose_guider=pg,
                              scheduler=make_scheduler(case))
    ref_img, poses, bks = inputs(SEED, SIZE, F)
    steps = case["steps"]
    seen = []
    with torch.no_grad():
        want = pipe(ref_img, poses, bks, SIZE, SIZE, F, steps, GUIDANCE, generator=torch.manual_seed(GEN_SEED),
                    callback=lambda i, t, lat: seen.append(lat.clone())).videos
    latents = seen[-1]  # the callback sees the latents after the last step

    # the oracle on the same pre-processed tensors and the same draws: latents, then (ancestral) one tensor per step
    vp = VaeImageProcessor(vae_scale_factor=8, do_convert_rgb=True)
    cp = VaeImageProcessor(vae_scale_factor=8, do_convert_rgb=True, do_normalize=False)
    with torch.no_grad():
        emb = clip(CLIPImageProcessor().preprocess(ref_img.resize((224, 224)), return_tensors="pt").pixel_values).image_embeds
        gen = torch.manual_seed(GEN_SEED)
        shape = (1, 4, F, SIZE // 8, SIZE // 8)
        lat0 = torch.randn(shape, generator=gen, dtype=emb.dtype)
        noise = ([torch.randn(shape, generator=gen, dtype=emb.dtype) for _ in range(steps)]
                 if case["scheduler"] == "EulerAncestralDiscreteScheduler" else None)
        W = O.Weights(sds["den"], sds["ref"], sds["pg"], sds["vae"], cfg, vae_cfg)
        got = SC.sample_clip(W, vp.preprocess(ref_img, height=SIZE, width=SIZE),
                             torch.stack([cp.preprocess(p, height=SIZE, width=SIZE)[0] for p in poses], dim=1).unsqueeze(0),
                             torch.cat([vp.preprocess(b, height=SIZE, width=SIZE) for b in bks]), emb, lat0, steps,
                             GUIDANCE, make_scheduler(case), step_noise=noise)
    assert want.shape == (1, 3, F, SIZE, SIZE), want.shape
    assert len(seen) == steps
    check(f"{case['name']}: latents", got["latents"], latents, 5e-5)
    check(f"{case['name']}: videos", got["videos"], want, 5e-5)
    return dict(**case, latents=latents.half(), videos=want[:, :, :, ::4, ::4].half())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--write", action="store_true", help="write tests/golden/pipeline_schedulers.pt")
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    bind_schedulers()
    out = [run_case(c) for c in CASES]
    if args.write:
        path = ROOT / "tests" / "golden" / "pipeline_schedulers.pt"
        torch.save({"seed": SEED, "generator_seed": GEN_SEED, "F": F, "size": SIZE, "guidance": GUIDANCE,
                    "widths": list(WIDTHS), "vae_widths": list(VAE_WIDTHS), "cases": out}, path)
        print("written", path)


if __name__ == "__main__":
    main()
