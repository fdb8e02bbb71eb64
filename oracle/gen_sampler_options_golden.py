"""Golden clips for the sampler options eta > 0 (stochastic DDIM) and interpolation_factor >= 2 (latent frame
interpolation), made by the reference's OWN Pose2VideoPipeline.__call__ (pipeline_pose2vid_long_edit_bkfill_roiclip.py
:338-578) on the CPU in fp32 with reduced widths, over oracle/diffusers_shim, whose DDIMScheduler is extended here by
the eta branch of diffusers' step (EtaDDIMScheduler: fresh noise from the caller's generator at every step). The
interpolation method is registered with the reference's own src/pipelines/utils.set_tensor_interpolation_method. Cases, 5 frames and 2 DDIM steps each, CFG 3.5, 64 x 64 pixels:

  eta = 1.0, interpolation_factor = 2, slerp
  eta = 0.5, interpolation_factor = 3, linear

The same clips are recomputed with oracle/sampler_options_oracle.sample_clip (fed the same draws) as a check, then the
denoised latents and the decoded videos (fp16, every 4th pixel) go to tests/golden/pipeline_sampler_options.pt.
Usage:  MIMO_REFERENCE=<checkout of the original project> python oracle/gen_sampler_options_golden.py [--write]
"""
from __future__ import annotations

import argparse
import os
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
REF = Path(os.environ.get("MIMO_REFERENCE") or sys.exit(__doc__))
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "oracle" / "diffusers_shim"))
sys.path.insert(0, str(REF))

from oracle import sampler_options_oracle as SO  # noqa: E402
from oracle import torch_oracle as O  # noqa: E402

CASES = [dict(name="eta1_k2_slerp", eta=1.0, k=2, slerp=True), dict(name="eta05_k3_linear", eta=0.5, k=3, slerp=False)]
F, SIZE, STEPS, GUIDANCE, SEED, GEN_SEED = 5, 64, 2, 3.5, 500, 42
WIDTHS, VAE_WIDTHS = (128, 256, 512, 512), (32, 64, 128, 128)


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


def eta_scheduler():
    """The shim's DDIMScheduler with diffusers 0.24 DDIMScheduler.step's eta > 0 branch [3P]: the noise is
    variance_noise or randn_tensor(model_output.shape, generator, dtype=model_output.dtype), drawn at every step."""
    from diffusers import DDIMScheduler
    from diffusers.utils.torch_utils import randn_tensor

    class EtaDDIMScheduler(DDIMScheduler):
        def step(self, model_output, timestep, sample, eta=0.0, use_clipped_model_output=False, generator=None,
                 variance_noise=None, return_dict=True):
            if not eta > 0:
                return super().step(model_output, timestep, sample, eta, use_clipped_model_output, generator,
                                    variance_noise, return_dict)
            assert not use_clipped_model_output
            if variance_noise is not None and generator is not None:
                raise ValueError("Cannot pass both generator and variance_noise.")
            if variance_noise is None:
                variance_noise = randn_tensor(model_output.shape, generator=generator, device=model_output.device,
                                              dtype=model_output.dtype)
            return SimpleNamespace(prev_sample=SO.ddim_step(self._d, model_output, int(timestep), sample, eta,
                                                            variance_noise))

    return EtaDDIMScheduler


def run_case(case):
    from diffusers import AutoencoderKL
    from diffusers.image_processor import VaeImageProcessor
    from src.pipelines import utils as ref_utils
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
    sched = eta_scheduler()(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
                            steps_offset=1, prediction_type="v_prediction", rescale_betas_zero_snr=True,
                            timestep_spacing="trailing")
    pipe = Pose2VideoPipeline(vae=vae, image_encoder=clip, reference_unet=ref, denoising_unet=den, pose_guider=pg,
                              scheduler=sched)
    ref_img, poses, bks = inputs(SEED, SIZE, F)
    ref_utils.set_tensor_interpolation_method(case["slerp"])
    method = ref_utils.get_tensor_interpolation_method()
    steps_seen = []
    with torch.no_grad():
        want = pipe(ref_img, poses, bks, SIZE, SIZE, F, STEPS, GUIDANCE, eta=case["eta"],
                    generator=torch.manual_seed(GEN_SEED), interpolation_factor=case["k"],
                    callback=lambda i, t, lat: steps_seen.append(lat.clone())).videos
    latents = steps_seen[-1]  # the callback sees the latents after the last step

    # the oracle on the same pre-processed tensors and the same draws: latents, then one noise tensor per step
    vp = VaeImageProcessor(vae_scale_factor=8, do_convert_rgb=True)
    cp = VaeImageProcessor(vae_scale_factor=8, do_convert_rgb=True, do_normalize=False)
    with torch.no_grad():
        emb = clip(CLIPImageProcessor().preprocess(ref_img.resize((224, 224)), return_tensors="pt").pixel_values).image_embeds
        gen = torch.manual_seed(GEN_SEED)
        shape = (1, 4, F, SIZE // 8, SIZE // 8)
        lat0 = torch.randn(shape, generator=gen, dtype=emb.dtype)
        noise = [torch.randn(shape, generator=gen, dtype=emb.dtype) for _ in range(STEPS)]
        W = O.Weights(sds["den"], sds["ref"], sds["pg"], sds["vae"], cfg, vae_cfg)
        got = SO.sample_clip(W, vp.preprocess(ref_img, height=SIZE, width=SIZE),
                             torch.stack([cp.preprocess(p, height=SIZE, width=SIZE)[0] for p in poses], dim=1).unsqueeze(0),
                             torch.cat([vp.preprocess(b, height=SIZE, width=SIZE) for b in bks]), emb, lat0, STEPS,
                             GUIDANCE, eta=case["eta"], step_noise=noise, interpolation_factor=case["k"], interpolation=method)
    assert want.shape == (1, 3, (F - 1) * case["k"] + 1, SIZE, SIZE), want.shape
    check(f"{case['name']}: latents", got["latents"], latents, 5e-5)
    check(f"{case['name']}: videos", got["videos"], want, 5e-5)
    return dict(name=case["name"], eta=case["eta"], k=case["k"], slerp=case["slerp"], latents=latents.half(),
                videos=want[:, :, :, ::4, ::4].half())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--write", action="store_true", help="write tests/golden/pipeline_sampler_options.pt")
    args = ap.parse_args()
    torch.set_grad_enabled(False)
    out = [run_case(c) for c in CASES]
    if args.write:
        path = ROOT / "tests" / "golden" / "pipeline_sampler_options.pt"
        torch.save({"seed": SEED, "generator_seed": GEN_SEED, "F": F, "size": SIZE, "steps": STEPS, "guidance": GUIDANCE,
                    "widths": list(WIDTHS), "vae_widths": list(VAE_WIDTHS), "cases": out}, path)
        print("written", path)


if __name__ == "__main__":
    main()
