"""CPU/fp32 ORACLE of the two sampler options eta > 0 (stochastic DDIM) and interpolation_factor >= 2 (latent frame
interpolation) — TEST INFRASTRUCTURE, NOT PRODUCT CODE. It extends oracle/torch_oracle.py (whose DDIM step and
sample_clip restate the reference's shipped configuration, eta = 0 and interpolation_factor = 1) without changing it:

  ddim_step           diffusers 0.24 DDIMScheduler.step [3P] for v-prediction with eta > 0 (pipeline :128-147, :421,
                      :551-553 with the caller's eta and generator)
  interpolate_latents Pose2VideoPipeline.interpolate_latents (pipeline_pose2vid_long_edit_bkfill_roiclip.py:294-334)
  sample_clip         torch_oracle.sample_clip with both options (pipeline :338-578, :566-567)

Pinned against the reference's own pipeline file by oracle/gen_sampler_options_golden.py.
"""
from __future__ import annotations

import time
from typing import Dict, List, Optional

import torch

from oracle import torch_oracle as O


def ddim_step(sched: O.DDIM, model_output: torch.Tensor, t: int, sample: torch.Tensor, eta: float,
              noise: Optional[torch.Tensor]) -> torch.Tensor:
    """eta > 0: `noise` is the step's randn_tensor(model_output.shape) draw:
    sigma = eta * sqrt((1 - abar_prev) / (1 - abar_t) * (1 - abar_t / abar_prev)),
    x_prev = sqrt(abar_prev) x0 + sqrt(1 - abar_prev - sigma^2) eps + sigma noise.  eta = 0: torch_oracle's DDIM.step."""
    if not eta > 0:
        return sched.step(model_output, t, sample)
    prev_t = t - sched.num_train_timesteps // sched.num_inference_steps
    a_t = sched.alphas_cumprod[t]
    a_p = sched.alphas_cumprod[prev_t] if prev_t >= 0 else sched.final_alpha_cumprod
    b_t = 1 - a_t
    x0 = (a_t ** 0.5) * sample - (b_t ** 0.5) * model_output  # v_prediction
    eps = (a_t ** 0.5) * model_output + (b_t ** 0.5) * sample
    std_dev_t = eta * (((1 - a_p) / b_t) * (1 - a_t / a_p)) ** 0.5  # DDIMScheduler._get_variance
    direction = (1 - a_p - std_dev_t ** 2) ** 0.5 * eps
    return a_p ** 0.5 * x0 + direction + std_dev_t * noise


def interpolate_latents(latents: torch.Tensor, interpolation_factor: int, method) -> torch.Tensor:
    """[b, c, F, h, w] -> [b, c, (F - 1) * k + 1, h, w]: frame i at i * k, method(v_i, v_{i+1}, j / k) at i * k + j."""
    if interpolation_factor < 2:
        return latents
    k = interpolation_factor
    b, c, fr, h, w = latents.shape
    assert fr >= 2, "the reference fails on a 1-frame clip here (v1 is None)"
    new = torch.zeros((b, c, (fr - 1) * k + 1, h, w), dtype=latents.dtype, device=latents.device)
    rate = [i / k for i in range(k)][1:]
    idx = 0
    for i0 in range(fr - 1):
        v0, v1 = latents[:, :, i0], latents[:, :, i0 + 1]
        new[:, :, idx] = v0
        idx += 1
        for t in rate:
            new[:, :, idx] = method(v0, v1, t)
            idx += 1
    new[:, :, idx] = latents[:, :, fr - 1]
    return new


def sample_clip(W: O.Weights, ref_image: torch.Tensor, pose: torch.Tensor, backgrounds: torch.Tensor,
                image_embeds: torch.Tensor, init_latents: torch.Tensor, num_inference_steps: int,
                guidance_scale: float, context_frames: int = 24, context_overlap: int = 4, eta: float = 0.0,
                step_noise: Optional[List[torch.Tensor]] = None, interpolation_factor: int = 1, interpolation=None,
                timing: Optional[dict] = None, decode: bool = True) -> Dict[str, torch.Tensor]:
    """torch_oracle.sample_clip (same inputs) with the two options: eta > 0 takes step i's noise from step_noise[i]
    ([1,4,F,h,w] each); interpolation_factor >= 2 decodes interpolate_latents(latents, k, interpolation) into
    "videos", while "latents" stays the denoised clip."""
    cfg_ = W.unet_cfg
    do_cfg = guidance_scale > 1.0
    dtype = init_latents.dtype
    sched = O.DDIM()
    timesteps = sched.set_timesteps(num_inference_steps)
    ehs = image_embeds.unsqueeze(1)
    if do_cfg:
        ehs = torch.cat([torch.zeros_like(ehs), ehs], dim=0)  # :385-391
    latents = init_latents * sched.init_noise_sigma
    Fr = latents.shape[2]
    tm = timing if timing is not None else {}

    t0 = time.perf_counter()
    ref_latents = O.vae_encode_mean(W.vae, ref_image, W.vae_cfg) * 0.18215  # :424-431
    bk = torch.stack([O.vae_encode_mean(W.vae, backgrounds[i:i + 1], W.vae_cfg)[0] * 0.18215 for i in range(Fr)], dim=1)
    vid_bk = bk.unsqueeze(0).to(dtype)  # [1,4,F,h,w]  :434-443
    tm["vae_encode_s"] = time.perf_counter() - t0
    pose_fea = O.pose_guider(W.pose_guider, pose)  # :446-457
    rl = ref_latents.repeat(2 if do_cfg else 1, 1, 1, 1)
    banks = O.reference_unet_banks(W.reference_unet, rl, ehs, cfg_)  # :480-490
    rep = 2 if do_cfg else 1
    for i, t in enumerate(timesteps):
        t = int(t)
        noise_pred = torch.zeros((latents.shape[0] * rep, *latents.shape[1:]), dtype=dtype, device=latents.device)
        counter = torch.zeros((1, 1, Fr, 1, 1), dtype=dtype, device=latents.device)
        for c in O.uniform_windows(0, Fr, context_frames, 1, context_overlap):  # :492-500
            lat_in = latents[:, :, c].repeat(rep, 1, 1, 1, 1)
            bk_in = vid_bk[:, :, c].repeat(rep, 1, 1, 1, 1)
            x = torch.cat([lat_in, bk_in], dim=1)
            pose_in = pose_fea[:, :, c].repeat(rep, 1, 1, 1, 1)
            pred = O.denoising_unet(W.denoising_unet, x, t, ehs[: x.shape[0]], pose_in, banks, cfg_, cfg=do_cfg)
            noise_pred[:, :, c] = noise_pred[:, :, c] + pred  # :540-542
            counter[:, :, c] = counter[:, :, c] + 1
        if do_cfg:
            u, cnd = (noise_pred / counter).chunk(2)
            noise_pred = u + guidance_scale * (cnd - u)
        noise = step_noise[i] if eta > 0 else None
        latents = ddim_step(sched, noise_pred, t, latents, eta, noise).to(dtype)  # :551-553
    out = {"latents": latents}
    if decode:
        vid_lat = interpolate_latents(latents, interpolation_factor, interpolation)  # :566-567
        z = (1 / 0.18215 * vid_lat)[0].permute(1, 0, 2, 3)  # "(b f) c h w"
        frames = torch.cat([O.vae_decode(W.vae, z[i:i + 1], W.vae_cfg) for i in range(z.shape[0])])  # :113-121
        video = frames.permute(1, 0, 2, 3).unsqueeze(0)
        out["videos"] = (video / 2 + 0.5).clamp(0, 1).float().cpu()
    return out
