"""CPU/fp32 ORACLE of rescaled classifier-free guidance (guidance_rescale) — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

  rescale_noise_cfg  a restatement of diffusers' rescale_noise_cfg [3P] (Lin et al., "Common Diffusion Noise Schedules
                     and Sample Steps are Flawed", arXiv 2305.08891, §3.4). diffusers is not a dependency here, so this is
                     not pinned against it; tests/test_guidance_rescale_cpu.py checks it against a second plain statement.
  sample_clip        the sampling loop of torch_oracle.sample_clip / schedulers_oracle.sample_clip (pipeline :338-578)
                     with the rescale where diffusers' pipelines apply it: after the guidance line (:545-549, including
                     the division by `counter`) and before scheduler.step (:551-553). scheduler=None is torch_oracle's
                     DDIM. With guidance_rescale = 0 it computes exactly what those two functions compute, which are
                     unchanged (the reference pipeline accepts the keyword and ignores it).
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Dict, List, Optional

import torch

from oracle import torch_oracle as O


def rescale_noise_cfg(noise_cfg: torch.Tensor, noise_pred_text: torch.Tensor, guidance_rescale: float = 0.0):
    """diffusers.pipelines.stable_diffusion.pipeline_stable_diffusion.rescale_noise_cfg [3P]: unbiased std over every
    dim but the batch, in the tensors' dtype."""
    std_text = noise_pred_text.std(dim=list(range(1, noise_pred_text.ndim)), keepdim=True)
    std_cfg = noise_cfg.std(dim=list(range(1, noise_cfg.ndim)), keepdim=True)
    noise_pred_rescaled = noise_cfg * (std_text / std_cfg)
    return guidance_rescale * noise_pred_rescaled + (1 - guidance_rescale) * noise_cfg


class DDIM(O.DDIM):
    """torch_oracle.DDIM with the object surface of schedulers_oracle's classes (integer timesteps, as its loop uses)."""

    def set_timesteps(self, num_inference_steps: int, device=None):
        self.timesteps = [int(t) for t in super().set_timesteps(num_inference_steps)]

    def scale_model_input(self, sample, timestep=None):
        return sample

    def step(self, model_output, timestep, sample, generator=None, noise=None, return_dict=True):
        return SimpleNamespace(prev_sample=super().step(model_output, timestep, sample))


def sample_clip(W: O.Weights, ref_image: torch.Tensor, pose: torch.Tensor, backgrounds: torch.Tensor,
                image_embeds: torch.Tensor, init_latents: torch.Tensor, num_inference_steps: int,
                guidance_scale: float, scheduler=None, step_noise: Optional[List[torch.Tensor]] = None,
                context_frames: int = 24, context_overlap: int = 4, decode: bool = True,
                guidance_rescale: float = 0.0) -> Dict[str, torch.Tensor]:
    """torch_oracle.sample_clip (scheduler None) or schedulers_oracle.sample_clip (same inputs), plus guidance_rescale."""
    cfg_ = W.unet_cfg
    do_cfg = guidance_scale > 1.0
    dtype = init_latents.dtype
    sched = scheduler if scheduler is not None else DDIM()
    sched.set_timesteps(num_inference_steps)
    ehs = image_embeds.unsqueeze(1)
    if do_cfg:
        ehs = torch.cat([torch.zeros_like(ehs), ehs], dim=0)  # :385-391
    latents = init_latents * sched.init_noise_sigma  # :182
    Fr = latents.shape[2]
    ref_latents = O.vae_encode_mean(W.vae, ref_image, W.vae_cfg) * 0.18215  # :424-431
    bk = torch.stack([O.vae_encode_mean(W.vae, backgrounds[i:i + 1], W.vae_cfg)[0] * 0.18215 for i in range(Fr)], dim=1)
    vid_bk = bk.unsqueeze(0).to(dtype)  # [1,4,F,h,w]  :434-443
    pose_fea = O.pose_guider(W.pose_guider, pose)  # :446-457
    rep = 2 if do_cfg else 1
    banks = O.reference_unet_banks(W.reference_unet, ref_latents.repeat(rep, 1, 1, 1), ehs, cfg_)  # :480-490
    for i, t in enumerate(sched.timesteps):
        noise_pred = torch.zeros((latents.shape[0] * rep, *latents.shape[1:]), dtype=dtype, device=latents.device)
        counter = torch.zeros((1, 1, Fr, 1, 1), dtype=dtype, device=latents.device)
        for c in O.uniform_windows(0, Fr, context_frames, 1, context_overlap):  # :492-500
            lat_in = sched.scale_model_input(latents[:, :, c].repeat(rep, 1, 1, 1, 1), t)  # :519-521
            x = torch.cat([lat_in, vid_bk[:, :, c].repeat(rep, 1, 1, 1, 1)], dim=1)
            pose_in = pose_fea[:, :, c].repeat(rep, 1, 1, 1, 1)
            pred = O.denoising_unet(W.denoising_unet, x, t, ehs[: x.shape[0]], pose_in, banks, cfg_, cfg=do_cfg)
            noise_pred[:, :, c] = noise_pred[:, :, c] + pred  # :540-542
            counter[:, :, c] = counter[:, :, c] + 1
        if do_cfg:
            u, cnd = (noise_pred / counter).chunk(2)
            noise_pred = u + guidance_scale * (cnd - u)
            if guidance_rescale > 0.0:  # diffusers: `if do_classifier_free_guidance and guidance_rescale > 0.0`
                noise_pred = rescale_noise_cfg(noise_pred, cnd, guidance_rescale)
        noise = step_noise[i] if step_noise is not None else None
        latents = sched.step(noise_pred, t, latents, noise=noise).prev_sample.to(dtype)  # :551-553
    out = {"latents": latents}
    if decode:
        z = (1 / 0.18215 * latents)[0].permute(1, 0, 2, 3)  # "(b f) c h w"
        frames = torch.cat([O.vae_decode(W.vae, z[i:i + 1], W.vae_cfg) for i in range(Fr)])  # :113-121
        video = frames.permute(1, 0, 2, 3).unsqueeze(0)
        out["videos"] = (video / 2 + 0.5).clamp(0, 1).float().cpu()
    return out
