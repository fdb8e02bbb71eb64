"""CPU/fp32 ORACLE of the schedulers DPM-Solver++ (multistep), Euler and Euler-ancestral — TEST INFRASTRUCTURE, NOT
PRODUCT CODE. A restatement of diffusers' DPMSolverMultistepScheduler (algorithm_type="dpmsolver++",
solver_type="midpoint", final_sigmas_type="zero", lower_order_final), EulerDiscreteScheduler and
EulerAncestralDiscreteScheduler [3P] for the reference's configuration (configs/inference/inference_v2.yaml:24-33:
scaled_linear 0.00085 -> 0.012, rescale_betas_zero_snr, trailing spacing, v-prediction), built on the abar table of
oracle/torch_oracle.DDIM (unchanged) with abar[-1] = 2^-24 as diffusers' later releases set it.

The scalar arithmetic is diffusers': fp32 sigma tables (sigma = sqrt((1 - abar) / abar), np.interp at the timesteps,
a final 0), fp32 0-dim tensors for alpha / sigma / lambda / h, tensor ops in the sample's dtype. The classes have the
object surface the reference's pipeline touches (set_timesteps / timesteps / init_noise_sigma / scale_model_input /
order / step(..., generator)); step() also takes this step's draw as `noise` so that a second run can be fed the same
draws.

  sample_clip   torch_oracle.sample_clip over one of these schedulers (pipeline :338-578: init_noise_sigma at :182,
                scale_model_input on the latent half at :519-521, the scheduler's step at :551-553)

Pinned against the reference's own pipeline file by oracle/gen_scheduler_golden.py.
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Dict, List, Optional

import numpy as np
import torch

from oracle import torch_oracle as O

T_TRAIN = 1000


def alphas_cumprod() -> torch.Tensor:
    a = O.DDIM().alphas_cumprod.clone()
    a[-1] = 2.0 ** -24
    return a


class _Sigmas:
    order = 1

    def __init__(self):
        self.alphas_cumprod = alphas_cumprod()
        table = ((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5
        self.sigmas = torch.cat([table.flip(0), torch.zeros(1)])
        self.timesteps = None
        self.step_index = None
        self.config = SimpleNamespace(num_train_timesteps=T_TRAIN, timestep_spacing="trailing")

    def _table(self, ts: np.ndarray, dtype) -> None:
        sig = np.interp(ts, np.arange(0, T_TRAIN), (((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5).numpy())
        self.sigmas = torch.from_numpy(np.concatenate([sig, [0.0]]).astype(np.float32))
        self.timesteps = torch.from_numpy(ts.astype(dtype))
        self.num_inference_steps = len(ts)
        self.step_index = None

    def _index(self, timestep) -> int:
        if self.step_index is None:
            idx = (self.timesteps == timestep).nonzero()
            self.step_index = int(idx[1 if len(idx) > 1 else 0])
        return self.step_index


class DPMSolverPP(_Sigmas):
    def __init__(self, solver_order: int = 2, lower_order_final: bool = True):
        super().__init__()
        self.solver_order, self.lower_order_final = solver_order, lower_order_final
        self.init_noise_sigma = 1.0

    def set_timesteps(self, num_inference_steps: int, device=None):
        ts = np.arange(T_TRAIN, 0, -T_TRAIN / num_inference_steps).round().copy().astype(np.int64) - 1
        self._table(ts, np.int64)
        self.model_outputs = [None] * self.solver_order
        self.lower_order_nums = 0

    def scale_model_input(self, sample, timestep=None):
        return sample

    @staticmethod
    def _alpha_sigma(sigma):
        alpha_t = 1 / ((sigma ** 2 + 1) ** 0.5)
        return alpha_t, sigma * alpha_t

    def _lam(self, i):
        a, s = self._alpha_sigma(self.sigmas[i])
        return a, s, torch.log(a) - torch.log(s)

    def step(self, model_output, timestep, sample, generator=None, noise=None, return_dict=True):
        i = self._index(timestep)
        n = len(self.timesteps)
        lower_final = i == n - 1  # final_sigmas_type = "zero"
        lower_second = i == n - 2 and self.lower_order_final and n < 15
        alpha_s0, sigma_s0, lam_s0 = self._lam(i)
        x0 = alpha_s0 * sample - sigma_s0 * model_output  # convert_model_output, v_prediction
        self.model_outputs = self.model_outputs[1:] + [x0]
        alpha_t, sigma_t, lam_t = self._lam(i + 1)
        h = lam_t - lam_s0
        m0 = x0
        if self.solver_order == 1 or self.lower_order_nums < 1 or lower_final:
            prev = (sigma_t / sigma_s0) * sample - (alpha_t * (torch.exp(-h) - 1.0)) * m0
        elif self.solver_order == 2 or self.lower_order_nums < 2 or lower_second:
            m1 = self.model_outputs[-2]
            r0 = (lam_s0 - self._lam(i - 1)[2]) / h
            D0, D1 = m0, (1.0 / r0) * (m0 - m1)
            prev = ((sigma_t / sigma_s0) * sample - (alpha_t * (torch.exp(-h) - 1.0)) * D0
                    - 0.5 * (alpha_t * (torch.exp(-h) - 1.0)) * D1)
        else:
            m1, m2 = self.model_outputs[-2], self.model_outputs[-3]
            lam_s1, lam_s2 = self._lam(i - 1)[2], self._lam(i - 2)[2]
            r0, r1 = (lam_s0 - lam_s1) / h, (lam_s1 - lam_s2) / h
            D1_0, D1_1 = (1.0 / r0) * (m0 - m1), (1.0 / r1) * (m1 - m2)
            D1 = D1_0 + (r0 / (r0 + r1)) * (D1_0 - D1_1)
            D2 = (1.0 / (r0 + r1)) * (D1_0 - D1_1)
            prev = ((sigma_t / sigma_s0) * sample - (alpha_t * (torch.exp(-h) - 1.0)) * m0
                    + (alpha_t * ((torch.exp(-h) - 1.0) / h + 1.0)) * D1
                    - (alpha_t * ((torch.exp(-h) - 1.0 + h) / h ** 2 - 0.5)) * D2)
        if self.lower_order_nums < self.solver_order:
            self.lower_order_nums += 1
        self.step_index += 1
        return SimpleNamespace(prev_sample=prev) if return_dict else (prev,)


class Euler(_Sigmas):
    ancestral = False

    @property
    def init_noise_sigma(self):
        return self.sigmas.max()  # trailing spacing

    def set_timesteps(self, num_inference_steps: int, device=None):
        ts = np.arange(T_TRAIN, 0, -T_TRAIN / num_inference_steps).round().copy().astype(np.float32) - 1
        self._table(ts, np.float32)

    def scale_model_input(self, sample, timestep):
        sigma = self.sigmas[self._index(timestep)]
        return sample / ((sigma ** 2 + 1) ** 0.5)

    def step(self, model_output, timestep, sample, generator=None, noise=None, return_dict=True):
        i = self._index(timestep)
        sigma, sigma_to = self.sigmas[i], self.sigmas[i + 1]
        sample = sample.to(torch.float32)
        x0 = model_output * (-sigma / (sigma ** 2 + 1) ** 0.5) + (sample / (sigma ** 2 + 1))
        derivative = (sample - x0) / sigma
        if self.ancestral:
            sigma_up = (sigma_to ** 2 * (sigma ** 2 - sigma_to ** 2) / sigma ** 2) ** 0.5
            sigma_down = (sigma_to ** 2 - sigma_up ** 2) ** 0.5
            prev = sample + derivative * (sigma_down - sigma)
            if noise is None:
                noise = torch.randn(model_output.shape, generator=generator, dtype=model_output.dtype)
            prev = prev + noise.to(prev.device) * sigma_up
        else:
            if noise is None:  # diffusers draws (for s_churn) even when nothing reads it
                torch.randn(model_output.shape, generator=generator, dtype=model_output.dtype)
            prev = sample + derivative * (sigma_to - sigma)
        prev = prev.to(model_output.dtype)
        self.step_index += 1
        return SimpleNamespace(prev_sample=prev) if return_dict else (prev,)


class EulerAncestral(Euler):
    ancestral = True


def sample_clip(W: O.Weights, ref_image: torch.Tensor, pose: torch.Tensor, backgrounds: torch.Tensor,
                image_embeds: torch.Tensor, init_latents: torch.Tensor, num_inference_steps: int,
                guidance_scale: float, scheduler, step_noise: Optional[List[torch.Tensor]] = None,
                context_frames: int = 24, context_overlap: int = 4, decode: bool = True) -> Dict[str, torch.Tensor]:
    """torch_oracle.sample_clip (same inputs) over `scheduler` (one of the classes above): init_latents are scaled by
    its init_noise_sigma, the latent half of every UNet input by scale_model_input, and step i of Euler-ancestral
    adds step_noise[i]."""
    cfg_ = W.unet_cfg
    do_cfg = guidance_scale > 1.0
    dtype = init_latents.dtype
    sched = scheduler
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
    rl = ref_latents.repeat(2 if do_cfg else 1, 1, 1, 1)
    banks = O.reference_unet_banks(W.reference_unet, rl, ehs, cfg_)  # :480-490
    rep = 2 if do_cfg else 1
    for i, t in enumerate(sched.timesteps):
        noise_pred = torch.zeros((latents.shape[0] * rep, *latents.shape[1:]), dtype=dtype, device=latents.device)
        counter = torch.zeros((1, 1, Fr, 1, 1), dtype=dtype, device=latents.device)
        for c in O.uniform_windows(0, Fr, context_frames, 1, context_overlap):  # :492-500
            lat_in = sched.scale_model_input(latents[:, :, c].repeat(rep, 1, 1, 1, 1), t)  # :519-521
            bk_in = vid_bk[:, :, c].repeat(rep, 1, 1, 1, 1)
            x = torch.cat([lat_in, bk_in], dim=1)
            pose_in = pose_fea[:, :, c].repeat(rep, 1, 1, 1, 1)
            pred = O.denoising_unet(W.denoising_unet, x, t, ehs[: x.shape[0]], pose_in, banks, cfg_, cfg=do_cfg)
            noise_pred[:, :, c] = noise_pred[:, :, c] + pred  # :540-542
            counter[:, :, c] = counter[:, :, c] + 1
        if do_cfg:
            u, cnd = (noise_pred / counter).chunk(2)
            noise_pred = u + guidance_scale * (cnd - u)
        noise = step_noise[i] if step_noise is not None else None
        latents = sched.step(noise_pred, t, latents, noise=noise).prev_sample.to(dtype)  # :551-553
    out = {"latents": latents}
    if decode:
        z = (1 / 0.18215 * latents)[0].permute(1, 0, 2, 3)  # "(b f) c h w"
        frames = torch.cat([O.vae_decode(W.vae, z[i:i + 1], W.vae_cfg) for i in range(z.shape[0])])  # :113-121
        video = frames.permute(1, 0, 2, 3).unsqueeze(0)
        out["videos"] = (video / 2 + 0.5).clamp(0, 1).float().cpu()
    return out
