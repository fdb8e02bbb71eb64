"""DDIM timestep / coefficient tables for the sampler loop.

The reference builds `diffusers.DDIMScheduler(**noise_scheduler_kwargs)` (run_animate.py:96-97,
configs/inference/inference_v2.yaml:24-33); diffusers is a third-party dependency that is not part of the
reference tree. This class accepts the same keyword arguments and exposes the attributes the pipeline touches
(set_timesteps / timesteps / init_noise_sigma / scale_model_input / order / alphas_cumprod), and — instead of
`step()` on tensors — the four scalars the fused CFG+DDIM kernel needs. The integer tables are pinned by
tests/golden/integer_tables.json.
"""
from __future__ import annotations

from types import SimpleNamespace

import numpy as np
import torch


class DDIMScheduler:
    order = 1

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", clip_sample: bool = True, set_alpha_to_one: bool = True,
                 steps_offset: int = 0, prediction_type: str = "epsilon", rescale_betas_zero_snr: bool = False,
                 timestep_spacing: str = "leading", **unused):
        if beta_schedule == "scaled_linear":
            betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
        elif beta_schedule == "linear":
            betas = torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
        else:
            raise NotImplementedError(f"{beta_schedule} is not implemented for DDIMScheduler")
        if rescale_betas_zero_snr:
            abar_sqrt = torch.cumprod(1.0 - betas, dim=0).sqrt()
            a0, aT = abar_sqrt[0].clone(), abar_sqrt[-1].clone()
            abar_sqrt = (abar_sqrt - aT) * (a0 / (a0 - aT))
            abar = abar_sqrt ** 2
            alphas = torch.cat([abar[0:1], abar[1:] / abar[:-1]])
            betas = 1 - alphas
        if clip_sample:
            raise NotImplementedError("clip_sample=True is not used by the reference and not implemented")
        if prediction_type != "v_prediction":
            # the fused CFG+DDIM kernel and step() implement the reference's shipped parameterisation only
            # (configs/inference/inference_v2.yaml:24-33); silently running v-prediction for "epsilon" would be wrong
            raise NotImplementedError(f"prediction_type={prediction_type!r}: only 'v_prediction' (the reference's "
                                      "inference_v2.yaml) is implemented")
        self.betas = betas
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        self.final_alpha_cumprod = torch.tensor(1.0) if set_alpha_to_one else self.alphas_cumprod[0]
        self.init_noise_sigma = 1.0
        self.config = SimpleNamespace(num_train_timesteps=num_train_timesteps, steps_offset=steps_offset,
                                      prediction_type=prediction_type, timestep_spacing=timestep_spacing)
        self.num_inference_steps = None
        self.timesteps = None

    def set_timesteps(self, num_inference_steps: int, device=None):
        T = self.config.num_train_timesteps
        if num_inference_steps > T:
            raise ValueError("num_inference_steps cannot exceed num_train_timesteps")
        self.num_inference_steps = num_inference_steps
        sp = self.config.timestep_spacing
        if sp == "trailing":
            ts = np.round(np.arange(T, 0, -T / num_inference_steps)).astype(np.int64) - 1
        elif sp == "leading":
            ratio = T // num_inference_steps
            ts = (np.arange(0, num_inference_steps) * ratio).round()[::-1].copy().astype(np.int64) + self.config.steps_offset
        else:
            raise ValueError(f"{sp} is not supported")
        self.timesteps = torch.from_numpy(ts).to(device)

    def scale_model_input(self, sample, timestep=None):
        return sample

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, eta: float = 0.0,
             use_clipped_model_output: bool = False, generator=None, variance_noise=None, return_dict: bool = True,
             **unused):
        """diffusers DDIMScheduler.step [3P] for v-prediction (pipeline :128-147, :551-553): tensor in, tensor out, in
        the dtype / on the device of `sample`. eta > 0 adds sigma * noise, the noise being `variance_noise` or drawn by
        randn_tensor(model_output.shape, generator, dtype=model_output.dtype) - at every call, also at the last step
        where sigma = 0. The engine's own sampler uses the fused kernels (step_coefficients / noise_coefficients);
        this method exists so that the reference's unmodified pipeline file runs over this scheduler."""
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating "
                             "the scheduler")
        if use_clipped_model_output:
            raise NotImplementedError("use_clipped_model_output is outside the reference's shipped configuration")
        if eta == 0.0 and variance_noise is not None:
            raise NotImplementedError("variance_noise at eta = 0 is outside the reference's shipped configuration")
        t = int(timestep)
        a_t, a_p = self._alphas(t)
        b_t = 1 - a_t
        x0 = (a_t ** 0.5) * sample - (b_t ** 0.5) * model_output
        eps = (a_t ** 0.5) * model_output + (b_t ** 0.5) * sample
        if eta > 0:
            if variance_noise is not None and generator is not None:
                raise ValueError("Cannot pass both generator and variance_noise. Please make sure that either "
                                 "`generator` or `variance_noise` stays `None`.")
            std_dev_t = eta * self._variance(a_t, a_p) ** 0.5
            direction = self._direction(a_p, std_dev_t) * eps
            prev = a_p ** 0.5 * x0 + direction
            if variance_noise is None:
                from .pipeline import _randn_tensor
                variance_noise = _randn_tensor(model_output.shape, generator, model_output.device, model_output.dtype)
            prev = prev + std_dev_t * variance_noise
        else:
            direction = (1 - a_p) ** 0.5 * eps  # std_dev_t = 0 at eta = 0
            prev = a_p ** 0.5 * x0 + direction
        if not return_dict:
            return (prev,)
        return SimpleNamespace(prev_sample=prev, pred_original_sample=x0)

    def step_coefficients(self, t: int):
        """(sqrt(abar_t), sqrt(1 - abar_t), sqrt(abar_prev), sqrt(1 - abar_prev)); prev_t = t - T // N (NOT the next
        table entry: for N = 30 they differ)."""
        prev_t = t - self.config.num_train_timesteps // self.num_inference_steps
        a_t = self.alphas_cumprod[t]
        a_p = self.alphas_cumprod[prev_t] if prev_t >= 0 else self.final_alpha_cumprod
        return float(a_t ** 0.5), float((1 - a_t) ** 0.5), float(a_p ** 0.5), float((1 - a_p) ** 0.5)

    def _alphas(self, t: int):
        prev_t = t - self.config.num_train_timesteps // self.num_inference_steps
        a_p = self.alphas_cumprod[prev_t] if prev_t >= 0 else self.final_alpha_cumprod
        return self.alphas_cumprod[t], a_p

    @staticmethod
    def _variance(a_t, a_p):
        """DDIMScheduler._get_variance [3P]: (1 - abar_prev) / (1 - abar_t) * (1 - abar_t / abar_prev), fp32."""
        return ((1 - a_p) / (1 - a_t)) * (1 - a_t / a_p)

    @staticmethod
    def _direction(a_p, std_dev_t):
        """sqrt(1 - abar_prev - sigma^2) in fp32, the radicand clamped at 0. At eta = 1 on a zero-terminal-SNR schedule
        (rescale_betas_zero_snr, abar = 0 at t = 999) the first step's radicand is exactly 0 in real arithmetic, and
        fp32 rounding can make it -1 ulp (at 20 and 25 steps): diffusers then returns NaN latents for the whole clip;
        here the square root is of 0, the exact value. Everywhere else the result is diffusers' to the bit."""
        return (1 - a_p - std_dev_t ** 2).clamp(min=0) ** 0.5

    def noise_coefficients(self, t: int, eta: float):
        """(sqrt(1 - abar_prev - sigma^2), sigma) with sigma = eta * sqrt(variance): the direction coefficient and the
        noise scale of a stochastic DDIM step (eta > 0), in the fp32 tensor arithmetic of DDIMScheduler.step [3P]."""
        a_t, a_p = self._alphas(t)
        std_dev_t = eta * self._variance(a_t, a_p) ** 0.5
        return float(self._direction(a_p, std_dev_t)), float(std_dev_t)
