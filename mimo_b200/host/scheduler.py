"""Schedulers of the sampler loop: DDIM, DPM-Solver++ (multistep), Euler and Euler-ancestral.

The reference builds `diffusers.DDIMScheduler(**noise_scheduler_kwargs)` (run_animate.py:96-97,
configs/inference/inference_v2.yaml:24-33) and its pipeline accepts six diffusers scheduler classes (pipeline :11-18,
:46-53); diffusers is a third-party dependency that is not part of the reference tree. The classes here accept the same
keyword arguments, expose what the pipeline touches (set_timesteps / timesteps / init_noise_sigma / scale_model_input /
order / alphas_cumprod / config / a tensor step()) and, for the engine's sampler, fused_step(): DDIM runs
mimo_cfg_ddim_step(_noise), the other three mimo_cfg_multistep with multistep_coefficients(i). The DDIM integer tables
are pinned by tests/golden/integer_tables.json. engine_scheduler() maps a caller's scheduler (an engine one, or a
diffusers instance read as a config container) to the engine's class.
"""
from __future__ import annotations

import math
from collections.abc import Mapping
from types import SimpleNamespace

import numpy as np
import torch

from .. import ops


def _betas(name: str, num_train_timesteps: int, beta_start: float, beta_end: float, beta_schedule: str,
           rescale_betas_zero_snr: bool) -> torch.Tensor:
    """diffusers' beta schedules [3P] in fp32, with rescale_zero_terminal_snr (abar at the last timestep becomes 0)."""
    if beta_schedule == "scaled_linear":
        betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
    elif beta_schedule == "linear":
        betas = torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
    else:
        raise NotImplementedError(f"{beta_schedule} is not implemented for {name}")
    if rescale_betas_zero_snr:
        abar_sqrt = torch.cumprod(1.0 - betas, dim=0).sqrt()
        a0, aT = abar_sqrt[0].clone(), abar_sqrt[-1].clone()
        abar_sqrt = (abar_sqrt - aT) * (a0 / (a0 - aT))
        abar = abar_sqrt ** 2
        alphas = torch.cat([abar[0:1], abar[1:] / abar[:-1]])
        betas = 1 - alphas
    return betas


def _check_v_prediction(prediction_type: str) -> None:
    if prediction_type != "v_prediction":
        # the fused kernels and step() implement the reference's shipped parameterisation only
        # (configs/inference/inference_v2.yaml:24-33); silently running v-prediction for "epsilon" would be wrong
        raise NotImplementedError(f"prediction_type={prediction_type!r}: only 'v_prediction' (the reference's "
                                  "inference_v2.yaml) is implemented")


class _Scheduler:
    """What the schedulers the engine runs share. The sampler loop (Pose2VideoPipeline._denoise) calls new_history()
    and step_draws() once per clip, then model_input_scale(i) and fused_step() at every step i."""
    order = 1

    @classmethod
    def from_config(cls, config, **overrides):
        items = config.items() if isinstance(config, Mapping) else vars(config).items()
        return cls(**{**{k: v for k, v in items if not k.startswith("_")}, **overrides})

    def scale_model_input(self, sample, timestep=None):
        return sample

    @staticmethod
    def _step_output(prev, x0, return_dict: bool):
        return SimpleNamespace(prev_sample=prev, pred_original_sample=x0) if return_dict else (prev,)

    def model_input_scale(self, i: int):
        return None  # the divisor scale_model_input applies at step i; None: the identity

    def new_history(self, latents: torch.Tensor):
        return None  # what fused_step() carries from one step of a clip to the next


class DDIMScheduler(_Scheduler):
    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", clip_sample: bool = True, set_alpha_to_one: bool = True,
                 steps_offset: int = 0, prediction_type: str = "epsilon", rescale_betas_zero_snr: bool = False,
                 timestep_spacing: str = "leading", **unused):
        betas = _betas("DDIMScheduler", num_train_timesteps, beta_start, beta_end, beta_schedule,
                       rescale_betas_zero_snr)
        if clip_sample:
            raise NotImplementedError("clip_sample=True is not used by the reference and not implemented")
        _check_v_prediction(prediction_type)
        self.betas = betas
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        self.final_alpha_cumprod = torch.tensor(1.0) if set_alpha_to_one else self.alphas_cumprod[0]
        self.init_noise_sigma = 1.0
        self.config = SimpleNamespace(num_train_timesteps=num_train_timesteps, beta_start=beta_start,
                                      beta_end=beta_end, beta_schedule=beta_schedule, clip_sample=clip_sample,
                                      set_alpha_to_one=set_alpha_to_one, steps_offset=steps_offset,
                                      prediction_type=prediction_type, rescale_betas_zero_snr=rescale_betas_zero_snr,
                                      timestep_spacing=timestep_spacing)
        self.num_inference_steps = self.timesteps = None

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

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, eta: float = 0.0,
             use_clipped_model_output: bool = False, generator=None, variance_noise=None, return_dict: bool = True,
             **unused):
        """diffusers DDIMScheduler.step [3P] for v-prediction (pipeline :128-147, :551-553): tensor in, tensor out, in
        the dtype / on the device of `sample`. eta > 0 adds sigma * noise, the noise being `variance_noise` or drawn by
        randn_tensor(model_output.shape, generator, dtype=model_output.dtype) - at every call, also at the last step
        where sigma = 0. The engine's own sampler runs fused_step() (step_coefficients / noise_coefficients);
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
        return self._step_output(prev, x0, return_dict)

    def step_coefficients(self, t: int):
        """(sqrt(abar_t), sqrt(1 - abar_t), sqrt(abar_prev), sqrt(1 - abar_prev)); prev_t = t - T // N (NOT the next
        table entry: for N = 30 they differ)."""
        a_t, a_p = self._alphas(t)
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

    def step_draws(self, eta: float) -> bool:
        return eta > 0  # step() draws randn_tensor(model_output.shape) at every step, also the last one

    def fused_step(self, i, t, pred_uncond, pred_cond, latents, guidance, *, eta, noise, history, counter, frame_stride):
        """CFG + DDIM step at timestep t, on `latents` in place; eta > 0 adds sigma * noise."""
        co = self.step_coefficients(t)
        if eta > 0:
            dir_c, sigma = self.noise_coefficients(t, eta)
            ops.cfg_ddim_step_noise(pred_uncond, pred_cond, latents, guidance, *co[:3], dir_c, noise, sigma,
                                    counter=counter, frame_stride=frame_stride)
        else:
            ops.cfg_ddim_step(pred_uncond, pred_cond, latents, guidance, *co, counter=counter, frame_stride=frame_stride)


# ------------------------------------------------------------------------------------------------
# DPM-Solver++ multistep, Euler and Euler-ancestral
# ------------------------------------------------------------------------------------------------
class _SigmaScheduler(_Scheduler):
    """What the three non-DDIM schedulers share: DDIMScheduler's betas and abar, except that with
    rescale_betas_zero_snr abar at the last timestep is 2^-24 instead of 0 (so sigma_max = sqrt((1 - abar) / abar) is
    about 4096, not infinite), step-index bookkeeping, and the affine form of a step that mimo_cfg_multistep runs:

        m  = a * x + b * v                                    (the solver's model quantity: the x0 prediction)
        x' = c_x * x + c_m * m + c_1 * h_1 + c_2 * h_2 + c_n * noise

    with v the guided v-prediction, h_1 / h_2 the m of the previous two steps and noise this step's draw.
    multistep_coefficients(i) gives (a, b, c_x, c_m, c_1, c_2, c_n) for step i in float64 (from the fp32 abar / sigma
    tables), which the caller casts to fp32 once."""
    draws_noise = False  # whether step() consumes one randn draw of the sample's shape per step

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", prediction_type: str = "epsilon", rescale_betas_zero_snr: bool = False,
                 timestep_spacing: str = "linspace", steps_offset: int = 0, trained_betas=None, **unused):
        name = type(self).__name__
        if trained_betas is not None:
            raise NotImplementedError(f"{name}: trained_betas is outside the reference's configuration")
        if timestep_spacing not in ("linspace", "leading", "trailing"):
            raise ValueError(f"{timestep_spacing} is not supported")
        _check_v_prediction(prediction_type)
        self.betas = _betas(name, num_train_timesteps, beta_start, beta_end, beta_schedule, rescale_betas_zero_snr)
        self.alphas_cumprod = torch.cumprod(1.0 - self.betas, dim=0)
        if rescale_betas_zero_snr:
            self.alphas_cumprod[-1] = 2.0 ** -24  # close to 0 without being 0 (diffusers' later releases)
        self.config = SimpleNamespace(num_train_timesteps=num_train_timesteps, beta_start=beta_start,
                                      beta_end=beta_end, beta_schedule=beta_schedule, prediction_type=prediction_type,
                                      rescale_betas_zero_snr=rescale_betas_zero_snr,
                                      timestep_spacing=timestep_spacing, steps_offset=steps_offset)
        self.num_inference_steps = self.timesteps = self._step_index = None

    @property
    def step_index(self):
        return self._step_index

    def index_for_timestep(self, timestep) -> int:
        """diffusers' _init_step_index: the position of `timestep` in the table (the second match if it repeats)."""
        if self.timesteps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating "
                             "the scheduler")
        t = timestep.item() if torch.is_tensor(timestep) else timestep
        idx = (self.timesteps == t).nonzero()
        if len(idx) == 0:
            raise ValueError(f"timestep {t} is not in this scheduler's table {self.timesteps.tolist()}")
        return int(idx[1 if len(idx) > 1 else 0])

    def _begin_step(self, timestep) -> int:
        if self._step_index is None:
            self._step_index = self.index_for_timestep(timestep)
        return self._step_index

    def _sigma_table(self) -> np.ndarray:
        """sqrt((1 - abar) / abar) over the training timesteps, in fp32 as diffusers computes it."""
        return (((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5).numpy()

    def step_draws(self, eta: float) -> bool:
        return self.draws_noise  # eta reaches DDIM only (prepare_extra_step_kwargs, pipeline :128-147)

    def new_history(self, latents: torch.Tensor) -> torch.Tensor:
        """The m of the last two steps, slot i % 2 written at step i (every rank of a sharded run keeps its own)."""
        return torch.empty((2,) + tuple(latents.shape), dtype=latents.dtype, device=latents.device)

    def fused_step(self, i, t, pred_uncond, pred_cond, latents, guidance, *, eta, noise, history, counter, frame_stride):
        """CFG + step i, on `latents` in place; h_1, h_2 and the noise are passed where their coefficient is not 0."""
        co = self.multistep_coefficients(i)
        ops.cfg_multistep(pred_uncond, pred_cond, latents, guidance, co, history[i % 2],
                          h1=history[(i - 1) % 2] if co[4] != 0 else None, h2=history[i % 2] if co[5] != 0 else None,
                          noise=noise if co[6] != 0 else None, counter=counter, frame_stride=frame_stride)


class DPMSolverMultistepScheduler(_SigmaScheduler):
    """diffusers DPMSolverMultistepScheduler [3P] with algorithm_type="dpmsolver++", solver_type="midpoint", orders
    1-3 and final_sigmas_type="zero", for v-prediction. In VP form: alpha = sqrt(abar), sigma = sqrt(1 - abar),
    lambda = log alpha - log sigma; the model quantity is the data prediction x0 = alpha_s * x - sigma_s * v. Warm-up:
    the first step is first order, the second at most second order; the last step lands on sigma = 0 (abar = 1) and is
    first order, so it returns the last x0 prediction; with lower_order_final and fewer than 15 steps the step before
    it is at most second order."""

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", trained_betas=None, solver_order: int = 2,
                 prediction_type: str = "epsilon", thresholding: bool = False, algorithm_type: str = "dpmsolver++",
                 solver_type: str = "midpoint", lower_order_final: bool = True, euler_at_final: bool = False,
                 use_karras_sigmas: bool = False, use_lu_lambdas: bool = False, final_sigmas_type: str = "zero",
                 lambda_min_clipped: float = -float("inf"), variance_type=None, timestep_spacing: str = "linspace",
                 steps_offset: int = 0, rescale_betas_zero_snr: bool = False, **unused):
        if algorithm_type != "dpmsolver++":
            raise NotImplementedError(f"algorithm_type={algorithm_type!r}: only 'dpmsolver++' is implemented")
        if solver_type != "midpoint":
            raise NotImplementedError(f"solver_type={solver_type!r}: only 'midpoint' is implemented")
        for flag, on in (("use_karras_sigmas", use_karras_sigmas), ("use_lu_lambdas", use_lu_lambdas),
                         ("thresholding", thresholding)):
            if on:
                raise NotImplementedError(f"{flag}=True is not implemented")
        if final_sigmas_type != "zero":
            raise NotImplementedError(f"final_sigmas_type={final_sigmas_type!r}: only 'zero' is implemented")
        if lambda_min_clipped != -float("inf") or variance_type is not None:
            raise NotImplementedError("lambda_min_clipped and variance_type are not implemented")
        if solver_order not in (1, 2, 3):
            raise ValueError(f"solver_order={solver_order}: DPM-Solver++ multistep runs orders 1 to 3")
        super().__init__(num_train_timesteps, beta_start, beta_end, beta_schedule, prediction_type,
                         rescale_betas_zero_snr, timestep_spacing, steps_offset, trained_betas)
        self.config.__dict__.update(solver_order=solver_order, algorithm_type=algorithm_type, solver_type=solver_type,
                                    lower_order_final=lower_order_final, euler_at_final=euler_at_final,
                                    final_sigmas_type=final_sigmas_type)
        self.init_noise_sigma = 1.0
        self.model_outputs = [None] * solver_order

    def set_timesteps(self, num_inference_steps: int, device=None):
        T, n = self.config.num_train_timesteps, num_inference_steps
        if not 0 < n <= T:
            raise ValueError(f"num_inference_steps={n}: must be in 1 .. {T}")
        sp = self.config.timestep_spacing
        if sp == "linspace":
            ts = np.linspace(0, T - 1, n + 1).round()[::-1][:-1].copy().astype(np.int64)
        elif sp == "leading":
            ratio = T // (n + 1)
            ts = (np.arange(0, n + 1) * ratio).round()[::-1][:-1].copy().astype(np.int64) + self.config.steps_offset
        else:  # trailing: DDIM's table
            ts = np.arange(T, 0, -T / n).round().copy().astype(np.int64) - 1
        sig = np.interp(ts, np.arange(0, T), self._sigma_table())
        self.sigmas = torch.from_numpy(np.concatenate([sig, [0.0]]).astype(np.float32))
        self.timesteps = torch.from_numpy(ts).to(device=device, dtype=torch.int64)
        self.num_inference_steps = len(ts)
        self.model_outputs = [None] * self.config.solver_order
        self._step_index = None

    def _vp(self, i: int):
        """(alpha, sigma, lambda) at table position i in float64; i = N is the final sigma = 0 (abar = 1)."""
        abar = 1.0 if i >= len(self.timesteps) else float(self.alphas_cumprod[int(self.timesteps[i])])
        a, s = math.sqrt(abar), math.sqrt(1.0 - abar)
        return a, s, (math.inf if s == 0.0 else math.log(a) - math.log(s))

    def solver_order_at(self, i: int) -> int:
        """The order step i runs (diffusers' step(): warm-up, lower_order_final, lower_order_second)."""
        n, order, cfg = len(self.timesteps), self.config.solver_order, self.config
        final = i == n - 1  # final_sigmas_type = "zero" makes the last step first order
        second = i == n - 2 and cfg.lower_order_final and n < 15
        if order == 1 or i < 1 or final:
            return 1
        if order == 2 or i < 2 or second:
            return 2
        return 3

    def _terms(self, i: int):
        """The scalars of step i: x0 = a * x + b * v, then the update's sigma ratio, alpha_t, exp(-h), h, r0, r1."""
        a0, s0, l0 = self._vp(i)
        at, st, lt = self._vp(i + 1)
        h = lt - l0
        r0 = (l0 - self._vp(i - 1)[2]) / h if i >= 1 and math.isfinite(h) else None
        r1 = (self._vp(i - 1)[2] - self._vp(i - 2)[2]) / h if i >= 2 and math.isfinite(h) else None
        return a0, -s0, st / s0, at, math.exp(-h), h, r0, r1

    def multistep_coefficients(self, i: int):
        """(a, b, c_x, c_m, c_1, c_2, c_n) of step i: the D0 / D1 / D2 combinations of diffusers' first-, second- and
        third-order dpmsolver++ updates expanded over the model outputs m (this step), h_1, h_2 (the two before)."""
        a, b, cx, at, eh, h, r0, r1 = self._terms(i)
        order = self.solver_order_at(i)
        A = at * (eh - 1.0)
        if order == 1:  # x' = cx x - A D0
            w = (-A, 0.0, 0.0)
        elif order == 2:  # x' = cx x - A D0 - A / 2 D1, D1 = (m0 - m1) / r0
            w = (-A - 0.5 * A / r0, 0.5 * A / r0, 0.0)
        else:  # x' = cx x - A D0 + B D1 - C D2
            B = at * ((eh - 1.0) / h + 1.0)
            Cc = at * ((eh - 1.0 + h) / h ** 2 - 0.5)
            d10 = (1.0 / r0, -1.0 / r0, 0.0)
            d11 = (0.0, 1.0 / r1, -1.0 / r1)
            k = r0 / (r0 + r1)
            d1 = tuple(p + k * (p - q) for p, q in zip(d10, d11))
            d2 = tuple((p - q) / (r0 + r1) for p, q in zip(d10, d11))
            w = tuple(-A * (j == 0) + B * p - Cc * q for j, (p, q) in enumerate(zip(d1, d2)))
        return a, b, cx, w[0], w[1], w[2], 0.0

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, generator=None, variance_noise=None,
             return_dict: bool = True, **unused):
        """diffusers DPMSolverMultistepScheduler.step [3P] (dpmsolver++, midpoint, v-prediction): tensor in, tensor
        out in the dtype of `sample`. `generator` is accepted (the reference's pipeline passes it) and not used: the
        ODE solver draws nothing."""
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating "
                             "the scheduler")
        i = self._begin_step(timestep)
        a, b, cx, at, eh, h, r0, r1 = self._terms(i)
        x0 = a * sample + b * model_output
        self.model_outputs = self.model_outputs[1:] + [x0]
        m0, m1, m2 = self.model_outputs[-1], self.model_outputs[-2] if len(self.model_outputs) > 1 else None, \
            self.model_outputs[-3] if len(self.model_outputs) > 2 else None
        order = self.solver_order_at(i)
        A = at * (eh - 1.0)
        if order == 1:
            prev = cx * sample - A * m0
        elif order == 2:
            D1 = (1.0 / r0) * (m0 - m1)
            prev = cx * sample - A * m0 - 0.5 * A * D1
        else:
            D1_0, D1_1 = (1.0 / r0) * (m0 - m1), (1.0 / r1) * (m1 - m2)
            D1 = D1_0 + (r0 / (r0 + r1)) * (D1_0 - D1_1)
            D2 = (1.0 / (r0 + r1)) * (D1_0 - D1_1)
            prev = (cx * sample - A * m0 + (at * ((eh - 1.0) / h + 1.0)) * D1
                    - (at * ((eh - 1.0 + h) / h ** 2 - 0.5)) * D2)
        self._step_index += 1
        return self._step_output(prev, x0, return_dict)


class EulerDiscreteScheduler(_SigmaScheduler):
    """diffusers EulerDiscreteScheduler [3P] for v-prediction, in sigma space: sigma = sqrt((1 - abar) / abar)
    interpolated at the timesteps (which are fp32 and, with linspace spacing, not integers), a final sigma = 0
    appended. scale_model_input is x / sqrt(sigma^2 + 1); x0 = v * (-sigma / sqrt(sigma^2 + 1)) + x / (sigma^2 + 1);
    x' = x + (sigma_next - sigma) * (x - x0) / sigma."""

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", trained_betas=None, prediction_type: str = "epsilon",
                 interpolation_type: str = "linear", use_karras_sigmas: bool = False, timestep_spacing: str = "linspace",
                 timestep_type: str = "discrete", steps_offset: int = 0, rescale_betas_zero_snr: bool = False,
                 **unused):
        if use_karras_sigmas or unused.get("use_exponential_sigmas") or unused.get("use_beta_sigmas"):
            raise NotImplementedError("Karras / exponential / beta sigmas are not implemented")
        if interpolation_type != "linear" or timestep_type != "discrete":
            raise NotImplementedError(f"interpolation_type={interpolation_type!r}, timestep_type={timestep_type!r}: "
                                      "only 'linear' / 'discrete' are implemented")
        if unused.get("sigma_min") is not None or unused.get("sigma_max") is not None:
            raise NotImplementedError("sigma_min / sigma_max are not implemented")
        super().__init__(num_train_timesteps, beta_start, beta_end, beta_schedule, prediction_type,
                         rescale_betas_zero_snr, timestep_spacing, steps_offset, trained_betas)
        self.config.__dict__.update(interpolation_type=interpolation_type, use_karras_sigmas=use_karras_sigmas,
                                    timestep_type=timestep_type)
        sig = self._sigma_table()
        self.sigmas = torch.cat([torch.from_numpy(sig[::-1].copy()).to(torch.float32), torch.zeros(1)])

    @property
    def init_noise_sigma(self):
        """sigma_max for linspace / trailing spacing, sqrt(sigma_max^2 + 1) otherwise (a 0-dim fp32 tensor)."""
        max_sigma = self.sigmas.max()
        if self.config.timestep_spacing in ("linspace", "trailing"):
            return max_sigma
        return (max_sigma ** 2 + 1) ** 0.5

    def set_timesteps(self, num_inference_steps: int, device=None):
        T, n = self.config.num_train_timesteps, num_inference_steps
        if not 0 < n <= T:
            raise ValueError(f"num_inference_steps={n}: must be in 1 .. {T}")
        sp = self.config.timestep_spacing
        if sp == "linspace":
            ts = np.linspace(0, T - 1, n, dtype=np.float32)[::-1].copy()
        elif sp == "leading":
            ratio = T // n
            ts = (np.arange(0, n) * ratio).round()[::-1].copy().astype(np.float32) + self.config.steps_offset
        else:
            ts = np.arange(T, 0, -T / n).round().copy().astype(np.float32) - 1
        sig = np.interp(ts, np.arange(0, T), self._sigma_table())
        self.sigmas = torch.from_numpy(np.concatenate([sig, [0.0]]).astype(np.float32))
        self.timesteps = torch.from_numpy(ts.astype(np.float32)).to(device=device)
        self.num_inference_steps = n
        self._step_index = None

    def model_input_scale(self, i: int):
        """sqrt(sigma_i^2 + 1) as the 0-dim fp32 tensor diffusers divides by: `x / s` is its own expression."""
        sigma = self.sigmas[i]
        return (sigma ** 2 + 1) ** 0.5

    def scale_model_input(self, sample, timestep):
        return sample / self.model_input_scale(self._begin_step(timestep))

    def _target(self, i: int):
        """(sigma at which the deterministic update lands, sigma_up of the added noise)."""
        return float(self.sigmas[i + 1]), 0.0

    def multistep_coefficients(self, i: int):
        """x' = (sd / sigma) x + (1 - sd / sigma) x0 + sigma_up noise, with sd = sigma_next (Euler) or sigma_down."""
        sigma = float(self.sigmas[i])
        sd, up = self._target(i)
        a, b = 1.0 / (sigma * sigma + 1.0), -sigma / math.sqrt(sigma * sigma + 1.0)
        return a, b, sd / sigma, 1.0 - sd / sigma, 0.0, 0.0, up

    def _noise(self, model_output, generator, variance_noise):
        return None

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, s_churn: float = 0.0,
             s_tmin: float = 0.0, s_tmax: float = float("inf"), s_noise: float = 1.0, generator=None,
             variance_noise=None, return_dict: bool = True, **unused):
        """diffusers' step [3P] for v-prediction: tensor in, tensor out in the dtype of `sample`."""
        if s_churn > 0:
            raise NotImplementedError("s_churn > 0 is not implemented")
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating "
                             "the scheduler")
        i = self._begin_step(timestep)
        sigma = float(self.sigmas[i])
        sd, up = self._target(i)
        x0 = model_output * (-sigma / math.sqrt(sigma * sigma + 1.0)) + sample / (sigma * sigma + 1.0)
        prev = sample + ((sample - x0) / sigma) * (sd - sigma)
        noise = self._noise(model_output, generator, variance_noise)
        if noise is not None:
            prev = prev + noise * up
        self._step_index += 1
        return self._step_output(prev, x0, return_dict)


class EulerAncestralDiscreteScheduler(EulerDiscreteScheduler):
    """diffusers EulerAncestralDiscreteScheduler [3P] for v-prediction: the Euler update lands on sigma_down and
    sigma_up * noise is added, sigma_up = sqrt(sigma_next^2 (sigma^2 - sigma_next^2) / sigma^2),
    sigma_down = sqrt(sigma_next^2 - sigma_up^2). One randn_tensor(model_output.shape, generator) draw per step, also
    at the last one (sigma_up = 0 there)."""
    draws_noise = True

    def _target(self, i: int):
        s, sn = float(self.sigmas[i]), float(self.sigmas[i + 1])
        up = math.sqrt(sn * sn * (s * s - sn * sn) / (s * s))
        return math.sqrt(max(sn * sn - up * up, 0.0)), up

    def _noise(self, model_output, generator, variance_noise):
        if variance_noise is not None and generator is not None:
            raise ValueError("Cannot pass both generator and variance_noise.")
        if variance_noise is not None:
            return variance_noise
        from .pipeline import _randn_tensor
        return _randn_tensor(model_output.shape, generator, model_output.device, model_output.dtype)


class _NotRun:
    def __init__(self, *args, **kwargs):
        raise NotImplementedError(f"{type(self).__name__} is not run by the engine; the schedulers it runs are "
                                  f"{', '.join(sorted(_RUN))}")

    @classmethod
    def from_config(cls, config, **overrides):
        return cls()


class LMSDiscreteScheduler(_NotRun):
    pass


class PNDMScheduler(_NotRun):
    pass


_RUN = {c.__name__: c for c in (DDIMScheduler, DPMSolverMultistepScheduler, EulerDiscreteScheduler,
                                EulerAncestralDiscreteScheduler)}
_ALL = {**_RUN, "LMSDiscreteScheduler": LMSDiscreteScheduler, "PNDMScheduler": PNDMScheduler}


def engine_scheduler(obj):
    """The engine's scheduler for the caller's `obj`: an engine scheduler is returned as it is; anything else is read as
    a config container, as a diffusers scheduler is: the engine class of the same name is built from `obj.config`
    (its `_`-prefixed keys dropped). LMS, PNDM and unknown classes are refused."""
    if isinstance(obj, _Scheduler):
        return obj
    name = type(obj).__name__
    cls = _ALL.get(name)
    if cls is None:
        raise NotImplementedError(f"scheduler {name}: the schedulers the engine runs are {', '.join(sorted(_RUN))}")
    config = getattr(obj, "config", None)
    if config is None:
        raise TypeError(f"scheduler {name} has no config to build the engine's {name} from")
    return cls.from_config(config)
