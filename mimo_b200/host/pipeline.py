"""Pose2VideoPipeline with the reference's call surface (src/pipelines/pipeline_pose2vid_long_edit_bkfill_roiclip.py:
36-80 constructor, :338-363 __call__ signature, :573-578 output), driving the sm_90a engine.

What stays as in the reference: PIL pre-processing semantics, CLIP through the HF module the caller passes, the CPU
generator noise (prepare_latents :149-183), context windows (:492-510), CFG (:545-549) and scheduler (:551-553) maths.
What changes is where the arithmetic runs: reference_unet / pose_guider / denoising_unet / VAE are engine objects
behind the C ABI; each step's CFG + scheduler update is one fused kernel that the scheduler runs itself
(host/scheduler.py: fused_step), latent frame interpolation another; the frames are decoded in batched VAE passes (one
pass up to DECODE_PIXELS_PER_PASS output pixels).

__call__ = preprocess() [host: PIL -> pinned tensors]  ->  H2D  ->  sample_tensors() [device]  ->  D2H, and
sample_tensors() = _check_sampling -> CLIP -> _encode_vae -> _pose_features -> _shard_plan + _reference_pass
-> _denoise -> [interpolation] -> _decode, each phase timed by CUDA events (timings).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Sequence, Union

import numpy as np
import PIL.Image
import torch
import torch.distributed as dist

from .. import engine as E
from .. import ops
from ..lib import MimoError
from .context import get_context_scheduler
from .modules import ReferenceAttentionControl
from .scheduler import engine_scheduler
from .shard import Exchange, ShardPlan, gather_layout


@dataclass
class Pose2VideoPipelineOutput:
    videos: Union[torch.Tensor, np.ndarray]


def pil_to_uint8(images, height: int, width: int, scale_factor: int = 8) -> torch.Tensor:
    """First half of diffusers VaeImageProcessor(do_convert_rgb=True).preprocess [3P] (pipeline :73-80, :424-426,
    :436, :448-450): RGB -> LANCZOS resize to (w, h) floored to multiples of 8, kept as uint8 [N, H, W, 3]."""
    imgs = images if isinstance(images, (list, tuple)) else [images]
    w, h = width - width % scale_factor, height - height % scale_factor
    return torch.from_numpy(np.stack([np.asarray(i.convert("RGB").resize((w, h), resample=PIL.Image.LANCZOS), dtype=np.uint8)
                                      for i in imgs]))


def uint8_to_tensor(u8: torch.Tensor, normalize: bool) -> torch.Tensor:
    """Second half, on whatever device `u8` lives on: [N, H, W, 3] uint8 -> fp32 NCHW in [0, 1], then 2x - 1 if
    `normalize`. The same IEEE fp32 division / multiply / subtract as the host version: results are bit-identical,
    the clip's images just cross PCIe as bytes and the 38 M-element conversion runs on the GPU instead of one core."""
    t = u8.permute(0, 3, 1, 2).to(torch.float32) / 255.0
    return 2.0 * t - 1.0 if normalize else t


def pil_to_tensor(images, height: int, width: int, normalize: bool, scale_factor: int = 8) -> torch.Tensor:
    """The full VaeImageProcessor.preprocess on the host (used by the tests and the oracle)."""
    return uint8_to_tensor(pil_to_uint8(images, height, width, scale_factor), normalize).contiguous()


def _dedupe_images(images) -> "tuple[list, torch.Tensor]":
    """Indices of the first occurrence of every distinct image (by size, mode and pixel bytes) and, per image, the
    index of its representative among those: animate mode passes one identical white background per frame
    (run_animate.py:174-177) and the VAE should see it once. CRC-32 only buckets the candidates; a hit is confirmed byte
    for byte, so two different frames can never share latents."""
    import zlib
    first, inverse, buckets, raws = [], [], {}, []
    for i, im in enumerate(images):
        raw = im.tobytes()
        key = (im.size, im.mode, len(raw), zlib.crc32(raw))
        j = next((k for k in buckets.get(key, ()) if raws[k] == raw), None)
        if j is None:
            j = len(first)
            buckets.setdefault(key, []).append(j)
            first.append(i)
            raws.append(raw)
        inverse.append(j)
    return first, torch.tensor(inverse, dtype=torch.long)


def shard_tokens(h: int, w: int, levels: int, motion_levels: Optional[Sequence[int]] = None) -> int:
    """Tokens per frame that every UNet level with a motion module splits evenly: the gcd of h_l * w_l over those levels
    (engine.latent_levels; `motion_levels` indexes them finest first, None = every level). A frame group of G GPUs cuts
    each motion module's tokens into G pixel shards, so G must divide it. For latents that are multiples of
    2^(levels - 1) and modules down to the coarsest level this is that level's count; at 98 x 98 (784 x 784 pixels) it
    is 1. Without any motion module nothing is split: 0, which every G divides."""
    import math
    lv = E.latent_levels(h, w, levels)
    idx = range(levels) if motion_levels is None else motion_levels
    return math.gcd(*(lv[i][0] * lv[i][1] for i in idx))


_POOL = None


def _pool():
    """Host threads for the pre-processing: PIL's resize / convert and torch's CPU random draw release the GIL."""
    global _POOL
    import os
    if _POOL is None or _POOL[0] != os.getpid():  # a forked child inherits the object but not its threads
        from concurrent.futures import ThreadPoolExecutor
        n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
        _POOL = (os.getpid(), ThreadPoolExecutor(max_workers=max(2, min(8, n)), thread_name_prefix="mimo-pre"))
    return _POOL[1]


def _sample_key(im, raw: bytes):
    """Bucket key of an image for the dedupe: geometry + CRC-32 of every 1021st byte (a prime stride visits every
    channel and column phase). Only a bucket: equality is always confirmed on the full bytes."""
    import zlib
    return (im.size, im.mode, len(raw), zlib.crc32(raw[::1021]))


def stage_frames_u8(images, height: int, width: int, pinned: bool, scale_factor: int = 8, raws=None) -> torch.Tensor:
    """pil_to_uint8() written straight into one (pinned) staging tensor [N, h, w, 3]: the same pixel values — PIL's
    `convert("RGB")` and `resize` return plain copies when the mode / size already match (Image.py: `return self.copy()`),
    so those two copies, the per-image ndarray and the np.stack + pin_memory copies of the simple version are skipped,
    and frames that do need the LANCZOS resize run on the host thread pool (PIL releases the GIL inside it).
    `raws[i]`, when given, is `images[i].tobytes()` (the dedupe already made it)."""
    imgs = images if isinstance(images, (list, tuple)) else [images]
    w, h = width - width % scale_factor, height - height % scale_factor
    out = torch.empty((len(imgs), h, w, 3), dtype=torch.uint8, pin_memory=pinned)
    dst = out.numpy().reshape(len(imgs), -1)

    def one(i):
        im = imgs[i]
        if im.mode == "RGB" and im.size == (w, h):
            raw = raws[i] if raws is not None else im.tobytes()
        else:
            raw = im.convert("RGB").resize((w, h), resample=PIL.Image.LANCZOS).tobytes()
        dst[i] = np.frombuffer(raw, dtype=np.uint8)

    heavy = [i for i, im in enumerate(imgs) if im.size != (w, h)]
    if len(heavy) > 1:
        list(_pool().map(one, range(len(imgs))))
    else:
        for i in range(len(imgs)):
            one(i)
    return out


def _dedupe_raws(images) -> "tuple[list, torch.Tensor, list]":
    """_dedupe_images() with a sampled bucket key, also returning the pixel bytes of the representatives."""
    first, inverse, buckets, raws = [], [], {}, []
    for i, im in enumerate(images):
        raw = im.tobytes()
        key = _sample_key(im, raw)
        j = next((k for k in buckets.get(key, ()) if raws[k] == raw), None)
        if j is None:
            j = len(first)
            buckets.setdefault(key, []).append(j)
            first.append(i)
            raws.append(raw)
        inverse.append(j)
    return first, torch.tensor(inverse, dtype=torch.long), raws


def _randn_tensor(shape, generator, device: torch.device, dtype) -> torch.Tensor:
    """diffusers.utils.torch_utils.randn_tensor [3P] (pipeline :175-177): the draw happens on the generator's device
    (CPU generator -> CPU draw in the target dtype, then moved: this is what defines seed parity); a list of
    generators draws one batch element each; no generator draws on the execution device."""
    gens = generator if isinstance(generator, (list, tuple)) else [generator]
    gdev = gens[0].device if gens[0] is not None else device
    if gdev.type != device.type and gdev.type != "cpu":
        raise ValueError(f"Cannot generate a {device} tensor from a generator of type {gdev.type}.")
    if isinstance(generator, (list, tuple)):
        one = (1,) + tuple(shape[1:])
        return torch.cat([torch.randn(one, generator=g, device=gdev, dtype=dtype) for g in generator], 0).to(device)
    return torch.randn(shape, generator=generator, device=gdev, dtype=dtype).to(device)


def _all_gather_rows(local: torch.Tensor, world: int, group) -> torch.Tensor:
    """[n, ...] of every rank -> [world * n, ...] in rank order: one all_gather_into_tensor."""
    out = torch.empty((world * local.shape[0],) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out, local.contiguous(), group=group)
    return out


class Pose2VideoPipeline:
    _optional_components: list = []

    def __init__(self, vae, image_encoder, reference_unet, denoising_unet, pose_guider, scheduler,
                 image_proj_model=None, tokenizer=None, text_encoder=None):
        self.vae, self.image_encoder = vae, image_encoder
        self.reference_unet, self.denoising_unet, self.pose_guider = reference_unet, denoising_unet, pose_guider
        self.scheduler = scheduler
        self.image_proj_model, self.tokenizer, self.text_encoder = image_proj_model, tokenizer, text_encoder
        self.vae_scale_factor = 2 ** (len(self.vae.config.block_out_channels) - 1)
        self._clip_image_processor = None
        self._vae_engines = None
        self.timings: Dict[str, float] = {}
        self.last_latents: Optional[torch.Tensor] = None
        self.io_bytes = {"h2d": 0, "d2h": 0}
        self._shard = (0, 1, None)  # (rank, world, process group): see enable_sharding()
        self.force_plan = None  # (cfg_ways, win_ways, frame_ways) instead of ShardPlan.make's: tests exercise every axis
        self._xchg_frame = self._xchg_world = self._xchg_key = None  # see _exchanges()
        self._xchg_retired, self._xchg_timeout_ms = [], 0

    def enable_sharding(self, rank: int, world: int, group=None, exchange_timeout_ms: int = 0):
        """Partition every clip over `world` GPUs (one process per GPU, torch.distributed already initialised):
        CFG branches x context windows x frames of a window, see host/shard.py. Per-frame work is local; each motion
        module re-shards frames <-> pixels with a peer-memory exchange kernel (no NCCL on the data path); the
        per-window predictions are all-gathered the same way once per step, so every rank holds the whole clip's
        latents (tiny); pose features and decoded frames are computed sharded and gathered once per clip."""
        self._shard = (rank, world, group)
        self._xchg_key = None  # the next clip re-creates the peer buffers (and frees the old ones, collectively)
        self._xchg_timeout_ms = exchange_timeout_ms

    enable_frame_sharding = enable_sharding  # round-1 name

    def release_exchanges(self):
        """Collective (every rank calls it): unmap and free the peer buffers of exchanges that were replaced because the
        clip geometry or the partitioning changed. The exchanges in use stay."""
        _, _, group = self._shard
        retired, self._xchg_retired = self._xchg_retired, []
        for x in retired:
            x.destroy(group)

    def _exchanges(self, plan, nb: int, n_my_windows: int, fl: int, h: int, w: int, dtype):
        """(frame-group exchange or None, world exchange): peer buffers sized for this geometry; collective."""
        rank, world, group = self._shard
        key = (plan, nb, n_my_windows, fl, h, w, dtype)
        if self._xchg_key != key:
            # captured forwards hold the old buffers' addresses: drop the graphs; the old exchanges are retired, not
            # freed (freeing peer-mapped memory is a collective: release_exchanges() does it when the caller wants to)
            self.denoising_unet.engine()._graphs.clear()
            self._xchg_retired += [x for x in (self._xchg_frame, self._xchg_world) if x is not None]
            self._xchg_frame = self._xchg_world = None
            esz = torch.empty((), dtype=dtype).element_size()
            c0 = self.denoising_unet.config.block_out_channels[0]
            tok = nb * fl * h * w * c0 * esz  # the widest token tensor of a forward: the first level's
            kw = dict(timeout_ms=self._xchg_timeout_ms)
            sizes = {"A": tok, "B": tok}
            if not getattr(self.denoising_unet, "use_inflated_groupnorm", True):
                # window GroupNorm: the per-frame partial tables of ResnetBlock3D norm1 / norm2 / conv_norm_out
                t = self._window_table_bytes(nb, fl, h, w)
                sizes.update(N0=t, N1=t, N2=t)
            self._xchg_frame = (Exchange.create(plan.frame_group(), rank, sizes, self.device, group, **kw)
                                if plan.frame_ways > 1 else None)
            # two gather sources used alternately: a source may only be rewritten once every peer has announced the NEXT
            # exchange (= finished pulling this one), i.e. after one exchange in between (csrc/exchange.cu)
            sz = n_my_windows * nb * 4 * fl * h * w * esz
            self._xchg_world = Exchange.create(list(range(world)), rank, {"S0": sz, "S1": sz}, self.device, group, **kw)
            self._xchg_key = key
        return self._xchg_frame, self._xchg_world

    def _window_table_bytes(self, nb: int, fl: int, h: int, w: int) -> int:
        """The largest window-GroupNorm partial table of one member's fl frames: every ResnetBlock3D input / output
        width (up-block inputs include the skip) at every level of an h x w latent."""
        cfg = self.denoising_unet.config
        ch = list(cfg.block_out_channels)
        widths = set(ch) | {a + b for a in ch for b in ch}
        return max(ops.groupnorm_window_table_bytes(nb, fl, lh * lw, c, cfg.norm_num_groups)
                   for lh, lw in E.latent_levels(h, w, len(ch)) for c in widths if c % cfg.norm_num_groups == 0)

    # ------------------------------------------------------------------------------------------------
    def to(self, device=None, dtype=None):
        for m in (self.vae, self.image_encoder, self.reference_unet, self.denoising_unet, self.pose_guider):
            if isinstance(m, torch.nn.Module):
                m.to(device=device, dtype=dtype)
        self._vae_engines = None
        return self

    @property
    def device(self) -> torch.device:
        return self.denoising_unet.device

    @property
    def _execution_device(self) -> torch.device:  # pipeline :98-112 (no accelerate hooks here: the models' device)
        return self.device

    def enable_vae_slicing(self):
        """pipeline :82-86. diffusers' slicing bounds the decoder's activation memory by decoding one image at a time; the
        engine decodes a clip's frames in one batched pass (per GPU: < 3 GB at 512 x 512 x 24 frames): nothing to switch."""

    def disable_vae_slicing(self):
        """See enable_vae_slicing()."""

    def _clip_pixels(self, ref_image: PIL.Image.Image) -> torch.Tensor:
        if self._clip_image_processor is None:
            from transformers import CLIPImageProcessor
            self._clip_image_processor = CLIPImageProcessor()
        return self._clip_image_processor.preprocess(ref_image.resize((224, 224)), return_tensors="pt").pixel_values

    def _clip(self):
        """The caller's transformers.CLIPVisionModelWithProjection is a parameter container here: its forward runs on
        the engine's kernels (mimo_b200/clip_engine.py), rebuilt when the parameters move or change dtype."""
        from ..clip_engine import CLIPVisionEngine
        p = next(self.image_encoder.parameters())
        key = (p.device, p.dtype, p.data_ptr())
        if getattr(self, "_clip_engine_key", None) != key:
            if p.device.type != "cuda":
                raise MimoError("the CLIP image encoder must be on a CUDA (sm_90a) device: no CPU fallback")
            self._clip_engine = CLIPVisionEngine(self.image_encoder.state_dict(), self.image_encoder.config, p.device, p.dtype)
            self._clip_engine_key = key
        return self._clip_engine

    def _clip_embeds(self, ref_image: PIL.Image.Image) -> torch.Tensor:
        return self._clip().image_embeds(self._clip_pixels(ref_image))

    def _vae(self):
        from .modules import AutoencoderKL as _OurVAE
        if isinstance(self.vae, _OurVAE):
            return self.vae.engine()
        if self._vae_engines is None:
            # a diffusers.AutoencoderKL (or anything with its state-dict layout): only weights and config are read
            sd = self.vae.state_dict()
            dt = self.denoising_unet.dtype
            self._vae_engines = (E.VAEEncoderEngine(sd, self.device, dt), E.VAEDecoderEngine(sd, self.device, dt))
        return self._vae_engines

    # Output pixels one batched VAE decode pass may cover: 48 frames at 768 x 768, the largest clip the benchmark decodes on
    # one GPU (its widest activation, 128 channels at full resolution, is then 3.6 G elements, ~7 GB in 16 bits). Every
    # clip up to that size keeps one pass; longer ones (e.g. an interpolated 784 x 784 clip) decode in chunks of frames.
    DECODE_PIXELS_PER_PASS = 48 * 768 * 768

    def decode_latents_device(self, latents: torch.Tensor, frames_per_pass: Optional[int] = None) -> torch.Tensor:
        """[1, 4, F, h, w] -> device tensor [1, 3, F, H, W] in [0, 1] (pipeline :113-123): batched engine passes of at
        most `frames_per_pass` frames (default: DECODE_PIXELS_PER_PASS worth). The decoder's arithmetic is per image,
        so the chunked result is byte-identical to one pass."""
        z = (1 / 0.18215 * latents)[0].permute(1, 0, 2, 3).contiguous()
        dec = self._vae()[1]
        n, s = z.shape[0], self.vae_scale_factor
        per = frames_per_pass or max(1, self.DECODE_PIXELS_PER_PASS // (z.shape[2] * s * z.shape[3] * s))
        if n <= per:
            frames = dec.decode(z)  # [F, 3, H, W]
        else:
            first = dec.decode(z[:per])
            frames = torch.empty((n,) + tuple(first.shape[1:]), dtype=first.dtype, device=first.device)
            frames[:per] = first
            del first
            for i in range(per, n, per):
                frames[i:i + per] = dec.decode(z[i:i + per])
        video = frames.permute(1, 0, 2, 3).unsqueeze(0)
        return (video / 2 + 0.5).clamp(0, 1)

    def decode_latents(self, latents: torch.Tensor) -> np.ndarray:
        return self.decode_latents_device(latents).cpu().float().numpy()  # :124-126

    def prepare_latents(self, batch_size, num_channels_latents, width, height, video_length, dtype, device, generator,
                        latents=None, scheduler=None):
        """pipeline :149-183; `scheduler` (default self.scheduler) gives init_noise_sigma: a float, or a 0-dim fp32
        tensor for Euler, whose multiply keeps the latents' dtype as the reference's does."""
        shape = (batch_size, num_channels_latents, video_length, height // self.vae_scale_factor,
                 width // self.vae_scale_factor)
        if isinstance(generator, list) and len(generator) != batch_size:
            raise ValueError(f"You have passed a list of generators of length {len(generator)}, but requested an "
                             f"effective batch size of {batch_size}.")
        if latents is None:
            latents = _randn_tensor(shape, generator, torch.device(device), dtype)
        else:
            latents = latents.to(device)  # pipeline :179
        return latents * (scheduler if scheduler is not None else self.scheduler).init_noise_sigma

    def check_size(self, width: int, height: int) -> None:
        """Whether the UNets' fused x2 upsampler serves every level: width and height multiples of 8 x 2^(UNet levels - 1)
        = 64 pixels. __call__ runs other sizes too (run_animate.py's default is 784 x 784): the levels that do not double
        exactly take the reference's `forward_upsample_size` path (unet_3d_edit_bkfill.py:430-435)."""
        m = self.vae_scale_factor << (len(self.denoising_unet.config.block_out_channels) - 1)
        if width % m or height % m:
            raise NotImplementedError(f"width x height = {width} x {height}: not both multiples of {m}, so some UNet up "
                                      "steps take the forward_upsample_size path instead of the fused x2 kernel; "
                                      f"the nearest sizes it serves are e.g. {width // m * m or m} x {height // m * m or m}")

    def latent_levels(self, width: int, height: int):
        """(h, w) of the latents at every UNet level for an image of width x height (engine.latent_levels)."""
        return E.latent_levels(height // self.vae_scale_factor, width // self.vae_scale_factor,
                               len(self.denoising_unet.config.block_out_channels))

    # ------------------------------------------------------------------------------------------------
    def _draw_noise(self, width, height, video_length, dtype, generator, num_inference_steps: int, eta: float,
                    pinned: bool, sched):
        """The clip's random draws in the reference's order: the initial latents (prepare_latents, scaled by `sched`'s
        init_noise_sigma), then, for schedulers whose steps consume a draw (step_draws) and with a generator, one
        randn_tensor(model_output.shape) per step (also at the last step), stacked in one (pinned) tensor
        [steps, 1, 4, F, h, w]. Without a generator the step noise is drawn on the device inside the loop, as
        randn_tensor does."""
        latents = self.prepare_latents(1, 4, width, height, video_length, dtype, "cpu", generator, scheduler=sched)
        if not (sched.step_draws(eta) and generator is not None and num_inference_steps > 0):
            return latents, None
        shape = tuple(latents.shape)
        noise = torch.empty((num_inference_steps,) + shape, dtype=dtype, pin_memory=pinned)
        for i in range(num_inference_steps):
            noise[i] = _randn_tensor(shape, generator, torch.device("cpu"), dtype)
        return latents, noise

    def preprocess(self, ref_image, pose_images, vid_bk_images, width, height, video_length, generator,
                   dtype, num_inference_steps: int = 0, eta: float = 0.0) -> Dict[str, torch.Tensor]:
        """Host side of __call__: PIL -> pinned CPU tensors (what the reference does at pipeline :379-381, :409-418,
        :424-426, :435-437, :446-453 before anything touches the device). With a generator, the per-step noise of DDIM
        with eta > 0 or of Euler-ancestral is drawn here too, right after the initial latents, as "step_noise"."""
        sched = engine_scheduler(self.scheduler)
        if num_inference_steps > 0:
            sched.set_timesteps(num_inference_steps, device="cpu")  # init_noise_sigma may depend on the table
        pinned = torch.cuda.is_available()
        pin = lambda t: t.contiguous().pin_memory() if pinned else t.contiguous()
        bks = list(vid_bk_images)
        if len(bks) != video_length or len(pose_images) != video_length:
            raise ValueError(f"video_length={video_length} but {len(pose_images)} pose images and {len(bks)} background "
                             "images were passed (pipeline :435-453 indexes both per frame)")
        # the noise draw (CPU generator, target dtype: ~10 ms of one core for a 24-frame clip) runs beside the image staging
        noise = _pool().submit(self._draw_noise, width, height, video_length, dtype, generator, num_inference_steps, eta,
                               pinned, sched)
        try:
            # identical background frames are converted, copied and encoded once; every frame is written straight into
            # its pinned staging tensor (stage_frames_u8: same bytes as pil_to_uint8, without the intermediate copies)
            first, inverse, raws = _dedupe_raws(bks)
            out = {
                "clip_pixels": pin(self._clip_pixels(ref_image)),
                "ref_u8": stage_frames_u8(ref_image, height, width, pinned),
                "bk_unique_u8": stage_frames_u8([bks[i] for i in first], height, width, pinned, raws=raws),
                "bk_inverse": inverse,
                "pose_u8": stage_frames_u8(list(pose_images), height, width, pinned),  # [F, H, W, 3]
            }
        finally:
            latents, step_noise = noise.result()  # also on an error above: the generator must not be left in use by a worker
        out["latents"] = pin(latents)
        if step_noise is not None:
            out["step_noise"] = step_noise
        return out

    @staticmethod
    def _interpolation_method(interpolation_factor: int, video_length: int) -> Optional[int]:
        """The mimo_interpolate_frames method for interpolation_factor (None: no interpolation, k <= 1 as in the
        reference). Checked before any work: the reference only fails after the whole denoising loop."""
        if interpolation_factor is None or interpolation_factor < 2:
            return None
        from .interpolation import get_tensor_interpolation_method, kernel_method
        method = kernel_method(get_tensor_interpolation_method())
        if video_length < 2:
            raise ValueError(f"interpolation_factor={interpolation_factor} needs at least 2 frames to interpolate "
                             f"between, got video_length={video_length}")
        return method

    @torch.no_grad()
    def sample_tensors(self, inp: Dict[str, torch.Tensor], num_inference_steps: int, guidance_scale: float,
                       context_schedule="uniform", context_frames=24, context_stride=1, context_overlap=4,
                       callback=None, callback_steps=1, decode: bool = True, eta: float = 0.0,
                       interpolation_factor: int = 1, guidance_rescale: float = 0.0) -> Dict[str, torch.Tensor]:
        """Device side: everything in `inp` already lives in HBM; returns device tensors. The scheduler is
        engine_scheduler(self.scheduler); each step is one fused kernel: mimo_cfg_ddim_step(_noise) for DDIM,
        mimo_cfg_multistep for DPM-Solver++, Euler and Euler-ancestral. The per-step noise of eta > 0 (stochastic DDIM)
        and of Euler-ancestral is inp["step_noise"] [steps, 1, 4, F, h, w] (preprocess draws it from the generator) or,
        without it, drawn on the device at every step. interpolation_factor k >= 2: the registered interpolation method
        inserts k-1 frames between neighbours before the decode; out["latents"] stays the denoised clip.
        guidance_rescale phi in [0, 1]: rescaled CFG (Lin et al. 2023 §3.4, diffusers' rescale_noise_cfg [3P]) between
        the guidance line and the step, with statistics over the whole clip (mimo_cfg_rescale); 0 or no CFG: not run."""
        sched, interp, step_noise = self._check_sampling(inp, num_inference_steps, eta, interpolation_factor,
                                                         guidance_rescale)
        dtype, do_cfg = self.denoising_unet.dtype, guidance_scale > 1.0
        marks = []

        def mark(name):
            marks.append((name, torch.cuda.Event(enable_timing=True)))
            marks[-1][1].record()

        mark("start")
        sched.set_timesteps(num_inference_steps, device="cpu")
        timesteps = [t.item() for t in sched.timesteps]  # DDIM / DPM-Solver++: int; Euler: fp32 values
        ehs = self._clip().image_embeds(inp["clip_pixels"]).to(dtype).unsqueeze(1)  # :378-385
        ehs = torch.cat([torch.zeros_like(ehs), ehs], dim=0) if do_cfg else ehs
        mark("clip")
        latents = inp["latents"].to(dtype).clone()
        F_, h, w = latents.shape[2:]
        ref_latents, vid_bk, pose_px = self._encode_vae(inp, dtype, h, w)
        mark("vae_encode")
        pose_fea = self._pose_features(pose_px, F_, h, w)
        mark("pose_guider")
        windows = list(get_context_scheduler(context_schedule)(0, num_inference_steps, F_, context_frames,
                                                               context_stride, context_overlap))
        plan = self._shard_plan(windows, do_cfg, h, w)
        branches = plan.branches(do_cfg) if plan else tuple(range(2 if do_cfg else 1))
        reader, writer = self._reference_pass(ref_latents, ehs, do_cfg, branches, dtype)
        mark("reference_unet")
        self._denoise(sched, timesteps, latents, windows, plan, branches, pose_fea, vid_bk, guidance_scale, eta,
                      step_noise, callback, callback_steps, guidance_rescale)
        mark("denoise")
        reader.clear()
        writer.clear()
        out = {"latents": latents}
        if decode:
            vid_lat = latents
            if interp is not None:  # pipeline :566-567: the frames to decode, (F - 1) * k + 1 of them
                vid_lat = ops.interpolate_frames(latents, interpolation_factor, interp)
                mark("interpolate")
            out["videos"] = self._decode(vid_lat)
            mark("vae_decode")
        self._marks = marks
        self.last_latents = latents
        return out

    @staticmethod
    def _check_guidance_rescale(guidance_rescale: float) -> None:
        """phi of rescaled CFG must lie in the paper's range [0, 1] (NaN and infinities refused)."""
        if not 0.0 <= float(guidance_rescale) <= 1.0:
            raise ValueError(f"guidance_rescale={guidance_rescale}: must be a finite value in [0, 1]")

    def _check_sampling(self, inp, num_inference_steps: int, eta: float, interpolation_factor: int,
                        guidance_rescale: float = 0.0):
        """The refusals, in this order, before any work -> (scheduler, interpolation method, step noise or None)."""
        if eta < 0:
            raise ValueError(f"eta={eta}: DDIM's eta is >= 0 (0 deterministic, 1 DDPM-like)")
        self._check_guidance_rescale(guidance_rescale)
        interp = self._interpolation_method(interpolation_factor, inp["latents"].shape[2])
        sched = engine_scheduler(self.scheduler)
        step_noise = inp.get("step_noise") if sched.step_draws(eta) else None
        if step_noise is not None and (step_noise.shape[0] < num_inference_steps
                                       or tuple(step_noise.shape[1:]) != tuple(inp["latents"].shape)):
            raise ValueError(f"step_noise {tuple(step_noise.shape)} does not hold {num_inference_steps} draws of "
                             f"{tuple(inp['latents'].shape)}")
        return sched, interp, step_noise

    def _encode_vae(self, inp, dtype, h: int, w: int):
        """-> (reference latents, background latents [1, 4, F, h, w], pose pixels [1, 3, F, H, W]): every image goes
        from bytes to normalised pixels on the device here (pipeline :424-426, :435-437, :446-453)."""
        enc, _ = self._vae()
        ref_px = uint8_to_tensor(inp["ref_u8"], True).to(dtype)
        bk_px = uint8_to_tensor(inp["bk_unique_u8"], True).to(dtype)
        pose_px = uint8_to_tensor(inp["pose_u8"], False).permute(1, 0, 2, 3).unsqueeze(0).to(dtype)
        rank, world, group = self._shard
        n_bk = bk_px.shape[0]
        if world > 1 and n_bk >= world:
            # edit mode: one distinct background per frame (run_edit.py:232-238) - every GPU encodes its share, one
            # all-gather per clip (per-image arithmetic: identical to encoding them all here)
            ref_latents = enc.encode_mean(ref_px) * 0.18215  # :424-431
            per = -(-n_bk // world)
            lo, hi = min(rank * per, n_bk), min((rank + 1) * per, n_bk)
            mine = torch.zeros((per, 4, h, w), device=self.device, dtype=dtype)
            if hi > lo:
                mine[:hi - lo] = enc.encode_mean(bk_px[lo:hi].contiguous()).to(dtype)
            bk_mean = _all_gather_rows(mine, world, group)[:n_bk]
        elif n_bk <= 4:
            # animate mode: the reference image and the (deduplicated) background go through the encoder together
            # (per-image arithmetic: the same values as two calls, one kernel chain instead of two)
            both = enc.encode_mean(torch.cat([ref_px, bk_px]))
            ref_latents, bk_mean = both[:1] * 0.18215, both[1:]
        else:
            ref_latents, bk_mean = enc.encode_mean(ref_px) * 0.18215, enc.encode_mean(bk_px)
        bk_lat = (bk_mean * 0.18215)[inp["bk_inverse"].to(self.device)]
        return ref_latents, bk_lat.permute(1, 0, 2, 3).unsqueeze(0).to(dtype).contiguous(), pose_px  # :434-443

    def _pose_features(self, pose_px: torch.Tensor, F_: int, h: int, w: int) -> torch.Tensor:
        """Channels-last pose features [F, h * w, C]; ranks that divide F compute their frames and all-gather."""
        rank, world, group = self._shard
        if world > 1 and F_ % world == 0:
            fl = F_ // world
            loc = self.pose_guider.forward_nhwc(pose_px[:, :, rank * fl:(rank + 1) * fl].contiguous())
            return _all_gather_rows(loc, world, group).reshape(F_, h * w, -1)
        return self.pose_guider.forward_nhwc(pose_px).reshape(F_, h * w, -1)

    def _shard_plan(self, windows, do_cfg: bool, h: int, w: int):
        """How the ranks divide the clip (host/shard.py: CFG branches x windows x frames), or None on one GPU."""
        rank, world, _ = self._shard
        if world <= 1:
            return None
        if len({len(c) for c in windows}) != 1:
            raise NotImplementedError("context windows of different lengths cannot be sharded")
        nb = len(self.denoising_unet.config.block_out_channels)
        plan = ShardPlan.make(world, rank, do_cfg, len(windows), len(windows[0]),
                              min_tokens=shard_tokens(h, w, nb, self.denoising_unet.motion_layout.levels(nb)))
        if self.force_plan is not None:
            assert self.force_plan[0] * self.force_plan[1] * self.force_plan[2] == world
            plan = ShardPlan(world, rank, *self.force_plan)
        return plan

    def _reference_pass(self, ref_latents, ehs, do_cfg: bool, branches, dtype):
        """Reference UNet once, banks -> denoising engine for this GPU's CFG `branches` (pipeline :393-406, :480-490)."""
        writer = ReferenceAttentionControl(self.reference_unet, do_classifier_free_guidance=do_cfg, mode="write",
                                           batch_size=1, fusion_blocks="full")
        reader = ReferenceAttentionControl(self.denoising_unet, do_classifier_free_guidance=do_cfg, mode="read",
                                           batch_size=1, fusion_blocks="full")
        self.reference_unet(ref_latents.to(dtype).repeat(2 if do_cfg else 1, 1, 1, 1), torch.zeros((), dtype=torch.int64),
                            encoder_hidden_states=ehs, return_dict=False)
        self.denoising_unet._branches = branches
        reader.update(writer)
        return reader, writer

    def _denoise(self, sched, timesteps, latents, windows, plan, branches, pose_fea, vid_bk, guidance_scale: float,
                 eta: float, step_noise, callback, callback_steps: int, guidance_rescale: float = 0.0) -> None:
        """The denoising loop (pipeline :492-561) on `latents`, in place: per step, this GPU's windows, then fused_step
        (after mimo_cfg_rescale when CFG is on and guidance_rescale > 0)."""
        device, dtype = self.device, latents.dtype
        F_, h, w = latents.shape[2:]
        do_cfg = guidance_scale > 1.0
        # every rank holds the whole clip's prediction here, so the clip-wide statistics need no communication
        rescaled = torch.empty_like(latents) if do_cfg and guidance_rescale > 0 else None
        rep, nb, single = 2 if do_cfg else 1, len(branches), len(windows) == 1
        den = self.denoising_unet.engine()
        my_windows = plan.windows_of(len(windows)) if plan else list(range(len(windows)))
        win_inputs = []
        for wi in my_windows:  # the windows and their pose features are the same at every step (pipeline :493-500)
            c = windows[wi]
            cl = plan.local_frames(c) if plan else c  # this rank's frames of the window, in window order
            pose_in = pose_fea[cl].reshape(1, len(cl) * h * w, -1).repeat(nb, 1, 1).reshape(nb * len(cl) * h * w, -1)
            win_inputs.append((c, cl, vid_bk[:, :, cl], pose_in.contiguous()))
        if plan:
            fl = len(win_inputs[0][1])
            den.xchg, xw = self._exchanges(plan, nb, len(my_windows), fl, h, w, dtype)
            stages = [xw.bufs[k].view(len(my_windows), nb * 4 * fl * h * w, dtype) for k in ("S0", "S1")]
            gathered = torch.empty((plan.world, len(my_windows), nb, 4, fl, h, w), dtype=dtype, device=device)
            gcols = next(c for c in (64, 32, 16, 8) if stages[0].numel() % c == 0)
            scatter = [(q, j, list(brs), torch.tensor(fr, dtype=torch.long, device=device))
                       for q, j, brs, fr in gather_layout(plan, windows, do_cfg)]
            counter_all = torch.zeros((F_,), device=device, dtype=dtype)
            for c in windows:
                counter_all[c] = counter_all[c] + 1
        elif den.xchg is not None:
            den._graphs.clear()  # graphs captured with exchange nodes must not serve an un-sharded run
            den.xchg = None
        history = sched.new_history(latents)
        draws = sched.step_draws(eta)
        for i, t in enumerate(timesteps):
            # scale_model_input (pipeline :519-521): the reference's own expression `x / s` with s a 0-dim fp32 tensor
            # for Euler; the identity for DDIM and DPM-Solver++
            s_in = sched.model_input_scale(i)
            lat_src = latents if s_in is None else latents / s_in
            if plan:
                par = xw.parity  # alternates across steps AND clips
                xw.parity = par ^ 1
                stage = stages[par]
                for j, (c, cl, bk_c, pose_in) in enumerate(win_inputs):
                    lat_in = torch.cat([lat_src[:, :, cl], bk_c], dim=1).repeat(nb, 1, 1, 1, 1)
                    stage[j].copy_(den.forward(lat_in, t, pose_in).reshape(-1))
                xw.pull(2, ("S0", "S1")[par], gathered.view(-1, gcols), 1, 1, stage.numel() // gcols, gcols)
                noise_pred = torch.zeros((rep, 4, F_, h, w), device=device, dtype=dtype)
                for q, j, brs, fidx in scatter:
                    noise_pred[brs[0]:brs[-1] + 1] = noise_pred[brs[0]:brs[-1] + 1].index_add(2, fidx, gathered[q, j])
                counter = None if single else counter_all
            else:
                if not single:
                    noise_pred = torch.zeros((rep, 4, F_, h, w), device=device, dtype=dtype)
                    counter = torch.zeros((F_,), device=device, dtype=dtype)
                for c, cl, bk_c, pose_in in win_inputs:
                    lat_in = torch.cat([lat_src[:, :, cl], bk_c], dim=1).repeat(rep, 1, 1, 1, 1)
                    pred = den.forward(lat_in, t, pose_in)
                    if single:
                        noise_pred, counter = pred, None
                    else:
                        noise_pred[:, :, c] = noise_pred[:, :, c] + pred  # :540-542
                        counter[c] = counter[c] + 1
            # the reference divides the window sums by `counter` only inside its guidance branch (pipeline :545-549):
            # without CFG, frames that two windows cover keep the SUM of both predictions - mirrored, not repaired
            pu, pc, g_, cnt = (noise_pred[0], noise_pred[1], guidance_scale, counter) if do_cfg else (
                noise_pred[0], noise_pred[0], 1.0, None)
            if rescaled is not None:
                # diffusers' rescale_noise_cfg sits between the guidance line and the step; the step kernels pass a
                # prediction given as both halves at guidance 1 through unchanged: rnd(v + rnd(1 * rnd(v - v))) = v
                ops.cfg_rescale(pu, pc, g_, guidance_rescale, out=rescaled, counter=cnt, frame_stride=h * w)
                pu, pc, g_, cnt = rescaled, rescaled, 1.0, None
            noise = None
            if draws:  # one draw per step, also at the last one where its coefficient is 0 (DDIMScheduler.step [3P])
                noise = (step_noise[i] if step_noise is not None
                         else torch.randn(tuple(latents.shape), device=device, dtype=dtype))
            sched.fused_step(i, t, pu, pc, latents, g_, eta=eta, noise=noise, history=history, counter=cnt,
                             frame_stride=h * w)
            # the reference's inner `for i in range(num_context_batches)` (pipeline :503-510) shadows the step index: its
            # callback test (:556-561) and the index it passes see the LAST CONTEXT BATCH's index, at every step
            i_ref = len(windows) - 1
            if callback is not None and i_ref % callback_steps == 0:
                callback(i_ref, t, latents)

    def _decode(self, vid_lat: torch.Tensor) -> torch.Tensor:
        """decode_latents_device(); ranks that divide the frames decode their frames and all-gather."""
        rank, world, group = self._shard
        Fv = vid_lat.shape[2]
        if world > 1 and Fv % world == 0:
            fl = Fv // world
            loc = self.decode_latents_device(vid_lat[:, :, rank * fl:(rank + 1) * fl])  # [1, 3, fl, H, W]
            return _all_gather_rows(loc, world, group).view((world,) + tuple(loc.shape)).permute(1, 2, 0, 3, 4, 5).reshape(
                1, 3, Fv, loc.shape[-2], loc.shape[-1])
        return self.decode_latents_device(vid_lat)

    def _collect_timings(self):
        m = self._marks
        self.timings = {m[k][0] + "_ms": m[k - 1][1].elapsed_time(m[k][1]) for k in range(1, len(m))}

    # ------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def __call__(self, ref_image, pose_images, vid_bk_images, width, height, video_length, num_inference_steps,
                 guidance_scale, num_images_per_prompt=1, eta: float = 0.0,
                 generator: Optional[Union[torch.Generator, List[torch.Generator]]] = None,
                 output_type: Optional[str] = "tensor", return_dict: bool = True,
                 callback: Optional[Callable[[int, int, torch.Tensor], None]] = None,
                 callback_steps: Optional[int] = 1, context_schedule="uniform", context_frames=24, context_stride=1,
                 context_overlap=4, context_batch_size=1, interpolation_factor=1, guidance_rescale: float = 0.0,
                 **kwargs):
        device = self.device
        if device.type != "cuda":
            raise MimoError("Pose2VideoPipeline needs its models on a CUDA (sm_90a) device: no CPU fallback")
        if context_batch_size != 1 or num_images_per_prompt != 1:
            raise NotImplementedError("context_batch_size != 1 and num_images_per_prompt != 1 are outside the "
                                      "reference's shipped configuration")
        if eta < 0:
            raise ValueError(f"eta={eta}: DDIM's eta is >= 0 (0 deterministic, 1 DDPM-like)")
        self._check_guidance_rescale(guidance_rescale)
        self._interpolation_method(interpolation_factor, video_length)  # before any work is done
        dtype = self.denoising_unet.dtype
        self.latent_levels(width, height)  # refuses only images smaller than one latent pixel
        engine_scheduler(self.scheduler)  # refuses LMS, PNDM and unknown schedulers before any work
        host = self.preprocess(ref_image, pose_images, vid_bk_images, width, height, video_length, generator, dtype,
                               num_inference_steps, eta)
        dev_in = {k: v.to(device, non_blocking=True) for k, v in host.items()}
        self.io_bytes["h2d"] = sum(v.numel() * v.element_size() for v in host.values())
        out = self.sample_tensors(dev_in, num_inference_steps, guidance_scale, context_schedule, context_frames,
                                  context_stride, context_overlap, callback, callback_steps, eta=eta,
                                  interpolation_factor=interpolation_factor, guidance_rescale=guidance_rescale)
        vid = out["videos"].float()  # :124-126 "always cast to float32": exact, and 20 ms cheaper here than on one host core
        host_vid = torch.empty(vid.shape, dtype=torch.float32, pin_memory=True)
        host_vid.copy_(vid, non_blocking=True)  # one D2H of the finished clip, into pinned memory
        torch.cuda.synchronize(device)
        images = host_vid.numpy()
        self.io_bytes["d2h"] = vid.numel() * vid.element_size()
        self._collect_timings()
        if output_type == "tensor":
            images = torch.from_numpy(images)
        if not return_dict:
            return images
        return Pose2VideoPipelineOutput(videos=images)
