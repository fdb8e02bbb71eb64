"""CPU/fp32 ORACLE of the MIMO denoising path — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A functional (state-dict driven) restatement, in plain PyTorch, of what the reference computes on its hot path.
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this module;
nothing under mimo_b200/ does. It runs on whatever device its tensors live on (CPU fp32 for the baseline; a
checker may also run it on the GPU in fp32 — it is still torch library code, never our kernels).

Pinning: the reference has no tests, fixtures or golden vectors for this path (SURVEY.md §4/§8c), so this file
is pinned against *outputs of the reference itself*: oracle/pin_against_reference.py imports the original project's src
verbatim (on oracle/diffusers_shim) in the build container, feeds both implementations the same seeded state
dicts and inputs, asserts agreement, and writes tests/golden/*.pt. diffusers==0.24.0 (install.sh:12) is absent
from the original project and this image; its Attention / FeedForward / ResnetBlock2D / AutoencoderKL / DDIMScheduler
arithmetic is restated here from the published algorithm and anchored on the reference's call sites.

Every function cites the reference file:line it follows (paths relative to the original project's root).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

SD = Dict[str, torch.Tensor]

TAPS: Optional[dict] = None  # debugging aid: when a dict, _unet_body records every block output [N, C, H, W] by path


def _tap(name: str, x: torch.Tensor) -> torch.Tensor:
    if TAPS is not None:
        TAPS[name] = x.detach().float().cpu()
    return x


# =====================================================================================================
# configuration (configs/inference/inference_v2.yaml + SD1.5 unet/config.json, SURVEY.md §5/§8c)
# =====================================================================================================
@dataclass
class UNetConfig:
    block_out_channels: Tuple[int, ...] = (320, 640, 1280, 1280)
    layers_per_block: int = 2
    heads: int = 8  # SD1.5 "attention_head_dim: 8" is the head COUNT (unet_3d_edit_bkfill.py:116-117,138)
    cross_attention_dim: int = 768
    norm_num_groups: int = 32
    norm_eps: float = 1e-5
    in_channels: int = 8  # denoising UNet: latents(4) + background latents(4) (unet_3d_edit_bkfill.py:88)
    out_channels: int = 4
    motion_max_len: int = 32  # temporal_position_encoding_max_len
    motion_groups: int = 32  # TemporalTransformer3DModel.norm_num_groups default (motion_module.py:106)

    @property
    def time_embed_dim(self) -> int:
        return self.block_out_channels[0] * 4


@dataclass
class VAEConfig:
    block_out_channels: Tuple[int, ...] = (128, 256, 512, 512)
    layers_per_block: int = 2
    latent_channels: int = 4
    norm_num_groups: int = 32
    in_channels: int = 3
    out_channels: int = 3


POSE_CHANNELS = (16, 32, 96, 256)  # run_animate.py:88-90


# =====================================================================================================
# leaf ops
# =====================================================================================================
def _lin(sd: SD, p: str, x: torch.Tensor) -> torch.Tensor:
    return F.linear(x, sd[p + ".weight"], sd.get(p + ".bias"))


def _conv(sd: SD, p: str, x: torch.Tensor, stride: int = 1, padding: int = 1) -> torch.Tensor:
    return F.conv2d(x, sd[p + ".weight"], sd.get(p + ".bias"), stride=stride, padding=padding)


def _gn(sd: SD, p: str, x: torch.Tensor, groups: int, eps: float) -> torch.Tensor:
    return F.group_norm(x, groups, sd[p + ".weight"], sd[p + ".bias"], eps)


def _ln(sd: SD, p: str, x: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    return F.layer_norm(x, (x.shape[-1],), sd[p + ".weight"], sd[p + ".bias"], eps)


def attention(sd: SD, p: str, x: torch.Tensor, ctx: Optional[torch.Tensor], heads: int) -> torch.Tensor:
    """diffusers Attention + AttnProcessor2_0 [3P]: to_q/k/v (no bias unless present), SDPA scale d^-1/2, to_out[0].
    Constructed at src/models/attention.py:321-345 and src/models/motion_module.py:282-292."""
    B, Lq, _ = x.shape
    kv = x if ctx is None else ctx
    q = _lin(sd, p + ".to_q", x)
    k = _lin(sd, p + ".to_k", kv)
    v = _lin(sd, p + ".to_v", kv)
    d = q.shape[-1] // heads
    q = q.view(B, -1, heads, d).transpose(1, 2)
    k = k.view(B, -1, heads, d).transpose(1, 2)
    v = v.view(B, -1, heads, d).transpose(1, 2)
    o = F.scaled_dot_product_attention(q, k, v, attn_mask=None, dropout_p=0.0, is_causal=False)
    o = o.transpose(1, 2).reshape(B, -1, heads * d).to(q.dtype)
    return _lin(sd, p + ".to_out.0", o)


def feed_forward(sd: SD, p: str, x: torch.Tensor) -> torch.Tensor:
    """diffusers FeedForward(activation_fn="geglu") [3P]: Linear(C, 8C) -> h * gelu_erf(gate) -> Linear(4C, C).
    Constructed at src/models/attention.py:359 and src/models/motion_module.py:235."""
    h, gate = _lin(sd, p + ".net.0.proj", x).chunk(2, dim=-1)
    return _lin(sd, p + ".net.2", h * F.gelu(gate))


def timestep_embedding(sd: SD, t: torch.Tensor, dim: int, dtype: torch.dtype) -> torch.Tensor:
    """Timesteps(dim, flip_sin_to_cos=True, freq_shift=0) -> TimestepEmbedding [3P]; call site
    src/models/unet_3d_edit_bkfill.py:447-468 (t_emb cast to the model dtype before the MLP)."""
    half = dim // 2
    exponent = -math.log(10000) * torch.arange(0, half, dtype=torch.float32, device=t.device) / (half - 0.0)
    emb = t[:, None].float() * torch.exp(exponent)[None, :]
    emb = torch.cat([torch.sin(emb), torch.cos(emb)], dim=-1)
    emb = torch.cat([emb[:, half:], emb[:, :half]], dim=-1)  # flip_sin_to_cos
    emb = emb.to(dtype)
    return _lin(sd, "time_embedding.linear_2", F.silu(_lin(sd, "time_embedding.linear_1", emb)))


def resnet_block(sd: SD, p: str, x: torch.Tensor, temb: Optional[torch.Tensor], groups: int, eps: float,
                 output_scale_factor: float = 1.0) -> torch.Tensor:
    """ResnetBlock3D.forward, src/models/resnet.py:217-247 (== diffusers ResnetBlock2D on (b f) frames).
    x: [N, C, H, W]; temb: [N, temb_dim] or None (VAE)."""
    h = F.silu(_gn(sd, p + ".norm1", x, groups, eps))
    h = _conv(sd, p + ".conv1", h)
    if temb is not None:
        h = h + _lin(sd, p + ".time_emb_proj", F.silu(temb))[:, :, None, None]
    h = F.silu(_gn(sd, p + ".norm2", h, groups, eps))
    h = _conv(sd, p + ".conv2", h)
    if (p + ".conv_shortcut.weight") in sd:
        x = _conv(sd, p + ".conv_shortcut", x, padding=0)
    return (x + h) / output_scale_factor


# =====================================================================================================
# spatial transformer (Transformer3DModel / Transformer2DModel) with the reference-attention hooks
# =====================================================================================================
def _tokens(x: torch.Tensor) -> torch.Tensor:
    n, c, h, w = x.shape
    return x.permute(0, 2, 3, 1).reshape(n, h * w, c)


def _untokens(t: torch.Tensor, h: int, w: int) -> torch.Tensor:
    n, _, c = t.shape
    return t.reshape(n, h, w, c).permute(0, 3, 1, 2).contiguous()


def transformer_block_write(sd: SD, p: str, x: torch.Tensor, ehs: torch.Tensor, heads: int, bank: list) -> torch.Tensor:
    """BasicTransformerBlock under hacked_basic_transformer_inner_forward, MODE == "write":
    src/models/mutual_self_attention.py:120-147, 241-276."""
    nh = _ln(sd, p + ".norm1", x)
    bank.append(nh.clone())
    x = attention(sd, p + ".attn1", nh, None, heads) + x
    x = attention(sd, p + ".attn2", _ln(sd, p + ".norm2", x), ehs, heads) + x
    return feed_forward(sd, p + ".ff", _ln(sd, p + ".norm3", x)) + x


def transformer_block_read(sd: SD, p: str, x: torch.Tensor, ehs: torch.Tensor, heads: int, bank: Sequence[torch.Tensor],
                           video_length: int, cfg: bool) -> torch.Tensor:
    """TemporalBasicTransformerBlock under hacked_basic_transformer_inner_forward, MODE == "read":
    src/models/mutual_self_attention.py:148-239 (unet_use_temporal_attention False -> :222 skipped)."""
    nh = _ln(sd, p + ".norm1", x)
    # :154-168  bank [B, L, C] -> repeat over frames "(b t) l c"; keys/values = [self | bank]
    bank_fea = [d.unsqueeze(1).repeat(1, video_length, 1, 1).flatten(0, 1) for d in bank]
    mod = torch.cat([nh] + bank_fea, dim=1)
    hs_uc = attention(sd, p + ".attn1", nh, mod, heads) + x
    if cfg:
        # :177-197 the first half of the batch (unconditional branch) is recomputed WITHOUT the bank
        hs_c = hs_uc.clone()
        half = x.shape[0] // 2
        hs_c[:half] = attention(sd, p + ".attn1", nh[:half], nh[:half], heads) + x[:half]
        x = hs_c
    else:
        x = hs_uc
    x = attention(sd, p + ".attn2", _ln(sd, p + ".norm2", x), ehs, heads) + x  # :202-216
    return feed_forward(sd, p + ".ff", _ln(sd, p + ".norm3", x)) + x  # :219


def spatial_transformer(sd: SD, p: str, x: torch.Tensor, ehs: torch.Tensor, cfg_: UNetConfig, block_fn) -> torch.Tensor:
    """Transformer3DModel.forward, src/models/transformer_3d.py:103-169 (2-D twin: transformer_2d.py:213-396):
    GN(eps 1e-6) -> 1x1 conv -> tokens -> block -> 1x1 conv -> + residual. x: [N, C, H, W]."""
    n, c, h, w = x.shape
    res = x
    hcur = _gn(sd, p + ".norm", x, cfg_.norm_num_groups, 1e-6)
    hcur = _conv(sd, p + ".proj_in", hcur, padding=0)
    t = _tokens(hcur)
    t = block_fn(p + ".transformer_blocks.0", t)
    hcur = _conv(sd, p + ".proj_out", _untokens(t, h, w), padding=0)
    return hcur + res


# =====================================================================================================
# motion module
# =====================================================================================================
def motion_module(sd: SD, p: str, x: torch.Tensor, video_length: int, cfg_: UNetConfig) -> torch.Tensor:
    """VanillaTemporalModule -> TemporalTransformer3DModel -> TemporalTransformerBlock -> VersatileAttention:
    src/models/motion_module.py:77-91, 146-184, 238-261, 353-390 (+ PositionalEncoding :277-279).
    x: [(b f), C, H, W]."""
    tp = p + ".temporal_transformer"
    n, c, h, w = x.shape
    res = x
    t = _tokens(_gn(sd, tp + ".norm", x, cfg_.motion_groups, 1e-6))
    t = _lin(sd, tp + ".proj_in", t)
    bp = tp + ".transformer_blocks.0"
    f = video_length
    b = n // f
    d = h * w
    for i in range(2):  # attention_block_types = (Temporal_Self, Temporal_Self)
        nh = _ln(sd, f"{bp}.norms.{i}", t)
        # "(b f) d c -> (b d) f c"
        seq = nh.reshape(b, f, d, c).permute(0, 2, 1, 3).reshape(b * d, f, c)
        pe = sd[f"{bp}.attention_blocks.{i}.pos_encoder.pe"]
        seq = seq + pe[:, :f].to(seq.dtype)
        o = attention(sd, f"{bp}.attention_blocks.{i}", seq, None, cfg_.heads)
        o = o.reshape(b, d, f, c).permute(0, 2, 1, 3).reshape(n, d, c)
        t = o + t
    t = feed_forward(sd, bp + ".ff", _ln(sd, bp + ".ff_norm", t)) + t
    t = _lin(sd, tp + ".proj_out", t)
    return _untokens(t, h, w) + res


# =====================================================================================================
# UNets
# =====================================================================================================
def transformer_paths(cfg_: UNetConfig) -> List[str]:
    """Spatial transformer block prefixes in the pairing order ReferenceAttentionControl uses: torch_dfs visits
    children as registered (down_blocks, up_blocks, mid_block — mid_block is assigned last in both UNets'
    __init__), then a stable sort by -channels (src/models/mutual_self_attention.py:288-297, 331-349)."""
    nb = len(cfg_.block_out_channels)
    paths = []
    for i in range(nb - 1):
        for j in range(cfg_.layers_per_block):
            paths.append((cfg_.block_out_channels[i], f"down_blocks.{i}.attentions.{j}"))
    rev = list(reversed(cfg_.block_out_channels))
    for i in range(1, nb):
        for j in range(cfg_.layers_per_block + 1):
            paths.append((rev[i], f"up_blocks.{i}.attentions.{j}"))
    paths.append((cfg_.block_out_channels[-1], "mid_block.attentions.0"))
    order = sorted(range(len(paths)), key=lambda k: -paths[k][0])  # python's sort is stable
    return [paths[k][1] for k in order]


def _unet_body(sd: SD, x: torch.Tensor, temb: torch.Tensor, cfg_: UNetConfig, xf_fn: Callable[[str, torch.Tensor], torch.Tensor],
               mm_fn: Optional[Callable[[str, torch.Tensor], torch.Tensor]], stop_after_last_attention: bool = False):
    """Shared down / mid / up skeleton: src/models/unet_3d_edit_bkfill.py:487-566 with the block forwards of
    src/models/unet_3d_blocks.py:269-293, 440-464, 563-583, 725-745, 848-862 (2-D twins in unet_2d_blocks.py)."""
    g, eps = cfg_.norm_num_groups, cfg_.norm_eps
    nb = len(cfg_.block_out_channels)
    skips = [x]
    for i in range(nb):
        has_attn = i < nb - 1
        for j in range(cfg_.layers_per_block):
            x = _tap(f"down_blocks.{i}.resnets.{j}", resnet_block(sd, f"down_blocks.{i}.resnets.{j}", x, temb, g, eps))
            if has_attn:
                x = _tap(f"down_blocks.{i}.attentions.{j}", xf_fn(f"down_blocks.{i}.attentions.{j}", x))
            if mm_fn is not None:
                x = _tap(f"down_blocks.{i}.motion_modules.{j}", mm_fn(f"down_blocks.{i}.motion_modules.{j}", x))
            skips.append(x)
        if i < nb - 1:
            x = _tap(f"down_blocks.{i}.down", _conv(sd, f"down_blocks.{i}.downsamplers.0.conv", x, stride=2, padding=1))
            skips.append(x)
    x = _tap("mid_block.resnets.0", resnet_block(sd, "mid_block.resnets.0", x, temb, g, eps))
    x = _tap("mid_block.attentions.0", xf_fn("mid_block.attentions.0", x))
    if mm_fn is not None:
        x = _tap("mid_block.motion_modules.0", mm_fn("mid_block.motion_modules.0", x))
    x = _tap("mid_block.resnets.1", resnet_block(sd, "mid_block.resnets.1", x, temb, g, eps))
    for i in range(nb):
        has_attn = i > 0
        for j in range(cfg_.layers_per_block + 1):
            x = torch.cat([x, skips.pop()], dim=1)
            x = _tap(f"up_blocks.{i}.resnets.{j}", resnet_block(sd, f"up_blocks.{i}.resnets.{j}", x, temb, g, eps))
            if has_attn:
                x = _tap(f"up_blocks.{i}.attentions.{j}", xf_fn(f"up_blocks.{i}.attentions.{j}", x))
            if mm_fn is not None:
                x = _tap(f"up_blocks.{i}.motion_modules.{j}", mm_fn(f"up_blocks.{i}.motion_modules.{j}", x))
        if i < nb - 1:
            x = F.interpolate(x, scale_factor=2.0, mode="nearest")  # Upsample3D: scale_factor=[1,2,2] over (f,h,w)
            x = _tap(f"up_blocks.{i}.up", _conv(sd, f"up_blocks.{i}.upsamplers.0.conv", x))
    return x


def reference_unet_banks(sd: SD, latents: torch.Tensor, ehs: torch.Tensor, cfg_: UNetConfig,
                         bank_dtype: Optional[torch.dtype] = torch.float16) -> Dict[str, torch.Tensor]:
    """reference_unet forward at t = 0 in "write" mode (pipeline :480-490; src/models/unet_2d_condition.py:872-1308,
    whose conv_norm_out/conv_out are removed, :645-653/:1295-1299). Returns {block prefix: norm1(x) [B, HW, C]}
    after ReferenceAttentionControl.update's cast `.to(float16)` (src/models/mutual_self_attention.py:313, 349),
    stored back in the compute dtype is NOT done here: the cast dtype is kept (torch.cat promotes in the reader)."""
    B = latents.shape[0]
    t = torch.zeros((B,), dtype=torch.int64, device=latents.device)
    temb = timestep_embedding(sd, t, cfg_.block_out_channels[0], latents.dtype)
    banks: Dict[str, torch.Tensor] = {}

    def xf(p: str, x: torch.Tensor) -> torch.Tensor:
        bank: list = []
        out = spatial_transformer(sd, p, x, ehs, cfg_,
                                  lambda bp, tok: transformer_block_write(sd, bp, tok, ehs, cfg_.heads, bank))
        banks[p] = bank[0].to(bank_dtype) if bank_dtype is not None else bank[0]
        return out

    x = _conv(sd, "conv_in", latents)
    _unet_body(sd, x, temb, cfg_, xf, None)
    return banks


def denoising_unet(sd: SD, sample: torch.Tensor, timestep, ehs: torch.Tensor, pose_fea: Optional[torch.Tensor],
                   banks: Dict[str, torch.Tensor], cfg_: UNetConfig, cfg: bool = True) -> torch.Tensor:
    """UNet3DConditionModel.forward, src/models/unet_3d_edit_bkfill.py:398-576, with every spatial block in
    "read" mode. sample [b, 8, f, h, w], ehs [b, 1, 768], pose_fea [b, 320, f, h, w] -> [b, 4, f, h, w]."""
    b, c, f, h, w = sample.shape
    t = timestep if torch.is_tensor(timestep) else torch.tensor([timestep], dtype=torch.int64, device=sample.device)
    t = t.reshape(-1).to(sample.device).expand(b)
    temb = timestep_embedding(sd, t, cfg_.block_out_channels[0], sample.dtype)  # [b, 1280]
    temb_n = temb.repeat_interleave(f, dim=0)  # broadcast over frames ([:, :, None, None, None] in resnet.py:226)
    ehs_n = ehs.repeat_interleave(f, dim=0)  # "b n c -> (b f) n c", transformer_3d.py:116-119

    def to4(x5):
        return x5.permute(0, 2, 1, 3, 4).reshape(b * f, x5.shape[1], x5.shape[3], x5.shape[4])

    x = _conv(sd, "conv_in", to4(sample))
    if pose_fea is not None:
        x = x + to4(pose_fea)  # :483-485

    def xf(p: str, xx: torch.Tensor) -> torch.Tensor:
        bank = [banks[p]] if p in banks else []
        return spatial_transformer(sd, p, xx, ehs_n, cfg_,
                                   lambda bp, tok: transformer_block_read(sd, bp, tok, ehs_n, cfg_.heads, bank, f, cfg))

    x = _unet_body(sd, x, temb_n, cfg_, xf, lambda p, xx: motion_module(sd, p, xx, f, cfg_))
    x = F.silu(_gn(sd, "conv_norm_out", x, cfg_.norm_num_groups, cfg_.norm_eps))  # :569-571
    x = _conv(sd, "conv_out", x)
    return x.reshape(b, f, x.shape[1], h, w).permute(0, 2, 1, 3, 4)


def pose_guider(sd: SD, cond: torch.Tensor) -> torch.Tensor:
    """PoseGuider.forward, src/models/pose_guider.py:47-57. cond [b, 3, f, H, W] in [0, 1] -> [b, 320, f, H/8, W/8]."""
    b, c, f, H, W = cond.shape
    x = cond.permute(0, 2, 1, 3, 4).reshape(b * f, c, H, W)
    x = F.silu(_conv(sd, "conv_in", x))
    for i in range(6):
        x = F.silu(_conv(sd, f"blocks.{i}", x, stride=2 if i % 2 == 1 else 1))
    x = _conv(sd, "conv_out", x)
    return x.reshape(b, f, x.shape[1], x.shape[2], x.shape[3]).permute(0, 2, 1, 3, 4)


# =====================================================================================================
# VAE (diffusers AutoencoderKL, sd-vae-ft-mse layout) [3P]; call sites pipeline :113-126, :430, :438
# =====================================================================================================
def _vae_attn(sd: SD, p: str, x: torch.Tensor, groups: int) -> torch.Tensor:
    """UNetMidBlock2D attention: 1 head of dim C, GroupNorm(eps 1e-6) on the input, biased q/k/v, residual."""
    n, c, h, w = x.shape
    t = x.view(n, c, h * w).transpose(1, 2)
    t = F.group_norm(t.transpose(1, 2), groups, sd[p + ".group_norm.weight"], sd[p + ".group_norm.bias"], 1e-6).transpose(1, 2)
    o = attention(sd, p, t, None, heads=1)
    return o.transpose(-1, -2).reshape(n, c, h, w) + x


def _vae_mid(sd: SD, p: str, x: torch.Tensor, groups: int) -> torch.Tensor:
    x = resnet_block(sd, p + ".resnets.0", x, None, groups, 1e-6)
    x = _vae_attn(sd, p + ".attentions.0", x, groups)
    return resnet_block(sd, p + ".resnets.1", x, None, groups, 1e-6)


def vae_encode_mean(sd: SD, x: torch.Tensor, cfg_: VAEConfig = VAEConfig()) -> torch.Tensor:
    """AutoencoderKL.encode(x).latent_dist.mean. Downsample = F.pad(0,1,0,1) + 3x3 stride-2 conv, padding 0."""
    g = cfg_.norm_num_groups
    nb = len(cfg_.block_out_channels)
    h = _conv(sd, "encoder.conv_in", x)
    for i in range(nb):
        for j in range(cfg_.layers_per_block):
            h = resnet_block(sd, f"encoder.down_blocks.{i}.resnets.{j}", h, None, g, 1e-6)
        if i < nb - 1:
            h = F.pad(h, (0, 1, 0, 1))
            h = _conv(sd, f"encoder.down_blocks.{i}.downsamplers.0.conv", h, stride=2, padding=0)
    h = _vae_mid(sd, "encoder.mid_block", h, g)
    h = _conv(sd, "encoder.conv_out", F.silu(_gn(sd, "encoder.conv_norm_out", h, g, 1e-6)))
    moments = _conv(sd, "quant_conv", h, padding=0)
    return moments[:, : cfg_.latent_channels]


def vae_decode(sd: SD, z: torch.Tensor, cfg_: VAEConfig = VAEConfig()) -> torch.Tensor:
    """AutoencoderKL.decode(z).sample: post_quant 1x1, conv_in, mid, 4 up blocks (3 resnets, nearest x2 + conv on
    the first 3), GN-SiLU-conv_out."""
    g = cfg_.norm_num_groups
    nb = len(cfg_.block_out_channels)
    h = _conv(sd, "post_quant_conv", z, padding=0)
    h = _conv(sd, "decoder.conv_in", h)
    h = _vae_mid(sd, "decoder.mid_block", h, g)
    for i in range(nb):
        for j in range(cfg_.layers_per_block + 1):
            h = resnet_block(sd, f"decoder.up_blocks.{i}.resnets.{j}", h, None, g, 1e-6)
        if i < nb - 1:
            h = F.interpolate(h, scale_factor=2.0, mode="nearest")
            h = _conv(sd, f"decoder.up_blocks.{i}.upsamplers.0.conv", h)
    return _conv(sd, "decoder.conv_out", F.silu(_gn(sd, "decoder.conv_norm_out", h, g, 1e-6)))


# =====================================================================================================
# DDIM scheduler [3P] with the reference's kwargs (configs/inference/inference_v2.yaml:24-33)
# =====================================================================================================
class DDIM:
    """DDIMScheduler(beta 0.00085->0.012 scaled_linear, v_prediction, rescale_betas_zero_snr, trailing spacing,
    steps_offset 1, clip_sample False, set_alpha_to_one True). Call sites: pipeline :373-374, :519-521, :551-553."""

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.00085, beta_end: float = 0.012):
        betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
        # rescale_zero_terminal_snr
        alphas_bar_sqrt = torch.cumprod(1.0 - betas, dim=0).sqrt()
        a0, aT = alphas_bar_sqrt[0].clone(), alphas_bar_sqrt[-1].clone()
        alphas_bar_sqrt = (alphas_bar_sqrt - aT) * (a0 / (a0 - aT))
        alphas_bar = alphas_bar_sqrt ** 2
        alphas = torch.cat([alphas_bar[0:1], alphas_bar[1:] / alphas_bar[:-1]])
        self.betas = 1 - alphas
        self.alphas_cumprod = torch.cumprod(1.0 - self.betas, dim=0)
        self.final_alpha_cumprod = torch.tensor(1.0)
        self.num_train_timesteps = num_train_timesteps
        self.init_noise_sigma = 1.0
        self.num_inference_steps = None
        self.timesteps = None

    def set_timesteps(self, n: int) -> np.ndarray:
        self.num_inference_steps = n
        ts = np.round(np.arange(self.num_train_timesteps, 0, -self.num_train_timesteps / n)).astype(np.int64) - 1
        self.timesteps = ts
        return ts

    def coefficients(self, t: int) -> Tuple[float, float, float, float]:
        """(sqrt(abar_t), sqrt(1-abar_t), sqrt(abar_prev), sqrt(1-abar_prev)) with prev_t = t - 1000 // N."""
        prev_t = t - self.num_train_timesteps // self.num_inference_steps
        a_t = self.alphas_cumprod[t]
        a_p = self.alphas_cumprod[prev_t] if prev_t >= 0 else self.final_alpha_cumprod
        return (float(a_t ** 0.5), float((1 - a_t) ** 0.5), float(a_p ** 0.5), float((1 - a_p) ** 0.5))

    def step(self, model_output: torch.Tensor, t: int, sample: torch.Tensor) -> torch.Tensor:
        prev_t = t - self.num_train_timesteps // self.num_inference_steps
        a_t = self.alphas_cumprod[t]
        a_p = self.alphas_cumprod[prev_t] if prev_t >= 0 else self.final_alpha_cumprod
        b_t = 1 - a_t
        x0 = (a_t ** 0.5) * sample - (b_t ** 0.5) * model_output  # v_prediction
        eps = (a_t ** 0.5) * model_output + (b_t ** 0.5) * sample
        direction = (1 - a_p) ** 0.5 * eps  # eta = 0
        return a_p ** 0.5 * x0 + direction


# =====================================================================================================
# context windows (src/pipelines/context.py:7-42) — integer logic, must be bit-exact
# =====================================================================================================
def ordered_halving(val: int) -> float:
    return int(f"{val:064b}"[::-1], 2) / (1 << 64)


def uniform_windows(step: int, num_frames: int, context_size: int = 24, context_stride: int = 1,
                    context_overlap: int = 4, closed_loop: bool = True) -> List[List[int]]:
    if num_frames <= context_size:
        return [list(range(num_frames))]
    out = []
    context_stride = min(context_stride, int(np.ceil(np.log2(num_frames / context_size))) + 1)
    for context_step in 1 << np.arange(context_stride):
        pad = int(round(num_frames * ordered_halving(step)))
        for j in range(int(ordered_halving(step) * context_step) + pad,
                       num_frames + pad + (0 if closed_loop else -context_overlap),
                       (context_size * context_step - context_overlap)):
            out.append([e % num_frames for e in range(j, j + context_size * context_step, context_step)])
    return out


# =====================================================================================================
# whole sampler (Pose2VideoPipeline.__call__, pipeline :338-578) on tensors
# =====================================================================================================
@dataclass
class Weights:
    denoising_unet: SD
    reference_unet: SD
    pose_guider: SD
    vae: SD
    unet_cfg: UNetConfig = field(default_factory=UNetConfig)
    vae_cfg: VAEConfig = field(default_factory=VAEConfig)


def sample_clip(W: Weights, ref_image: torch.Tensor, pose: torch.Tensor, backgrounds: torch.Tensor,
                image_embeds: torch.Tensor, init_latents: torch.Tensor, num_inference_steps: int,
                guidance_scale: float, context_frames: int = 24, context_overlap: int = 4,
                timing: Optional[dict] = None, decode: bool = True) -> Dict[str, torch.Tensor]:
    """Tensor-level restatement of the pipeline after its PIL pre-processing:
      ref_image [1,3,H,W] in [-1,1]; pose [1,3,F,H,W] in [0,1]; backgrounds [F,3,H,W] in [-1,1];
      image_embeds [1,768] (CLIP output); init_latents [1,4,F,h,w] (randn_tensor result)."""
    import time
    cfg_ = W.unet_cfg
    do_cfg = guidance_scale > 1.0
    dtype = init_latents.dtype
    sched = DDIM()
    timesteps = sched.set_timesteps(num_inference_steps)
    ehs = image_embeds.unsqueeze(1)
    if do_cfg:
        ehs = torch.cat([torch.zeros_like(ehs), ehs], dim=0)  # :385-391
    latents = init_latents * sched.init_noise_sigma
    Fr = latents.shape[2]
    tm = timing if timing is not None else {}

    t0 = time.perf_counter()
    ref_latents = vae_encode_mean(W.vae, ref_image, W.vae_cfg) * 0.18215  # :424-431
    bk = torch.stack([vae_encode_mean(W.vae, backgrounds[i:i + 1], W.vae_cfg)[0] * 0.18215 for i in range(Fr)], dim=1)
    vid_bk = bk.unsqueeze(0).to(dtype)  # [1,4,F,h,w]  :434-443
    tm["vae_encode_s"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    pose_fea = pose_guider(W.pose_guider, pose)  # :446-457
    tm["pose_s"] = time.perf_counter() - t0

    banks = None
    tm["unet_s"] = 0.0
    for i, t in enumerate(timesteps):
        t = int(t)
        if i == 0:  # :480-490
            t0 = time.perf_counter()
            rl = ref_latents.repeat(2 if do_cfg else 1, 1, 1, 1)
            banks = reference_unet_banks(W.reference_unet, rl, ehs, cfg_)
            tm["ref_unet_s"] = time.perf_counter() - t0
        noise_pred = torch.zeros((latents.shape[0] * (2 if do_cfg else 1), *latents.shape[1:]), dtype=dtype, device=latents.device)
        counter = torch.zeros((1, 1, Fr, 1, 1), dtype=dtype, device=latents.device)
        t0 = time.perf_counter()
        for c in uniform_windows(0, Fr, context_frames, 1, context_overlap):  # :492-500 (step arg is always 0)
            rep = 2 if do_cfg else 1
            lat_in = latents[:, :, c].repeat(rep, 1, 1, 1, 1)
            bk_in = vid_bk[:, :, c].repeat(rep, 1, 1, 1, 1)
            x = torch.cat([lat_in, bk_in], dim=1)
            pose_in = pose_fea[:, :, c].repeat(rep, 1, 1, 1, 1)
            pred = denoising_unet(W.denoising_unet, x, t, ehs[: x.shape[0]], pose_in, banks, cfg_, cfg=do_cfg)
            noise_pred[:, :, c] = noise_pred[:, :, c] + pred  # :540-542
            counter[:, :, c] = counter[:, :, c] + 1
        tm["unet_s"] += time.perf_counter() - t0
        if do_cfg:
            u, cnd = (noise_pred / counter).chunk(2)
            noise_pred = u + guidance_scale * (cnd - u)
        latents = sched.step(noise_pred, t, latents).to(dtype)  # :551-553
    out = {"latents": latents}
    if decode:
        t0 = time.perf_counter()
        z = (1 / 0.18215 * latents)[0].permute(1, 0, 2, 3)  # "(b f) c h w"
        frames = torch.cat([vae_decode(W.vae, z[i:i + 1], W.vae_cfg) for i in range(Fr)])  # :113-121
        video = frames.permute(1, 0, 2, 3).unsqueeze(0)
        out["videos"] = (video / 2 + 0.5).clamp(0, 1).float().cpu()
        tm["vae_decode_s"] = time.perf_counter() - t0
    return out


# =====================================================================================================
# seeded random weights with the reference's state-dict key schema (SURVEY.md §8b)
# =====================================================================================================
def _rand(gen: torch.Generator, shape, std: float) -> torch.Tensor:
    return torch.randn(shape, generator=gen, dtype=torch.float32) * std


class _Maker:
    def __init__(self, seed: int):
        self.gen = torch.Generator().manual_seed(seed)
        self.sd: SD = {}

    def conv(self, p, cin, cout, k=3, bias=True, gain=1.0):
        self.sd[p + ".weight"] = _rand(self.gen, (cout, cin, k, k), gain / math.sqrt(cin * k * k))
        if bias:
            self.sd[p + ".bias"] = _rand(self.gen, (cout,), 0.02)

    def lin(self, p, cin, cout, bias=True, gain=1.0):
        self.sd[p + ".weight"] = _rand(self.gen, (cout, cin), gain / math.sqrt(cin))
        if bias:
            self.sd[p + ".bias"] = _rand(self.gen, (cout,), 0.02)

    def norm(self, p, c):
        self.sd[p + ".weight"] = 1.0 + _rand(self.gen, (c,), 0.1)
        self.sd[p + ".bias"] = _rand(self.gen, (c,), 0.05)

    def resnet(self, p, cin, cout, temb=None):
        self.norm(p + ".norm1", cin)
        self.conv(p + ".conv1", cin, cout)
        if temb:
            self.lin(p + ".time_emb_proj", temb, cout)
        self.norm(p + ".norm2", cout)
        self.conv(p + ".conv2", cout, cout, gain=0.5)
        if cin != cout:
            self.conv(p + ".conv_shortcut", cin, cout, k=1)

    def attn(self, p, c, ctx=None, bias=False):
        self.lin(p + ".to_q", c, c, bias=bias)
        self.lin(p + ".to_k", ctx or c, c, bias=bias)
        self.lin(p + ".to_v", ctx or c, c, bias=bias)
        self.lin(p + ".to_out.0", c, c, gain=0.5)

    def ff(self, p, c):
        self.lin(p + ".net.0.proj", c, 8 * c)
        self.lin(p + ".net.2", 4 * c, c, gain=0.5)

    def spatial_transformer(self, p, c, ctx):
        self.norm(p + ".norm", c)
        self.conv(p + ".proj_in", c, c, k=1)
        b = p + ".transformer_blocks.0"
        self.norm(b + ".norm1", c)
        self.attn(b + ".attn1", c)
        self.norm(b + ".norm2", c)
        self.attn(b + ".attn2", c, ctx=ctx)
        self.norm(b + ".norm3", c)
        self.ff(b + ".ff", c)
        self.conv(p + ".proj_out", c, c, k=1, gain=0.5)

    def motion(self, p, c, max_len):
        t = p + ".temporal_transformer"
        self.norm(t + ".norm", c)
        self.lin(t + ".proj_in", c, c)
        b = t + ".transformer_blocks.0"
        for i in range(2):
            self.attn(f"{b}.attention_blocks.{i}", c)
            self.sd[f"{b}.attention_blocks.{i}.pos_encoder.pe"] = positional_encoding(c, max_len)
            self.norm(f"{b}.norms.{i}", c)
        self.ff(b + ".ff", c)
        self.norm(b + ".ff_norm", c)
        # zero-initialised in the reference (motion_module.py:72-75); re-randomised so the path is live (SURVEY §4)
        self.lin(t + ".proj_out", c, c, gain=0.5)


def positional_encoding(d_model: int, max_len: int) -> torch.Tensor:
    """PositionalEncoding buffer, src/models/motion_module.py:264-275."""
    position = torch.arange(max_len).unsqueeze(1)
    div_term = torch.exp(torch.arange(0, d_model, 2) * (-math.log(10000.0) / d_model))
    pe = torch.zeros(1, max_len, d_model)
    pe[0, :, 0::2] = torch.sin(position * div_term)
    pe[0, :, 1::2] = torch.cos(position * div_term)
    return pe


def make_unet_state_dict(cfg_: UNetConfig, seed: int, motion: bool, in_channels: int, out_head: bool) -> SD:
    m = _Maker(seed)
    ch = cfg_.block_out_channels
    temb = cfg_.time_embed_dim
    nb = len(ch)
    m.conv("conv_in", in_channels, ch[0])
    m.lin("time_embedding.linear_1", ch[0], temb)
    m.lin("time_embedding.linear_2", temb, temb)
    out_c = ch[0]
    for i in range(nb):
        in_c, out_c = out_c, ch[i]
        for j in range(cfg_.layers_per_block):
            m.resnet(f"down_blocks.{i}.resnets.{j}", in_c if j == 0 else out_c, out_c, temb)
            if i < nb - 1:
                m.spatial_transformer(f"down_blocks.{i}.attentions.{j}", out_c, cfg_.cross_attention_dim)
            if motion:
                m.motion(f"down_blocks.{i}.motion_modules.{j}", out_c, cfg_.motion_max_len)
        if i < nb - 1:
            m.conv(f"down_blocks.{i}.downsamplers.0.conv", out_c, out_c)
    m.resnet("mid_block.resnets.0", ch[-1], ch[-1], temb)
    m.spatial_transformer("mid_block.attentions.0", ch[-1], cfg_.cross_attention_dim)
    if motion:
        m.motion("mid_block.motion_modules.0", ch[-1], cfg_.motion_max_len)
    m.resnet("mid_block.resnets.1", ch[-1], ch[-1], temb)
    rev = list(reversed(ch))
    out_c = rev[0]
    for i in range(nb):
        prev_out = out_c
        out_c = rev[i]
        in_c = rev[min(i + 1, nb - 1)]
        for j in range(cfg_.layers_per_block + 1):
            skip_c = in_c if j == cfg_.layers_per_block else out_c
            res_in = prev_out if j == 0 else out_c
            m.resnet(f"up_blocks.{i}.resnets.{j}", res_in + skip_c, out_c, temb)
            if i > 0:
                m.spatial_transformer(f"up_blocks.{i}.attentions.{j}", out_c, cfg_.cross_attention_dim)
            if motion:
                m.motion(f"up_blocks.{i}.motion_modules.{j}", out_c, cfg_.motion_max_len)
        if i < nb - 1:
            m.conv(f"up_blocks.{i}.upsamplers.0.conv", out_c, out_c)
    if out_head:
        m.norm("conv_norm_out", ch[0])
        m.conv("conv_out", ch[0], cfg_.out_channels, gain=0.5)
    return m.sd


def make_denoising_unet_sd(cfg_: UNetConfig = UNetConfig(), seed: int = 1) -> SD:
    return make_unet_state_dict(cfg_, seed, motion=True, in_channels=cfg_.in_channels, out_head=True)


def make_reference_unet_sd(cfg_: UNetConfig = UNetConfig(), seed: int = 2) -> SD:
    return make_unet_state_dict(cfg_, seed, motion=False, in_channels=4, out_head=False)


def make_pose_guider_sd(seed: int = 3, out_channels: int = 320, channels: Sequence[int] = POSE_CHANNELS) -> SD:
    m = _Maker(seed)
    m.conv("conv_in", 3, channels[0], gain=1.4)
    k = 0
    for i in range(len(channels) - 1):
        m.conv(f"blocks.{k}", channels[i], channels[i], gain=1.4)
        m.conv(f"blocks.{k + 1}", channels[i], channels[i + 1], gain=1.4)
        k += 2
    m.conv("conv_out", channels[-1], out_channels, gain=0.5)  # zero-init in the reference (pose_guider.py:38-45)
    return m.sd


def make_vae_sd(cfg_: VAEConfig = VAEConfig(), seed: int = 4) -> SD:
    m = _Maker(seed)
    ch = cfg_.block_out_channels
    nb = len(ch)
    m.conv("encoder.conv_in", cfg_.in_channels, ch[0])
    out_c = ch[0]
    for i in range(nb):
        in_c, out_c = out_c, ch[i]
        for j in range(cfg_.layers_per_block):
            m.resnet(f"encoder.down_blocks.{i}.resnets.{j}", in_c if j == 0 else out_c, out_c)
        if i < nb - 1:
            m.conv(f"encoder.down_blocks.{i}.downsamplers.0.conv", out_c, out_c)
    for side in ("encoder", "decoder"):
        m.resnet(f"{side}.mid_block.resnets.0", ch[-1], ch[-1])
        a = f"{side}.mid_block.attentions.0"
        m.norm(a + ".group_norm", ch[-1])
        m.attn(a, ch[-1], bias=True)
        m.resnet(f"{side}.mid_block.resnets.1", ch[-1], ch[-1])
    m.norm("encoder.conv_norm_out", ch[-1])
    m.conv("encoder.conv_out", ch[-1], 2 * cfg_.latent_channels)
    m.conv("quant_conv", 2 * cfg_.latent_channels, 2 * cfg_.latent_channels, k=1)
    m.conv("post_quant_conv", cfg_.latent_channels, cfg_.latent_channels, k=1)
    rev = list(reversed(ch))
    m.conv("decoder.conv_in", cfg_.latent_channels, rev[0])
    out_c = rev[0]
    for i in range(nb):
        in_c, out_c = out_c, rev[i]
        for j in range(cfg_.layers_per_block + 1):
            m.resnet(f"decoder.up_blocks.{i}.resnets.{j}", in_c if j == 0 else out_c, out_c)
        if i < nb - 1:
            m.conv(f"decoder.up_blocks.{i}.upsamplers.0.conv", out_c, out_c)
    m.norm("decoder.conv_norm_out", rev[-1])
    m.conv("decoder.conv_out", rev[-1], cfg_.out_channels, gain=0.5)
    return m.sd


def cast_sd(sd: SD, dtype: torch.dtype, device=None) -> SD:
    return {k: v.to(device=device, dtype=dtype) for k, v in sd.items()}
