"""The denoising UNet3D built with use_inflated_groupnorm=False, on top of oracle/torch_oracle.py (which is unchanged).
TEST INFRASTRUCTURE, NOT PRODUCT CODE.

With the flag off, every ResnetBlock3D builds norm1 / norm2 as a plain torch.nn.GroupNorm, and so does conv_norm_out
(src/models/resnet.py:155-163, 185-192; src/models/unet_3d_edit_bkfill.py:71, 236-247). On the [b, C, f, h, w] video
tensor its statistics cover every frame of a sample. The GroupNorms of Transformer3DModel and of the motion module stay
per frame (transformer_3d.py:115-124, motion_module.py:151-156); the reference UNet2D and the VAE do not change.

`denoising_unet` below is torch_oracle.denoising_unet with those three GroupNorms over the window. Inside
`window_groupnorm()`, torch_oracle.denoising_unet is this function, so torch_oracle.sample_clip and
scripts/oracle_any_size.py's cases (which call it) compute the non-inflated network; the two context managers nest.
"""
from __future__ import annotations

import contextlib
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from oracle import torch_oracle as O

_RESNET_BLOCK = O.resnet_block
_DENOISING_UNET = O.denoising_unet


def group_norm_frames(sd: O.SD, p: str, x: torch.Tensor, groups: int, eps: float, frames: int) -> torch.Tensor:
    """nn.GroupNorm of the [b, C, f, H, W] video tensor whose frames are x's [(b f), C, H, W] images."""
    n, c, h, w = x.shape
    v = x.reshape(n // frames, frames, c, h, w).transpose(1, 2)
    return O._gn(sd, p, v, groups, eps).transpose(1, 2).reshape(n, c, h, w)


def resnet_block(sd: O.SD, p: str, x: torch.Tensor, temb: Optional[torch.Tensor], groups: int, eps: float,
                 frames: int, output_scale_factor: float = 1.0) -> torch.Tensor:
    """torch_oracle.resnet_block (ResnetBlock3D.forward, resnet.py:217-247) with norm1 / norm2 over `frames` frames."""
    h = F.silu(group_norm_frames(sd, p + ".norm1", x, groups, eps, frames))
    h = O._conv(sd, p + ".conv1", h)
    if temb is not None:
        h = h + O._lin(sd, p + ".time_emb_proj", F.silu(temb))[:, :, None, None]
    h = F.silu(group_norm_frames(sd, p + ".norm2", h, groups, eps, frames))
    h = O._conv(sd, p + ".conv2", h)
    if (p + ".conv_shortcut.weight") in sd:
        x = O._conv(sd, p + ".conv_shortcut", x, padding=0)
    return (x + h) / output_scale_factor


def denoising_unet(sd: O.SD, sample: torch.Tensor, timestep, ehs: torch.Tensor, pose_fea: Optional[torch.Tensor],
                   banks: Dict[str, torch.Tensor], cfg_: O.UNetConfig, cfg: bool = True) -> torch.Tensor:
    """UNet3DConditionModel(use_inflated_groupnorm=False).forward: torch_oracle.denoising_unet with the ResBlocks'
    norm1 / norm2 and conv_norm_out over all f frames of each sample. sample [b, 8, f, h, w] -> [b, 4, f, h, w]."""
    b, c, f, h, w = sample.shape
    t = timestep if torch.is_tensor(timestep) else torch.tensor([timestep], dtype=torch.int64, device=sample.device)
    t = t.reshape(-1).to(sample.device).expand(b)
    temb = O.timestep_embedding(sd, t, cfg_.block_out_channels[0], sample.dtype)
    temb_n = temb.repeat_interleave(f, dim=0)
    ehs_n = ehs.repeat_interleave(f, dim=0)

    def to4(x5):
        return x5.permute(0, 2, 1, 3, 4).reshape(b * f, x5.shape[1], x5.shape[3], x5.shape[4])

    x = O._conv(sd, "conv_in", to4(sample))
    if pose_fea is not None:
        x = x + to4(pose_fea)

    def xf(p: str, xx: torch.Tensor) -> torch.Tensor:
        bank = [banks[p]] if p in banks else []
        return O.spatial_transformer(sd, p, xx, ehs_n, cfg_,
                                     lambda bp, tok: O.transformer_block_read(sd, bp, tok, ehs_n, cfg_.heads, bank, f, cfg))

    # the UNet body (torch_oracle's, or scripts/oracle_any_size.py's when it is swapped in) looks resnet_block up in
    # torch_oracle at call time: for this body only, it is the window block
    O.resnet_block = lambda sd_, p, xx, te, g, eps: resnet_block(sd_, p, xx, te, g, eps, f)
    try:
        x = O._unet_body(sd, x, temb_n, cfg_, xf, lambda p, xx: O.motion_module(sd, p, xx, f, cfg_))
    finally:
        O.resnet_block = _RESNET_BLOCK
    x = F.silu(group_norm_frames(sd, "conv_norm_out", x, cfg_.norm_num_groups, cfg_.norm_eps, f))  # :569-571
    x = O._conv(sd, "conv_out", x)
    return x.reshape(b, f, x.shape[1], h, w).permute(0, 2, 1, 3, 4)


@contextlib.contextmanager
def window_groupnorm():
    """Within the block, torch_oracle.denoising_unet (and sample_clip, which calls it) is the non-inflated network."""
    O.denoising_unet = denoising_unet
    try:
        yield
    finally:
        O.denoising_unet = _DENOISING_UNET
