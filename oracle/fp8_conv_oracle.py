"""FP8 emulation of the denoising UNet3D's ResnetBlock3D convolutions, on top of oracle/torch_oracle.py and
oracle/window_gn_oracle.py (both unchanged). TEST INFRASTRUCTURE, NOT PRODUCT CODE.

With UNet3DConditionModel.enable_fp8(convs=True), the engine runs every ResnetBlock3D conv1 and conv2 from e4m3
operands: the GroupNorm + SiLU in front of each writes e4m3 with one scale per frame (an upper bound on the frame's
amax, built from the per-group min / max of the GroupNorm input), the weights have one scale per output channel. Here
each of them takes the fp32 SiLU(GroupNorm) output through mimo_b200.ops.groupnorm_silu_e4m3_host, the host statement of
that rule, and the weight through ops.quantize_e4m3_rows (the rule that packs the engine's weights), and convolves the
DEQUANTIZED values in fp32. Everything else is the wrapped oracle's code.

Inside `fp8_conv_emulation()`, torch_oracle.denoising_unet computes the network with FP8 convolutions. It composes with
fp8_oracle.fp8_emulation() in either order; with window_gn_oracle.window_groupnorm() (statistics over the window) it is
entered inside that context, as the latter replaces torch_oracle.denoising_unet itself. The reference UNet and the VAE,
which the engine never runs in FP8, are not affected.
"""
from __future__ import annotations

import contextlib
from typing import Optional

import torch
import torch.nn.functional as F

from mimo_b200.ops import groupnorm_silu_e4m3_host, quantize_e4m3_rows
from oracle import torch_oracle as O
from oracle import window_gn_oracle as W


def gn_silu8(sd: O.SD, p: str, x: torch.Tensor, groups: int, eps: float, frames: int = 1) -> torch.Tensor:
    """SiLU(GroupNorm) of x [N, C, H, W] quantized per image (statistics per image, or per sample over `frames`
    consecutive images) and dequantized, in fp32"""
    n, c, h, w = x.shape
    xc = x.float().permute(0, 2, 3, 1).reshape(n, h * w, c)
    q, scale, _ = groupnorm_silu_e4m3_host(xc, sd[p + ".weight"], sd[p + ".bias"], groups, eps, frames)
    return (q.float() * scale[:, None, None]).reshape(n, h, w, c).permute(0, 3, 1, 2)


def conv8(sd: O.SD, p: str, x: torch.Tensor) -> torch.Tensor:
    """3x3 conv with the weight quantized per output channel (over all its 9 Cin taps, as the packed row) and
    dequantized"""
    wt = sd[p + ".weight"]
    q, s = quantize_e4m3_rows(wt.reshape(wt.shape[0], -1))
    return F.conv2d(x, (q.float() * s[:, None]).reshape(wt.shape), sd.get(p + ".bias"), padding=1)


def resnet_block(sd: O.SD, p: str, x: torch.Tensor, temb: Optional[torch.Tensor], groups: int, eps: float,
                 frames: int = 1, output_scale_factor: float = 1.0) -> torch.Tensor:
    """torch_oracle.resnet_block (or window_gn_oracle's, frames > 1) with conv1 and conv2 in FP8"""
    h = conv8(sd, p + ".conv1", gn_silu8(sd, p + ".norm1", x, groups, eps, frames))
    if temb is not None:
        h = h + O._lin(sd, p + ".time_emb_proj", F.silu(temb))[:, :, None, None]
    h = conv8(sd, p + ".conv2", gn_silu8(sd, p + ".norm2", h, groups, eps, frames))
    if (p + ".conv_shortcut.weight") in sd:
        x = O._conv(sd, p + ".conv_shortcut", x, padding=0)
    return (x + h) / output_scale_factor


@contextlib.contextmanager
def fp8_conv_emulation():
    """torch_oracle.denoising_unet (and everything calling it) computes the network with FP8 ResBlock convs inside this
    context; the ResBlocks of other networks keep their code"""
    inner = O.denoising_unet

    def denoising_unet(*args, **kw):
        saved = O.resnet_block, W.resnet_block
        O.resnet_block = lambda sd, p, x, temb, groups, eps, output_scale_factor=1.0: resnet_block(
            sd, p, x, temb, groups, eps, 1, output_scale_factor)
        W.resnet_block = resnet_block  # window_gn_oracle's body passes its frame count
        try:
            return inner(*args, **kw)
        finally:
            O.resnet_block, W.resnet_block = saved

    O.denoising_unet = denoising_unet
    try:
        yield
    finally:
        O.denoising_unet = inner
