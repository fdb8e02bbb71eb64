"""FP8 emulation of the denoising UNet3D's feed-forward output projections, on top of oracle/fp8_oracle.py and
oracle/torch_oracle.py (both unchanged). TEST INFRASTRUCTURE, NOT PRODUCT CODE.

With UNet3DConditionModel.enable_fp8(ff_out=True), the engine runs every FeedForward's ff.net.2 Linear(4C, C) - in the
spatial transformers and in the motion modules' transformer blocks - from e4m3 operands: the e4m3 GEGLU in front of it
writes its fp32 output as e4m3 with one scale per row and 128-column block, the weight has one scale per output channel.
Here the fp32 GEGLU output goes through mimo_b200.ops.quantize_e4m3_blocks (the host statement of the block rule) and the
weight through ops.quantize_e4m3_rows (the rule that packs the engine's weights), and the DEQUANTIZED values are
multiplied in fp32.

The FP8 feed-forward output only exists on top of the FP8 projections, so `fp8_ff_out_emulation()` replaces the feed-
forward of fp8_oracle's transformer block and motion module: it takes effect inside fp8_oracle.fp8_emulation(), entered
in either order. It composes with fp8_conv_oracle.fp8_conv_emulation() and window_gn_oracle.window_groupnorm() as those
do with fp8_emulation().
"""
from __future__ import annotations

import contextlib

import torch
import torch.nn.functional as F

from mimo_b200.ops import E4M3_BLOCK, quantize_e4m3_blocks
from oracle import fp8_oracle as F8
from oracle import torch_oracle as O


def fake_quant_blocks(y: torch.Tensor) -> torch.Tensor:
    """y [..., K] quantized per row and 128-column block and dequantized, in fp32"""
    y2 = y.float().reshape(-1, y.shape[-1])
    q, s = quantize_e4m3_blocks(y2, E4M3_BLOCK)
    deq = q.float().reshape(y2.shape[0], -1, E4M3_BLOCK) * s.t()[:, :, None]
    return deq.reshape(y.shape)


def _feed_forward8(sd: O.SD, p: str, x: torch.Tensor) -> torch.Tensor:
    """fp8_oracle's feed-forward (FP8 GEGLU) with ff.net.2 in FP8: block-quantized GEGLU output, per-channel weight"""
    h, gate = F8._lin8(sd, p + ".net.0.proj", F8.fake_quant(x)).chunk(2, dim=-1)
    return F8._lin8(sd, p + ".net.2", fake_quant_blocks(h * F.gelu(gate)))


@contextlib.contextmanager
def fp8_ff_out_emulation():
    """inside this context (and fp8_oracle.fp8_emulation()), the FP8 network's feed-forward output projections run in FP8"""
    saved = F8._feed_forward8
    F8._feed_forward8 = _feed_forward8
    try:
        yield
    finally:
        F8._feed_forward8 = saved
