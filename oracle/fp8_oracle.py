"""FP8 emulation of the denoising UNet3D's LN-fed projections, on top of oracle/torch_oracle.py (which is unchanged).
TEST INFRASTRUCTURE, NOT PRODUCT CODE.

With FP8 on (UNet3DConditionModel.enable_fp8), the engine runs four projections from e4m3 operands: the spatial
transformer's q|k|v after norm1 and GEGLU after norm3, and the motion module's two q|k|v after norm + PE and its GEGLU
after ff_norm. Here each of them takes the fp32 LN(+PE) output and the weight through the per-row rule (amax / 448,
round to nearest, saturate) and multiplies the DEQUANTIZED values in fp32. The rule is mimo_b200.ops.quantize_e4m3_rows,
the host statement that also packs the engine's weights; tests/test_fp8_cpu.py pins it to hand-computed e4m3 bytes and
tests/test_fp8_gpu.py pins the LayerNorm kernel to it. Everything else - including the bank keys / values, which the
engine projects in the model dtype - is torch_oracle's code.

Inside `fp8_emulation()`, torch_oracle.transformer_block_read and torch_oracle.motion_module are the functions below, so
torch_oracle.denoising_unet computes the FP8 network.
"""
from __future__ import annotations

import contextlib
from typing import Optional, Sequence

import torch
import torch.nn.functional as F

from mimo_b200.ops import quantize_e4m3_rows
from oracle import torch_oracle as O


def fake_quant(y: torch.Tensor) -> torch.Tensor:
    """y [..., K] quantized per row of K and dequantized, in fp32"""
    q, s = quantize_e4m3_rows(y.reshape(-1, y.shape[-1]))
    return (q.float() * s[:, None]).reshape(y.shape)


def _lin8(sd: O.SD, p: str, x: torch.Tensor) -> torch.Tensor:
    """Linear on fake-quantized activations (x is already dequantized) and a per-output-channel fake-quantized weight"""
    return F.linear(x, fake_quant(sd[p + ".weight"]), sd.get(p + ".bias"))


def _attention8(sd: O.SD, p: str, xq: torch.Tensor, extra_kv: Optional[torch.Tensor], heads: int) -> torch.Tensor:
    """torch_oracle.attention for self-attention whose q / k / v of the tokens xq come from e4m3; keys / values of the
    `extra_kv` tokens (the reference bank) are projected in full precision, as the engine does."""
    B = xq.shape[0]
    q, k, v = (_lin8(sd, f"{p}.to_{n}", xq) for n in "qkv")
    if extra_kv is not None:
        extra_kv = extra_kv.to(xq.dtype)  # banks may be stored in fp16 (reference_unet_banks); torch.cat promotes there
        k = torch.cat([k, O._lin(sd, p + ".to_k", extra_kv)], 1)
        v = torch.cat([v, O._lin(sd, p + ".to_v", extra_kv)], 1)
    d = q.shape[-1] // heads
    q, k, v = (t.view(B, -1, heads, d).transpose(1, 2) for t in (q, k, v))
    o = F.scaled_dot_product_attention(q, k, v, attn_mask=None, dropout_p=0.0, is_causal=False)
    return O._lin(sd, p + ".to_out.0", o.transpose(1, 2).reshape(B, -1, heads * d).to(q.dtype))


def _feed_forward8(sd: O.SD, p: str, x: torch.Tensor) -> torch.Tensor:
    h, gate = _lin8(sd, p + ".net.0.proj", fake_quant(x)).chunk(2, dim=-1)
    return O._lin(sd, p + ".net.2", h * F.gelu(gate))


def transformer_block_read(sd: O.SD, p: str, x: torch.Tensor, ehs: torch.Tensor, heads: int,
                           bank: Sequence[torch.Tensor], video_length: int, cfg: bool) -> torch.Tensor:
    """torch_oracle.transformer_block_read with the q|k|v of attn1 and the GEGLU projection in FP8"""
    nh = O._ln(sd, p + ".norm1", x)
    nq = fake_quant(nh)
    bank_fea = [d.unsqueeze(1).repeat(1, video_length, 1, 1).flatten(0, 1) for d in bank]
    extra = torch.cat(bank_fea, dim=1) if bank_fea else None
    hs_uc = _attention8(sd, p + ".attn1", nq, extra, heads) + x
    if cfg:
        hs_c = hs_uc.clone()
        half = x.shape[0] // 2
        hs_c[:half] = _attention8(sd, p + ".attn1", nq[:half], None, heads) + x[:half]
        x = hs_c
    else:
        x = hs_uc
    x = O.attention(sd, p + ".attn2", O._ln(sd, p + ".norm2", x), ehs, heads) + x
    return _feed_forward8(sd, p + ".ff", O._ln(sd, p + ".norm3", x)) + x


def motion_module(sd: O.SD, p: str, x: torch.Tensor, video_length: int, cfg_: O.UNetConfig) -> torch.Tensor:
    """torch_oracle.motion_module with both q|k|v projections (after LN + PE) and the GEGLU projection in FP8"""
    tp = p + ".temporal_transformer"
    n, c, h, w = x.shape
    res = x
    t = O._tokens(O._gn(sd, tp + ".norm", x, cfg_.motion_groups, 1e-6))
    t = O._lin(sd, tp + ".proj_in", t)
    bp = tp + ".transformer_blocks.0"
    f = video_length
    b = n // f
    d = h * w
    for i in range(2):
        nh = O._ln(sd, f"{bp}.norms.{i}", t)
        seq = nh.reshape(b, f, d, c).permute(0, 2, 1, 3).reshape(b * d, f, c)
        seq = seq + sd[f"{bp}.attention_blocks.{i}.pos_encoder.pe"][:, :f].to(seq.dtype)
        o = _attention8(sd, f"{bp}.attention_blocks.{i}", fake_quant(seq), None, cfg_.heads)
        t = o.reshape(b, d, f, c).permute(0, 2, 1, 3).reshape(n, d, c) + t
    t = _feed_forward8(sd, bp + ".ff", O._ln(sd, bp + ".ff_norm", t)) + t
    t = O._lin(sd, tp + ".proj_out", t)
    return O._untokens(t, h, w) + res


@contextlib.contextmanager
def fp8_emulation():
    """torch_oracle.denoising_unet (and everything calling it) computes the FP8 network inside this context"""
    saved = O.transformer_block_read, O.motion_module
    O.transformer_block_read, O.motion_module = transformer_block_read, motion_module
    try:
        yield
    finally:
        O.transformer_block_read, O.motion_module = saved
