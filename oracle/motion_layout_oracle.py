"""The denoising UNet3D with other motion-module layouts, on top of oracle/torch_oracle.py (which is unchanged).
TEST INFRASTRUCTURE, NOT PRODUCT CODE.

torch_oracle builds and runs configs/inference/inference_v2.yaml's layout: a motion module after every layer of every
block, each one TemporalTransformerBlock of two Temporal_Self attentions with positional encoding. The reference builds
others from the same config keys:

  * motion_module_resolutions / motion_module_decoder_only / motion_module_mid_block choose the blocks that get modules
    (src/models/unet_3d_edit_bkfill.py:145-230: down level i is resolution 2^i, up level i is 2^(3 - i));
  * num_transformer_block stacks TemporalTransformerBlocks between proj_in and proj_out (motion_module.py:119-144,
    170-176);
  * attention_block_types gives one norms.i + attention_blocks.i per entry, each followed by its residual
    (motion_module.py:212-261);
  * temporal_position_encoding adds pos_encoder.pe before each attention, or not (motion_module.py:320-329);
  * num_attention_heads sets the heads of the temporal attention, independently of the spatial ones (:58-61).

Inside `motion_layout(layout)`, torch_oracle.motion_module is the module of that layout (identity where the layout has
none), so torch_oracle.denoising_unet, window_gn_oracle.denoising_unet and sample_clip compute the layout's network.
"""
from __future__ import annotations

import contextlib
from dataclasses import dataclass
from typing import Tuple

import torch

from oracle import torch_oracle as O

_MOTION_MODULE = O.motion_module


@dataclass(frozen=True)
class Layout:
    resolutions: Tuple[int, ...] = (1, 2, 4, 8)
    mid_block: bool = True
    decoder_only: bool = False
    blocks: int = 1
    attn_blocks: int = 2
    pe: bool = True
    max_len: int = 32
    heads: int = 8

    def has_module(self, path: str) -> bool:
        """Whether the motion module at `path` (e.g. "up_blocks.2.motion_modules.1") exists: the reference's four
        levels, down resolution 2^i, up resolution 2^(3 - i), the mid block by its own flag."""
        parts = path.split(".")
        if parts[0] == "mid_block":
            return self.mid_block
        i = int(parts[1])
        if parts[0] == "down_blocks":
            return not self.decoder_only and 2 ** i in self.resolutions
        return 2 ** (3 - i) in self.resolutions


def motion_module(sd: O.SD, p: str, x: torch.Tensor, video_length: int, lay: Layout, fp8: bool = False) -> torch.Tensor:
    """VanillaTemporalModule -> TemporalTransformer3DModel with `lay.blocks` TemporalTransformerBlocks of
    `lay.attn_blocks` Temporal_Self attentions each (motion_module.py:146-184, 238-261, 353-390). x: [(b f), C, H, W].
    fp8: every q|k|v (after LN (+ PE)) and GEGLU projection in FP8, emulated as oracle/fp8_oracle.py does."""
    attention, feed_forward = O.attention, O.feed_forward
    if fp8:
        from oracle import fp8_oracle as F8
        attention = lambda sd_, p_, seq, ctx, heads: F8._attention8(sd_, p_, F8.fake_quant(seq), ctx, heads)
        feed_forward = F8._feed_forward8
    tp = p + ".temporal_transformer"
    n, c, h, w = x.shape
    res = x
    t = O._tokens(O._gn(sd, tp + ".norm", x, 32, 1e-6))
    t = O._lin(sd, tp + ".proj_in", t)
    f = video_length
    b = n // f
    d = h * w
    for k in range(lay.blocks):
        bp = f"{tp}.transformer_blocks.{k}"
        for i in range(lay.attn_blocks):
            nh = O._ln(sd, f"{bp}.norms.{i}", t)
            seq = nh.reshape(b, f, d, c).permute(0, 2, 1, 3).reshape(b * d, f, c)  # "(b f) d c -> (b d) f c"
            if lay.pe:
                seq = seq + sd[f"{bp}.attention_blocks.{i}.pos_encoder.pe"][:, :f].to(seq.dtype)
            o = attention(sd, f"{bp}.attention_blocks.{i}", seq, None, lay.heads)
            t = o.reshape(b, d, f, c).permute(0, 2, 1, 3).reshape(n, d, c) + t
        t = feed_forward(sd, bp + ".ff", O._ln(sd, bp + ".ff_norm", t)) + t
    t = O._lin(sd, tp + ".proj_out", t)
    return O._untokens(t, h, w) + res


def make_denoising_unet_sd(cfg_: O.UNetConfig, lay: Layout, seed: int) -> O.SD:
    """torch_oracle.make_denoising_unet_sd(cfg_, seed) with its motion modules replaced by `lay`'s, drawn from seed + 500
    in module order (the other weights are those of the inference_v2 state dict of the same seed)."""
    sd = {k: v for k, v in O.make_denoising_unet_sd(cfg_, seed=seed).items() if ".motion_modules." not in k}
    m = O._Maker(seed + 500)
    ch = list(cfg_.block_out_channels)
    nb = len(ch)
    paths = [(f"down_blocks.{i}.motion_modules.{j}", ch[i]) for i in range(nb) for j in range(cfg_.layers_per_block)]
    paths += [("mid_block.motion_modules.0", ch[-1])]
    paths += [(f"up_blocks.{i}.motion_modules.{j}", ch[nb - 1 - i]) for i in range(nb)
              for j in range(cfg_.layers_per_block + 1)]
    for p, c in paths:
        if not lay.has_module(p):
            continue
        t = p + ".temporal_transformer"
        m.norm(t + ".norm", c)
        m.lin(t + ".proj_in", c, c)
        for k in range(lay.blocks):
            b = f"{t}.transformer_blocks.{k}"
            for i in range(lay.attn_blocks):
                m.attn(f"{b}.attention_blocks.{i}", c)
                if lay.pe:
                    m.sd[f"{b}.attention_blocks.{i}.pos_encoder.pe"] = O.positional_encoding(c, lay.max_len)
                m.norm(f"{b}.norms.{i}", c)
            m.ff(b + ".ff", c)
            m.norm(b + ".ff_norm", c)
        # zero-initialised in the reference (motion_module.py:72-75); random here so the module is live
        m.lin(t + ".proj_out", c, c, gain=0.5)
    sd.update(m.sd)
    return sd


@contextlib.contextmanager
def motion_layout(lay: Layout, fp8: bool = False):
    """Within the block, torch_oracle.motion_module runs `lay`'s module (fp8: with the FP8 projections), or passes x
    through where `lay` has none. Nests inside fp8_oracle.fp8_emulation(), which covers the spatial transformers."""
    saved = O.motion_module
    O.motion_module = lambda sd, p, x, f, cfg_: motion_module(sd, p, x, f, lay, fp8) if lay.has_module(p) else x
    try:
        yield
    finally:
        O.motion_module = saved
