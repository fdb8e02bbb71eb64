"""State-dict key schema of the reference's networks (diffusers key names, OIHW / [out, in] shapes).

The reference's modules are the source of truth (src/models/unet_3d_edit_bkfill.py:87-251, unet_3d_blocks.py,
transformer_3d.py:58-95, attention.py:321-360, motion_module.py:119-144, 212-236, 298-306, pose_guider.py:20-45,
unet_2d_condition.py); tests/test_host_cpu.py checks these enumerations key-for-key and shape-for-shape against
the oracle's generator, which oracle/pin_against_reference.py loads into the reference's own modules with
strict=True.
"""
from __future__ import annotations

from collections import OrderedDict
from dataclasses import dataclass
from typing import Dict, List, Sequence, Tuple

Shape = Tuple[int, ...]


class _S:
    def __init__(self):
        self.d: "OrderedDict[str, Shape]" = OrderedDict()

    def conv(self, p, cin, cout, k=3):
        self.d[p + ".weight"] = (cout, cin, k, k)
        self.d[p + ".bias"] = (cout,)

    def lin(self, p, cin, cout, bias=True):
        self.d[p + ".weight"] = (cout, cin)
        if bias:
            self.d[p + ".bias"] = (cout,)

    def norm(self, p, c):
        self.d[p + ".weight"] = (c,)
        self.d[p + ".bias"] = (c,)

    def resnet(self, p, cin, cout, temb):
        self.norm(p + ".norm1", cin)
        self.conv(p + ".conv1", cin, cout)
        if temb:
            self.lin(p + ".time_emb_proj", temb, cout)
        self.norm(p + ".norm2", cout)
        self.conv(p + ".conv2", cout, cout)
        if cin != cout:
            self.conv(p + ".conv_shortcut", cin, cout, k=1)

    def attn(self, p, c, ctx=None, bias=False):
        self.lin(p + ".to_q", c, c, bias)
        self.lin(p + ".to_k", ctx or c, c, bias)
        self.lin(p + ".to_v", ctx or c, c, bias)
        self.lin(p + ".to_out.0", c, c, True)

    def ff(self, p, c):
        self.lin(p + ".net.0.proj", c, 8 * c)
        self.lin(p + ".net.2", 4 * c, c)

    def xf(self, p, c, ctx):
        self.norm(p + ".norm", c)
        self.conv(p + ".proj_in", c, c, k=1)
        b = p + ".transformer_blocks.0"
        self.norm(b + ".norm1", c)
        self.attn(b + ".attn1", c)
        self.norm(b + ".norm2", c)
        self.attn(b + ".attn2", c, ctx=ctx)
        self.norm(b + ".norm3", c)
        self.ff(b + ".ff", c)
        self.conv(p + ".proj_out", c, c, k=1)

    def motion(self, p, c, lay: "MotionLayout"):
        t = p + ".temporal_transformer"
        self.norm(t + ".norm", c)
        self.lin(t + ".proj_in", c, c)
        for k in range(lay.blocks):
            b = f"{t}.transformer_blocks.{k}"
            for i in range(lay.attn_blocks):
                self.attn(f"{b}.attention_blocks.{i}", c)
                if lay.pe:
                    self.d[f"{b}.attention_blocks.{i}.pos_encoder.pe"] = (1, lay.max_len, c)
                self.norm(f"{b}.norms.{i}", c)
            self.ff(b + ".ff", c)
            self.norm(b + ".ff_norm", c)
        self.lin(t + ".proj_out", c, c)


@dataclass(frozen=True)
class MotionLayout:
    """Where the denoising UNet3D has a VanillaTemporalModule and what each one holds (unet_3d_edit_bkfill.py:145-230,
    motion_module.py:45-55, 98-144, 212-236). The defaults are configs/inference/inference_v2.yaml's."""
    resolutions: Tuple[int, ...] = (1, 2, 4, 8)  # motion_module_resolutions
    mid_block: bool = True                        # motion_module_mid_block
    decoder_only: bool = False                    # motion_module_decoder_only
    blocks: int = 1                               # num_transformer_block
    attn_blocks: int = 2                          # len(attention_block_types), all "Temporal_Self"
    pe: bool = True                               # temporal_position_encoding
    max_len: int = 32                             # temporal_position_encoding_max_len
    heads: int = 8                                # num_attention_heads

    def placed(self, path: str, levels: int) -> bool:
        """Whether the block at `path` ("down_blocks.i", "mid_block" or "up_blocks.i") has motion modules. Down level i
        is resolution 2^i, up level i is 2^(3 - i) whatever the number of levels, as the reference computes them
        (unet_3d_edit_bkfill.py:124, 188)."""
        if path == "mid_block":
            return self.mid_block
        kind, i = path.split(".")
        if kind == "down_blocks":
            return not self.decoder_only and 2 ** int(i) in self.resolutions
        return 2 ** (3 - int(i)) in self.resolutions

    def levels(self, levels: int) -> List[int]:
        """The UNet levels (0 = finest) at which some block has motion modules."""
        return [lv for lv in range(levels) if self.placed(f"down_blocks.{lv}", levels)
                or self.placed(f"up_blocks.{levels - 1 - lv}", levels) or (lv == levels - 1 and self.mid_block)]

    def head_widths(self, block_out_channels: Sequence[int]) -> Dict[int, float]:
        """{module width: channels per temporal-attention head} over the levels that have motion modules"""
        ch = list(block_out_channels)
        return {ch[lv]: ch[lv] / self.heads for lv in self.levels(len(ch))}


def unet_schema(block_out_channels: Sequence[int] = (320, 640, 1280, 1280), layers_per_block: int = 2,
                cross_attention_dim: int = 768, in_channels: int = 8, out_channels: int = 4, motion: bool = True,
                out_head: bool = True, motion_layout: MotionLayout = MotionLayout()) -> Dict[str, Shape]:
    """motion: the denoising UNet3D, with motion modules where `motion_layout` places them; False: the UNet2D."""
    s = _S()
    lay = motion_layout
    ch = list(block_out_channels)
    nb = len(ch)
    temb = ch[0] * 4
    s.conv("conv_in", in_channels, ch[0])
    s.lin("time_embedding.linear_1", ch[0], temb)
    s.lin("time_embedding.linear_2", temb, temb)
    out_c = ch[0]
    for i in range(nb):
        in_c, out_c = out_c, ch[i]
        for j in range(layers_per_block):
            s.resnet(f"down_blocks.{i}.resnets.{j}", in_c if j == 0 else out_c, out_c, temb)
            if i < nb - 1:
                s.xf(f"down_blocks.{i}.attentions.{j}", out_c, cross_attention_dim)
            if motion and lay.placed(f"down_blocks.{i}", nb):
                s.motion(f"down_blocks.{i}.motion_modules.{j}", out_c, lay)
        if i < nb - 1:
            s.conv(f"down_blocks.{i}.downsamplers.0.conv", out_c, out_c)
    s.resnet("mid_block.resnets.0", ch[-1], ch[-1], temb)
    s.xf("mid_block.attentions.0", ch[-1], cross_attention_dim)
    if motion and lay.placed("mid_block", nb):
        s.motion("mid_block.motion_modules.0", ch[-1], lay)
    s.resnet("mid_block.resnets.1", ch[-1], ch[-1], temb)
    rev = ch[::-1]
    out_c = rev[0]
    for i in range(nb):
        prev_out, out_c = out_c, rev[i]
        in_c = rev[min(i + 1, nb - 1)]
        for j in range(layers_per_block + 1):
            skip_c = in_c if j == layers_per_block else out_c
            res_in = prev_out if j == 0 else out_c
            s.resnet(f"up_blocks.{i}.resnets.{j}", res_in + skip_c, out_c, temb)
            if i > 0:
                s.xf(f"up_blocks.{i}.attentions.{j}", out_c, cross_attention_dim)
            if motion and lay.placed(f"up_blocks.{i}", nb):
                s.motion(f"up_blocks.{i}.motion_modules.{j}", out_c, lay)
        if i < nb - 1:
            s.conv(f"up_blocks.{i}.upsamplers.0.conv", out_c, out_c)
    if out_head:
        s.norm("conv_norm_out", ch[0])
        s.conv("conv_out", ch[0], out_channels)
    return s.d


def pose_guider_schema(conditioning_embedding_channels: int = 320, conditioning_channels: int = 3,
                       block_out_channels: Sequence[int] = (16, 32, 96, 256)) -> Dict[str, Shape]:
    s = _S()
    c = list(block_out_channels)
    s.conv("conv_in", conditioning_channels, c[0])
    k = 0
    for i in range(len(c) - 1):
        s.conv(f"blocks.{k}", c[i], c[i])
        s.conv(f"blocks.{k + 1}", c[i], c[i + 1])
        k += 2
    s.conv("conv_out", c[-1], conditioning_embedding_channels)
    return s.d


def vae_schema(block_out_channels: Sequence[int] = (128, 256, 512, 512), layers_per_block: int = 2,
               latent_channels: int = 4, in_channels: int = 3, out_channels: int = 3) -> Dict[str, Shape]:
    """diffusers AutoencoderKL (sd-vae-ft-mse layout) [3P]: the checkpoint the reference loads at run_animate.py:70-73."""
    s = _S()
    ch = list(block_out_channels)
    nb = len(ch)
    s.conv("encoder.conv_in", in_channels, ch[0])
    out_c = ch[0]
    for i in range(nb):
        in_c, out_c = out_c, ch[i]
        for j in range(layers_per_block):
            s.resnet(f"encoder.down_blocks.{i}.resnets.{j}", in_c if j == 0 else out_c, out_c, None)
        if i < nb - 1:
            s.conv(f"encoder.down_blocks.{i}.downsamplers.0.conv", out_c, out_c)
    for side in ("encoder", "decoder"):
        s.resnet(f"{side}.mid_block.resnets.0", ch[-1], ch[-1], None)
        a = f"{side}.mid_block.attentions.0"
        s.norm(a + ".group_norm", ch[-1])
        s.attn(a, ch[-1], bias=True)
        s.resnet(f"{side}.mid_block.resnets.1", ch[-1], ch[-1], None)
    s.norm("encoder.conv_norm_out", ch[-1])
    s.conv("encoder.conv_out", ch[-1], 2 * latent_channels)
    s.conv("quant_conv", 2 * latent_channels, 2 * latent_channels, k=1)
    s.conv("post_quant_conv", latent_channels, latent_channels, k=1)
    rev = ch[::-1]
    s.conv("decoder.conv_in", latent_channels, rev[0])
    out_c = rev[0]
    for i in range(nb):
        in_c, out_c = out_c, rev[i]
        for j in range(layers_per_block + 1):
            s.resnet(f"decoder.up_blocks.{i}.resnets.{j}", in_c if j == 0 else out_c, out_c, None)
        if i < nb - 1:
            s.conv(f"decoder.up_blocks.{i}.upsamplers.0.conv", out_c, out_c)
    s.norm("decoder.conv_norm_out", rev[-1])
    s.conv("decoder.conv_out", rev[-1], out_channels)
    return s.d
