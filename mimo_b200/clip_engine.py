"""CLIP ViT image encoder on the engine's kernels (SURVEY.md §8f rank 4).

The reference calls `self.image_encoder(clip_image).image_embeds` once per clip with a
transformers.CLIPVisionModelWithProjection (pipeline_pose2vid_long_edit_bkfill_roiclip.py:378-385; the module is built at
run_animate.py:92-94). The caller still passes that module; only its state dict and config are read here, and the
forward runs as C-ABI kernel calls: patch embedding as one GEMM over unfolded 14x14 patches, then per layer
LN -> fused q|k|v GEMM (+bias) -> flash attention (wgmma, d = 64) -> out-proj GEMM (+bias, +residual) -> LN ->
fc1 GEMM (+bias) -> quick-GELU -> fc2 GEMM (+bias, +residual); pooled = post-LN of the class token; projection GEMM.
"""
from __future__ import annotations

from typing import Dict

import torch

from . import lib as L
from . import ops


class CLIPVisionEngine:
    def __init__(self, sd: Dict[str, torch.Tensor], config, device, dtype=torch.float16):
        L.check(L.load().mimo_device_check(torch.device(device).index or 0), "mimo_device_check")
        if getattr(config, "hidden_act", "quick_gelu") != "quick_gelu":
            raise NotImplementedError(f"CLIP hidden_act={config.hidden_act!r}: the reference's image encoder "
                                      "(sd-image-variations CLIP ViT-L/14) uses quick_gelu")
        self.device, self.dtype = torch.device(device), dtype
        self.hidden, self.heads = config.hidden_size, config.num_attention_heads
        self.patch, self.image = config.patch_size, config.image_size
        self.eps = config.layer_norm_eps
        self.layers = config.num_hidden_layers
        if (self.hidden // self.heads) % 8 or self.hidden % 8:
            raise NotImplementedError("CLIP head dim must be a multiple of 8")
        t = lambda k: sd[k].detach().to(device=self.device, dtype=dtype).contiguous()
        p = "vision_model."
        wpe = t(p + "embeddings.patch_embedding.weight")  # [hidden, 3, P, P]
        k = wpe[0].numel()
        self.kpad = (k + 7) // 8 * 8
        self.w_patch = torch.zeros((self.hidden, self.kpad), device=self.device, dtype=dtype)
        self.w_patch[:, :k] = wpe.reshape(self.hidden, k)
        self.cls = t(p + "embeddings.class_embedding")
        self.pos = t(p + "embeddings.position_embedding.weight")  # [1 + n_patches, hidden]
        self.pre_ln = (t(p + "pre_layrnorm.weight"), t(p + "pre_layrnorm.bias"))
        self.post_ln = (t(p + "post_layernorm.weight"), t(p + "post_layernorm.bias"))
        self.proj = t("visual_projection.weight")
        self.blocks = []
        for i in range(self.layers):
            b = f"{p}encoder.layers.{i}."
            qkv_w = torch.cat([t(b + f"self_attn.{x}_proj.weight") for x in "qkv"], 0).contiguous()
            qkv_b = torch.cat([t(b + f"self_attn.{x}_proj.bias") for x in "qkv"], 0).contiguous()
            self.blocks.append({
                "ln1": (t(b + "layer_norm1.weight"), t(b + "layer_norm1.bias")),
                "ln2": (t(b + "layer_norm2.weight"), t(b + "layer_norm2.bias")),
                "qkv": (qkv_w, qkv_b), "o": (t(b + "self_attn.out_proj.weight"), t(b + "self_attn.out_proj.bias")),
                "fc1": (t(b + "mlp.fc1.weight"), t(b + "mlp.fc1.bias")),
                "fc2": (t(b + "mlp.fc2.weight"), t(b + "mlp.fc2.bias")),
            })

    def image_embeds(self, pixel_values: torch.Tensor) -> torch.Tensor:
        """pixel_values [n, 3, S, S] (CLIPImageProcessor output) -> image_embeds [n, projection_dim]."""
        n, c, H, W = pixel_values.shape
        P, C = self.patch, self.hidden
        gh, gw = H // P, W // P
        tok = gh * gw + 1
        if tok != self.pos.shape[0]:
            raise L.MimoError(f"CLIP: {gh}x{gw} patches + class token != {self.pos.shape[0]} position embeddings")
        # unfold (pure data movement of the 0.6 MB input): [n, 3, gh, P, gw, P] -> [n * gh * gw, 3 * P * P]
        x = pixel_values.to(device=self.device, dtype=self.dtype).reshape(n, c, gh, P, gw, P)
        cols = torch.zeros((n * gh * gw, self.kpad), device=self.device, dtype=self.dtype)
        cols[:, :c * P * P] = x.permute(0, 2, 4, 1, 3, 5).reshape(n * gh * gw, c * P * P)
        # class token + position embeddings enter through the patch GEMM's residual: build the additive term once
        add = self.pos.unsqueeze(0).repeat(n, 1, 1)
        add[:, 0] += self.cls
        h = torch.empty((n, tok, C), device=self.device, dtype=self.dtype)
        h[:, 0] = add[:, 0]
        patches = ops.gemm(cols, self.w_patch, residual=add[:, 1:].reshape(n * gh * gw, C).contiguous())
        h[:, 1:] = patches.reshape(n, gh * gw, C)
        h = h.reshape(n * tok, C)
        h = ops.layernorm(h, *self.pre_ln, eps=self.eps)
        for b in self.blocks:
            y = ops.layernorm(h, *b["ln1"], eps=self.eps)
            qkv = ops.gemm(y, b["qkv"][0], bias=b["qkv"][1])
            att = ops.attn_spatial(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], n, tok, self.heads)
            h = ops.gemm(att, b["o"][0], bias=b["o"][1], residual=h)
            y = ops.layernorm(h, *b["ln2"], eps=self.eps)
            y = ops.quick_gelu(ops.gemm(y, b["fc1"][0], bias=b["fc1"][1]))
            h = ops.gemm(y, b["fc2"][0], bias=b["fc2"][1], residual=h)
        pooled = h.reshape(n, tok, C)[:, 0].contiguous()
        pooled = ops.layernorm(pooled, *self.post_ln, eps=self.eps)
        return ops.gemm(pooled, self.proj)
