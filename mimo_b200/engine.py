"""The H100 denoising engine: packs a reference-layout state dict once, then runs the reference's module graph
(src/models/unet_3d_edit_bkfill.py:398-576 and friends) as a straight line of C-ABI kernel calls over
channels-last fp16/bf16 activations. No torch math on the hot path: torch only owns memory and the stream.

Layout: every activation is a 2-D tensor [rows, C], rows = ((b f), y, x) flattened, so
  * InflatedConv3d / InflatedGroupNorm's "b c f h w <-> (b f) c h w" copies (resnet.py:13-15, 24-26) vanish,
  * spatial-transformer tokens are the same buffer (transformer_3d.py:128-130 is a no-op view),
  * the motion module's "(b f) d c <-> (b d) f c" (motion_module.py:363-365, 388) becomes strided addressing.

Algebraic folds (identical results up to rounding order; see DESIGN.md):
  * cross-attention over the single CLIP token (attention.py:412-426): softmax over one key is 1, so
    attn2(x) == to_out(to_v(e)) for every token -> one vector per CFG branch, added in attn1's to_out epilogue;
  * the unconditional half attends to itself only (mutual_self_attention.py:177-197): expressed with
    bank_index = -1 instead of running attn1 twice;
  * bank keys/values are projected once per clip instead of once per frame per step;
  * q/k/v projections are one [3C, C] GEMM; GEGLU is a GEMM epilogue.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import lib as L
from . import ops

SD = Dict[str, torch.Tensor]


@dataclass
class UNetSpec:
    block_out_channels: Tuple[int, ...] = (320, 640, 1280, 1280)
    layers_per_block: int = 2
    heads: int = 8
    cross_attention_dim: int = 768
    norm_num_groups: int = 32
    norm_eps: float = 1e-5
    motion_groups: int = 32
    in_channels: int = 8
    out_channels: int = 4
    motion: bool = True
    out_head: bool = True


def _dev(sd: SD, key: str, device, dtype) -> torch.Tensor:
    return sd[key].detach().to(device=device, dtype=dtype).contiguous()


class _Packer:
    """Repack reference-layout weights (OIHW convs, [out, in] linears) for the kernels."""

    def __init__(self, sd: SD, device, dtype):
        self.sd, self.device, self.dtype = sd, device, dtype

    def t(self, key):
        return _dev(self.sd, key, self.device, self.dtype)

    def has(self, key):
        return key in self.sd

    def conv3(self, p, cin_pad=None, cout_pad=None):
        w = self.t(p + ".weight")
        b = self.t(p + ".bias")
        wp = ops.pack_conv3x3_weight(w, cin_pad, cout_pad)
        if wp.shape[0] != b.shape[0]:
            bp = torch.zeros(wp.shape[0], device=self.device, dtype=self.dtype)
            bp[: b.shape[0]] = b
            b = bp
        return wp, b

    def conv1(self, p):
        w = self.t(p + ".weight")
        return w.reshape(w.shape[0], -1).contiguous(), self.t(p + ".bias")

    def lin(self, p, bias=True):
        return self.t(p + ".weight"), (self.t(p + ".bias") if bias and self.has(p + ".bias") else None)

    def norm(self, p):
        return self.t(p + ".weight"), self.t(p + ".bias")

    def geglu(self, p):
        w, b = self.lin(p)
        return ops.pack_geglu_weight(w, b)

    def conv_up(self, p):
        """the 3x3 conv behind a nearest-x2 upsampling, as four 2x2-tap parity classes (ops.pack_conv_up2x_weight)"""
        return ops.pack_conv_up2x_weight(self.t(p + ".weight")), self.t(p + ".bias")


def bank_index_rows(branches: Sequence[int], frames: int, cfg: bool, nbank: int):
    """Bank routing of every frame-sample row of a forward (mutual_self_attention.py:154-197): -1 = attend to self only
    (the unconditional CFG branch), else the index of the bank feature map to append. With CFG the conditional bank is the
    LAST of the `nbank` maps the writer handed over (both halves -> index 1; conditional half only -> index 0); without
    CFG every row reads bank 0. Returns (indices, index of the conditional bank)."""
    cond = nbank - 1
    if not cfg:
        return [0] * (len(branches) * frames), cond
    return sum(([-1 if br == 0 else cond] * frames for br in branches), []), cond


class UNetEngine:
    """Executes the denoising UNet3D (motion=True) or the reference UNet2D bank pass (motion=False)."""

    def __init__(self, sd: SD, spec: UNetSpec, device, dtype=torch.float16):
        L.check(L.load().mimo_device_check(torch.device(device).index or 0), "mimo_device_check")
        self.spec, self.device, self.dtype = spec, torch.device(device), dtype
        self.clip_state: Optional[dict] = None
        self._persist: Dict[str, Dict[str, torch.Tensor]] = {}
        self._graphs: Dict[tuple, dict] = {}
        self.use_graphs = True
        self._launches_per_forward = 0
        # packed weights: from the on-disk cache when MIMO_B200_WEIGHT_CACHE is set and holds this state dict
        from .host import weight_cache as WC
        cache = WC.cache_dir()
        cfile = None
        if cache is not None:
            key = WC.fingerprint(sd, f"unet|{spec}|{dtype}|{L.load().mimo_version().decode()}")
            cfile = cache / f"unet-{key}.safetensors"
            if cfile.exists():
                st = WC.load(cfile, self.device)
                self.w, self.resnets, self.xf_paths = st["w"], st["resnets"], st["xf_paths"]
                self.temb_off = {k: tuple(v) for k, v in st["temb_off"].items()}
                self.from_cache = True
                return
        self.from_cache = False
        self._pack(sd, spec, device, dtype)
        if cfile is not None:
            WC.save(cfile, {"w": self.w, "resnets": self.resnets, "xf_paths": self.xf_paths,
                            "temb_off": {k: list(v) for k, v in self.temb_off.items()}})

    def _pack(self, sd: SD, spec: UNetSpec, device, dtype):
        pk = _Packer(sd, device, dtype)
        ch = spec.block_out_channels
        nb = len(ch)
        self.w: Dict[str, object] = {}
        W = self.w
        cin_pad = (spec.in_channels + 7) // 8 * 8
        W["conv_in"] = pk.conv3("conv_in", cin_pad=cin_pad)
        W["time1"] = pk.lin("time_embedding.linear_1")
        W["time2"] = pk.lin("time_embedding.linear_2")
        self.resnets: List[str] = []
        self.temb_off: Dict[str, Tuple[int, int]] = {}

        def add_resnet(p):
            r = {
                "n1": pk.norm(p + ".norm1"), "c1": pk.conv3(p + ".conv1"), "n2": pk.norm(p + ".norm2"),
                "c2": pk.conv3(p + ".conv2"),
                "sc": pk.conv1(p + ".conv_shortcut") if pk.has(p + ".conv_shortcut.weight") else None,
            }
            W[p] = r
            self.resnets.append(p)

        def add_xf(p):
            b = p + ".transformer_blocks.0"
            C = sd[p + ".norm.weight"].shape[0]
            wq, wk, wv = (pk.t(f"{b}.attn1.to_{x}.weight") for x in "qkv")
            W[p] = {
                "C": C, "gn": pk.norm(p + ".norm"), "pin": pk.conv1(p + ".proj_in"), "pout": pk.conv1(p + ".proj_out"),
                "ln1": pk.norm(b + ".norm1"), "ln3": pk.norm(b + ".norm3"),
                "qkv": torch.cat([wq, wk, wv], 0).contiguous(), "kv": torch.cat([wk, wv], 0).contiguous(),
                "o1": pk.lin(b + ".attn1.to_out.0"),
                "xv": pk.t(b + ".attn2.to_v.weight"), "xo": pk.lin(b + ".attn2.to_out.0"),
                "geglu": pk.geglu(b + ".ff.net.0.proj"), "ffo": pk.lin(b + ".ff.net.2"),
            }

        def add_mm(p):
            t = p + ".temporal_transformer"
            b = t + ".transformer_blocks.0"
            m = {"gn": pk.norm(t + ".norm"), "pin": pk.lin(t + ".proj_in"), "pout": pk.lin(t + ".proj_out"),
                 "ffn": pk.norm(b + ".ff_norm"), "geglu": pk.geglu(b + ".ff.net.0.proj"), "ffo": pk.lin(b + ".ff.net.2"),
                 "attn": []}
            for i in range(2):
                a = f"{b}.attention_blocks.{i}"
                qkv = torch.cat([pk.t(f"{a}.to_{x}.weight") for x in "qkv"], 0).contiguous()
                pe = pk.t(a + ".pos_encoder.pe")[0].contiguous()  # [max_len, C]
                m["attn"].append({"ln": pk.norm(f"{b}.norms.{i}"), "qkv": qkv, "o": pk.lin(a + ".to_out.0"), "pe": pe})
            W[p] = m

        self.xf_paths: List[str] = []
        for i in range(nb):
            for j in range(spec.layers_per_block):
                add_resnet(f"down_blocks.{i}.resnets.{j}")
                if i < nb - 1:
                    add_xf(f"down_blocks.{i}.attentions.{j}")
                    self.xf_paths.append(f"down_blocks.{i}.attentions.{j}")
                if spec.motion:
                    add_mm(f"down_blocks.{i}.motion_modules.{j}")
            if i < nb - 1:
                W[f"down_blocks.{i}.down"] = pk.conv3(f"down_blocks.{i}.downsamplers.0.conv")
        add_resnet("mid_block.resnets.0")
        add_xf("mid_block.attentions.0")
        self.xf_paths.append("mid_block.attentions.0")
        if spec.motion:
            add_mm("mid_block.motion_modules.0")
        add_resnet("mid_block.resnets.1")
        for i in range(nb):
            for j in range(spec.layers_per_block + 1):
                add_resnet(f"up_blocks.{i}.resnets.{j}")
                if i > 0:
                    add_xf(f"up_blocks.{i}.attentions.{j}")
                    self.xf_paths.append(f"up_blocks.{i}.attentions.{j}")
                if spec.motion:
                    add_mm(f"up_blocks.{i}.motion_modules.{j}")
            if i < nb - 1:
                W[f"up_blocks.{i}.up"] = pk.conv_up(f"up_blocks.{i}.upsamplers.0.conv")
        if spec.out_head:
            W["norm_out"] = pk.norm("conv_norm_out")
            W["conv_out"] = pk.conv3("conv_out")
        # all time_emb_proj layers as one GEMM: [sum(Cout), temb]
        ws, bs, off = [], [], 0
        for p in self.resnets:
            w, b = pk.lin(p + ".time_emb_proj")
            self.temb_off[p] = (off, w.shape[0])
            off += w.shape[0]
            ws.append(w)
            bs.append(b)
        W["temb_all"] = (torch.cat(ws, 0).contiguous(), torch.cat(bs, 0).contiguous())

    # ------------------------------------------------------------------------------------------------
    def _sinusoid(self, timesteps: torch.Tensor) -> torch.Tensor:
        """Timesteps(flip_sin_to_cos, shift 0) in fp32, cast to the model dtype (unet_3d_edit_bkfill.py:462-467)."""
        c0 = self.spec.block_out_channels[0]
        half = c0 // 2
        t = timesteps.to(device=self.device, dtype=torch.float32).reshape(-1)
        exponent = -math.log(10000) * torch.arange(0, half, dtype=torch.float32, device=self.device) / half
        emb = t[:, None] * torch.exp(exponent)[None, :]
        return torch.cat([torch.cos(emb), torch.sin(emb)], dim=-1).to(self.dtype).contiguous()

    def _time_embed_from(self, emb: torch.Tensor) -> torch.Tensor:
        """TimestepEmbedding MLP and ALL resnets' time_emb_proj(silu(emb)) as three GEMMs. -> [b, sum(Cout)]"""
        w1, b1 = self.w["time1"]
        w2, b2 = self.w["time2"]
        h = ops.gemm(emb, w1, bias=b1, act=L.ACT_SILU)
        h = ops.gemm(h, w2, bias=b2, act=L.ACT_SILU)  # only silu(emb) is ever consumed (resnet.py:226)
        wa, ba = self.w["temb_all"]
        return ops.gemm(h, wa, bias=ba)

    def _time_embed(self, timesteps: torch.Tensor) -> torch.Tensor:
        return self._time_embed_from(self._sinusoid(timesteps))

    def _resnet(self, p, x0, x1, tembs, n, h, w, rows_per_branch):
        r = self.w[p]
        g, eps = self.spec.norm_num_groups, self.spec.norm_eps
        hw = h * w
        t = ops.groupnorm(x0, *r["n1"], n, hw, groups=g, eps=eps, silu=True, x1=x1)
        off, cout = self.temb_off[p]
        t = ops.conv3x3(t, r["c1"][0], n, h, w, bias=r["c1"][1], rowvec=tembs[:, off:off + cout],
                        rows_per_group=rows_per_branch)
        t = ops.groupnorm(t, *r["n2"], n, hw, groups=g, eps=eps, silu=True)
        if r["sc"] is not None:
            res = ops.gemm(x0, r["sc"][0], a1=x1, bias=r["sc"][1])
        else:
            assert x1 is None
            res = x0
        return ops.conv3x3(t, r["c2"][0], n, h, w, bias=r["c2"][1], residual=res)

    def _ff(self, x, ln, geglu, ffo):
        nh = ops.layernorm(x, *ln)
        gg = ops.gemm(nh, geglu[0], bias=geglu[1], act=L.ACT_GEGLU)
        return ops.gemm(gg, ffo[0], bias=ffo[1], residual=x)

    def _xf_read(self, p, x, n, hw, rows_per_branch, st):
        m = self.w[p]
        C = m["C"]
        hcur = ops.groupnorm(x, *m["gn"], n, hw, groups=self.spec.norm_num_groups, eps=1e-6)
        hcur = ops.gemm(hcur, m["pin"][0], bias=m["pin"][1])
        nh = ops.layernorm(hcur, *m["ln1"])
        qkv = ops.gemm(nh, m["qkv"])
        bank = st["banks"].get(p)
        if bank is not None:
            att = ops.attn_spatial(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], n, hw, self.spec.heads,
                                   bank_k=bank[:, :, :C], bank_v=bank[:, :, C:], bank_index=st["bank_index"],
                                   n_bank_frames=st["n_bank_frames"])
        else:
            att = ops.attn_spatial(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], n, hw, self.spec.heads)
        hcur = ops.gemm(att, m["o1"][0], bias=m["o1"][1], residual=hcur, rowvec=st["xattn"][p],
                        rows_per_group=rows_per_branch)
        hcur = self._ff(hcur, m["ln3"], m["geglu"], m["ffo"])
        return ops.gemm(hcur, m["pout"][0], bias=m["pout"][1], residual=x)

    def _motion(self, p, x, b, f, hw):
        """VanillaTemporalModule (motion_module.py:77-91, 146-184, 238-261). Single GPU: f = all frames of the window.
        Frame-sharded (self.xchg, G GPUs): this GPU holds f = F / G frames; the tokens are re-sharded to pixels for the
        transformer block (every GPU then owns all F frames of hw / G pixels, so LN + PE, q/k/v, the attention over
        frames, out-proj and the feed-forward are all local) and back, each by one peer-memory exchange kernel."""
        m = self.w[p]
        n = b * f
        xg = self.xchg
        G = xg.G if xg is not None else 1
        F_ = f * G
        if F_ > m["attn"][0]["pe"].shape[0]:
            # the reference fails here with a shape error (motion_module.py:277-279: x + pe[:, :x.size(1)])
            raise L.MimoError(f"{F_} frames in a window exceed temporal_position_encoding_max_len="
                              f"{m['attn'][0]['pe'].shape[0]}")
        hcur = ops.groupnorm(x, *m["gn"], n, hw, groups=self.spec.motion_groups, eps=1e-6)
        C = m["pin"][0].shape[0]
        if G == 1:
            hw_l = hw
            hcur = ops.gemm(hcur, m["pin"][0], bias=m["pin"][1])
        else:
            if hw % G:
                raise L.MimoError(f"{hw} tokens per frame cannot be split over a frame group of {G} GPUs")
            hw_l = hw // G
            ops.gemm(hcur, m["pin"][0], out=xg.bufs["A"].view(n * hw, C, x.dtype), bias=m["pin"][1])
            hcur = xg.pull(0, "A", torch.empty((b * F_ * hw_l, C), dtype=x.dtype, device=x.device), b, f, hw, C)
        for a in m["attn"]:
            nh = ops.layernorm(hcur, *a["ln"], pe=a["pe"], rows_per_frame=hw_l, frames=F_)
            qkv = ops.gemm(nh, a["qkv"])
            att = ops.attn_temporal(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], b, F_, hw_l, self.spec.heads)
            hcur = ops.gemm(att, a["o"][0], bias=a["o"][1], residual=hcur)
        hcur = self._ff(hcur, m["ffn"], m["geglu"], m["ffo"])
        if G == 1:
            return ops.gemm(hcur, m["pout"][0], bias=m["pout"][1], residual=x)
        ops.gemm(hcur, m["pout"][0], out=xg.bufs["B"].view(b * F_ * hw_l, C, x.dtype), bias=m["pout"][1])
        return xg.pull(1, "B", torch.empty_like(x), b, f, hw, C, residual=x)

    def _down(self, p, x, n, h, w):
        wp, b = self.w[p]
        col = ops.im2col3x3(x, n, h, w, stride=2)
        return ops.gemm(col, wp, bias=b)

    def _up(self, p, x, n, h, w):
        wp, b = self.w[p]
        return ops.conv_up2x(x, wp, n, h, w, bias=b)  # Upsample3D (resnet.py:53-90) without the 4x tensor

    def check_latent_size(self, h: int, w: int) -> None:
        """The down path halves h and w once per level and the up path doubles them back exactly. The reference also
        accepts sizes that do not divide (its script default 784 x 784 -> 98 x 98 latents) by interpolating every upsampler
        to the skip connection's size (unet_3d_edit_bkfill.py:430-435, :544-545 `forward_upsample_size`); the fused
        nearest-x2 + 3x3 kernel (mimo_conv_up2x) has no such mode: refuse instead of reading past the skip tensors."""
        m = 1 << (len(self.spec.block_out_channels) - 1)
        if h <= 0 or w <= 0 or h % m or w % m:
            raise L.MimoError(f"latent size {h} x {w} is not a multiple of {m} (pixels: {8 * m}): the reference's "
                              "forward_upsample_size path (unet_3d_edit_bkfill.py:430-435) is not implemented; "
                              f"use a width and height that are multiples of {8 * m}")

    xchg = None  # host.shard.Exchange of this GPU's frame group (None / G == 1: all frames of a window are local)
    taps: Optional[dict] = None  # debugging aid (scripts/gpu_probe.py): block outputs as [N, C, H, W] fp32 on CPU

    def _tap(self, name, x, n, h, w):
        if self.taps is not None:
            self.taps[name] = x.float().reshape(n, h, w, -1).permute(0, 3, 1, 2).cpu()
        return x

    def _body(self, x, tembs, b, f, h, w, xf_fn, stop_at: Optional[str] = None):
        sp = self.spec
        nb = len(sp.block_out_channels)
        n = b * f
        skips = [(x, h, w)]
        rpb = lambda hh, ww: f * hh * ww  # rows per CFG branch at this resolution
        for i in range(nb):
            for j in range(sp.layers_per_block):
                x = self._tap(f"down_blocks.{i}.resnets.{j}", self._resnet(f"down_blocks.{i}.resnets.{j}", x, None, tembs, n, h, w, rpb(h, w)), n, h, w)
                if i < nb - 1:
                    x = self._tap(f"down_blocks.{i}.attentions.{j}", xf_fn(f"down_blocks.{i}.attentions.{j}", x, n, h * w, rpb(h, w)), n, h, w)
                if sp.motion:
                    x = self._tap(f"down_blocks.{i}.motion_modules.{j}", self._motion(f"down_blocks.{i}.motion_modules.{j}", x, b, f, h * w), n, h, w)
                skips.append((x, h, w))
            if i < nb - 1:
                x = self._down(f"down_blocks.{i}.down", x, n, h, w)
                h, w = h // 2, w // 2
                self._tap(f"down_blocks.{i}.down", x, n, h, w)
                skips.append((x, h, w))
        x = self._tap("mid_block.resnets.0", self._resnet("mid_block.resnets.0", x, None, tembs, n, h, w, rpb(h, w)), n, h, w)
        x = self._tap("mid_block.attentions.0", xf_fn("mid_block.attentions.0", x, n, h * w, rpb(h, w)), n, h, w)
        if sp.motion:
            x = self._tap("mid_block.motion_modules.0", self._motion("mid_block.motion_modules.0", x, b, f, h * w), n, h, w)
        x = self._tap("mid_block.resnets.1", self._resnet("mid_block.resnets.1", x, None, tembs, n, h, w, rpb(h, w)), n, h, w)
        for i in range(nb):
            for j in range(sp.layers_per_block + 1):
                s, _, _ = skips.pop()
                x = self._tap(f"up_blocks.{i}.resnets.{j}", self._resnet(f"up_blocks.{i}.resnets.{j}", x, s, tembs, n, h, w, rpb(h, w)), n, h, w)
                if i > 0:
                    pth = f"up_blocks.{i}.attentions.{j}"
                    x = xf_fn(pth, x, n, h * w, rpb(h, w))
                    if stop_at == pth:
                        return x, h, w
                    self._tap(pth, x, n, h, w)
                if sp.motion:
                    x = self._tap(f"up_blocks.{i}.motion_modules.{j}", self._motion(f"up_blocks.{i}.motion_modules.{j}", x, b, f, h * w), n, h, w)
            if i < nb - 1:
                x = self._up(f"up_blocks.{i}.up", x, n, h, w)
                h, w = 2 * h, 2 * w
                self._tap(f"up_blocks.{i}.up", x, n, h, w)
        return x, h, w

    # ------------------------------------------------------------------------------------------------
    def cross_attn_vectors(self, ehs: torch.Tensor) -> Dict[str, torch.Tensor]:
        """attn2 over one key: out = to_out(to_v(e)) per CFG branch (attention.py:412-426). ehs [b, 1, 768]."""
        e = ehs.reshape(ehs.shape[0], -1).to(device=self.device, dtype=self.dtype).contiguous()
        out = {}
        for p in self.xf_paths:
            m = self.w[p]
            v = ops.gemm(e, m["xv"])
            out[p] = ops.gemm(v, m["xo"][0], bias=m["xo"][1])
        return out

    def write_banks(self, latents: torch.Tensor, ehs: torch.Tensor, reader: "UNetEngine") -> Dict[str, torch.Tensor]:
        """reference_unet pass at t = 0 ("write" mode, pipeline :480-490): returns, per spatial block, the bank's
        keys|values already projected with the READER's to_k/to_v: {path: [nb, hw, 2C]}. `self` is the reference
        UNet (motion=False). latents [nb, 4, h, w]."""
        nbr, c, h, w = latents.shape
        self.check_latent_size(h, w)
        x_in = ops.ncfhw_to_nhwc(latents.to(self.device).unsqueeze(2).contiguous(), 8, self.dtype)
        tembs = self._time_embed(torch.zeros(nbr, device=self.device))
        st = {"xattn": self.cross_attn_vectors(ehs)}
        banks: Dict[str, torch.Tensor] = {}
        last = [p for p in self.xf_paths if p.startswith("up_blocks")][-1]

        def xf_write(p, x, n, hw, rows_per_branch):
            m = self.w[p]
            C = m["C"]
            hcur = ops.groupnorm(x, *m["gn"], n, hw, groups=self.spec.norm_num_groups, eps=1e-6)
            hcur = ops.gemm(hcur, m["pin"][0], bias=m["pin"][1])
            nh = ops.layernorm(hcur, *m["ln1"])
            # mutual_self_attention.py:137-139 + :349 — the bank is norm1(x) cast to fp16; project it with the reader
            banks[p] = ops.gemm(nh, reader.w[p]["kv"]).reshape(n, hw, 2 * C)
            if p == last:
                return x  # everything after the last bank write is dead code in the reference (SURVEY §3.4)
            qkv = ops.gemm(nh, m["qkv"])
            att = ops.attn_spatial(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], n, hw, self.spec.heads)
            hcur = ops.gemm(att, m["o1"][0], bias=m["o1"][1], residual=hcur, rowvec=st["xattn"][p],
                            rows_per_group=rows_per_branch)
            hcur = self._ff(hcur, m["ln3"], m["geglu"], m["ffo"])
            return ops.gemm(hcur, m["pout"][0], bias=m["pout"][1], residual=x)

        wci, bci = self.w["conv_in"]
        x = ops.conv3x3(x_in, wci, nbr, h, w, bias=bci)
        self._body(x, tembs, nbr, 1, h, w, xf_write, stop_at=last)
        return banks

    # ------------------------------------------------------------------------------------------------
    # per-clip state lives in PERSISTENT buffers (same addresses for every clip) so that captured CUDA graphs of the
    # forward stay valid: begin_clip / set_cross_attn copy new values in place.
    def _store(self, slot: str, new: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        cur = self._persist.get(slot)
        if cur is not None and cur.keys() == new.keys() and all(cur[k].shape == new[k].shape for k in new):
            for k in new:
                cur[k].copy_(new[k])
            return cur
        self._persist[slot] = new
        self._graphs.clear()  # addresses changed: captured graphs are stale
        return new

    def set_cross_attn(self, ehs: torch.Tensor):
        br = list(self.clip_state["branches"])
        vec = {p: v[br].contiguous() for p, v in self.cross_attn_vectors(ehs).items()}  # this GPU's CFG branch(es)
        self.clip_state["xattn"] = self._store("xattn", vec)

    def begin_clip(self, ehs: torch.Tensor, banks: Dict[str, torch.Tensor], cfg: bool, frames: int,
                   branches: Optional[Sequence[int]] = None):
        """Per-clip state of the denoising UNet: folded cross-attention vectors, projected banks, bank routing.
        `branches`: which rows of `ehs` (CFG branches: 0 = unconditional, 1 = conditional) this GPU evaluates; the
        batch dimension of forward()'s sample is len(branches). Default: all of them."""
        branches = tuple(range(ehs.shape[0])) if branches is None else tuple(branches)
        self.clip_state = {"banks": self._store("banks", banks), "cfg": cfg, "frames": 0, "batch": len(branches),
                           "branches": branches, "bank_index": None, "n_bank_frames": 0}
        self.set_cross_attn(ehs)
        self.begin_clip_frames(frames, len(branches))

    def begin_clip_frames(self, frames: int, b: int):
        st = self.clip_state
        if b != len(st["branches"]):
            raise L.MimoError(f"forward() got a batch of {b} but this engine evaluates branches {st['branches']}")
        # unconditional rows ignore the bank (mutual_self_attention.py:177-197); conditional rows read bank 1
        nbank = next(iter(st["banks"].values())).shape[0] if st["banks"] else 1
        idx, cond = bank_index_rows(st["branches"], frames, st["cfg"], nbank)
        new = torch.tensor(idx, dtype=torch.int32, device=self.device)
        st["bank_index"] = self._store(f"bank_index_{len(idx)}_{st['branches']}_{cond}", {"i": new})["i"]
        st["n_bank_frames"] = sum(1 for i in idx if i >= 0)
        st["frames"] = frames

    def _forward_impl(self, sample: torch.Tensor, emb: torch.Tensor, pose_nhwc: Optional[torch.Tensor]) -> torch.Tensor:
        st = self.clip_state
        b, c, f, h, w = sample.shape
        x_in = ops.ncfhw_to_nhwc(sample, (c + 7) // 8 * 8, self.dtype)
        tembs = self._time_embed_from(emb)
        wci, bci = self.w["conv_in"]
        x = ops.conv3x3(x_in, wci, b * f, h, w, bias=bci, residual=pose_nhwc)
        xf = lambda p, xx, n, hw, rpb: self._xf_read(p, xx, n, hw, rpb, st)
        x, h2, w2 = self._body(x, tembs, b, f, h, w, xf)
        x = ops.groupnorm(x, *self.w["norm_out"], b * f, h * w, groups=self.spec.norm_num_groups,
                          eps=self.spec.norm_eps, silu=True)
        wco, bco = self.w["conv_out"]
        y = ops.conv3x3(x, wco, b * f, h, w, bias=bco)
        return ops.nhwc_to_ncfhw(y, b, self.spec.out_channels, f, h, w)

    def forward(self, sample: torch.Tensor, timestep, pose_nhwc: Optional[torch.Tensor]) -> torch.Tensor:
        """UNet3DConditionModel.forward (unet_3d_edit_bkfill.py:398-576). sample [b, 8, f, h, w] (reference layout,
        any float dtype); pose_nhwc [(b f) h w, 320] channels-last or None. Returns [b, 4, f, h, w].
        The ~1 400 kernel launches of one forward are a fixed graph per input shape: after one eager run they are
        captured into a CUDA graph and replayed (the returned tensor is then a static buffer, valid until the next
        forward of the same shape)."""
        st = self.clip_state
        assert st is not None, "begin_clip() must run before forward()"
        b, c, f, h, w = sample.shape
        self.check_latent_size(h, w)
        if st["bank_index"] is None or st["bank_index"].numel() != b * f:
            self.begin_clip_frames(f, b)
        t = timestep if torch.is_tensor(timestep) else torch.tensor([timestep])
        emb = self._sinusoid(t.reshape(-1).expand(b) if t.numel() == 1 else t)
        sample = sample.contiguous()
        if not self.use_graphs or self.taps is not None or ops.PROFILE is not None:
            return self._forward_impl(sample, emb, pose_nhwc)
        key = (tuple(sample.shape), sample.dtype, pose_nhwc is not None, st["bank_index"].data_ptr(), id(self.xchg))
        g = self._graphs.get(key)
        if g is None:
            g = {"calls": 0}
            self._graphs[key] = g
        if "graph" not in g:
            g["calls"] += 1
            if g["calls"] < 2:  # first call of a shape runs eagerly (lazy one-time setup inside the C library)
                return self._forward_impl(sample, emb, pose_nhwc)
            g["sample"] = sample.clone()
            g["emb"] = emb.clone()
            g["pose"] = pose_nhwc.clone() if pose_nhwc is not None else None
            graph = torch.cuda.CUDAGraph()
            torch.cuda.synchronize()
            l0 = ops.launches()
            with torch.cuda.graph(graph):
                g["out"] = self._forward_impl(g["sample"], g["emb"], g["pose"])
            g["graph"] = graph
            g["launches"] = ops.launches() - l0  # kernels recorded in the graph (nothing ran during capture)
            ops.add_launches(-g["launches"])
        g["sample"].copy_(sample)
        g["emb"].copy_(emb)
        if pose_nhwc is not None:
            # always copied: neither data_ptr nor torch's version counter identify the CONTENT of a tensor that is
            # written through raw pointers and recycled by the caching allocator (a stale-pose replay otherwise)
            g["pose"].copy_(pose_nhwc)
        g["graph"].replay()
        ops.add_launches(g["launches"])
        return g["out"]


class PoseGuiderEngine:
    """PoseGuider.forward (src/models/pose_guider.py:47-57): 8 convs + SiLU; stride-2 layers via im2col + GEMM."""

    def __init__(self, sd: SD, device, dtype=torch.float16):
        pk = _Packer(sd, device, dtype)
        self.device, self.dtype = torch.device(device), dtype
        self.layers = [("conv_in", 1)] + [(f"blocks.{i}", 2 if i % 2 == 1 else 1) for i in range(6)] + [("conv_out", 1)]
        self.w = {name: pk.conv3(name) for name, _ in self.layers}
        self.cout = sd["conv_out.weight"].shape[0]

    def forward(self, cond: torch.Tensor) -> torch.Tensor:
        """cond [1, 3, F, H, W] -> channels-last [(F) H/8 W/8, 320]."""
        b, c, f, H, W = cond.shape
        if H % 8 or W % 8:  # three stride-2 convolutions; the pipeline floors its images to multiples of 8 (:73-80)
            raise L.MimoError(f"pose frames of {H} x {W}: height and width must be multiples of 8")
        x = ops.ncfhw_to_nhwc(cond.to(self.device).contiguous(), 8, self.dtype)
        n, h, w = b * f, H, W
        for name, stride in self.layers:
            wp, bias = self.w[name]
            act = L.ACT_NONE if name == "conv_out" else L.ACT_SILU
            if stride == 1:
                x = ops.conv3x3(x, wp, n, h, w, bias=bias, act=act)
            else:
                col = ops.im2col3x3(x, n, h, w, stride=2)
                x = ops.gemm(col, wp, bias=bias, act=act)
                h, w = h // 2, w // 2
        return x


class _VAEBlocks:
    """ResnetBlock2D (no time embedding) and the 1-head mid-block attention shared by encoder and decoder."""

    def _add_res(self, pk, p):
        self.w[p] = {"n1": pk.norm(p + ".norm1"), "c1": pk.conv3(p + ".conv1"), "n2": pk.norm(p + ".norm2"),
                     "c2": pk.conv3(p + ".conv2"),
                     "sc": pk.conv1(p + ".conv_shortcut") if pk.has(p + ".conv_shortcut.weight") else None}

    def _add_attn(self, pk, a):
        self.w[a] = {"gn": pk.norm(a + ".group_norm"), "q": pk.lin(a + ".to_q"), "k": pk.lin(a + ".to_k"),
                     "v": pk.lin(a + ".to_v"), "o": pk.lin(a + ".to_out.0")}

    def _res(self, p, x, n, h, w):
        r = self.w[p]
        t = ops.groupnorm(x, *r["n1"], n, h * w, groups=self.groups, eps=1e-6, silu=True)
        t = ops.conv3x3(t, r["c1"][0], n, h, w, bias=r["c1"][1])
        t = ops.groupnorm(t, *r["n2"], n, h * w, groups=self.groups, eps=1e-6, silu=True)
        resid = ops.gemm(x, r["sc"][0], bias=r["sc"][1]) if r["sc"] is not None else x
        return ops.conv3x3(t, r["c2"][0], n, h, w, bias=r["c2"][1], residual=resid)

    def _attn(self, key, x, n, hw):
        a = self.w[key]
        C = x.shape[1]
        t = ops.groupnorm(x, *a["gn"], n, hw, groups=self.groups, eps=1e-6)
        q = ops.gemm(t, a["q"][0], bias=a["q"][1])
        k = ops.gemm(t, a["k"][0], bias=a["k"][1])
        out = torch.empty_like(x)
        scale = C ** -0.5
        for i in range(n):
            sl = slice(i * hw, (i + 1) * hw)
            s = ops.gemm(q[sl], k[sl], scale=scale)                      # [hw, hw] logits
            ops.softmax_rows_(s)
            vt = ops.gemm(a["v"][0], t[sl])                              # V^T (bias folded below: rows of P sum to 1)
            o = ops.gemm(s, vt, bias=a["v"][1])                          # P V + b_v
            ops.gemm(o, a["o"][0], out=out[sl], bias=a["o"][1], residual=x[sl])
        return out


class VAEEncoderEngine(_VAEBlocks):
    """AutoencoderKL.encode(x).latent_dist.mean for sd-vae-ft-mse (diffusers [3P]; call sites pipeline :430, :438).
    Downsampling is F.pad(0,1,0,1) + 3x3 stride-2 conv without padding: im2col(pad_lo=0) + GEMM."""

    def __init__(self, sd: SD, device, dtype=torch.float16, groups: int = 32):
        pk = _Packer(sd, device, dtype)
        self.device, self.dtype, self.groups = torch.device(device), dtype, groups
        self.w: Dict[str, object] = {}
        W = self.w
        W["conv_in"] = pk.conv3("encoder.conv_in", cin_pad=8)
        self.n_down = len({k.split(".")[2] for k in sd if k.startswith("encoder.down_blocks.")})
        self.n_res = len({k.split(".")[4] for k in sd if k.startswith("encoder.down_blocks.0.resnets.")})
        for i in range(self.n_down):
            for j in range(self.n_res):
                self._add_res(pk, f"encoder.down_blocks.{i}.resnets.{j}")
            if pk.has(f"encoder.down_blocks.{i}.downsamplers.0.conv.weight"):
                W[f"down{i}"] = pk.conv3(f"encoder.down_blocks.{i}.downsamplers.0.conv")
        self._add_res(pk, "encoder.mid_block.resnets.0")
        self._add_res(pk, "encoder.mid_block.resnets.1")
        self._add_attn(pk, "encoder.mid_block.attentions.0")
        W["norm_out"] = pk.norm("encoder.conv_norm_out")
        W["conv_out"] = pk.conv3("encoder.conv_out")
        self.latent = sd["quant_conv.weight"].shape[0] // 2
        W["quant"] = pk.conv1("quant_conv")

    def encode_mean(self, x: torch.Tensor) -> torch.Tensor:
        """x [n, 3, H, W] in [-1, 1] -> latent mean [n, 4, H/8, W/8] (not yet scaled by 0.18215)."""
        n, c, h, w = x.shape
        m = 1 << sum(1 for i in range(self.n_down) if f"down{i}" in self.w)
        if h % m or w % m:
            raise L.MimoError(f"images of {h} x {w}: height and width must be multiples of {m} (VaeImageProcessor floors "
                              "to multiples of the VAE scale factor, pipeline :73-80)")
        t = ops.ncfhw_to_nhwc(x.to(self.device).unsqueeze(2).contiguous(), 8, self.dtype)
        t = ops.conv3x3(t, self.w["conv_in"][0], n, h, w, bias=self.w["conv_in"][1])
        for i in range(self.n_down):
            for j in range(self.n_res):
                t = self._res(f"encoder.down_blocks.{i}.resnets.{j}", t, n, h, w)
            if f"down{i}" in self.w:
                col = ops.im2col3x3(t, n, h, w, stride=2, pad_lo=0)
                t = ops.gemm(col, self.w[f"down{i}"][0], bias=self.w[f"down{i}"][1])
                h, w = h // 2, w // 2
        t = self._res("encoder.mid_block.resnets.0", t, n, h, w)
        t = self._attn("encoder.mid_block.attentions.0", t, n, h * w)
        t = self._res("encoder.mid_block.resnets.1", t, n, h, w)
        t = ops.groupnorm(t, *self.w["norm_out"], n, h * w, groups=self.groups, eps=1e-6, silu=True)
        t = ops.conv3x3(t, self.w["conv_out"][0], n, h, w, bias=self.w["conv_out"][1])
        t = ops.gemm(t, self.w["quant"][0], bias=self.w["quant"][1])
        return ops.nhwc_to_ncfhw(t, n, self.latent, 1, h, w)[:, :, 0]


class VAEDecoderEngine(_VAEBlocks):
    """AutoencoderKL.decode for sd-vae-ft-mse (diffusers [3P]; call site pipeline :113-126), all frames of a
    shard batched. The mid-block attention (1 head, d = 512) runs as GEMM -> row softmax -> GEMM."""

    def __init__(self, sd: SD, device, dtype=torch.float16, groups: int = 32):
        pk = _Packer(sd, device, dtype)
        self.device, self.dtype, self.groups = torch.device(device), dtype, groups
        self.w: Dict[str, object] = {}
        W = self.w
        lat = sd["post_quant_conv.weight"].shape[0]
        wq = torch.zeros(8, 8, device=device, dtype=dtype)
        wq[:lat, :lat] = pk.t("post_quant_conv.weight").reshape(lat, lat)
        bq = torch.zeros(8, device=device, dtype=dtype)
        bq[:lat] = pk.t("post_quant_conv.bias")
        W["pq"] = (wq, bq)
        W["conv_in"] = pk.conv3("decoder.conv_in", cin_pad=8)
        self.n_up = len({k.split(".")[2] for k in sd if k.startswith("decoder.up_blocks.")})
        self.n_res = len({k.split(".")[4] for k in sd if k.startswith("decoder.up_blocks.0.resnets.")})

        self._add_res(pk, "decoder.mid_block.resnets.0")
        self._add_res(pk, "decoder.mid_block.resnets.1")
        self._add_attn(pk, "decoder.mid_block.attentions.0")
        for i in range(self.n_up):
            for j in range(self.n_res):
                self._add_res(pk, f"decoder.up_blocks.{i}.resnets.{j}")
            if pk.has(f"decoder.up_blocks.{i}.upsamplers.0.conv.weight"):
                W[f"up{i}"] = pk.conv_up(f"decoder.up_blocks.{i}.upsamplers.0.conv")
        W["norm_out"] = pk.norm("decoder.conv_norm_out")
        W["conv_out"] = pk.conv3("decoder.conv_out")
        self.out_channels = sd["decoder.conv_out.weight"].shape[0]

    def decode(self, z: torch.Tensor) -> torch.Tensor:
        """z [n, 4, h, w] (already divided by 0.18215) -> [n, 3, 8h, 8w] in the engine dtype."""
        n, c, h, w = z.shape
        x = ops.ncfhw_to_nhwc(z.to(self.device).unsqueeze(2).contiguous(), 8, self.dtype)  # [n,4,1,h,w]: "f" = 1
        x = ops.gemm(x, self.w["pq"][0], bias=self.w["pq"][1])
        x = ops.conv3x3(x, self.w["conv_in"][0], n, h, w, bias=self.w["conv_in"][1])
        x = self._res("decoder.mid_block.resnets.0", x, n, h, w)
        x = self._attn("decoder.mid_block.attentions.0", x, n, h * w)
        x = self._res("decoder.mid_block.resnets.1", x, n, h, w)
        for i in range(self.n_up):
            for j in range(self.n_res):
                x = self._res(f"decoder.up_blocks.{i}.resnets.{j}", x, n, h, w)
            if f"up{i}" in self.w:
                x = ops.conv_up2x(x, self.w[f"up{i}"][0], n, h, w, bias=self.w[f"up{i}"][1])
                h, w = 2 * h, 2 * w
        x = ops.groupnorm(x, *self.w["norm_out"], n, h * w, groups=self.groups, eps=1e-6, silu=True)
        y = ops.conv3x3(x, self.w["conv_out"][0], n, h, w, bias=self.w["conv_out"][1])
        out = ops.nhwc_to_ncfhw(y, n, self.out_channels, 1, h, w)  # [n, 3, 1, H, W]
        return out[:, :, 0]
