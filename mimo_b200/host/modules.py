"""Host-side mirror of the reference's module surface (SURVEY.md §8b): same class names, constructor arguments,
state-dict keys, forward signatures and error behaviour as

  src/models/unet_3d_edit_bkfill.py  UNet3DConditionModel   (:30-81, :398-409, :573-682)
  src/models/unet_2d_condition.py    UNet2DConditionModel   (:872-887)
  src/models/pose_guider.py          PoseGuider             (:12-57)
  src/models/mutual_self_attention.py ReferenceAttentionControl (:19-50, :313, :352)

but the modules are only parameter containers: forward() hands the tensors to the sm_90a engine
(mimo_b200/engine.py) through the C ABI. On a non-CUDA device forward() raises — there is no CPU path.
"""
from __future__ import annotations

import json
import math
from dataclasses import dataclass
from pathlib import Path
from types import SimpleNamespace
from typing import Dict, Optional, Tuple, Union

import torch
from torch import nn

from .. import engine as E
from ..lib import MimoError
from . import schema


class _Tree(nn.Module):
    """Nested containers so that state_dict() yields exactly the reference's dotted keys."""

    def put(self, parts, tensor: torch.Tensor, buffer: bool):
        if len(parts) == 1:
            if buffer:
                self.register_buffer(parts[0], tensor)
            else:
                self.register_parameter(parts[0], nn.Parameter(tensor, requires_grad=False))
            return
        if parts[0] not in self._modules:
            self.add_module(parts[0], _Tree())
        self._modules[parts[0]].put(parts[1:], tensor, buffer)


def _pe(d_model: int, max_len: int) -> torch.Tensor:
    # PositionalEncoding buffer (src/models/motion_module.py:264-275)
    position = torch.arange(max_len).unsqueeze(1)
    div_term = torch.exp(torch.arange(0, d_model, 2) * (-math.log(10000.0) / d_model))
    pe = torch.zeros(1, max_len, d_model)
    pe[0, :, 0::2] = torch.sin(position * div_term)
    pe[0, :, 1::2] = torch.cos(position * div_term)
    return pe


class _EngineModel(nn.Module):
    """Parameter container + lazily built engine (rebuilt when the parameters move or change dtype)."""

    def _materialise(self, shapes: Dict[str, Tuple[int, ...]]):
        gen = torch.Generator().manual_seed(0)
        for k, shp in shapes.items():
            parts = k.split(".")
            if parts[-1] == "pe":
                t, buf = _pe(shp[2], shp[1]), True
            elif parts[-1] == "bias":
                t, buf = torch.zeros(shp), False
            elif len(shp) == 1:
                t, buf = torch.ones(shp), False
            else:
                fan_in = 1
                for s in shp[1:]:
                    fan_in *= s
                t, buf = torch.randn(shp, generator=gen) / math.sqrt(fan_in), False
            self._tree.put(parts, t, buf)

    def __init__(self):
        super().__init__()
        self._tree = _Tree()
        self._engine = None
        self._engine_key = None

    # state-dict keys must not carry the container's name
    def state_dict(self, *args, destination=None, prefix="", keep_vars=False):
        return self._tree.state_dict(*args, destination=destination, prefix=prefix, keep_vars=keep_vars)

    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):
        self._engine = None
        return self._tree.load_state_dict(state_dict, strict=strict, assign=assign)

    @property
    def dtype(self) -> torch.dtype:
        return next(self._tree.parameters()).dtype

    @property
    def device(self) -> torch.device:
        return next(self._tree.parameters()).device

    def _require_cuda(self):
        if self.device.type != "cuda":
            raise MimoError(f"{type(self).__name__}.forward needs the model on a CUDA (sm_90a) device; it is on "
                            f"{self.device}. mimo_b200 has no CPU fallback.")
        if self.dtype not in (torch.float16, torch.bfloat16):
            raise MimoError(f"{type(self).__name__}: engine dtypes are float16 / bfloat16, got {self.dtype}")

    def _key(self):
        p = next(self._tree.parameters())
        return (p.device, p.dtype, p.data_ptr())


class PoseGuider(_EngineModel):
    def __init__(self, conditioning_embedding_channels: int, conditioning_channels: int = 3,
                 block_out_channels: Tuple[int, ...] = (16, 32, 64, 128)):
        super().__init__()
        self._materialise(schema.pose_guider_schema(conditioning_embedding_channels, conditioning_channels,
                                                    block_out_channels))

    def engine(self) -> E.PoseGuiderEngine:
        self._require_cuda()
        if self._engine is None or self._engine_key != self._key():
            self._engine = E.PoseGuiderEngine(self.state_dict(), self.device, self.dtype)
            self._engine_key = self._key()
        return self._engine

    def forward_nhwc(self, conditioning: torch.Tensor) -> torch.Tensor:
        return self.engine().forward(conditioning)

    def forward(self, conditioning: torch.Tensor) -> torch.Tensor:
        """[b, 3, f, H, W] -> [b, C, f, H/8, W/8] (src/models/pose_guider.py:47-57)."""
        b, c, f, H, W = conditioning.shape
        y = self.forward_nhwc(conditioning)
        from .. import ops
        return ops.nhwc_to_ncfhw(y, b, y.shape[1], f, H // 8, W // 8)


@dataclass
class UNet3DConditionOutput:
    sample: torch.Tensor

    def __getitem__(self, i):
        return (self.sample,)[i]


class _UNetBase(_EngineModel):
    _motion = False
    _out_head = False

    def _init_unet(self, block_out_channels, layers_per_block, cross_attention_dim, attention_head_dim, norm_num_groups,
                   norm_eps, in_channels, out_channels, extra: dict, motion_max_len: int = 32):
        if isinstance(attention_head_dim, (tuple, list)):
            if len(set(attention_head_dim)) != 1:
                raise NotImplementedError("per-level attention_head_dim is not used by the reference's SD1.5 config")
            attention_head_dim = attention_head_dim[0]
        self.config = SimpleNamespace(block_out_channels=tuple(block_out_channels), layers_per_block=layers_per_block,
                                      cross_attention_dim=cross_attention_dim, attention_head_dim=attention_head_dim,
                                      norm_num_groups=norm_num_groups, norm_eps=norm_eps, in_channels=in_channels,
                                      out_channels=out_channels, center_input_sample=False, **extra)
        self._spec = E.UNetSpec(block_out_channels=tuple(block_out_channels), layers_per_block=layers_per_block,
                                heads=attention_head_dim, cross_attention_dim=cross_attention_dim,
                                norm_num_groups=norm_num_groups, norm_eps=norm_eps, in_channels=in_channels,
                                out_channels=out_channels, motion=self._motion, out_head=self._out_head)
        self._materialise(schema.unet_schema(block_out_channels, layers_per_block, cross_attention_dim, in_channels,
                                             out_channels, motion=self._motion, out_head=self._out_head,
                                             motion_max_len=motion_max_len))
        self._ref_mode: Optional[str] = None
        self._ref_cfg = False

    def engine(self) -> E.UNetEngine:
        self._require_cuda()
        if self._engine is None or self._engine_key != self._key():
            self._engine = E.UNetEngine(self.state_dict(), self._spec, self.device, self.dtype)
            self._engine_key = self._key()
        return self._engine

    @classmethod
    def _config_from_dir(cls, path, subfolder):
        p = Path(path)
        if subfolder is not None:
            p = p / subfolder
        cfg_file = p / "config.json"
        if not (cfg_file.exists() and cfg_file.is_file()):
            raise RuntimeError(f"{cfg_file} does not exist or is not a file")
        return p, json.loads(cfg_file.read_text())

    @staticmethod
    def _load_weights_file(p: Path):
        st = p / "diffusion_pytorch_model.safetensors"
        if st.exists():
            from safetensors.torch import load_file
            return load_file(str(st), device="cpu")
        pt = p / "diffusion_pytorch_model.bin"
        if pt.exists():
            return torch.load(pt, map_location="cpu", weights_only=True)
        raise FileNotFoundError(f"no weights file found in {p}")


class UNet2DConditionModel(_UNetBase):
    """The reference UNet: run once per clip at t = 0 to fill the banks (pipeline :480-490). Its output head is
    removed in the reference (unet_2d_condition.py:645-653, 1295-1299), so forward() returns nothing useful there
    either: the side effect (banks) is what counts."""

    def __init__(self, sample_size=None, in_channels=4, out_channels=4, block_out_channels=(320, 640, 1280, 1280),
                 layers_per_block=2, cross_attention_dim=1280, attention_head_dim=8, norm_num_groups=32, norm_eps=1e-5,
                 **unused):
        super().__init__()
        self._init_unet(block_out_channels, layers_per_block, cross_attention_dim, attention_head_dim, norm_num_groups,
                        norm_eps, in_channels, out_channels, dict(sample_size=sample_size))
        self._pending = None  # (latents, ehs) of the last write-mode forward

    @classmethod
    def from_pretrained(cls, path, subfolder=None, **kw):
        p, cfg = cls._config_from_dir(path, subfolder)
        keys = ("sample_size", "in_channels", "out_channels", "block_out_channels", "layers_per_block",
                "cross_attention_dim", "attention_head_dim", "norm_num_groups", "norm_eps")
        model = cls(**{k: cfg[k] for k in keys if k in cfg})
        sd = cls._load_weights_file(p)
        sd = {k: v for k, v in sd.items() if not k.startswith(("conv_norm_out.", "conv_out."))}
        model.load_state_dict(sd, strict=True)
        return model

    def forward(self, sample, timestep, encoder_hidden_states=None, return_dict: bool = True, **unused):
        self._require_cuda()
        if self._ref_mode != "write":
            raise MimoError("UNet2DConditionModel is only executed as the reference ('write') network; wrap it in "
                            "ReferenceAttentionControl(mode='write') first (pipeline :393-399)")
        t = timestep if torch.is_tensor(timestep) else torch.tensor(timestep)
        if int(t.reshape(-1)[0]) != 0:
            raise MimoError("the reference network is evaluated at timestep 0 only (pipeline :481-489)")
        self._pending = (sample, encoder_hidden_states)
        out = sample  # the reference's return value is unused (pipeline :481-489)
        return SimpleNamespace(sample=out) if return_dict else (out,)


class UNet3DConditionModel(_UNetBase):
    _motion = True
    _out_head = True

    def __init__(self, sample_size=None, in_channels=4, out_channels=4, center_input_sample=False, flip_sin_to_cos=True,
                 freq_shift=0, down_block_types=None, mid_block_type="UNetMidBlock3DCrossAttn", up_block_types=None,
                 only_cross_attention=False, block_out_channels=(320, 640, 1280, 1280), layers_per_block=2,
                 downsample_padding=1, mid_block_scale_factor=1, act_fn="silu", norm_num_groups=32, norm_eps=1e-5,
                 cross_attention_dim=1280, attention_head_dim=8, dual_cross_attention=False,
                 use_linear_projection=False, class_embed_type=None, num_class_embeds=None, upcast_attention=False,
                 resnet_time_scale_shift="default", use_inflated_groupnorm=False, use_motion_module=False,
                 motion_module_resolutions=(1, 2, 4, 8), motion_module_mid_block=False,
                 motion_module_decoder_only=False, motion_module_type=None, motion_module_kwargs=None,
                 unet_use_cross_frame_attention=None, unet_use_temporal_attention=None):
        super().__init__()
        mk = dict(motion_module_kwargs or {})
        # the engine implements the reference's shipped inference configuration (configs/inference/inference_v2.yaml)
        unsupported = []
        if not (use_motion_module and motion_module_mid_block and not motion_module_decoder_only
                and tuple(motion_module_resolutions) == (1, 2, 4, 8) and motion_module_type == "Vanilla"):
            unsupported.append("motion-module placement other than inference_v2.yaml")
        if unet_use_cross_frame_attention or unet_use_temporal_attention:
            unsupported.append("unet_use_cross_frame_attention / unet_use_temporal_attention")
        if mk.get("num_attention_heads", 8) != attention_head_dim or mk.get("num_transformer_block", 1) != 1 \
                or list(mk.get("attention_block_types", ["Temporal_Self", "Temporal_Self"])) != ["Temporal_Self"] * 2 \
                or not mk.get("temporal_position_encoding", True) or mk.get("temporal_attention_dim_div", 1) != 1:
            unsupported.append("motion_module_kwargs other than inference_v2.yaml")
        if dual_cross_attention or use_linear_projection or class_embed_type or num_class_embeds or upcast_attention \
                or resnet_time_scale_shift != "default" or center_input_sample or not flip_sin_to_cos or freq_shift:
            unsupported.append("non-SD1.5 UNet options")
        if unsupported:
            raise NotImplementedError("mimo_b200.UNet3DConditionModel: " + "; ".join(unsupported))
        self._motion_max_len = mk.get("temporal_position_encoding_max_len", 32)
        self._init_unet(block_out_channels, layers_per_block, cross_attention_dim, attention_head_dim, norm_num_groups,
                        norm_eps, 8, out_channels,  # in_channels is forced to 8 (unet_3d_edit_bkfill.py:88)
                        dict(sample_size=sample_size), motion_max_len=self._motion_max_len)

    @classmethod
    def from_pretrained_2d(cls, pretrained_model_path, motion_module_path, subfolder=None,
                           unet_additional_kwargs=None, mm_zero_proj_out=False):
        """SD1.5 UNet weights + motion-module weights, conv_in zero-padded 4 -> 8 input channels
        (src/models/unet_3d_edit_bkfill.py:578-682)."""
        p, cfg = cls._config_from_dir(pretrained_model_path, subfolder)
        keys = ("sample_size", "out_channels", "block_out_channels", "layers_per_block", "cross_attention_dim",
                "attention_head_dim", "norm_num_groups", "norm_eps")
        model = cls(**{k: cfg[k] for k in keys if k in cfg}, **dict(unet_additional_kwargs or {}))
        sd = dict(cls._load_weights_file(p))
        mp = Path(motion_module_path)
        if mp.exists() and mp.is_file():
            if mp.suffix.lower() in (".pth", ".pt", ".ckpt"):
                msd = torch.load(mp, map_location="cpu", weights_only=True)
            elif mp.suffix.lower() == ".safetensors":
                from safetensors.torch import load_file
                msd = load_file(str(mp), device="cpu")
            else:
                raise RuntimeError(f"unknown file format for motion module weights: {mp.suffix}")
            if mm_zero_proj_out:
                msd = {k: v for k, v in msd.items() if "proj_out" not in k}
            sd.update(msd)
        w = sd["conv_in.weight"]
        if w.shape[1] != 8:
            sd["conv_in.weight"] = torch.cat([w, torch.zeros(w.shape[0], 8 - w.shape[1], *w.shape[2:], dtype=w.dtype)], 1)
        model.load_state_dict(sd, strict=False)
        return model

    def forward(self, sample, timestep, encoder_hidden_states, class_labels=None, pose_cond_fea=None,
                attention_mask=None, down_block_additional_residuals=None, mid_block_additional_residual=None,
                return_dict: bool = True):
        """[b, 8, f, h, w] -> [b, 4, f, h, w] (src/models/unet_3d_edit_bkfill.py:398-576)."""
        self._require_cuda()
        if attention_mask is not None or down_block_additional_residuals is not None \
                or mid_block_additional_residual is not None or class_labels is not None:
            raise NotImplementedError("attention_mask / additional residuals / class labels are unused by the reference "
                                      "pipeline and not implemented by the engine")
        eng = self.engine()
        if eng.clip_state is None:
            raise MimoError("denoising_unet.forward before ReferenceAttentionControl.update(): no reference banks")
        b, c, f, h, w = sample.shape
        # re-folded on every call (32 one-row GEMMs, ~0.4 % of a forward): neither data_ptr nor torch's version counter
        # identify the CONTENT of a tensor whose storage the caching allocator recycles, and a stale vector is silent
        eng.set_cross_attn(encoder_hidden_states)
        pose = None
        if pose_cond_fea is not None:
            from .. import ops
            pose = ops.ncfhw_to_nhwc(pose_cond_fea.contiguous(), pose_cond_fea.shape[1], self.dtype)
        out = eng.forward(sample, timestep, pose)
        return UNet3DConditionOutput(sample=out) if return_dict else (out,)


class ReferenceAttentionControl:
    """Same constructor / update / clear surface as src/models/mutual_self_attention.py:19-50, 313-374. The
    reference monkey-patches 16 + 16 transformer blocks; here the two modes are engine states:
      writer ("write"): reference_unet.forward records (latents, ehs)
      reader.update(writer): runs the reference UNet, projects every bank with the reader's to_k / to_v and arms
                             the denoising engine (banks are stored in fp16 there too, :349).
      clear(): drops the banks."""

    def __init__(self, unet, mode="write", do_classifier_free_guidance=False, attention_auto_machine_weight=float("inf"),
                 gn_auto_machine_weight=1.0, style_fidelity=1.0, reference_attn=True, reference_adain=False,
                 fusion_blocks="midup", batch_size=1):
        assert mode in ["read", "write"]
        assert fusion_blocks in ["midup", "full"]
        if fusion_blocks != "full" or not reference_attn or reference_adain:
            raise NotImplementedError("the engine implements fusion_blocks='full', reference_attn only (pipeline :393-406)")
        self.unet, self.mode, self.cfg = unet, mode, bool(do_classifier_free_guidance)
        unet._ref_mode, unet._ref_cfg = mode, self.cfg

    def update(self, writer: "ReferenceAttentionControl", dtype=torch.float16):
        if self.mode != "read" or writer.mode != "write":
            raise MimoError("update() is called on the reader with the writer as argument (pipeline :490)")
        pending = writer.unet._pending
        if pending is None:
            raise MimoError("update() before the reference UNet's forward pass")
        latents, ehs = pending
        den, ref = self.unet.engine(), writer.unet.engine()
        if self.cfg and latents.shape[0] == 2:
            # Only the conditional half of the reference pass is ever read: unconditional rows of the denoising UNet
            # skip the bank (mutual_self_attention.py:177-197), so the writer's unconditional half (which the reference
            # computes and stores, :137-147) is dead work here - the engine runs the conditional row alone.
            banks = ref.write_banks(latents[1:2].contiguous(), ehs[1:2].contiguous(), den)
        else:
            banks = ref.write_banks(latents, ehs, den)
        den.begin_clip(ehs, banks, cfg=self.cfg, frames=1, branches=getattr(self.unet, "_branches", None))

    def clear(self):
        eng = self.unet._engine
        if eng is not None:
            eng.clip_state = None
        if self.mode == "write":
            self.unet._pending = None


class AutoencoderKL(_EngineModel):
    """Stand-in for diffusers.AutoencoderKL (sd-vae-ft-mse) [3P] with the surface the pipeline touches:
    .config.block_out_channels, .encode(x).latent_dist.mean, .decode(z).sample, .dtype/.device, state_dict in the
    diffusers key layout. A real diffusers AutoencoderKL can be passed to the pipeline instead: only its state_dict
    and config are read."""

    def __init__(self, block_out_channels=(128, 256, 512, 512), layers_per_block=2, latent_channels=4, in_channels=3,
                 out_channels=3, norm_num_groups=32, scaling_factor=0.18215, **unused):
        super().__init__()
        self.config = SimpleNamespace(block_out_channels=tuple(block_out_channels), layers_per_block=layers_per_block,
                                      latent_channels=latent_channels, norm_num_groups=norm_num_groups,
                                      scaling_factor=scaling_factor)
        self._materialise(schema.vae_schema(block_out_channels, layers_per_block, latent_channels, in_channels,
                                            out_channels))

    @classmethod
    def from_pretrained(cls, path, subfolder=None, **unused):
        """diffusers layout: <path>/config.json + diffusion_pytorch_model.{safetensors,bin} (run_animate.py:70-72)."""
        p, cfg = _UNetBase._config_from_dir(path, subfolder)
        keys = ("block_out_channels", "layers_per_block", "latent_channels", "in_channels", "out_channels",
                "norm_num_groups", "scaling_factor")
        model = cls(**{k: cfg[k] for k in keys if k in cfg})
        model.load_state_dict(_UNetBase._load_weights_file(p), strict=True)
        return model

    def engine(self):
        self._require_cuda()
        if self._engine is None or self._engine_key != self._key():
            sd = self.state_dict()
            g = self.config.norm_num_groups
            self._engine = (E.VAEEncoderEngine(sd, self.device, self.dtype, g), E.VAEDecoderEngine(sd, self.device, self.dtype, g))
            self._engine_key = self._key()
        return self._engine

    def encode(self, x):
        mean = self.engine()[0].encode_mean(x)
        return SimpleNamespace(latent_dist=SimpleNamespace(mean=mean))

    def decode(self, z):
        return SimpleNamespace(sample=self.engine()[1].decode(z))
