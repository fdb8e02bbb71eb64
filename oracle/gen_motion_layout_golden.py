"""Fixture of the denoising UNet3D with motion-module layouts other than inference_v2.yaml's, run by the reference's own
modules.

Usage:  MIMO_REFERENCE=<checkout of the original project> python oracle/gen_motion_layout_golden.py [--write]

Same recipe as oracle/pin_against_reference.py: the reference's src/** verbatim on oracle/diffusers_shim, fp32 on CPU,
UNet2D "write" pass -> ReferenceAttentionControl.update -> UNet3D "read" pass with 2 CFG branches, for each layout of
LAYOUTS at reduced widths with seeded weights (oracle/motion_layout_oracle.py makes them). The state dict is loaded
with strict=True, so the reference's key set is the oracle's. Checks the oracle against the reference and, with --write,
stores per layout the constructor arguments, the inputs, the reference's fp32 output and its sorted state-dict keys
(zlib-compressed, newline-joined) in tests/golden/unet_motion_layouts.pt.
"""
from __future__ import annotations

import argparse
import os
import sys
import zlib
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from oracle import motion_layout_oracle as ML  # noqa: E402
from oracle import torch_oracle as O  # noqa: E402
from oracle import window_gn_oracle as WG  # noqa: E402

WIDTHS = (128, 256, 512, 512)
F_, H, W = 4, 8, 8
_V2_KW = dict(num_attention_heads=8, num_transformer_block=1, attention_block_types=["Temporal_Self", "Temporal_Self"],
              temporal_position_encoding=True, temporal_position_encoding_max_len=32, temporal_attention_dim_div=1)
# each: UNet3DConditionModel keyword arguments beyond the SD1.5 ones, the layout they mean, a seed
LAYOUTS = [
    # AnimateDiff v1 inference config: no mid-block module, PE table of 24, plain GroupNorm over the window
    dict(name="v1", seed=1100, kwargs=dict(use_inflated_groupnorm=False, motion_module_mid_block=False,
                                            motion_module_kwargs=dict(_V2_KW, temporal_position_encoding_max_len=24)),
         layout=ML.Layout(mid_block=False, max_len=24)),
    # AnimateDiff v3: no mid-block module, per-frame GroupNorm
    dict(name="v3", seed=1200, kwargs=dict(use_inflated_groupnorm=True, motion_module_mid_block=False,
                                            motion_module_kwargs=_V2_KW),
         layout=ML.Layout(mid_block=False)),
    # decoder-only at the two finest resolutions, 2 transformer blocks of 3 attentions, no PE, 4 heads
    dict(name="stress", seed=1300,
         kwargs=dict(use_inflated_groupnorm=True, motion_module_mid_block=True, motion_module_decoder_only=True,
                     motion_module_resolutions=[1, 2],
                     motion_module_kwargs=dict(num_attention_heads=4, num_transformer_block=2,
                                               attention_block_types=["Temporal_Self"] * 3,
                                               temporal_position_encoding=False)),
         layout=ML.Layout(resolutions=(1, 2), decoder_only=True, blocks=2, attn_blocks=3, pe=False, max_len=24,
                          heads=4)),
    # every optional motion_module_kwargs key left out: VanillaTemporalModule's defaults (2 blocks, no PE, max_len 24)
    dict(name="omitted", seed=1400, kwargs=dict(use_inflated_groupnorm=True, motion_module_mid_block=True,
                                                 motion_module_kwargs={}),
         layout=ML.Layout(blocks=2, pe=False, max_len=24)),
]


def case_inputs(cfg: O.UNetConfig, seed: int):
    g = torch.Generator().manual_seed(seed + 10)
    ref_lat = torch.randn(1, 4, H, W, generator=g)
    emb = torch.randn(1, 1, cfg.cross_attention_dim, generator=g)
    ehs = torch.cat([torch.zeros_like(emb), emb])
    x = torch.randn(1, 8, F_, H, W, generator=g).repeat(2, 1, 1, 1, 1)
    return ref_lat, ehs, x


def oracle_case(cfg: O.UNetConfig, lay: ML.Layout, inflated: bool, sd_den, sd_ref, ref_lat, ehs, x,
                bank_dtype=torch.float16, fp8: bool = False) -> torch.Tensor:
    """UNet2D write -> UNet3D read of the layout's network, no pose features (every up step doubles at 8 x 8).
    fp8: the motion modules' LN-fed projections in FP8 (the spatial ones need fp8_oracle.fp8_emulation() around)."""
    with torch.no_grad(), ML.motion_layout(lay, fp8):
        banks = O.reference_unet_banks(sd_ref, ref_lat.repeat(2, 1, 1, 1), ehs, cfg, bank_dtype=bank_dtype)
        if inflated:
            return O.denoising_unet(sd_den, x, 499, ehs, None, banks, cfg, cfg=True)
        with WG.window_groupnorm():
            return O.denoising_unet(sd_den, x, 499, ehs, None, banks, cfg, cfg=True)


def reference_case(PIN, cfg: O.UNetConfig, kwargs: dict, sd_den, sd_ref, ref_lat, ehs, x):
    from src.models.mutual_self_attention import ReferenceAttentionControl
    from src.models.unet_3d_edit_bkfill import UNet3DConditionModel
    _, ref, _ = PIN.build_reference_models(cfg)
    common = dict(sample_size=64, in_channels=4, out_channels=4, block_out_channels=tuple(cfg.block_out_channels),
                  layers_per_block=cfg.layers_per_block, cross_attention_dim=cfg.cross_attention_dim,
                  attention_head_dim=cfg.heads, norm_num_groups=cfg.norm_num_groups, norm_eps=cfg.norm_eps,
                  flip_sin_to_cos=True, freq_shift=0, unet_use_cross_frame_attention=False,
                  unet_use_temporal_attention=False, use_motion_module=True, motion_module_type="Vanilla")
    den = UNet3DConditionModel(**common, **kwargs).eval()
    keys = sorted(den.state_dict().keys())
    den.load_state_dict(sd_den, strict=True)
    ref.load_state_dict(sd_ref, strict=True)
    t = torch.tensor(499)
    writer = ReferenceAttentionControl(ref, do_classifier_free_guidance=True, mode="write", batch_size=1,
                                       fusion_blocks="full")
    reader = ReferenceAttentionControl(den, do_classifier_free_guidance=True, mode="read", batch_size=1,
                                       fusion_blocks="full")
    ref(ref_lat.repeat(2, 1, 1, 1), torch.zeros_like(t), encoder_hidden_states=ehs, return_dict=False)
    reader.update(writer)
    want = den(x, t, encoder_hidden_states=ehs, return_dict=False)[0]
    reader.clear()
    writer.clear()
    return want, keys


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--write", action="store_true", help="write tests/golden/unet_motion_layouts.pt")
    args = ap.parse_args()
    if not os.environ.get("MIMO_REFERENCE"):
        sys.exit(__doc__)
    sys.path.insert(0, str(ROOT / "oracle" / "diffusers_shim"))
    sys.path.insert(0, os.environ["MIMO_REFERENCE"])
    from oracle import pin_against_reference as PIN  # the reference's modules, built and loaded as for every fixture
    torch.set_grad_enabled(False)
    cfg = O.UNetConfig(block_out_channels=WIDTHS)
    out = {"widths": list(WIDTHS), "f": F_, "h": H, "w": W, "cases": []}
    for c in LAYOUTS:
        lay, inflated = c["layout"], c["kwargs"]["use_inflated_groupnorm"]
        sd_den = ML.make_denoising_unet_sd(cfg, lay, c["seed"])
        sd_ref = O.make_reference_unet_sd(cfg, seed=c["seed"] + 1)
        ref_lat, ehs, x = case_inputs(cfg, c["seed"])
        want, keys = reference_case(PIN, cfg, c["kwargs"], sd_den, sd_ref, ref_lat, ehs, x)
        got = oracle_case(cfg, lay, inflated, sd_den, sd_ref, ref_lat, ehs, x)
        PIN.check(f"denoising_unet read-mode, layout {c['name']}", got, want, 2e-5)
        out["cases"].append(dict(name=c["name"], seed=c["seed"], kwargs=c["kwargs"], layout=vars(lay).copy(),
                                 ref_lat=ref_lat.clone(), ehs=ehs.clone(), x=x[:1].clone(), out=want.float().clone(),
                                 keys_zlib=zlib.compress("\n".join(keys).encode(), 9), n_keys=len(keys)))
    if args.write:
        path = ROOT / "tests" / "golden" / "unet_motion_layouts.pt"
        torch.save(out, path)
        print("wrote", path, path.stat().st_size, "bytes")


if __name__ == "__main__":
    main()
