"""Fixture of the denoising UNet3D built with use_inflated_groupnorm=False, run by the reference's own modules.

With the flag off, every ResnetBlock3D builds norm1 / norm2 as a plain torch.nn.GroupNorm, and so does conv_norm_out
(src/models/resnet.py:155-163, 185-192; src/models/unet_3d_edit_bkfill.py:236-247): on the [b, C, f, h, w] video tensor
its statistics cover every frame of a CFG branch. The GroupNorms of Transformer3DModel and of the motion module stay
per frame (transformer_3d.py:115-124, motion_module.py:151-156).

Usage:  MIMO_REFERENCE=<checkout of the original project> python oracle/gen_clip_gn_golden.py [--write]

Same recipe as oracle/pin_against_reference.py: the reference's src/** verbatim on oracle/diffusers_shim, fp32 on CPU,
UNet2D "write" pass -> ReferenceAttentionControl.update -> UNet3D "read" pass with 2 CFG branches. Two cases:
  * 16 x 16 latent, 4 frames (every up step doubles exactly);
  * 14 x 10 latent, 3 frames (levels 7 x 5, 4 x 3, 2 x 2: the up steps take the forward_upsample_size path, as
    784 x 784 images do).
Checks oracle/window_gn_oracle.py against both and, with --write, stores the reference's fp32 outputs in
tests/golden/unet_clip_gn_read.pt.
"""
from __future__ import annotations

import argparse
import os
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from oracle import torch_oracle as O  # noqa: E402
from oracle import window_gn_oracle as WG  # noqa: E402
from scripts import oracle_any_size as OA  # noqa: E402

WIDTHS = (128, 256, 512, 512)
CASES = [dict(name="even", f=4, h=16, w=16, seed=700), dict(name="odd", f=3, h=14, w=10, seed=710)]


def oracle_case(cfg: O.UNetConfig, f: int, h: int, w: int, seed: int, window: bool = True) -> torch.Tensor:
    """The oracle's UNet2D-write -> UNet3D-read output of one case (forwarded upsample sizes: the same graph as the
    scale-factor body wherever every level halves exactly); window=False: the per-frame (inflated) network."""
    if not window:
        return OA.oracle_odd_case(cfg, f, h, w, seed)
    with WG.window_groupnorm():
        return OA.oracle_odd_case(cfg, f, h, w, seed)


def reference_case(PIN, cfg: O.UNetConfig, f: int, h: int, w: int, seed: int) -> torch.Tensor:
    from src.models.mutual_self_attention import ReferenceAttentionControl
    from src.models.unet_3d_edit_bkfill import UNet3DConditionModel
    _, ref, pg = PIN.build_reference_models(cfg)
    common = dict(sample_size=64, in_channels=4, out_channels=4, block_out_channels=tuple(cfg.block_out_channels),
                  layers_per_block=cfg.layers_per_block, cross_attention_dim=cfg.cross_attention_dim,
                  attention_head_dim=cfg.heads, norm_num_groups=cfg.norm_num_groups, norm_eps=cfg.norm_eps,
                  flip_sin_to_cos=True, freq_shift=0)
    den = UNet3DConditionModel(**common, **dict(PIN.UNET_EXTRA, use_inflated_groupnorm=False)).eval()
    assert type(den.conv_norm_out) is torch.nn.GroupNorm
    (sd_den, sd_ref, sd_pg), ref_lat, ehs, x, pose_img = OA.odd_case_inputs(cfg, f, h, w, seed)
    den.load_state_dict(sd_den, strict=True)
    ref.load_state_dict(sd_ref, strict=True)
    pg.load_state_dict(sd_pg, strict=True)
    t = torch.tensor(499)
    writer = ReferenceAttentionControl(ref, do_classifier_free_guidance=True, mode="write", batch_size=1,
                                       fusion_blocks="full")
    reader = ReferenceAttentionControl(den, do_classifier_free_guidance=True, mode="read", batch_size=1,
                                       fusion_blocks="full")
    ref(ref_lat.repeat(2, 1, 1, 1), torch.zeros_like(t), encoder_hidden_states=ehs, return_dict=False)
    reader.update(writer)
    want = den(x, t, encoder_hidden_states=ehs, pose_cond_fea=pg(pose_img).repeat(2, 1, 1, 1, 1), return_dict=False)[0]
    reader.clear()
    writer.clear()
    return want


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--write", action="store_true", help="write tests/golden/unet_clip_gn_read.pt")
    args = ap.parse_args()
    if not os.environ.get("MIMO_REFERENCE"):
        sys.exit(__doc__)
    sys.path.insert(0, str(ROOT / "oracle" / "diffusers_shim"))
    sys.path.insert(0, os.environ["MIMO_REFERENCE"])
    from oracle import pin_against_reference as PIN  # the reference's modules, built and loaded as for every fixture
    torch.set_grad_enabled(False)
    cfg = O.UNetConfig(block_out_channels=WIDTHS)
    out = {"cfg": list(WIDTHS), "cases": []}
    for c in CASES:
        want = reference_case(PIN, cfg, c["f"], c["h"], c["w"], c["seed"])
        got = oracle_case(cfg, c["f"], c["h"], c["w"], c["seed"])
        PIN.check(f"denoising_unet read-mode, use_inflated_groupnorm=False, f={c['f']}, latent {c['h']}x{c['w']}",
                  got, want, 2e-5)
        # the per-frame network is a different one: the fixture must tell the two apart
        per_frame = oracle_case(cfg, c["f"], c["h"], c["w"], c["seed"], window=False)
        print(f"       per-frame GroupNorm differs from it by rel_l2 = {PIN.rel(per_frame, want):.3e}")
        out["cases"].append(dict(c, out=want.float().clone()))
    if args.write:
        path = ROOT / "tests" / "golden" / "unet_clip_gn_read.pt"
        torch.save(out, path)
        print("wrote", path)


if __name__ == "__main__":
    main()
