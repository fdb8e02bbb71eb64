"""The oracle (oracle/torch_oracle.py) at image sizes whose latents are not multiples of 2^(UNet levels - 1), and the
generator of the fixture that pins it against the reference's own modules at such a size.

oracle/torch_oracle.py upsamples with scale_factor=2, which is the reference's graph only when every level halves
exactly. The reference itself forwards the skip tensor's size to every upsampler when a latent side does not divide
(`forward_upsample_size`, src/models/unet_3d_edit_bkfill.py:427-435, 544-545; unet_2d_condition.py:946-955, 1269-1270;
F.interpolate(size=...) in resnet.py:75-77). `unet_body` below is torch_oracle._unet_body with that one difference, and
`forwarded_upsample_size()` makes torch_oracle's reference_unet_banks / denoising_unet / sample_clip use it. At sizes
that halve exactly both bodies compute the same thing.

Fixture:  MIMO_REFERENCE=<checkout of the original project> python scripts/oracle_any_size.py [--write]
runs the reference's UNet2D "write" pass -> ReferenceAttentionControl.update -> UNet3D "read" pass verbatim (on
oracle/diffusers_shim, fp32, CPU) at a 14 x 10 latent (levels 7 x 5, 4 x 3, 2 x 2), checks the oracle against it and,
with --write, stores tests/golden/unet_odd_read.pt. No other fixture is written.
"""
from __future__ import annotations

import argparse
import contextlib
import os
import sys
from pathlib import Path
from typing import Callable, Optional

import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from oracle import torch_oracle as O  # noqa: E402

ODD_CASE = dict(widths=(128, 256, 512, 512), f=4, h=14, w=10, seed=500)


def unet_body(sd, x: torch.Tensor, temb: torch.Tensor, cfg_: O.UNetConfig, xf_fn: Callable[[str, torch.Tensor], torch.Tensor],
              mm_fn: Optional[Callable[[str, torch.Tensor], torch.Tensor]], stop_after_last_attention: bool = False):
    """torch_oracle._unet_body, every upsampler interpolating to the size of the skip left on the stack."""
    g, eps = cfg_.norm_num_groups, cfg_.norm_eps
    nb = len(cfg_.block_out_channels)
    skips = [x]
    for i in range(nb):
        for j in range(cfg_.layers_per_block):
            x = O._tap(f"down_blocks.{i}.resnets.{j}", O.resnet_block(sd, f"down_blocks.{i}.resnets.{j}", x, temb, g, eps))
            if i < nb - 1:
                x = O._tap(f"down_blocks.{i}.attentions.{j}", xf_fn(f"down_blocks.{i}.attentions.{j}", x))
            if mm_fn is not None:
                x = O._tap(f"down_blocks.{i}.motion_modules.{j}", mm_fn(f"down_blocks.{i}.motion_modules.{j}", x))
            skips.append(x)
        if i < nb - 1:
            x = O._tap(f"down_blocks.{i}.down", O._conv(sd, f"down_blocks.{i}.downsamplers.0.conv", x, stride=2, padding=1))
            skips.append(x)
    x = O._tap("mid_block.resnets.0", O.resnet_block(sd, "mid_block.resnets.0", x, temb, g, eps))
    x = O._tap("mid_block.attentions.0", xf_fn("mid_block.attentions.0", x))
    if mm_fn is not None:
        x = O._tap("mid_block.motion_modules.0", mm_fn("mid_block.motion_modules.0", x))
    x = O._tap("mid_block.resnets.1", O.resnet_block(sd, "mid_block.resnets.1", x, temb, g, eps))
    for i in range(nb):
        for j in range(cfg_.layers_per_block + 1):
            x = torch.cat([x, skips.pop()], dim=1)
            x = O._tap(f"up_blocks.{i}.resnets.{j}", O.resnet_block(sd, f"up_blocks.{i}.resnets.{j}", x, temb, g, eps))
            if i > 0:
                x = O._tap(f"up_blocks.{i}.attentions.{j}", xf_fn(f"up_blocks.{i}.attentions.{j}", x))
            if mm_fn is not None:
                x = O._tap(f"up_blocks.{i}.motion_modules.{j}", mm_fn(f"up_blocks.{i}.motion_modules.{j}", x))
        if i < nb - 1:
            x = F.interpolate(x, size=tuple(skips[-1].shape[-2:]), mode="nearest")  # :544-545, resnet.py:75-77
            x = O._tap(f"up_blocks.{i}.up", O._conv(sd, f"up_blocks.{i}.upsamplers.0.conv", x))
    return x


@contextlib.contextmanager
def forwarded_upsample_size():
    """Within the block, torch_oracle's UNet functions (and sample_clip, which calls them) follow the skip sizes."""
    saved = O._unet_body
    O._unet_body = unet_body
    try:
        yield
    finally:
        O._unet_body = saved


def odd_case_inputs(cfg: O.UNetConfig, f: int, h: int, w: int, seed: int):
    """Seeded state dicts and inputs of the fixture case (the same draw order as pin_against_reference.unet_case)."""
    sds = (O.make_denoising_unet_sd(cfg, seed=seed), O.make_reference_unet_sd(cfg, seed=seed + 1),
           O.make_pose_guider_sd(seed=seed + 2, out_channels=cfg.block_out_channels[0]))
    g = torch.Generator().manual_seed(seed + 10)
    ref_lat = torch.randn(1, 4, h, w, generator=g)
    emb = torch.randn(1, 1, cfg.cross_attention_dim, generator=g)
    ehs = torch.cat([torch.zeros_like(emb), emb])
    x = torch.randn(1, 8, f, h, w, generator=g).repeat(2, 1, 1, 1, 1)
    pose_img = torch.rand(1, 3, f, h * 8, w * 8, generator=g)
    return sds, ref_lat, ehs, x, pose_img


def oracle_odd_case(cfg: O.UNetConfig, f: int, h: int, w: int, seed: int) -> torch.Tensor:
    (sd_den, sd_ref, sd_pg), ref_lat, ehs, x, pose_img = odd_case_inputs(cfg, f, h, w, seed)
    with torch.no_grad(), forwarded_upsample_size():
        banks = O.reference_unet_banks(sd_ref, ref_lat.repeat(2, 1, 1, 1), ehs, cfg)
        pose = O.pose_guider(sd_pg, pose_img)
        return O.denoising_unet(sd_den, x, 499, ehs, pose.repeat(2, 1, 1, 1, 1), banks, cfg, cfg=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--write", action="store_true", help="write tests/golden/unet_odd_read.pt")
    args = ap.parse_args()
    if not os.environ.get("MIMO_REFERENCE"):
        sys.exit(__doc__)
    sys.path.insert(0, str(ROOT / "oracle" / "diffusers_shim"))
    sys.path.insert(0, os.environ["MIMO_REFERENCE"])
    from oracle import pin_against_reference as PIN  # the reference's modules, built and loaded as for every fixture
    from src.models.mutual_self_attention import ReferenceAttentionControl
    torch.set_grad_enabled(False)
    c = ODD_CASE
    cfg = O.UNetConfig(block_out_channels=c["widths"])
    den, ref, pg = PIN.build_reference_models(cfg)
    (sd_den, sd_ref, sd_pg), ref_lat, ehs, x, pose_img = odd_case_inputs(cfg, c["f"], c["h"], c["w"], c["seed"])
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
    got = oracle_odd_case(cfg, c["f"], c["h"], c["w"], c["seed"])
    PIN.check(f"denoising_unet read-mode, widths {c['widths']}, f={c['f']}, latent {c['h']}x{c['w']} "
              "(forward_upsample_size)", got, want, 2e-5)
    if args.write:
        out = ROOT / "tests" / "golden" / "unet_odd_read.pt"
        torch.save({"cfg": list(c["widths"]), "seed": c["seed"], "f": c["f"], "h": c["h"], "w": c["w"],
                    "out": want.half()}, out)
        print("wrote", out)


if __name__ == "__main__":
    main()
