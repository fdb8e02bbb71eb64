"""Motion-module layouts other than inference_v2.yaml's on the GPU: per layout of tests/golden/unet_motion_layouts.pt,
the engine's forward in fp16 and bf16 against the fp32 oracle (PyTorch in the same dtype sets the bar, as in
test_parity_gpu.py) with eager, captured and replayed forwards bit-identical; the temporal attention at the head widths
these layouts add; FP8 on two layouts; a two-window __call__ with the AnimateDiff-v1-style UNet against
oracle.sample_clip; and frame-sharded clips when the box has 2 GPUs."""
import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import gen_motion_layout_golden as GL

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
DEV = "cuda"
_NAMES = [c["name"] for c in GL.LAYOUTS]


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(golden_dir / "unet_motion_layouts.pt")


def _den_model(widths, kwargs):
    from mimo_b200.host import modules as M
    return M.UNet3DConditionModel(block_out_channels=widths, cross_attention_dim=768, use_motion_module=True,
                                  motion_module_type="Vanilla", **kwargs)


def _layout_case(golden, name, dtype, fp8=False):
    """(engine outputs: eager, eager -> capture, replay), PyTorch in `dtype`, the fp32 oracle (and its FP8 emulation)"""
    from mimo_b200 import engine as E
    from oracle import fp8_oracle as F8
    from oracle import motion_layout_oracle as ML
    from oracle import torch_oracle as O
    c = next(x for x in golden["cases"] if x["name"] == name)
    widths = tuple(golden["widths"])
    cfg = O.UNetConfig(block_out_channels=widths)
    lay = ML.Layout(**c["layout"])
    inflated = c["kwargs"]["use_inflated_groupnorm"]
    sd_den = ML.make_denoising_unet_sd(cfg, lay, c["seed"])
    sd_ref = O.make_reference_unet_sd(cfg, seed=c["seed"] + 1)
    ref_lat, ehs, x = c["ref_lat"], c["ehs"], c["x"].repeat(2, 1, 1, 1, 1)
    dev = torch.device(DEV)
    lo = lambda v: v.to(dtype)
    r32 = lambda sd: {k: lo(v).float().to(dev) for k, v in sd.items()}
    rlo = lambda sd: {k: lo(v).to(dev) for k, v in sd.items()}
    with torch.no_grad():
        want = GL.oracle_case(cfg, lay, inflated, r32(sd_den), r32(sd_ref), lo(ref_lat).float().to(dev),
                              lo(ehs).float().to(dev), lo(x).float().to(dev))
        want8 = None
        if fp8:
            with F8.fp8_emulation():
                want8 = GL.oracle_case(cfg, lay, inflated, r32(sd_den), r32(sd_ref), lo(ref_lat).float().to(dev),
                                       lo(ehs).float().to(dev), lo(x).float().to(dev), fp8=True)
        torch_lo = GL.oracle_case(cfg, lay, inflated, rlo(sd_den), rlo(sd_ref), lo(ref_lat).to(dev), lo(ehs).to(dev),
                                  lo(x).to(dev), bank_dtype=torch.float16 if dtype == torch.float16 else dtype).float()
    spec = _den_model(widths, c["kwargs"])._spec  # the layout as the public module reads the config
    assert spec.motion_layout.heads == lay.heads and spec.inflated_groupnorm == inflated
    den = E.UNetEngine(sd_den, spec, dev, dtype)
    ref = E.UNetEngine(sd_ref, E.UNetSpec(block_out_channels=widths, in_channels=4, motion=False, out_head=False), dev,
                       dtype)
    banks = ref.write_banks(lo(ref_lat).to(dev).repeat(2, 1, 1, 1), lo(ehs).to(dev), den)
    den.begin_clip(lo(ehs).to(dev), banks, cfg=True, frames=x.shape[2])
    run = lambda: den.forward(lo(x).to(dev), 499, None).float().clone()
    outs = [run() for _ in range(3)]  # eager, eager -> capture, replay
    outs8 = None
    if fp8:
        den.set_fp8(True)
        outs8 = [run() for _ in range(3)]
        den.set_fp8(False)
        outs8.append(run())  # back to the model dtype
    torch.cuda.synchronize()
    return dict(outs=outs, outs8=outs8, torch_lo=torch_lo, want=want, want8=want8, den=den)


@pytest.mark.parametrize("dtype,floor", [(torch.float16, 1e-3), (torch.bfloat16, 8e-3)], ids=["f16", "bf16"])
@pytest.mark.parametrize("name", _NAMES)
def test_layout_forward_vs_oracle(golden, name, dtype, floor):
    r = _layout_case(golden, name, dtype)
    outs, want = r["outs"], r["want"]
    assert outs[0].shape == (2, 4, golden["f"], golden["h"], golden["w"])
    e_eng, e_ref = _rel(outs[0], want), _rel(r["torch_lo"], want)
    print(f"UNet3D layout {name} {dtype}: engine {e_eng:.3e}  torch {e_ref:.3e} (vs the fp32 oracle)")
    assert e_eng <= max(floor, e_ref), (e_eng, e_ref)
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[1], outs[2])
    # the engine ran the layout: the module count of the forward is the layout's
    mms = [p for p in r["den"].w if ".motion_modules." in p]
    c = next(x for x in golden["cases"] if x["name"] == name)
    keys = {k.split(".temporal_transformer.")[0] for k in _den_model(tuple(golden["widths"]), c["kwargs"]).state_dict()
            if ".motion_modules." in k}
    assert sorted(mms) == sorted(keys)


@pytest.mark.parametrize("name", ["v1", "stress"])
def test_layout_fp8_forward(golden, name):
    """enable_fp8 on the layout: rel(engine_fp8, fp32) <= rel(oracle_fp8, fp32) + max(1e-3, e_ref), the bound of
    test_fp8_gpu.py; eager, capture and replay bit-identical; FP8 off again gives the fp16 bytes."""
    r = _layout_case(golden, name, torch.float16, fp8=True)
    e8, want = r["outs8"], r["want"]
    e_eng8, e_q, e_ref = _rel(e8[0], want), _rel(r["want8"], want), _rel(r["torch_lo"], want)
    print(f"UNet3D layout {name}: engine_fp8 {e_eng8:.3e}  oracle_fp8 {e_q:.3e}  torch-fp16 {e_ref:.3e} (vs the fp32 "
          f"oracle); engine_fp8 vs oracle_fp8 {_rel(e8[0], r['want8']):.3e}")
    assert torch.isfinite(e8[0]).all()
    assert e_eng8 <= e_q + max(1e-3, e_ref), (e_eng8, e_q, e_ref)
    assert torch.equal(e8[0], e8[1]) and torch.equal(e8[1], e8[2])
    assert torch.equal(e8[3], r["outs"][0])
    # one e4m3 copy per transformer block of every module, each with one q|k|v per attention block
    lay = r["den"].spec.motion_layout
    mms = [p for p in r["den"].w if ".motion_modules." in p]
    w8 = {k: v for k, v in r["den"].w8.items() if ".motion_modules." in k}
    assert len(w8) == len(mms) * lay.blocks and all(len(v["qkv"]) == lay.attn_blocks for v in w8.values())


def test_window_longer_than_the_pe_table_raises(golden):
    """v1's PE table has 24 rows: a 25-frame window fails as the reference does (motion_module.py:277-279), one without
    PE (stress) runs it."""
    from mimo_b200 import engine as E
    from mimo_b200.lib import MimoError
    from oracle import motion_layout_oracle as ML
    from oracle import torch_oracle as O
    widths = tuple(golden["widths"])
    cfg = O.UNetConfig(block_out_channels=widths)
    for name, ok in (("v1", False), ("stress", True)):
        c = next(x for x in golden["cases"] if x["name"] == name)
        den = E.UNetEngine(ML.make_denoising_unet_sd(cfg, ML.Layout(**c["layout"]), c["seed"]),
                           _den_model(widths, c["kwargs"])._spec, DEV)
        den.use_graphs = False
        den.begin_clip(c["ehs"].half().to(DEV), {}, cfg=True, frames=25)
        x = torch.randn(2, 8, 25, 8, 8, device=DEV).half()
        if ok:
            assert torch.isfinite(den.forward(x, 499, None).float()).all()
        else:
            with pytest.raises(MimoError, match="temporal_position_encoding_max_len=24"):
                den.forward(x, 499, None)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("heads,d", [(4, 32), (4, 64), (8, 16), (8, 64), (1, 256), (32, 8), (16, 40), (2, 160),
                                     (5, 224), (5, 256), (3, 96)], ids=lambda v: str(v))
def test_attn_temporal_at_layout_head_widths(heads, d, dtype):
    """mimo_attn_temporal at the head counts / widths motion layouts use (the stress layout's 4 heads of 32 and 64,
    omitted keys' 8 heads at reduced widths, the extremes, and odd head counts whose rows are too wide for one CTA to
    stage every head: 5 heads of 224 or 256 channels), 24 frames, against fp32 softmax attention."""
    from mimo_b200 import ops
    b, f, hw = 2, 24, 37
    C = heads * d
    g = torch.Generator().manual_seed(heads * 1000 + d)
    qkv = (torch.randn(b * f * hw, 3 * C, generator=g) * 1.5).to(dtype).to(DEV)
    q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    got = ops.attn_temporal(q, k, v, b, f, hw, heads).float()
    seq = lambda t: t.float().reshape(b, f, hw, heads, d).permute(0, 2, 3, 1, 4)  # [b, hw, heads, f, d]
    o = torch.nn.functional.scaled_dot_product_attention(seq(q), seq(k), seq(v))
    want = o.permute(0, 3, 1, 2, 4).reshape(b * f * hw, C)
    assert _rel(got, want) < (2e-3 if dtype == torch.float16 else 1.2e-2)


def _pipe(widths, sds, kwargs, seed):
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection

    from mimo_b200.host import modules as M
    from mimo_b200.host.pipeline import Pose2VideoPipeline
    from mimo_b200.host.scheduler import DDIMScheduler
    den = _den_model(widths, kwargs)
    ref = M.UNet2DConditionModel(block_out_channels=widths, cross_attention_dim=768)
    pg = M.PoseGuider(widths[0], 3, (16, 32, 96, 256))
    vae = M.AutoencoderKL()
    for m, k in ((den, "den"), (ref, "ref"), (pg, "pg"), (vae, "vae")):
        m.load_state_dict(sds[k], strict=True)
    torch.manual_seed(seed)
    clip = CLIPVisionModelWithProjection(CLIPVisionConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=2,
                                                          num_attention_heads=4, image_size=224, patch_size=32,
                                                          projection_dim=768)).eval()
    sched = DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
                          steps_offset=1, prediction_type="v_prediction", rescale_betas_zero_snr=True,
                          timestep_spacing="trailing")
    return Pose2VideoPipeline(vae=vae, image_encoder=clip, reference_unet=ref, denoising_unet=den, pose_guider=pg,
                              scheduler=sched).to(DEV, dtype=torch.float16)


def test_call_two_windows_v1_vs_oracle():
    """__call__ with the AnimateDiff-v1-style UNet (no mid-block module, PE table of 24, GroupNorm over the window): 26
    frames at 128 x 128 (two context windows), 2 DDIM steps, CFG 3.5, against oracle.sample_clip in fp32."""
    import PIL.Image

    from mimo_b200.host.pipeline import pil_to_tensor
    from oracle import motion_layout_oracle as ML
    from oracle import torch_oracle as O
    from oracle.window_gn_oracle import window_groupnorm
    case = next(c for c in GL.LAYOUTS if c["name"] == "v1")
    widths = GL.WIDTHS
    F_, size, steps, seed = 26, 128, 2, 960
    cfg, vcfg = O.UNetConfig(block_out_channels=widths), O.VAEConfig()
    sds = dict(den=ML.make_denoising_unet_sd(cfg, case["layout"], seed), ref=O.make_reference_unet_sd(cfg, seed + 1),
               pg=O.make_pose_guider_sd(seed + 2, widths[0]), vae=O.make_vae_sd(vcfg, seed + 3))
    pipe = _pipe(widths, sds, case["kwargs"], seed + 4)
    rng = np.random.RandomState(seed)
    ref_img = PIL.Image.fromarray(rng.randint(0, 256, (size, size, 3), dtype=np.uint8))
    poses, bks = [], []
    for i in range(F_):
        a = np.zeros((size, size, 3), np.uint8)
        a[size // 4: size // 2 + i % 8, size // 3: size // 3 + 20] = rng.randint(11, 256, 3)
        poses.append(PIL.Image.fromarray(a))
        bks.append(PIL.Image.fromarray(rng.randint(0, 256, (size, size, 3), dtype=np.uint8)))
    out = pipe(ref_img, poses, bks, size, size, F_, steps, 3.5, generator=torch.manual_seed(42))
    dev = torch.device(DEV)
    with torch.no_grad(), window_groupnorm(), ML.motion_layout(case["layout"]):
        emb = pipe._clip_embeds(ref_img).float()
        lat0 = torch.randn((1, 4, F_, size // 8, size // 8), generator=torch.manual_seed(42), dtype=torch.float16)
        args = lambda cast: (cast(pil_to_tensor(ref_img, size, size, True).to(dev)),
                             cast(pil_to_tensor(poses, size, size, False).permute(1, 0, 2, 3).unsqueeze(0).to(dev)),
                             cast(pil_to_tensor(bks, size, size, True).to(dev)))
        r32 = lambda sd: {k: v.half().float().to(dev) for k, v in sd.items()}
        h16 = lambda sd: {k: v.half().to(dev) for k, v in sd.items()}
        W = O.Weights(r32(sds["den"]), r32(sds["ref"]), r32(sds["pg"]), r32(sds["vae"]), cfg, vcfg)
        want = O.sample_clip(W, *args(lambda t: t), emb.half().float(), lat0.float().to(dev), steps, 3.5)
        del W
        W16 = O.Weights(h16(sds["den"]), h16(sds["ref"]), h16(sds["pg"]), h16(sds["vae"]), cfg, vcfg)
        t16 = O.sample_clip(W16, *args(lambda t: t.half()), emb.half(), lat0.to(dev), steps, 3.5)
    le, ve = _rel(pipe.last_latents, want["latents"]), _rel(out.videos, want["videos"])
    le16, ve16 = _rel(t16["latents"], want["latents"]), _rel(t16["videos"], want["videos"])
    print(f"clip 128x128x26f v1 layout: latents {le:.3e} videos {ve:.3e}   torch-fp16: {le16:.3e} {ve16:.3e}")
    assert le <= max(1e-3, le16) and ve <= max(1e-3, ve16), (le, ve, le16, ve16)


@pytest.mark.parametrize("layout", ["v1", "stress"])
def test_frame_sharded_layout_clip_equals_single_gpu(layout, tmp_path):
    """The layout's UNet partitioned over 2 GPUs (one exchange pair per motion module the layout has, window GroupNorm
    all-gathers for v1) vs un-sharded, eager / captured / replayed (scripts/mgpu_check.py --motion-layout). Needs 2
    GPUs on this box."""
    world = 2
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs, this box has {torch.cuda.device_count()}")
    out = tmp_path / "mgpu.json"
    port = 29800 + (os.getpid() + len(layout)) % 90
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
           "127.0.0.1", "--master-port", str(port), str(ROOT / "scripts" / "mgpu_check.py"), "--out", str(out),
           "--frames", "24", "48", "--motion-layout", layout]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, cwd=ROOT)
    print(r.stdout[-3000:], r.stderr[-3000:])
    assert r.returncode == 0, "sharded clip differs from the single-GPU clip (see stdout)"
    res = json.loads(out.read_text())
    assert res["ok"] and all(c["latents_rel_l2"] <= 5e-3 and c["videos_rel_l2"] <= 2e-3 for c in res["cases"])
