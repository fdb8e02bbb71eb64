"""Window-mode GroupNorm (use_inflated_groupnorm=False) on the GPU: the kernel against fp64 torch.nn.GroupNorm on
[b, C, f, h, w], emulated frame shards (bit-identical by construction), graph capture, a whole UNet3D forward and a
two-window __call__ against the fp32 oracle (PyTorch-fp16's own error sets the bar, as in test_parity_gpu.py), and the
per-frame network byte-identical to the previous version (tests/golden/inflated_groupnorm_digests.json)."""
import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
DEV = "cuda"
WIDTHS = (128, 256, 512, 512)


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())


def _video(b, c, f, h, w, dtype, seed, offset=0.0):
    """Channels-last [b * f * h * w, c] activations and the same values as an fp64 [b, c, f, h, w] tensor; `offset`
    adds a mean that differs per frame (mean >> std: the shifted sums must not cancel)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, f, h * w, c, generator=g) * 1.5 + 0.3
    if offset:
        x = x + offset * (1 + torch.arange(f, dtype=torch.float32).view(1, f, 1, 1) / f)
    x = x.to(dtype)
    return x.reshape(b * f * h * w, c).to(DEV), x.double().reshape(b, f, h, w, c).permute(0, 4, 1, 2, 3)


def _affine(c, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    return ((torch.rand(c, generator=g) + 0.5).to(dtype).to(DEV), (torch.randn(c, generator=g) * 0.2).to(dtype).to(DEV))


def _want(x64, gamma, beta, groups, eps, silu):
    y = torch.nn.functional.group_norm(x64, groups, gamma.double().cpu(), beta.double().cpu(), eps)
    return torch.nn.functional.silu(y) if silu else y


def _nhwc(y):  # [b, c, f, h, w] -> [b * f * h * w, c]
    b, c = y.shape[:2]
    return y.permute(0, 2, 3, 4, 1).reshape(-1, c)


_SHAPES = [  # (h, w, c0, c1): 512 x 512 latent levels and a 98-wide latent; concat at 960 and 1920 channels
    (64, 64, 320, 0), (32, 32, 640, 320), (16, 16, 1280, 640), (98, 98, 320, 0), (25, 25, 1280, 640), (13, 13, 1280, 1280)]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("h,w,c0,c1", _SHAPES, ids=lambda v: str(v))
def test_window_groupnorm_vs_fp64(h, w, c0, c1, dtype):
    from mimo_b200 import ops
    b, f, groups, eps = 2, 6, 32, 1e-5
    c = c0 + c1
    x, x64 = _video(b, c, f, h, w, dtype, seed=h * 7 + c)
    gamma, beta = _affine(c, dtype, seed=c)
    tol = 2e-3 if dtype == torch.float16 else 1e-2
    for silu in (False, True):
        want = _nhwc(_want(x64, gamma, beta, groups, eps, silu))
        if c1:
            x0, x1 = x[:, :c0].contiguous(), x[:, c0:].contiguous()
            got = ops.groupnorm_window(x0, gamma, beta, b, f, h * w, groups=groups, eps=eps, silu=silu, x1=x1)
        else:
            got = ops.groupnorm_window(x, gamma, beta, b, f, h * w, groups=groups, eps=eps, silu=silu)
        e = _rel(got.cpu(), want)
        # the output is rounded once to the storage type: the error is that rounding
        assert e < tol / 4, (silu, e)
        assert float((got.cpu().double() - want).abs().max()) < tol * float(want.abs().max()), silu


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_window_groupnorm_offset_frames(dtype):
    """Every frame has its own mean, 30-60 std away from zero: the records' K_g shifts are moved to frame 0's exactly
    enough that the variance does not cancel."""
    from mimo_b200 import ops
    b, f, h, w, c = 2, 8, 16, 16, 320
    x, x64 = _video(b, c, f, h, w, dtype, seed=5, offset=40.0)
    gamma, beta = _affine(c, dtype, seed=6)
    want = _nhwc(_want(x64, gamma, beta, 32, 1e-6, False))
    got = ops.groupnorm_window(x, gamma, beta, b, f, h * w, groups=32, eps=1e-6)
    assert _rel(got.cpu(), want) < (5e-4 if dtype == torch.float16 else 4e-3)


@pytest.mark.parametrize("h,w,c0,c1", [(64, 64, 320, 0), (25, 25, 1280, 640), (13, 13, 640, 1280)], ids=str)
def test_emulated_shards_are_bit_identical(h, w, c0, c1):
    """Partials of G = 2 / 4 / 8 frame slices, concatenated, applied slice by slice: the same bytes as one call."""
    from mimo_b200 import ops
    b, f = 2, 8
    c = c0 + c1
    x, _ = _video(b, c, f, h, w, torch.float16, seed=9)
    gamma, beta = _affine(c, torch.float16, seed=10)
    x0, x1 = x[:, :c0].contiguous(), (x[:, c0:].contiguous() if c1 else None)
    kw = dict(groups=32, eps=1e-5, silu=True)
    whole = ops.groupnorm_window(x0, gamma, beta, b, f, h * w, x1=x1, **kw)
    hw = h * w
    sl = lambda t, k, fl: None if t is None else t.view(b, f, hw, -1)[:, k * fl:(k + 1) * fl].reshape(-1, t.shape[1]).contiguous()
    for G in (2, 4, 8):
        fl = f // G
        tables = [ops.groupnorm_window_partials(sl(x0, k, fl), b, fl, hw, groups=32, x1=sl(x1, k, fl)) for k in range(G)]
        table = torch.cat(tables)
        assert torch.equal(table, ops.groupnorm_window_partials(x0, b, f, hw, groups=32, x1=x1))
        for k in range(G):
            part = ops.groupnorm_window_apply(sl(x0, k, fl), gamma, beta, table, b, fl, f, hw, x1=sl(x1, k, fl), **kw)
            assert torch.equal(part.view(b, fl, hw, c), whole.view(b, f, hw, c)[:, k * fl:(k + 1) * fl]), (G, k)


def test_window_groupnorm_in_a_cuda_graph():
    from mimo_b200 import ops
    b, f, h, w, c = 2, 6, 32, 32, 640
    x, _ = _video(b, c, f, h, w, torch.float16, seed=11)
    gamma, beta = _affine(c, torch.float16, seed=12)
    eager = ops.groupnorm_window(x, gamma, beta, b, f, h * w, silu=True)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        table = ops.groupnorm_window_partials(x, b, f, h * w)
        out = ops.groupnorm_window_apply(x, gamma, beta, table, b, f, f, h * w, silu=True)
        out2 = ops.groupnorm_window(x, gamma, beta, b, f, h * w, silu=True)
    for _ in range(2):
        out.zero_()
        out2.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, eager) and torch.equal(out2, eager)


# ------------------------------------------------------------------------------------------------
# whole networks against the fp32 oracle
# ------------------------------------------------------------------------------------------------
def _unet_case(f, h, w, seed, dtype):
    from mimo_b200 import engine as E
    from oracle import torch_oracle as O
    from oracle.window_gn_oracle import window_groupnorm
    from scripts.oracle_any_size import forwarded_upsample_size, odd_case_inputs
    dev = torch.device(DEV)
    cfg = O.UNetConfig(block_out_channels=WIDTHS)
    (sd_den, sd_ref, sd_pg), ref_lat, ehs, x, pose_img = odd_case_inputs(cfg, f, h, w, seed)
    lo = lambda v: v.to(dtype)
    r32 = lambda sd: {k: lo(v).float().to(dev) for k, v in sd.items()}
    rlo = lambda sd: {k: lo(v).to(dev) for k, v in sd.items()}
    t = 499
    with torch.no_grad(), forwarded_upsample_size(), window_groupnorm():
        o_banks = O.reference_unet_banks(r32(sd_ref), lo(ref_lat).float().to(dev).repeat(2, 1, 1, 1),
                                         lo(ehs).float().to(dev), cfg)
        o_pose = O.pose_guider(r32(sd_pg), lo(pose_img).float().to(dev))
        want = O.denoising_unet(r32(sd_den), lo(x).float().to(dev), t, lo(ehs).float().to(dev),
                                o_pose.repeat(2, 1, 1, 1, 1), o_banks, cfg, cfg=True)
        l_banks = O.reference_unet_banks(rlo(sd_ref), lo(ref_lat).to(dev).repeat(2, 1, 1, 1), lo(ehs).to(dev), cfg,
                                         bank_dtype=torch.float16 if dtype == torch.float16 else dtype)
        l_pose = O.pose_guider(rlo(sd_pg), lo(pose_img).to(dev))
        torch_lo = O.denoising_unet(rlo(sd_den), lo(x).to(dev), t, lo(ehs).to(dev), l_pose.repeat(2, 1, 1, 1, 1),
                                    l_banks, cfg, cfg=True).float()
    den = E.UNetEngine(sd_den, E.UNetSpec(block_out_channels=WIDTHS, inflated_groupnorm=False), dev, dtype)
    ref = E.UNetEngine(sd_ref, E.UNetSpec(block_out_channels=WIDTHS, in_channels=4, motion=False, out_head=False), dev,
                       dtype)
    pg = E.PoseGuiderEngine(sd_pg, dev, dtype)
    banks = ref.write_banks(lo(ref_lat).to(dev).repeat(2, 1, 1, 1), lo(ehs).to(dev), den)  # one row per CFG branch
    den.begin_clip(lo(ehs).to(dev), banks, cfg=True, frames=f)
    pose = pg.forward(lo(pose_img).to(dev))
    pose2 = pose.reshape(1, f * h * w, -1).repeat(2, 1, 1).reshape(2 * f * h * w, -1).contiguous()
    outs = [den.forward(lo(x).to(dev), t, pose2).float().clone() for _ in range(3)]  # eager, eager->capture, replay
    torch.cuda.synchronize()
    return outs, torch_lo, want


@pytest.mark.parametrize("f,h,w,seed,dtype,floor", [
    (8, 16, 16, 760, torch.float16, 1e-3),
    (3, 14, 10, 770, torch.float16, 1e-3),   # forward_upsample_size path (784 x 784-style odd latent)
    (6, 16, 16, 780, torch.bfloat16, 8e-3),
], ids=["f8_16x16_f16", "f3_14x10_f16", "f6_16x16_bf16"])
def test_unet_forward_vs_oracle(f, h, w, seed, dtype, floor):
    outs, torch_lo, want = _unet_case(f, h, w, seed, dtype)
    assert outs[0].shape == (2, 4, f, h, w)
    e_eng, e_ref = _rel(outs[0], want), _rel(torch_lo, want)
    print(f"UNet3D window GroupNorm f={f} {h}x{w} {dtype}: engine {e_eng:.3e}  torch {e_ref:.3e} (vs the fp32 oracle)")
    assert e_eng <= max(floor, e_ref), (e_eng, e_ref)
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[1], outs[2])


def _pipe(widths, sds, inflated, seed):
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection

    from mimo_b200.host import modules as M
    from mimo_b200.host.pipeline import Pose2VideoPipeline
    from mimo_b200.host.scheduler import DDIMScheduler
    mk = dict(num_attention_heads=8, num_transformer_block=1, attention_block_types=["Temporal_Self", "Temporal_Self"],
              temporal_position_encoding=True, temporal_position_encoding_max_len=32, temporal_attention_dim_div=1)
    den = M.UNet3DConditionModel(block_out_channels=widths, cross_attention_dim=768, use_inflated_groupnorm=inflated,
                                 use_motion_module=True, motion_module_mid_block=True, motion_module_type="Vanilla",
                                 motion_module_kwargs=mk)
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


def test_call_two_windows_vs_oracle():
    """__call__ with use_inflated_groupnorm=False: 26 frames at 128 x 128 (two context windows, each normalised over its
    own 24 frames), 2 DDIM steps, CFG 3.5, against oracle.sample_clip in fp32 with the window network swapped in."""
    import PIL.Image

    from mimo_b200.host.pipeline import pil_to_tensor
    from oracle import torch_oracle as O
    from oracle.window_gn_oracle import window_groupnorm
    F_, size, steps, seed = 26, 128, 2, 950
    cfg, vcfg = O.UNetConfig(block_out_channels=WIDTHS), O.VAEConfig()
    sds = dict(den=O.make_denoising_unet_sd(cfg, seed), ref=O.make_reference_unet_sd(cfg, seed + 1),
               pg=O.make_pose_guider_sd(seed + 2, WIDTHS[0]), vae=O.make_vae_sd(vcfg, seed + 3))
    pipe = _pipe(WIDTHS, sds, False, seed + 4)
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
    with torch.no_grad(), window_groupnorm():
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
    print(f"clip 128x128x26f window GroupNorm: latents {le:.3e} videos {ve:.3e}   torch-fp16: {le16:.3e} {ve16:.3e}")
    assert le <= max(1e-3, le16) and ve <= max(1e-3, ve16), (le, ve, le16, ve16)


def test_flag_on_is_byte_identical_to_previous_version():
    """use_inflated_groupnorm=True: a seeded two-window __call__ and an engine forward (eager, capture, replay) give the
    bytes the previous version gave (digests written by scripts/window_gn_digests.py from that version's build)."""
    sys.path.insert(0, str(ROOT))
    from scripts.window_gn_digests import digests
    want = json.loads((ROOT / "tests" / "golden" / "inflated_groupnorm_digests.json").read_text())
    assert digests() == want


@pytest.mark.parametrize("world", [2, 4])
def test_frame_sharded_window_clip_equals_single_gpu(world, tmp_path):
    """use_inflated_groupnorm=False partitioned over `world` GPUs (frame groups all-gather the partial tables over peer
    memory) vs un-sharded (scripts/mgpu_check.py --window-groupnorm). Needs `world` GPUs on this box."""
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs, this box has {torch.cuda.device_count()}")
    out = tmp_path / "mgpu.json"
    port = 29900 + (os.getpid() + world) % 90
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
           "127.0.0.1", "--master-port", str(port), str(ROOT / "scripts" / "mgpu_check.py"), "--out", str(out),
           "--frames", "24", "48", "--window-groupnorm"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, cwd=ROOT)
    print(r.stdout[-3000:], r.stderr[-3000:])
    assert r.returncode == 0, "sharded clip differs from the single-GPU clip (see stdout)"
    res = json.loads(out.read_text())
    assert res["ok"] and all(c["latents_rel_l2"] <= 5e-3 and c["videos_rel_l2"] <= 2e-3 for c in res["cases"])
