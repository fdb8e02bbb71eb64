"""Image sizes whose latents are not multiples of 8 on an H100: the nearest-resize kernel, the general up step (resize +
3x3 conv) and the stride-2 down conv at odd sides, the UNet3D at the reference's 784 x 784 default (98 x 98 latents) and
at smaller odd and non-square sizes against the tolerance contract of test_parity_gpu.py, and the public __call__.
The fp32 oracle and PyTorch's fp16 execution of the same graph follow the reference's forwarded upsample sizes
(scripts/oracle_any_size.py).

Contract: rel_l2(engine, fp32 oracle) <= max(1e-3, rel_l2(PyTorch executing the same graph in fp16, fp32 oracle)); bf16
uses 8e-3 as the floor (8 mantissa bits). Every comparison prints both numbers."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = "cuda"
WIDTHS = (320, 640, 1280, 1280)
DTYPES = [torch.float16, torch.bfloat16]
SENTINEL = -77.0


def _dn(dt):
    return "f16" if dt == torch.float16 else "bf16"


def _rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-12))


@pytest.fixture(scope="module", autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device: the product path has no CPU fallback")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


def _nhwc(x):
    n, c, h, w = x.shape
    return x.permute(0, 2, 3, 1).reshape(n * h * w, c).contiguous()


def _ints(shape, dtype, lo=-3, hi=4):
    return torch.randint(lo, hi, shape, device=DEV).to(dtype)


# ------------------------------------------------------------------------------------------------
# mimo_upsample_nearest: bit-identical to F.interpolate(mode="nearest", size=...)
# ------------------------------------------------------------------------------------------------
RESIZE_CASES = [  # (h, w) -> (oh, ow)
    ((13, 13), (25, 25)), ((25, 25), (49, 49)), ((49, 49), (98, 98)),   # the up steps at 784 x 784
    ((1, 1), (1, 1)), ((7, 7), (3, 3)), ((5, 5), (12, 12)),               # identity, downscale, ratio 2.4
    ((13, 7), (25, 14)), ((4, 3), (7, 5)), ((3, 5), (8, 2)), ((2, 9), (1, 17)), ((9, 13), (17, 26)),
]


@pytest.mark.parametrize("dtype", DTYPES, ids=_dn)
@pytest.mark.parametrize("c", [8, 320, 1280])
@pytest.mark.parametrize("case", RESIZE_CASES, ids=lambda s: "{}x{}_to_{}x{}".format(*s[0], *s[1]))
def test_upsample_nearest_bit_exact(case, c, dtype):
    from mimo_b200 import ops
    (h, w), (oh, ow) = case
    n = 3
    torch.manual_seed(h * 100 + w * 10 + oh + c)
    x = torch.randn(n, c, h, w, device=DEV).to(dtype)
    want = _nhwc(F.interpolate(x.float(), size=(oh, ow), mode="nearest").to(dtype))  # a copy: exact in fp32
    rows = n * oh * ow
    buf = torch.full((rows + 64, c), SENTINEL, dtype=dtype, device=DEV)
    got = ops.upsample_nearest(_nhwc(x), n, h, w, oh, ow, out=buf[:rows])
    assert torch.equal(got, want), f"{int((got != want).sum())} of {want.numel()} elements differ"
    assert bool((buf[rows:] == SENTINEL).all()), "the kernel wrote past its output"


# ------------------------------------------------------------------------------------------------
# the general up step and the stride-2 down conv at odd sides: bit-exact on integer inputs
# ------------------------------------------------------------------------------------------------
UP_CASES = [  # n, (h, w) -> (th, tw), cin, cout
    (2, (13, 13), (25, 25), 64, 72), (2, (25, 25), (49, 49), 64, 64), (3, (4, 3), (7, 5), 72, 64),
    (2, (2, 2), (4, 3), 64, 64), (2, (7, 5), (14, 10), 64, 64), (2, (1, 1), (1, 1), 64, 64), (1, (5, 7), (9, 14), 64, 136),
]


@pytest.mark.parametrize("dtype", DTYPES, ids=_dn)
@pytest.mark.parametrize("case", UP_CASES, ids=lambda c: "n{}_{}x{}_to_{}x{}_c{}_o{}".format(c[0], *c[1], *c[2], c[3], c[4]))
def test_up_step_exact(case, dtype):
    """UNetEngine._up as the engine runs it (the fused kernel for exact x2, resize + conv3x3 otherwise) against
    F.interpolate(size=skip size) + F.conv2d(padding=1) in fp64, rounded once."""
    from mimo_b200 import engine as E
    from mimo_b200 import ops
    n, (h, w), (th, tw), cin, co = case
    torch.manual_seed(h * 31 + w + th)
    x = _ints((n, cin, h, w), dtype)
    W = _ints((co, cin, 3, 3), dtype)
    b = _ints((co,), dtype)
    want = _nhwc(F.conv2d(F.interpolate(x.double(), size=(th, tw), mode="nearest"), W.double(), b.double(), padding=1))
    eng = SimpleNamespace(w={"u": (ops.pack_conv_up2x_weight(W), b), "u_conv": (ops.pack_conv3x3_weight(W), b)})
    got = E.UNetEngine._up(eng, "u", _nhwc(x), n, h, w, th, tw)
    assert torch.equal(got, want.to(dtype)), f"{int((got != want.to(dtype)).sum())} of {want.numel()} differ"


@pytest.mark.parametrize("dtype", DTYPES, ids=_dn)
@pytest.mark.parametrize("hw", [(98, 98), (49, 49), (25, 25), (13, 13), (7, 5), (1, 3), (17, 25)],
                         ids=lambda s: f"{s[0]}x{s[1]}")
def test_down_conv_at_odd_sides_exact(hw, dtype):
    """UNetEngine._down (im2col stride 2 + GEMM) against F.conv2d(stride=2, padding=1): ceil(s / 2) outputs per side."""
    from mimo_b200 import engine as E
    from mimo_b200 import ops
    h, w = hw
    n, cin, co = 2, 64, 64
    torch.manual_seed(h * 7 + w)
    x = _ints((n, cin, h, w), dtype)
    W = _ints((co, cin, 3, 3), dtype)
    b = _ints((co,), dtype)
    want = _nhwc(F.conv2d(x.double(), W.double(), b.double(), stride=2, padding=1))
    eng = SimpleNamespace(w={"d": (ops.pack_conv3x3_weight(W), b)})
    got = E.UNetEngine._down(eng, "d", _nhwc(x), n, h, w)
    assert want.shape[0] == n * E.latent_levels(h, w, 2)[1][0] * E.latent_levels(h, w, 2)[1][1]
    assert torch.equal(got, want.to(dtype))


# ------------------------------------------------------------------------------------------------
# the denoising UNet3D with banks and pose features
# ------------------------------------------------------------------------------------------------
def _unet_case(f, h, w, seed, dtype=torch.float16):
    """(engine outputs [eager, eager -> capture, replay], torch low-precision execution, fp32 oracle) of one CFG window,
    as test_parity_gpu.py::_unet_case, at a latent of h x w."""
    from mimo_b200 import engine as E
    from oracle import torch_oracle as O
    from scripts.oracle_any_size import forwarded_upsample_size
    dev = torch.device(DEV)
    cfg = O.UNetConfig(block_out_channels=WIDTHS)
    sd_den = O.make_denoising_unet_sd(cfg, seed=seed)
    sd_ref = O.make_reference_unet_sd(cfg, seed=seed + 1)
    sd_pg = O.make_pose_guider_sd(seed=seed + 2, out_channels=WIDTHS[0])
    g = torch.Generator().manual_seed(seed + 10)
    ref_lat = torch.randn(1, 4, h, w, generator=g).repeat(2, 1, 1, 1)
    emb = torch.randn(1, 1, cfg.cross_attention_dim, generator=g)
    ehs = torch.cat([torch.zeros_like(emb), emb])
    x = torch.randn(1, 8, f, h, w, generator=g).repeat(2, 1, 1, 1, 1)
    pose_img = torch.rand(1, 3, f, h * 8, w * 8, generator=g)
    t = 499
    lo = lambda v: v.to(dtype)
    r32 = lambda sd: {k: lo(v).float().to(dev) for k, v in sd.items()}
    rlo = lambda sd: {k: lo(v).to(dev) for k, v in sd.items()}
    with torch.no_grad(), forwarded_upsample_size():
        o_banks = O.reference_unet_banks(r32(sd_ref), lo(ref_lat).float().to(dev), lo(ehs).float().to(dev), cfg)
        o_pose = O.pose_guider(r32(sd_pg), lo(pose_img).float().to(dev))
        want = O.denoising_unet(r32(sd_den), lo(x).float().to(dev), t, lo(ehs).float().to(dev),
                                o_pose.repeat(2, 1, 1, 1, 1), o_banks, cfg, cfg=True)
        l_banks = O.reference_unet_banks(rlo(sd_ref), lo(ref_lat).to(dev), lo(ehs).to(dev), cfg,
                                         bank_dtype=torch.float16 if dtype == torch.float16 else dtype)
        l_pose = O.pose_guider(rlo(sd_pg), lo(pose_img).to(dev))
        torch_lo = O.denoising_unet(rlo(sd_den), lo(x).to(dev), t, lo(ehs).to(dev), l_pose.repeat(2, 1, 1, 1, 1),
                                    l_banks, cfg, cfg=True).float()
        del o_banks, l_banks, l_pose, o_pose
        torch.cuda.empty_cache()
    den = E.UNetEngine(sd_den, E.UNetSpec(block_out_channels=WIDTHS), dev, dtype)
    ref = E.UNetEngine(sd_ref, E.UNetSpec(block_out_channels=WIDTHS, in_channels=4, motion=False, out_head=False), dev,
                       dtype)
    pg = E.PoseGuiderEngine(sd_pg, dev, dtype)
    banks = ref.write_banks(lo(ref_lat).to(dev), lo(ehs).to(dev), den)
    den.begin_clip(lo(ehs).to(dev), banks, cfg=True, frames=f)
    pose = pg.forward(lo(pose_img).to(dev))
    pose2 = pose.reshape(1, f * h * w, -1).repeat(2, 1, 1).reshape(2 * f * h * w, -1).contiguous()
    outs = [den.forward(lo(x).to(dev), t, pose2).float().clone() for _ in range(3)]  # eager, eager->capture, replay
    torch.cuda.synchronize()
    return outs, torch_lo, want


@pytest.mark.parametrize("f,h,w,seed,dtype,floor", [
    (24, 98, 98, 720, torch.float16, 1e-3),   # 784 x 784, 24 frames: the reference's script default
    (3, 25, 17, 730, torch.float16, 1e-3),    # 200 x 136: non-square, every up step but the last is general
    (3, 13, 21, 740, torch.bfloat16, 8e-3),   # bf16, non-square
], ids=["f24_98x98_f16", "f3_25x17_f16", "f3_13x21_bf16"])
def test_unet_forward_at_odd_sizes(f, h, w, seed, dtype, floor):
    outs, torch_lo, want = _unet_case(f, h, w, seed, dtype)
    assert outs[0].shape == (2, 4, f, h, w)
    e_eng, e_ref = _rel(outs[0], want), _rel(torch_lo, want)
    print(f"UNet3D f={f} {h}x{w} {_dn(dtype)} full width: engine {e_eng:.3e}  torch-{_dn(dtype)} {e_ref:.3e}  "
          "(both vs the fp32 oracle)")
    assert e_eng <= max(floor, e_ref), (e_eng, e_ref)
    # the eager run, the run that captures the CUDA graph of this shape, and its replay: bit-identical
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[1], outs[2])


# ------------------------------------------------------------------------------------------------
# the VAE at a latent whose token count is not a multiple of 8 (its mid-block attention pads the key axis)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hw", [(17, 25), (13, 13)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_vae_at_odd_latent_sizes(hw):
    """AutoencoderKL encode (pixels 8h x 8w) and decode (latent h x w), 3 images batched, hw = 425 / 169 tokens in the
    mid-block attention, against the fp32 oracle with PyTorch-fp16's own error as the bar (test_parity_gpu.py)."""
    from mimo_b200 import engine as E
    from oracle import torch_oracle as O
    h, w = hw
    dev = torch.device(DEV)
    cfg = O.VAEConfig()
    sd = O.make_vae_sd(cfg, seed=17)
    r32 = {k: v.half().float().to(dev) for k, v in sd.items()}
    r16 = {k: v.half().to(dev) for k, v in sd.items()}
    x = torch.rand(3, 3, 8 * h, 8 * w, generator=torch.Generator().manual_seed(18)) * 2 - 1
    z = torch.randn(3, 4, h, w, generator=torch.Generator().manual_seed(19)) * 4
    with torch.no_grad():
        enc_want = O.vae_encode_mean(r32, x.half().float().to(dev), cfg)
        enc_t16 = O.vae_encode_mean(r16, x.half().to(dev), cfg).float()
        dec_want = O.vae_decode(r32, z.half().float().to(dev), cfg)
        dec_t16 = O.vae_decode(r16, z.half().to(dev), cfg).float()
    enc = E.VAEEncoderEngine(sd, dev).encode_mean(x.half().to(dev)).float()
    dec = E.VAEDecoderEngine(sd, dev).decode(z.half().to(dev)).float()
    assert enc.shape == (3, 4, h, w) and dec.shape == (3, 3, 8 * h, 8 * w)
    for name, got, want, t16 in (("encode", enc, enc_want, enc_t16), ("decode", dec, dec_want, dec_t16)):
        e_eng, e_ref = _rel(got, want), _rel(t16, want)
        print(f"VAE {name} latent {h}x{w}: engine {e_eng:.3e}  torch-fp16 {e_ref:.3e}")
        assert e_eng <= max(3e-3, e_ref), (name, e_eng, e_ref)


# ------------------------------------------------------------------------------------------------
# the public __call__
# ------------------------------------------------------------------------------------------------
def _build_pipe(widths, sds, clip, dtype=torch.float16):
    from mimo_b200.host import modules as M
    from mimo_b200.host.pipeline import Pose2VideoPipeline
    from mimo_b200.host.scheduler import DDIMScheduler
    mk = dict(num_attention_heads=8, num_transformer_block=1, attention_block_types=["Temporal_Self", "Temporal_Self"],
              temporal_position_encoding=True, temporal_position_encoding_max_len=32, temporal_attention_dim_div=1)
    den = M.UNet3DConditionModel(block_out_channels=widths, cross_attention_dim=768, use_inflated_groupnorm=True,
                                 use_motion_module=True, motion_module_mid_block=True, motion_module_type="Vanilla",
                                 motion_module_kwargs=mk, unet_use_cross_frame_attention=False,
                                 unet_use_temporal_attention=False)
    ref = M.UNet2DConditionModel(block_out_channels=widths, cross_attention_dim=768)
    pg = M.PoseGuider(widths[0], 3, (16, 32, 96, 256))
    vae = M.AutoencoderKL()
    if sds is not None:
        for m, k in ((den, "den"), (ref, "ref"), (pg, "pg"), (vae, "vae")):
            m.load_state_dict(sds[k], strict=True)
    sched = DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
                          steps_offset=1, prediction_type="v_prediction", rescale_betas_zero_snr=True,
                          timestep_spacing="trailing")
    return Pose2VideoPipeline(vae=vae, image_encoder=clip, reference_unet=ref, denoising_unet=den, pose_guider=pg,
                              scheduler=sched).to(DEV, dtype=dtype)


def _small_clip(seed):
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection
    torch.manual_seed(seed)
    return CLIPVisionModelWithProjection(CLIPVisionConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=2,
                                                          num_attention_heads=4, image_size=224, patch_size=32,
                                                          projection_dim=768)).eval()


def _images(F_, width, height, seed):
    import PIL.Image
    rng = np.random.RandomState(seed)
    ref_img = PIL.Image.fromarray(rng.randint(0, 256, (height, width, 3), dtype=np.uint8))
    poses = []
    for i in range(F_):
        a = np.zeros((height, width, 3), np.uint8)
        a[height // 4: height // 2 + i % 16, width // 3: width // 3 + width // 6] = (200, 40 + 5 * i, 90)
        poses.append(PIL.Image.fromarray(a))
    bks = [PIL.Image.fromarray(np.full((height, width, 3), 255, np.uint8)) for _ in range(F_)]
    return ref_img, poses, bks


def test_call_at_200x136_two_windows_vs_oracle():
    """__call__ at 200 x 136 pixels (latents 17 x 25: levels 9 x 13, 5 x 7, 3 x 4), 26 frames = two context windows,
    2 DDIM steps, CFG 3.5, against oracle.sample_clip in fp32; PyTorch-fp16 on the same graph sets the bar."""
    from mimo_b200.host.pipeline import pil_to_tensor
    from oracle import torch_oracle as O
    from scripts.oracle_any_size import forwarded_upsample_size
    F_, width, height, steps, seed = 26, 200, 136, 2, 910
    cfg, vcfg = O.UNetConfig(block_out_channels=WIDTHS), O.VAEConfig()
    sds = dict(den=O.make_denoising_unet_sd(cfg, seed), ref=O.make_reference_unet_sd(cfg, seed + 1),
               pg=O.make_pose_guider_sd(seed + 2, WIDTHS[0]), vae=O.make_vae_sd(vcfg, seed + 3))
    pipe = _build_pipe(WIDTHS, sds, _small_clip(seed + 4))
    ref_img, poses, bks = _images(F_, width, height, seed)
    out = pipe(ref_img, poses, bks, width, height, F_, steps, 3.5, generator=torch.manual_seed(42))
    assert out.videos.shape == (1, 3, F_, height, width) and out.videos.dtype == torch.float32
    dev = torch.device(DEV)
    with torch.no_grad(), forwarded_upsample_size():
        emb = pipe._clip_embeds(ref_img).float()
        lat0 = torch.randn((1, 4, F_, height // 8, width // 8), generator=torch.manual_seed(42), dtype=torch.float16)
        args = lambda cast: (cast(pil_to_tensor(ref_img, height, width, True).to(dev)),
                             cast(pil_to_tensor(poses, height, width, False).permute(1, 0, 2, 3).unsqueeze(0).to(dev)),
                             cast(pil_to_tensor(bks[:1], height, width, True).to(dev)).expand(F_, -1, -1, -1))
        r32 = lambda sd: {k: v.half().float().to(dev) for k, v in sd.items()}
        h16 = lambda sd: {k: v.half().to(dev) for k, v in sd.items()}
        W = O.Weights(r32(sds["den"]), r32(sds["ref"]), r32(sds["pg"]), r32(sds["vae"]), cfg, vcfg)
        want = O.sample_clip(W, *args(lambda t: t), emb.half().float(), lat0.float().to(dev), steps, 3.5)
        del W
        W16 = O.Weights(h16(sds["den"]), h16(sds["ref"]), h16(sds["pg"]), h16(sds["vae"]), cfg, vcfg)
        t16 = O.sample_clip(W16, *args(lambda t: t.half()), emb.half(), lat0.to(dev), steps, 3.5)
    le, ve = _rel(pipe.last_latents, want["latents"]), _rel(out.videos, want["videos"])
    le16, ve16 = _rel(t16["latents"], want["latents"]), _rel(t16["videos"], want["videos"])
    print(f"clip 200x136x26f, 2 steps: latents {le:.3e} videos {ve:.3e}   torch-fp16: latents {le16:.3e} videos {ve16:.3e}")
    assert le <= max(1e-3, le16) and ve <= max(1e-3, ve16), (le, ve, le16, ve16)


def test_call_at_784x784_is_finite_and_deterministic():
    """The reference's default size, full-size modules (seeded default init), 24 frames, 2 steps: two calls with the same
    seed (the second replays the captured graphs) return the same bytes."""
    F_, size, steps = 24, 784, 2
    torch.manual_seed(42)
    pipe = _build_pipe(WIDTHS, None, _small_clip(5))
    ref_img, poses, bks = _images(F_, size, size, 11)
    vids = []
    for _ in range(2):
        out = pipe(ref_img, poses, bks, size, size, F_, steps, 3.5, generator=torch.manual_seed(7))
        assert out.videos.shape == (1, 3, F_, size, size) and out.videos.dtype == torch.float32
        assert bool(torch.isfinite(out.videos).all())
        vids.append(out.videos.clone())
    lat = pipe.last_latents
    assert lat.shape == (1, 4, F_, 98, 98) and bool(torch.isfinite(lat).all())
    print(f"clip 784x784x24f, 2 steps: video mean {float(vids[0].mean()):.4f}, std {float(vids[0].std()):.4f}")
    assert torch.equal(vids[0], vids[1])
