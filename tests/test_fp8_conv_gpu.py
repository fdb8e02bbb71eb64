"""FP8 ResBlock convolutions on the H100: GroupNorm + SiLU -> e4m3 with one scale per image (exact rule and accuracy, per
frame, over the window and frame-sharded), the e4m3 3x3 conv (bit-exact on integer operands), and the denoising UNet3D
with enable_fp8(convs=True) against the fp32 oracle and its FP8 emulation."""
import pytest
import torch
import torch.nn.functional as F

from mimo_b200 import lib as L
from mimo_b200 import ops

pytestmark = pytest.mark.gpu

DT = [torch.float16, torch.bfloat16]


@pytest.fixture(scope="module", autouse=True)
def _setup():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device: the product path has no CPU fallback")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    L.load().mimo_debug_force_bn(0)


def _rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-12))


def _split(x, c0):
    return x[:, :c0].contiguous(), x[:, c0:].contiguous()


# ------------------------------------------------------------------------------------------------
# GroupNorm + SiLU -> e4m3
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("window", [False, True])
def test_groupnorm_e4m3_exact_when_gamma_is_zero(dtype, window):
    """gamma = 0: every element of channel c is silu(beta_c). With beta 0 or an integer in 17..40, silu is exact (1 +
    exp(-beta) rounds to 1), so bytes and scales follow the host rule bit for bit: scale = max beta / 448."""
    dev = torch.device("cuda")
    g = torch.Generator(device="cuda").manual_seed(3 + window)
    n, hw, C = 6, 13 * 13, 640
    x = torch.randn(n * hw, C, device=dev, generator=g).to(dtype)
    gamma = torch.zeros(C, device=dev, dtype=dtype)
    mag = torch.randint(17, 41, (C,), device=dev, generator=g).float()
    beta = (mag * torch.randint(0, 2, (C,), device=dev, generator=g).float()).to(dtype)
    q, s = ops.groupnorm_e4m3(x, gamma, beta, n, hw, window_frames=3 if window else None)
    amax = beta.float().clamp(min=0).max()
    want_s = (amax / torch.tensor(448.0, device=dev)).expand(n)
    want_q = torch.clamp(beta.float() * (torch.tensor(448.0, device=dev) / amax), -448, 448)
    assert torch.equal(s, want_s)
    assert torch.equal(q.view(torch.uint8), want_q.to(torch.float8_e4m3fn).expand(n * hw, C).view(torch.uint8))
    # an all-zero bound: scale 1, zero bytes
    q, s = ops.groupnorm_e4m3(x, gamma, torch.zeros_like(beta), n, hw, window_frames=3 if window else None)
    assert torch.all(s == 1) and not q.view(torch.uint8).any()


def _gn_case(dtype, n, side, c0, c1, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    hw, C = side * side, c0 + c1
    x = (torch.randn(n * hw, C, device="cuda", generator=g) * 2 + torch.randn(C, device="cuda", generator=g)).to(dtype)
    gamma = (torch.randn(C, device="cuda", generator=g) + 0.5).to(dtype)
    beta = torch.randn(C, device="cuda", generator=g).to(dtype)
    return x, gamma, beta, hw


def _check_e4m3(q, s, y, scale_want):
    """scales match the host rule to a few ulp (the kernel's statistics and SiLU round differently), and every
    dequantized value lies within one e4m3 step (at its magnitude, times the image scale) of the fp32 result"""
    n = s.numel()
    err = float(((s - scale_want).abs() / scale_want).max())
    print(f"max rel scale difference {err:.2e} ({err / 2 ** -24:.1f} ulp)")
    assert err <= 2e-6
    y = y.reshape(n, -1)
    deq = q.float().reshape(n, -1) * s[:, None]
    v = (y / s[:, None]).abs().clamp(min=2.0 ** -6)
    step = torch.exp2(torch.floor(torch.log2(v)) - 3) * s[:, None]
    assert torch.all((deq - y).abs() <= step * 1.01 + 1e-6 * s[:, None] * 448), float(((deq - y).abs() / step).max())
    assert torch.all(q.float().abs() <= 448)


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("C,c1,side", [(320, 0, 49), (640, 0, 13), (960, 320, 49), (1280, 0, 8), (1920, 640, 13),
                                       (2560, 1280, 8), (2560, 0, 13), (640, 320, 8)])
def test_groupnorm_e4m3_random(dtype, C, c1, side):
    """per frame, one or two sources (the up blocks' concat): against the host statement of the rule on the same input"""
    n = 4
    x, gamma, beta, hw = _gn_case(dtype, n, side, C - c1, c1, seed=C + side)
    x0, x1 = _split(x, C - c1) if c1 else (x, None)
    q, s = ops.groupnorm_e4m3(x0, gamma, beta, n, hw, x1=x1)
    _, sw, y = ops.groupnorm_silu_e4m3_host(x.float().reshape(n, hw, C), gamma, beta, 32, 1e-5)
    _check_e4m3(q, s, y, sw)


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("C,c1,side", [(320, 0, 49), (1920, 640, 13), (2560, 1280, 8)])
def test_groupnorm_e4m3_window_and_frame_sharded(dtype, C, c1, side):
    """window statistics: against the host rule with frames, and the 16-bit groupnorm_window (+ SiLU) output within one
    step; the two halves of the window run as partials -> concatenated table -> apply give the same bytes and scales"""
    samples, frames = 2, 4
    n = samples * frames
    x, gamma, beta, hw = _gn_case(dtype, n, side, C - c1, c1, seed=7 * C + side)
    x0, x1 = _split(x, C - c1) if c1 else (x, None)
    q, s = ops.groupnorm_e4m3(x0, gamma, beta, n, hw, x1=x1, window_frames=frames)
    _, sw, y = ops.groupnorm_silu_e4m3_host(x.float().reshape(n, hw, C), gamma, beta, 32, 1e-5, frames)
    _check_e4m3(q, s, y, sw)
    y16 = ops.groupnorm_window(x0, gamma, beta, samples, frames, hw, x1=x1, silu=True).float()
    assert _rel(q.float().reshape(n, -1) * s[:, None], y16.reshape(n, -1)) < 0.04
    # frame-sharded: each half of every sample's frames on its own, as two ranks of a frame group would run them
    rows = lambda t, k: t.reshape(samples, frames, hw, -1)[:, 2 * k:2 * k + 2].reshape(samples * 2 * hw, -1).contiguous()
    halves = [(rows(x0, k), rows(x1, k) if x1 is not None else None) for k in range(2)]
    parts = [ops.groupnorm_e4m3_partials(a, samples, 2, hw, x1=b) for a, b in halves]
    table = torch.cat([t for t, _ in parts])
    outs = [ops.groupnorm_e4m3_apply(a, gamma, beta, table, w, samples, 2, frames, hw, x1=b)
            for (a, b), (_, w) in zip(halves, parts)]
    qs = torch.stack([o[0].view(torch.uint8).reshape(samples, 2, hw, C) for o in outs], 1).reshape(n * hw, C)
    ss = torch.stack([o[1].reshape(samples, 2) for o in outs], 1).reshape(n)
    assert torch.equal(qs, q.view(torch.uint8)) and torch.equal(ss, s)


# ------------------------------------------------------------------------------------------------
# e4m3 3x3 conv
# ------------------------------------------------------------------------------------------------
def _conv_case(n, h, w, cin, cout, g, img_scales=None):
    dev = torch.device("cuda")
    x = torch.randint(-2, 3, (n * h * w, cin), device=dev, generator=g).float()
    wt = torch.randint(-2, 3, (cout, 9 * cin), device=dev, generator=g).float()
    sx = img_scales if img_scales is not None else torch.exp2(torch.randint(-12, -8, (n,), device=dev, generator=g).float())
    sw = torch.exp2(torch.randint(-4, 0, (cout,), device=dev, generator=g).float())
    # fp64 conv of the integer operands (exact), times the power-of-two scales
    xi = x.double().reshape(n, h, w, cin).permute(0, 3, 1, 2)
    wi = wt.double().reshape(cout, 3, 3, cin).permute(0, 3, 1, 2)
    acc = F.conv2d(xi, wi, padding=1).permute(0, 2, 3, 1).reshape(n * h * w, cout)
    acc = acc * sx.double().repeat_interleave(h * w)[:, None] * sw.double()[None]
    return x.to(torch.float8_e4m3fn), sx, wt.to(torch.float8_e4m3fn), sw, acc.float()


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("bn", [160, 256])
@pytest.mark.parametrize("cin,cout,n,side", [(320, 320, 2, 49), (640, 640, 2, 25), (960, 640, 3, 13),
                                             (1280, 1280, 6, 8), (1920, 1280, 2, 13), (2560, 1280, 6, 8),
                                             (640, 320, 1, 98), (960, 320, 4, 64)])
def test_conv3x3_e4m3_exact_integers(dtype, bn, cin, cout, n, side):
    """|v| <= 2 integers are exact in e4m3 and power-of-two scales keep every product exact; the sums are exact in fp32,
    so the output equals the fp64 conv rounded once to `dtype`. (The e4m3 wgmma does not keep all of fp32's bits while it
    accumulates: with |v| <= 8, one output of a 9 x 2560-term sum came out one fp16 ulp off, so the operands stay small
    enough that the running sums, a few hundred here, keep every bit.) Covers every ResBlock Cin / Cout, half
    K blocks in each tap (Cin = 320, 960), both tile widths, 8 x 8 tiles of two whole images (TN = 2), ragged footprints
    (98, 49, 25, 13), and a persistent wrap (4 x 64 x 64 pixels: 128 row tiles, 256 or more tiles)."""
    g = torch.Generator(device="cuda").manual_seed(cin + cout + side + bn)
    x8, sx, w8, sw, acc = _conv_case(n, side, side, cin, cout, g)
    L.load().mimo_debug_force_bn(bn)
    try:
        got = ops.conv3x3_e4m3(x8, sx, w8, sw, n, side, side, dtype)
    finally:
        L.load().mimo_debug_force_bn(0)
    assert torch.equal(got, acc.to(dtype))


@pytest.mark.parametrize("dtype", DT)
def test_conv3x3_e4m3_image_scales_follow_the_output_pixel(dtype):
    """8 x 8 images, two per 128-row tile: distinct power-of-two scale per image (a row read with its neighbour image's
    scale would be off by a power of two)"""
    g = torch.Generator(device="cuda").manual_seed(11)
    n = 10
    sx = torch.exp2(-torch.arange(n, device="cuda").float() - 6)
    x8, sx, w8, sw, acc = _conv_case(n, 8, 8, 640, 320, g, img_scales=sx)
    assert torch.equal(ops.conv3x3_e4m3(x8, sx, w8, sw, n, 8, 8, dtype), acc.to(dtype))


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("bn", [160, 256])
@pytest.mark.parametrize("side,n", [(8, 6), (49, 2), (32, 4)])
def test_conv3x3_e4m3_epilogues(dtype, bn, side, n):
    """conv1's bias + per-branch time-embedding row (rows_per_group = 1 or several images, straddling tiles at 49 x 49)
    and conv2's residual: fmaf(acc, 1, bias + rowvec), then + residual, in that order"""
    g = torch.Generator(device="cuda").manual_seed(side + bn)
    cin, cout = 640, 1280
    x8, sx, w8, sw, acc = _conv_case(n, side, side, cin, cout, g)
    hw = side * side
    bias = torch.randint(-8, 9, (cout,), device="cuda", generator=g).to(dtype)
    rpg = hw * (n // 2)
    rowvec = torch.randint(-8, 9, (2, cout), device="cuda", generator=g).to(dtype)
    res = torch.randint(-8, 9, (n * hw, cout), device="cuda", generator=g).to(dtype)
    L.load().mimo_debug_force_bn(bn)
    try:
        got1 = ops.conv3x3_e4m3(x8, sx, w8, sw, n, side, side, dtype, bias=bias, rowvec=rowvec, rows_per_group=rpg)
        got2 = ops.conv3x3_e4m3(x8, sx, w8, sw, n, side, side, dtype, bias=bias, residual=res)
    finally:
        L.load().mimo_debug_force_bn(0)
    rv = rowvec.float().repeat_interleave(rpg, 0)
    assert torch.equal(got1, (acc + (bias.float() + rv)).to(dtype))
    assert torch.equal(got2, (acc + bias.float() + res.float()).to(dtype))


# ------------------------------------------------------------------------------------------------
# the denoising UNet3D
# ------------------------------------------------------------------------------------------------
def _den_case(f, hw, seed, widths=(320, 640, 1280, 1280), dtype=torch.float16, inflated=True):
    """engine outputs (fp16, FP8 projections, FP8 projections + convs, ...) and the oracle's fp32 / emulated references
    of one CFG window"""
    from mimo_b200 import engine as E
    from oracle import fp8_conv_oracle as F8C
    from oracle import fp8_oracle as F8
    from oracle import torch_oracle as O
    from oracle import window_gn_oracle as WG
    dev = torch.device("cuda")
    cfg = O.UNetConfig(block_out_channels=widths)
    sd_den = O.make_denoising_unet_sd(cfg, seed=seed)
    sd_ref = O.make_reference_unet_sd(cfg, seed=seed + 1)
    sd_pg = O.make_pose_guider_sd(seed=seed + 2, out_channels=widths[0])
    g = torch.Generator().manual_seed(seed + 10)
    ref_lat = torch.randn(1, 4, hw, hw, generator=g).repeat(2, 1, 1, 1)
    emb = torch.randn(1, 1, cfg.cross_attention_dim, generator=g)
    ehs = torch.cat([torch.zeros_like(emb), emb])
    x = torch.randn(1, 8, f, hw, hw, generator=g).repeat(2, 1, 1, 1, 1)
    pose_img = torch.rand(1, 3, f, hw * 8, hw * 8, generator=g)
    lo = lambda v: v.to(dtype)
    r32 = lambda sd: {k: lo(v).float().to(dev) for k, v in sd.items()}
    rlo = lambda sd: {k: lo(v).to(dev) for k, v in sd.items()}
    window = WG.window_groupnorm() if not inflated else __import__("contextlib").nullcontext()
    with torch.no_grad(), window:
        o_banks = O.reference_unet_banks(r32(sd_ref), lo(ref_lat).float().to(dev), lo(ehs).float().to(dev), cfg)
        o_pose = O.pose_guider(r32(sd_pg), lo(pose_img).float().to(dev)).repeat(2, 1, 1, 1, 1)
        args = (lo(x).float().to(dev), 499, lo(ehs).float().to(dev), o_pose, o_banks, cfg)
        want = O.denoising_unet(r32(sd_den), *args, cfg=True)
        with F8.fp8_emulation(), F8C.fp8_conv_emulation():
            want8 = O.denoising_unet(r32(sd_den), *args, cfg=True)
        l_banks = O.reference_unet_banks(rlo(sd_ref), lo(ref_lat).to(dev), lo(ehs).to(dev), cfg)
        l_pose = O.pose_guider(rlo(sd_pg), lo(pose_img).to(dev))
        torch_lo = O.denoising_unet(rlo(sd_den), lo(x).to(dev), 499, lo(ehs).to(dev), l_pose.repeat(2, 1, 1, 1, 1),
                                    l_banks, cfg, cfg=True).float()
        del o_banks, l_banks, l_pose
        torch.cuda.empty_cache()
    den = E.UNetEngine(sd_den, E.UNetSpec(block_out_channels=widths, inflated_groupnorm=inflated), dev, dtype)
    ref = E.UNetEngine(sd_ref, E.UNetSpec(block_out_channels=widths, in_channels=4, motion=False, out_head=False), dev,
                       dtype)
    pg = E.PoseGuiderEngine(sd_pg, dev, dtype)
    banks = ref.write_banks(lo(ref_lat).to(dev), lo(ehs).to(dev), den)
    den.begin_clip(lo(ehs).to(dev), banks, cfg=True, frames=f)
    pose = pg.forward(lo(pose_img).to(dev))
    pose2 = pose.reshape(1, f * hw * hw, -1).repeat(2, 1, 1).reshape(2 * f * hw * hw, -1).contiguous()
    run = lambda: den.forward(lo(x).to(dev), 499, pose2).float().clone()
    out = {"fp16": [run() for _ in range(3)]}
    den.set_fp8(True)
    out["proj"] = [run() for _ in range(3)]
    bytes_proj = den.fp8_bytes()
    den.set_fp8(True, convs=True)
    out["convs"] = [run() for _ in range(4)]  # eager, eager -> capture, replay, replay
    out["conv_bytes"] = den.fp8_bytes() - bytes_proj
    den.set_fp8(True)
    out["proj_again"] = [run() for _ in range(3)]
    den.set_fp8(False)
    out["fp16_again"] = [run() for _ in range(3)]
    torch.cuda.synchronize()
    return out, want, want8, torch_lo


def _check_forward(out, want, want8, torch_lo, label):
    e8 = out["convs"][0]
    e_eng8, e_q, e_ref = _rel(e8, want), _rel(want8, want), _rel(torch_lo, want)
    print(f"{label}: engine_fp8+convs {e_eng8:.3e}  oracle_fp8+convs {e_q:.3e}  torch-lo {e_ref:.3e}  (vs fp32 oracle); "
          f"engine_fp8+convs vs engine_fp8 {_rel(e8, out['proj'][0]):.3e}, vs engine_fp16 {_rel(e8, out['fp16'][0]):.3e}; "
          f"e4m3 conv weights {out['conv_bytes'] / 1e6:.1f} MB")
    assert torch.isfinite(e8).all()
    assert e_eng8 <= e_q + max(1e-3, e_ref), (e_eng8, e_q, e_ref)
    # eager, capture and replays are bit-identical; turning the convs off gives the projections-only FP8 bytes back,
    # and turning FP8 off the fp16 bytes
    for o in out["convs"][1:]:
        assert torch.equal(o, e8)
    for o in out["proj_again"]:
        assert torch.equal(o, out["proj"][0])
    for o in out["fp16_again"] + out["fp16"][1:]:
        assert torch.equal(o, out["fp16"][0])


def test_unet_fp8_convs_forward_at_bench_shape():
    """[2, 8, 24, 64, 64]: rel(engine, fp32) <= rel(emulation, fp32) + max(1e-3, e_ref)"""
    out, want, want8, torch_lo = _den_case(f=24, hw=64, seed=700)
    _check_forward(out, want, want8, torch_lo, "UNet3D f=24 64x64")
    # every ResBlock conv1 / conv2 of the SD1.5 UNet: 488 M e4m3 bytes plus one fp32 scale per output channel
    assert 0.45e9 < out["conv_bytes"] < 0.52e9


def test_unet_fp8_convs_forward_window_groupnorm():
    """a v1-style model (use_inflated_groupnorm=False): the ResBlocks' GroupNorms over the window, same bound"""
    out, want, want8, torch_lo = _den_case(f=8, hw=32, seed=710, inflated=False)
    _check_forward(out, want, want8, torch_lo, "UNet3D window-GN f=8 32x32")


def test_module_fp8_convs_api():
    """UNet3DConditionModel.enable_fp8(convs=True) / fp8_convs_enabled / disable_fp8() and the engine's set_fp8"""
    from mimo_b200.host import modules as M
    from oracle import torch_oracle as O
    widths = (128, 256, 512, 512)
    cfg = O.UNetConfig(block_out_channels=widths)
    mk = dict(num_attention_heads=8, num_transformer_block=1, attention_block_types=["Temporal_Self", "Temporal_Self"],
              temporal_position_encoding=True, temporal_position_encoding_max_len=32, temporal_attention_dim_div=1)
    den = M.UNet3DConditionModel(block_out_channels=widths, cross_attention_dim=768, use_inflated_groupnorm=True,
                                 use_motion_module=True, motion_module_mid_block=True, motion_module_type="Vanilla",
                                 motion_module_kwargs=mk, unet_use_cross_frame_attention=False,
                                 unet_use_temporal_attention=False)
    den.load_state_dict(O.make_denoising_unet_sd(cfg, 41), strict=True)
    den = den.to("cuda", torch.float16)
    assert not den.fp8_convs_enabled
    den.enable_fp8(convs=True)
    eng = den.engine()
    assert den.fp8_enabled and den.fp8_convs_enabled and eng.fp8 and eng.fp8_convs
    den.enable_fp8()
    assert den.fp8_enabled and not den.fp8_convs_enabled and eng.fp8 and not eng.fp8_convs
    den.enable_fp8(convs=True)
    den.disable_fp8()
    assert not den.fp8_enabled and not den.fp8_convs_enabled and not eng.fp8 and not eng.fp8_convs
    with pytest.raises(ValueError):
        eng.set_fp8(False, convs=True)


def test_pipeline_clip_with_fp8_convs_gives_finite_frames():
    """a two-step 64 x 64, 4-frame clip through Pose2VideoPipeline.__call__ with enable_fp8(convs=True)"""
    import numpy as np
    import PIL.Image
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection

    from mimo_b200.host import modules as M
    from mimo_b200.host.pipeline import Pose2VideoPipeline
    from mimo_b200.host.scheduler import DDIMScheduler
    from oracle import torch_oracle as O
    widths, F_, size, seed = (128, 256, 512, 512), 4, 64, 910
    cfg = O.UNetConfig(block_out_channels=widths)
    mk = dict(num_attention_heads=8, num_transformer_block=1, attention_block_types=["Temporal_Self", "Temporal_Self"],
              temporal_position_encoding=True, temporal_position_encoding_max_len=32, temporal_attention_dim_div=1)
    den = M.UNet3DConditionModel(block_out_channels=widths, cross_attention_dim=768, use_inflated_groupnorm=True,
                                 use_motion_module=True, motion_module_mid_block=True, motion_module_type="Vanilla",
                                 motion_module_kwargs=mk, unet_use_cross_frame_attention=False,
                                 unet_use_temporal_attention=False)
    ref = M.UNet2DConditionModel(block_out_channels=widths, cross_attention_dim=768)
    den.load_state_dict(O.make_denoising_unet_sd(cfg, seed), strict=True)
    ref.load_state_dict(O.make_reference_unet_sd(cfg, seed + 1), strict=True)
    pg = M.PoseGuider(widths[0], 3, (16, 32, 96, 256))
    pg.load_state_dict(O.make_pose_guider_sd(seed + 2, widths[0]), strict=True)
    vae = M.AutoencoderKL()
    vae.load_state_dict(O.make_vae_sd(O.VAEConfig(), seed + 3), strict=True)
    torch.manual_seed(seed + 4)
    clip = CLIPVisionModelWithProjection(CLIPVisionConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=2,
                                                          num_attention_heads=4, image_size=224, patch_size=32,
                                                          projection_dim=768)).eval()
    sched = DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
                          steps_offset=1, prediction_type="v_prediction", rescale_betas_zero_snr=True,
                          timestep_spacing="trailing")
    pipe = Pose2VideoPipeline(vae=vae, image_encoder=clip, reference_unet=ref, denoising_unet=den, pose_guider=pg,
                              scheduler=sched).to("cuda", dtype=torch.float16)
    pipe.denoising_unet.enable_fp8(convs=True)
    rng = np.random.RandomState(seed)
    img = lambda: PIL.Image.fromarray(rng.randint(0, 256, (size, size, 3), dtype=np.uint8))
    out = pipe(img(), [img() for _ in range(F_)], [img() for _ in range(F_)], size, size, F_, 2, 3.5,
               generator=torch.manual_seed(42))
    assert pipe.denoising_unet.fp8_convs_enabled and pipe.denoising_unet.engine().fp8_convs
    assert out.videos.shape == (1, 3, F_, size, size) and torch.isfinite(out.videos).all()
