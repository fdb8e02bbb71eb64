"""FP8 feed-forward output projections on the H100: the e4m3 GEGLU with an e4m3 output and one scale per row and
128-column block (exact rule and accuracy), the block-scaled e4m3 GEMM (bit-exact on integer operands), the whole FP8
feed-forward against its emulation, and the denoising UNet3D with enable_fp8(ff_out=True) against the fp32 oracle and
its FP8 emulation."""
import pytest
import torch
import torch.nn.functional as F

from mimo_b200 import lib as L
from mimo_b200 import ops

pytestmark = pytest.mark.gpu

DT = [torch.float16, torch.bfloat16]
WIDTHS = [320, 640, 1280]


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


def _pack_tiles(v, gt):
    """value rows v [4C, ...] and gate rows gt [4C, ...] -> the 256-row GEGLU tile interleave (128 value rows, 128 gate)"""
    n = v.shape[0] // 128
    return torch.stack([v.reshape(n, 128, *v.shape[1:]), gt.reshape(n, 128, *gt.shape[1:])], 1).reshape(2 * v.shape[0],
                                                                                                       *v.shape[1:])


# ------------------------------------------------------------------------------------------------
# GEGLU -> e4m3 blocks
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("C", WIDTHS)
def test_geglu_e4m3_zero_values_give_zero_bytes_and_unit_scales(dtype, C):
    """zero value weights and value bias: every GEGLU value is a zero (of the gate's GELU sign), every scale 1"""
    g = torch.Generator(device="cuda").manual_seed(C)
    M, K, inner = 333, C, 4 * C
    a = torch.randint(-4, 5, (M, K), device="cuda", generator=g).float().to(torch.float8_e4m3fn)
    sa = torch.rand(M, device="cuda", generator=g) + 0.5
    wv = torch.zeros(inner, K, device="cuda")
    wg = torch.randint(-4, 5, (inner, K), device="cuda", generator=g).float()
    w = _pack_tiles(wv, wg).to(torch.float8_e4m3fn)
    sw = torch.rand(2 * inner, device="cuda", generator=g) + 0.5
    bias = _pack_tiles(torch.zeros(inner, device="cuda"), torch.randn(inner, device="cuda", generator=g)).to(dtype)
    q, s = ops.gemm_e4m3_geglu_e4m3(a, sa, w, sw, dtype, bias=bias)
    assert q.shape == (M, inner) and s.shape == (inner // 128, M)
    assert torch.all(q.view(torch.uint8) & 0x7F == 0) and torch.all(s == 1)


def _exact_case(C, M, dtype, seed):
    """integer operands, power-of-two scales, gates of 8..15 from the bias alone: GELU(g) == g in fp32, so every GEGLU
    value is exact and the host rule sees the kernel's own fp32 values"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    K, inner = C, 4 * C
    a = torch.randint(-2, 3, (M, K), device="cuda", generator=g).float()
    sa = torch.exp2(torch.randint(-3, 1, (M,), device="cuda", generator=g).float())
    wv = torch.randint(-2, 3, (inner, K), device="cuda", generator=g).float()
    swv = torch.exp2(torch.randint(-6, -2, (inner,), device="cuda", generator=g).float())
    bv = torch.randint(-4, 5, (inner,), device="cuda", generator=g).float()
    bg = torch.randint(8, 16, (inner,), device="cuda", generator=g).float()
    w = _pack_tiles(wv, torch.zeros_like(wv)).to(torch.float8_e4m3fn)
    sw = _pack_tiles(swv, torch.ones_like(swv))
    bias = _pack_tiles(bv, bg).to(dtype)
    y = ((a.double() @ wv.double().t()) * sa.double()[:, None] * swv.double()[None] + bv.double()) * bg.double()
    return a.to(torch.float8_e4m3fn), sa, w, sw, bias, y.float()


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("C", WIDTHS)
@pytest.mark.parametrize("M", [333, 128 * 140])
def test_geglu_e4m3_matches_the_host_rule_bit_for_bit(dtype, C, M):
    """ragged rows (333) and a persistent wrap (140 row tiles x 10-40 column tiles over the SMs)"""
    a, sa, w, sw, bias, y = _exact_case(C, M, dtype, seed=C + M)
    q, s = ops.gemm_e4m3_geglu_e4m3(a, sa, w, sw, dtype, bias=bias)
    rq, rs = ops.quantize_e4m3_blocks(y, 128)
    assert torch.equal(s, rs)
    assert torch.equal(q.view(torch.uint8), rq.view(torch.uint8))


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("C", WIDTHS)
def test_geglu_e4m3_random_within_one_step(dtype, C):
    """random operands. The e4m3 wgmma keeps fewer bits than fp32 while it accumulates (the GEGLU values differ from an
    fp32 matmul by up to ~5e-3 relative at K = 1280), so the reference is the kernel's own GEGLU values as the 16-bit
    GEGLU of mimo_gemm_e4m3 writes them: the same tile, the same wgmma sequence and epilogue, rounded once to `dtype`.
    Scales agree to that rounding, and each dequantized value lies within one e4m3 step (at its magnitude, times its
    block scale) of the rounded value, plus the rounding"""
    g = torch.Generator(device="cuda").manual_seed(31 * C)
    M, K, N = 1000, C, 8 * C
    a, sa = ops.quantize_e4m3_rows(torch.randn(M, K, device="cuda", generator=g))
    w, sw = ops.pack_e4m3_weight(torch.randn(N, K, device="cuda", generator=g) / K ** 0.5)
    bias = (torch.randn(N, device="cuda", generator=g) * 0.3).to(dtype)
    q, s = ops.gemm_e4m3_geglu_e4m3(a, sa, w, sw, dtype, bias=bias)
    y = ops.gemm_e4m3(a, sa, w, sw, dtype, bias=bias, act=L.ACT_GEGLU).float()
    eps = 2.0 ** -11 if dtype == torch.float16 else 2.0 ** -8
    _, rs = ops.quantize_e4m3_blocks(y, 128)
    err = float(((s - rs).abs() / rs).max())
    print(f"C={C}: max rel scale difference to the 16-bit GEGLU's {err:.2e}")
    assert err <= eps
    sc = s.t().repeat_interleave(128, 1)
    deq = q.float() * sc
    v = (y / sc).abs().clamp(min=2.0 ** -6)
    step = torch.exp2(torch.floor(torch.log2(v)) - 3) * sc
    assert torch.all((deq - y).abs() <= step * 1.01 + eps * y.abs() + 1e-6 * sc * 448), float(((deq - y).abs() / step).max())
    # and the fp32 GEGLU on the host, within the accumulation's precision
    acc = ((a.float() * sa[:, None]) @ (w.float() * sw[:, None]).t() + bias.float()).reshape(M, N // 256, 2, 128)
    y32 = (acc[:, :, 0] * F.gelu(acc[:, :, 1])).reshape(M, N // 2)
    assert _rel(deq, y32) < 0.05


# ------------------------------------------------------------------------------------------------
# block-scaled e4m3 GEMM
# ------------------------------------------------------------------------------------------------
def _bs_case(M, N, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randint(-2, 3, (M, K), device="cuda", generator=g).float()
    w = torch.randint(-2, 3, (N, K), device="cuda", generator=g).float()
    # a different power of two per (block, row): a per-row (or per-block) scale would be off by a power of two
    sa = torch.exp2(torch.randint(-12, -7, (K // 128, M), device="cuda", generator=g).float())
    sw = torch.exp2(torch.randint(-4, 0, (N,), device="cuda", generator=g).float())
    acc = torch.zeros(M, N, device="cuda", dtype=torch.float64)
    for b in range(K // 128):
        acc += (a[:, 128 * b:128 * b + 128].double() @ w[:, 128 * b:128 * b + 128].double().t()) * sa[b].double()[:, None]
    acc = acc * sw.double()[None]
    return a.to(torch.float8_e4m3fn), sa, w.to(torch.float8_e4m3fn), sw, acc


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("M,N,K", [(333, 320, 1280), (1000, 640, 2560), (300, 1280, 5120), (128 * 60, 1280, 5120),
                                   (128 * 150, 320, 1280), (77, 640, 128)])
def test_blockscaled_exact_integers(dtype, bn, M, N, K):
    """|v| <= 2 integers and power-of-two scales: every block's product and every fma into the sum is exact in fp32, so
    the output is the fp64 result rounded once to `dtype`. Every FF-out K / N, ragged M, persistent wraps (600 and 750
    tiles), a single K block, both tile widths; then bias + residual"""
    a, sa, w, sw, acc = _bs_case(M, N, K, seed=M + N + K + bn)
    g = torch.Generator(device="cuda").manual_seed(bn)
    bias = torch.randint(-8, 9, (N,), device="cuda", generator=g).to(dtype)
    res = torch.randint(-8, 9, (M, N), device="cuda", generator=g).to(dtype)
    L.load().mimo_debug_force_bn(bn)
    try:
        got = ops.gemm_e4m3_blockscaled(a, sa, w, sw, dtype)
        got2 = ops.gemm_e4m3_blockscaled(a, sa, w, sw, dtype, bias=bias, residual=res)
    finally:
        L.load().mimo_debug_force_bn(0)
    assert torch.equal(got, acc.to(dtype))
    assert torch.equal(got2, (acc + bias.double() + res.double()).to(dtype))


def test_blockscaled_default_width_and_padded_scale_rows():
    """the default tile width (128 at every FF-out width) and scales in rows of whole 16-byte groups (M = 333 pads to
    336, the padding NaN) give the same bytes as a contiguous scale tensor"""
    for N in (320, 640, 1280):
        a, sa, w, sw, acc = _bs_case(333, N, 4 * N, seed=N)
        got = ops.gemm_e4m3_blockscaled(a, sa, w, sw, torch.float16)
        padded = torch.full((sa.shape[0], 336), float("nan"), device="cuda")[:, :333]
        padded.copy_(sa)
        got2 = ops.gemm_e4m3_blockscaled(a, padded, w, sw, torch.float16)
        assert torch.equal(got, acc.to(torch.float16)) and torch.equal(got2, got)


# ------------------------------------------------------------------------------------------------
# the FP8 feed-forward
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("C", WIDTHS)
def test_ff_chain_matches_the_emulation(dtype, C):
    """LN -> e4m3 rows -> GEGLU -> e4m3 blocks -> block-scaled FF-out + bias + residual, against the same chain in fp32 on
    the host from the kernel's LN output (oracle/fp8_ff_oracle.py's rule)"""
    from oracle import fp8_ff_oracle as F8F
    from oracle import fp8_oracle as F8
    g = torch.Generator(device="cuda").manual_seed(7 * C)
    M = 2 * 4 * 32 * 32
    x = torch.randn(M, C, device="cuda", generator=g).to(dtype)
    ln = ((torch.rand(C, device="cuda", generator=g) + 0.5).to(dtype), (torch.randn(C, device="cuda", generator=g) * 0.1).to(dtype))
    w1 = torch.randn(8 * C, C, device="cuda", generator=g) / C ** 0.5
    b1 = torch.randn(8 * C, device="cuda", generator=g) * 0.1
    w2 = torch.randn(C, 4 * C, device="cuda", generator=g) / (4 * C) ** 0.5
    b2 = torch.randn(C, device="cuda", generator=g) * 0.1
    wp, bp = ops.pack_geglu_weight(w1.to(dtype), b1.to(dtype))
    q, sc = ops.layernorm_e4m3(x, *ln)
    g8, gs = ops.gemm_e4m3_geglu_e4m3(q, sc, *ops.pack_e4m3_weight(wp), dtype, bias=bp)
    out = ops.gemm_e4m3_blockscaled(g8, gs, *ops.pack_e4m3_weight(w2.to(dtype)), dtype, bias=b2.to(dtype), residual=x)
    sd = {"ff.net.0.proj.weight": w1.to(dtype).float(), "ff.net.0.proj.bias": b1.to(dtype).float(),
          "ff.net.2.weight": w2.to(dtype).float(), "ff.net.2.bias": b2.to(dtype).float()}
    h, gate = F8._lin8(sd, "ff.net.0.proj", q.float() * sc[:, None]).chunk(2, dim=-1)
    want = F8._lin8(sd, "ff.net.2", F8F.fake_quant_blocks(h * F.gelu(gate))) + x.float()
    exact = F.linear(h * F.gelu(gate), sd["ff.net.2.weight"], sd["ff.net.2.bias"]) + x.float()
    e, e_q = _rel(out.float() - x.float(), want - x.float()), _rel(want - x.float(), exact - x.float())
    print(f"C={C} {dtype}: engine vs emulation {e:.2e}, emulation vs fp32 FF-out {e_q:.2e}")
    # the difference is the e4m3 wgmma's accumulation, which keeps fewer bits than fp32 (5e-3 to 9e-3 measured on an
    # H100, growing with K), and the output's rounding to 16 bits: well below the FP8 error itself
    assert e < 0.3 * e_q


# ------------------------------------------------------------------------------------------------
# the denoising UNet3D
# ------------------------------------------------------------------------------------------------
def _den_case(f, hw, seed, widths=(320, 640, 1280, 1280), dtype=torch.float16, inflated=True):
    """engine outputs (fp16, FP8 projections + convs, + FF-out, FF-out without convs, ...) and the oracle's fp32 /
    emulated references of one CFG window"""
    from mimo_b200 import engine as E
    from oracle import fp8_conv_oracle as F8C
    from oracle import fp8_ff_oracle as F8F
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
    want8 = {}
    with torch.no_grad(), window:
        o_banks = O.reference_unet_banks(r32(sd_ref), lo(ref_lat).float().to(dev), lo(ehs).float().to(dev), cfg)
        o_pose = O.pose_guider(r32(sd_pg), lo(pose_img).float().to(dev)).repeat(2, 1, 1, 1, 1)
        args = (lo(x).float().to(dev), 499, lo(ehs).float().to(dev), o_pose, o_banks, cfg)
        want = O.denoising_unet(r32(sd_den), *args, cfg=True)
        with F8.fp8_emulation(), F8C.fp8_conv_emulation(), F8F.fp8_ff_out_emulation():
            want8["convs_ffo"] = O.denoising_unet(r32(sd_den), *args, cfg=True)
        with F8.fp8_emulation(), F8F.fp8_ff_out_emulation():
            want8["ffo"] = O.denoising_unet(r32(sd_den), *args, cfg=True)
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
    out = {"fp16": [run() for _ in range(2)]}
    den.set_fp8(True, convs=True)
    out["convs"] = [run() for _ in range(2)]
    bytes_convs = den.fp8_bytes()
    den.set_fp8(True, convs=True, ff_out=True)
    out["convs_ffo"] = [run() for _ in range(4)]  # eager, eager -> capture, replay, replay
    out["ffo_bytes"] = den.fp8_bytes() - bytes_convs
    den.set_fp8(True, ff_out=True)
    out["ffo"] = [run() for _ in range(2)]
    den.set_fp8(True, convs=True)
    out["convs_again"] = [run() for _ in range(2)]
    den.set_fp8(False)
    out["fp16_again"] = [run() for _ in range(2)]
    torch.cuda.synchronize()
    return out, want, want8, torch_lo


def _check_forward(out, want, want8, torch_lo, label):
    e_ref = _rel(torch_lo, want)
    for key in ("convs_ffo", "ffo"):
        e8 = out[key][0]
        e_eng8, e_q = _rel(e8, want), _rel(want8[key], want)
        print(f"{label} {key}: engine {e_eng8:.3e}  emulation {e_q:.3e}  torch-lo {e_ref:.3e}  (vs fp32 oracle); "
              f"vs engine without FF-out {_rel(out['convs_ffo'][0], out['convs'][0]):.3e}; "
              f"e4m3 ff.net.2 weights {out['ffo_bytes'] / 1e6:.1f} MB")
        assert torch.isfinite(e8).all()
        assert e_eng8 <= e_q + max(1e-3, e_ref), (key, e_eng8, e_q, e_ref)
    # eager, capture and replays are bit-identical; turning the FF-out off gives the earlier FP8 bytes back, and turning
    # FP8 off the fp16 bytes
    for o in out["convs_ffo"][1:]:
        assert torch.equal(o, out["convs_ffo"][0])
    assert torch.equal(out["ffo"][1], out["ffo"][0])
    for o in out["convs_again"] + out["convs"][1:]:
        assert torch.equal(o, out["convs"][0])
    for o in out["fp16_again"] + out["fp16"][1:]:
        assert torch.equal(o, out["fp16"][0])
    assert not torch.equal(out["convs_ffo"][0], out["convs"][0])


def test_unet_fp8_ff_out_forward_at_bench_shape():
    """[2, 8, 24, 64, 64]: rel(engine, fp32) <= rel(emulation, fp32) + max(1e-3, e_ref), with and without the convs"""
    out, want, want8, torch_lo = _den_case(f=24, hw=64, seed=720)
    _check_forward(out, want, want8, torch_lo, "UNet3D f=24 64x64")
    # every ff.net.2 of the SD1.5 UNet (16 spatial transformers, 21 motion blocks): [C, 4C] e4m3 bytes + C fp32 scales
    want_bytes = sum(n * (4 * c * c + 4 * c) for n, c in ((5, 320), (5, 640), (6, 1280))) \
        + sum(n * (4 * c * c + 4 * c) for n, c in ((5, 320), (5, 640), (5, 1280), (6, 1280)))
    assert out["ffo_bytes"] == want_bytes, (out["ffo_bytes"], want_bytes)


def test_unet_fp8_ff_out_forward_window_groupnorm():
    """a v1-style model (use_inflated_groupnorm=False): the ResBlocks' GroupNorms over the window, same bound"""
    out, want, want8, torch_lo = _den_case(f=8, hw=32, seed=730, inflated=False)
    _check_forward(out, want, want8, torch_lo, "UNet3D window-GN f=8 32x32")


def test_pipeline_clip_with_fp8_ff_out_gives_finite_frames():
    """a two-step 64 x 64, 4-frame clip through Pose2VideoPipeline.__call__ with enable_fp8(convs=True, ff_out=True)"""
    import numpy as np
    import PIL.Image
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection

    from mimo_b200.host import modules as M
    from mimo_b200.host.pipeline import Pose2VideoPipeline
    from mimo_b200.host.scheduler import DDIMScheduler
    from oracle import torch_oracle as O
    widths, F_, size, seed = (128, 256, 512, 512), 4, 64, 920
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
    pipe.denoising_unet.enable_fp8(convs=True, ff_out=True)
    rng = np.random.RandomState(seed)
    img = lambda: PIL.Image.fromarray(rng.randint(0, 256, (size, size, 3), dtype=np.uint8))
    out = pipe(img(), [img() for _ in range(F_)], [img() for _ in range(F_)], size, size, F_, 2, 3.5,
               generator=torch.manual_seed(42))
    eng = pipe.denoising_unet.engine()
    assert pipe.denoising_unet.fp8_ff_out_enabled and eng.fp8_ff_out and eng.fp8_convs
    assert out.videos.shape == (1, 3, F_, size, size) and torch.isfinite(out.videos).all()
