"""FP8 (e4m3) path on the H100: LayerNorm -> e4m3 rows + scales (exact rule and accuracy), the e4m3 GEMM (bit-exact on
integer operands), and the denoising UNet3D with enable_fp8() against the fp32 oracle and its FP8 emulation."""
import pytest
import torch

from mimo_b200 import lib as L
from mimo_b200 import ops

pytestmark = pytest.mark.gpu

DT = [torch.float16, torch.bfloat16]


@pytest.fixture(scope="module", autouse=True)
def _setup():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device: the product path has no CPU fallback")
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


def _rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-12))


def _torch_rule(y):
    y = y.float()
    amax = y.abs().amax(dim=1)
    inv = torch.where(amax == 0, torch.ones_like(amax), torch.full_like(amax, 448.0) / amax)
    scale = torch.where(amax == 0, torch.ones_like(amax), amax / torch.full_like(amax, 448.0))
    return torch.clamp(y * inv[:, None], -448, 448).to(torch.float8_e4m3fn), scale


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("c", [320, 640, 1280, 96])
def test_layernorm_e4m3_exact_rows(dtype, c):
    """gamma = 0: every row is beta (+ the PE row of its frame), so bytes and scales follow the torch rule bit for bit."""
    dev = torch.device("cuda")
    g = torch.Generator(device="cuda").manual_seed(c)
    rows, hw, frames, off = 4 * 24 * 7 + 3, 7, 24, 5
    x = torch.randn(rows, c, device=dev, generator=g).to(dtype)
    gamma = torch.zeros(c, device=dev, dtype=dtype)
    beta = (torch.randn(c, device=dev, generator=g) * 3).to(dtype)
    q, s = ops.layernorm_e4m3(x, gamma, beta)
    rq, rs = _torch_rule(beta.float().expand(rows, c))
    assert torch.equal(q.view(torch.uint8), rq.view(torch.uint8)) and torch.equal(s, rs)
    pe = torch.randn(32, c, device=dev, generator=g).to(dtype)
    q, s = ops.layernorm_e4m3(x, gamma, beta, pe=pe, rows_per_frame=hw, frames=frames, pe_frame_offset=off)
    fr = off + (torch.arange(rows, device=dev) // hw) % frames
    rq, rs = _torch_rule(beta.float()[None] + pe.float()[fr])
    assert torch.equal(q.view(torch.uint8), rq.view(torch.uint8)) and torch.equal(s, rs)
    # a zero row (beta = 0, no PE): scale 1 and zero bytes
    q, s = ops.layernorm_e4m3(x, gamma, torch.zeros_like(beta))
    assert torch.all(s == 1) and not q.view(torch.uint8).any()


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("c", [320, 640, 1280, 96])
def test_layernorm_e4m3_random_rows(dtype, c):
    """every dequantized value lies within one e4m3 step (at its magnitude, times the row scale) of the fp32 LN"""
    dev = torch.device("cuda")
    g = torch.Generator(device="cuda").manual_seed(100 + c)
    rows = 3001
    x = (torch.randn(rows, c, device=dev, generator=g) * 2 + 0.3).to(dtype)
    gamma = (torch.randn(c, device=dev, generator=g) + 1).to(dtype)
    beta = torch.randn(c, device=dev, generator=g).to(dtype)
    q, s = ops.layernorm_e4m3(x, gamma, beta)
    y = torch.nn.functional.layer_norm(x.float(), (c,), gamma.float(), beta.float(), 1e-5)
    deq = q.float() * s[:, None]
    # e4m3 step at |v| in [2^e, 2^(e+1)): 2^(e-3); subnormals (|v| < 2^-6): 2^-9
    v = (y / s[:, None]).abs().clamp(min=2.0 ** -6)
    step = torch.exp2(torch.floor(torch.log2(v)) - 3) * s[:, None]
    assert torch.all((deq - y).abs() <= step * 1.0001), float(((deq - y).abs() / step).max())
    assert torch.allclose(s, y.abs().amax(1) / 448, rtol=1e-5, atol=0)


def _int_case(M, N, K, g):
    dev = torch.device("cuda")
    a = torch.randint(-16, 17, (M, K), device=dev, generator=g).float()
    w = torch.randint(-16, 17, (N, K), device=dev, generator=g).float()
    sa = torch.exp2(torch.randint(-8, 0, (M,), device=dev, generator=g).float())
    sw = torch.exp2(torch.randint(-8, 0, (N,), device=dev, generator=g).float())
    return a, w, sa, sw


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("M,N,K", [(128, 192, 320), (300, 200, 640), (1000, 384, 1280), (133 * 128 + 5, 960, 320),
                                   (257, 3840, 640), (64, 376, 1280)])
def test_gemm_e4m3_exact_integers(dtype, M, N, K):
    """|v| <= 16 integers are exact in e4m3, power-of-two scales keep every product exact, and the sums (<= 16 * 16 * K
    * 2^4) stay exact in fp32: the output must equal torch's fp32 result rounded once to `dtype`. Covers the K tails
    (320, 640 = 2.5, 5 K blocks of 128), ragged M and N, a persistent wrap (133 * 128 + 5 rows) and both tile widths
    (N = 3840 -> 256; 192 / 960 / 376 -> 192; 200 -> 256)."""
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    a, w, sa, sw = _int_case(M, N, K, g)
    a8, w8 = a.to(torch.float8_e4m3fn), w.to(torch.float8_e4m3fn)
    acc = (a @ w.t()) * sa[:, None] * sw[None, :]
    # plain
    assert torch.equal(ops.gemm_e4m3(a8, sa, w8, sw, dtype), acc.to(dtype))
    # bias + residual: fmaf(acc, 1, bias) then fmaf(res, 1, .)
    bias = torch.randint(-8, 9, (N,), device="cuda", generator=g).to(dtype)
    res = torch.randint(-8, 9, (M, N), device="cuda", generator=g).to(dtype)
    got = ops.gemm_e4m3(a8, sa, w8, sw, dtype, bias=bias, residual=res)
    assert torch.equal(got, (acc + bias.float() + res.float()).to(dtype))


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("scaled", [False, True])
def test_gemm_e4m3_geglu(dtype, scaled):
    """GEGLU epilogue on exact products: (value + bias_v) * gelu(gate + bias_g), against the 16-bit GEMM's own GEGLU
    epilogue fed the dequantized operands. With `scaled`, row and column scales are powers of two, so the dequantized
    operands a * sa and w * sw are exact in fp16 / bf16 and both kernels reach the epilogue with the same accumulators;
    this also checks that each gate column is scaled by its own (tile-interleaved) w_scale."""
    g = torch.Generator(device="cuda").manual_seed(77)
    M, inner, K = 700, 1280, 320
    N = 2 * inner
    a = torch.randint(-1, 2, (M, K), device="cuda", generator=g).float()  # small sums: h * gelu(gate) stays in fp16 range
    w = torch.randint(-1, 2, (N, K), device="cuda", generator=g).float()
    b = (torch.randint(-8, 9, (N,), device="cuda", generator=g).float() / 4).to(dtype)
    pw = lambda n: (torch.exp2(torch.randint(-3, 1, (n,), device="cuda", generator=g).float()) if scaled
                    else torch.ones(n, device="cuda"))
    sa, sw = pw(M), pw(N)
    wp, bp = ops.pack_geglu_weight(w.to(dtype), b)
    swp, _ = ops.pack_geglu_weight(sw[:, None], None)  # the column scales in the packed row order
    swp = swp[:, 0].contiguous()
    got = ops.gemm_e4m3(a.to(torch.float8_e4m3fn), sa, wp.float().to(torch.float8_e4m3fn), swp, dtype, bias=bp,
                        act=L.ACT_GEGLU)
    want = ops.gemm((a * sa[:, None]).to(dtype), (wp.float() * swp[:, None]).to(dtype), bias=bp, act=L.ACT_GEGLU)
    assert torch.equal(got, want)
    h, gate = ((a * sa[:, None]) @ (w * sw[:, None]).t() + b.float()).chunk(2, dim=-1)
    assert _rel(got, h * torch.nn.functional.gelu(gate)) < 1e-2


def _den_case(f, hw, seed, widths=(320, 640, 1280, 1280), dtype=torch.float16):
    """(engine fp16, engine fp8, oracle fp32, oracle fp8 emulation, torch low-precision execution) of one CFG window."""
    from mimo_b200 import engine as E
    from oracle import fp8_oracle as F8
    from oracle import torch_oracle as O
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
    with torch.no_grad():
        o_banks = O.reference_unet_banks(r32(sd_ref), lo(ref_lat).float().to(dev), lo(ehs).float().to(dev), cfg)
        o_pose = O.pose_guider(r32(sd_pg), lo(pose_img).float().to(dev)).repeat(2, 1, 1, 1, 1)
        args = (lo(x).float().to(dev), 499, lo(ehs).float().to(dev), o_pose, o_banks, cfg)
        want = O.denoising_unet(r32(sd_den), *args, cfg=True)
        with F8.fp8_emulation():
            want8 = O.denoising_unet(r32(sd_den), *args, cfg=True)
        l_banks = O.reference_unet_banks(rlo(sd_ref), lo(ref_lat).to(dev), lo(ehs).to(dev), cfg)
        l_pose = O.pose_guider(rlo(sd_pg), lo(pose_img).to(dev))
        torch_lo = O.denoising_unet(rlo(sd_den), lo(x).to(dev), 499, lo(ehs).to(dev), l_pose.repeat(2, 1, 1, 1, 1),
                                    l_banks, cfg, cfg=True).float()
        del o_banks, l_banks, l_pose
        torch.cuda.empty_cache()
    den = E.UNetEngine(sd_den, E.UNetSpec(block_out_channels=widths), dev, dtype)
    ref = E.UNetEngine(sd_ref, E.UNetSpec(block_out_channels=widths, in_channels=4, motion=False, out_head=False), dev,
                       dtype)
    pg = E.PoseGuiderEngine(sd_pg, dev, dtype)
    banks = ref.write_banks(lo(ref_lat).to(dev), lo(ehs).to(dev), den)
    den.begin_clip(lo(ehs).to(dev), banks, cfg=True, frames=f)
    pose = pg.forward(lo(pose_img).to(dev))
    pose2 = pose.reshape(1, f * hw * hw, -1).repeat(2, 1, 1).reshape(2 * f * hw * hw, -1).contiguous()
    run = lambda: den.forward(lo(x).to(dev), 499, pose2).float().clone()
    e16 = run()
    den.set_fp8(True)
    e8 = [run() for _ in range(4)]  # eager, eager -> capture, replay, replay
    den.set_fp8(False)
    back = [run() for _ in range(3)]
    torch.cuda.synchronize()
    return e16, e8, back, want, want8, torch_lo


def test_unet_fp8_forward_at_bench_shape():
    """[2, 8, 24, 64, 64]: the engine in FP8 may add no more error on top of the FP8 quantization itself than the fp16
    path's budget: rel(engine_fp8, fp32) <= rel(oracle_fp8, fp32) + max(1e-3, e_ref)."""
    e16, e8, back, want, want8, torch16 = _den_case(f=24, hw=64, seed=700)
    e_eng8, e_q, e_ref = _rel(e8[0], want), _rel(want8, want), _rel(torch16, want)
    print(f"UNet3D f=24 64x64: engine_fp8 {e_eng8:.3e}  oracle_fp8 {e_q:.3e}  torch-fp16 {e_ref:.3e}  (vs fp32 oracle); "
          f"engine_fp8 vs engine_fp16 {_rel(e8[0], e16):.3e}; engine_fp8 vs oracle_fp8 {_rel(e8[0], want8):.3e}")
    assert torch.isfinite(e8[0]).all()
    assert e_eng8 <= e_q + max(1e-3, e_ref), (e_eng8, e_q, e_ref)
    # eager, capture and replays are bit-identical; after disable_fp8 the fp16 path is byte-identical to before
    for o in e8[1:]:
        assert torch.equal(o, e8[0])
    for o in back:
        assert torch.equal(o, e16)


def _modules(widths, seed):
    from mimo_b200.host import modules as M
    from oracle import torch_oracle as O
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
    return den, ref


def _module_forward(den, ref, dtype, fp8_mode):
    """one CFG window through the public modules (reference write -> update -> denoising read), three forwards"""
    from mimo_b200.host.modules import ReferenceAttentionControl
    den, ref = den.to("cuda", dtype), ref.to("cuda", dtype)
    g = torch.Generator().manual_seed(3)
    ehs = torch.randn(2, 1, 768, generator=g).to("cuda", dtype)
    ref_lat = torch.randn(1, 4, 16, 16, generator=g).repeat(2, 1, 1, 1).to("cuda", dtype)
    x = torch.randn(2, 8, 4, 16, 16, generator=g).to("cuda", dtype)
    writer = ReferenceAttentionControl(ref, do_classifier_free_guidance=True, mode="write", fusion_blocks="full")
    reader = ReferenceAttentionControl(den, do_classifier_free_guidance=True, mode="read", fusion_blocks="full")
    ref(ref_lat, torch.zeros_like(ref_lat[:, 0, 0, 0]), encoder_hidden_states=ehs, return_dict=False)
    reader.update(writer)
    if fp8_mode != "never":
        den.enable_fp8()
        assert den.fp8_enabled and den.engine().fp8
        y8 = [den(x, 499, ehs).sample.float().clone() for _ in range(3)]
        assert torch.isfinite(y8[0]).all() and torch.equal(y8[0], y8[1]) and torch.equal(y8[1], y8[2])
        if fp8_mode == "on":
            return y8[0]
        den.disable_fp8()
        assert not den.fp8_enabled
    return torch.stack([den(x, 499, ehs).sample.float().clone() for _ in range(3)])


@pytest.mark.parametrize("dtype", DT)
def test_enable_disable_fp8_matches_a_model_that_never_enabled_it(dtype):
    """UNet3DConditionModel.enable_fp8() then disable_fp8(): outputs byte-identical to a model that never enabled FP8
    (eager, capture and replay); with FP8 on, the forwards are finite and bit-identical run to run"""
    widths = (128, 256, 512, 512)
    outs = {mode: _module_forward(*_modules(widths, 31), dtype, mode) for mode in ("never", "on_off", "on")}
    assert torch.equal(outs["never"], outs["on_off"])
    err = _rel(outs["on"], outs["never"][0])
    print(f"{dtype}: rel_l2(module fp8, module {dtype}) = {err:.3e}")
    assert err < 0.1


def test_pipeline_clip_with_fp8_gives_finite_frames():
    """a two-step 64 x 64, 4-frame clip through Pose2VideoPipeline.__call__ with pipe.denoising_unet.enable_fp8()"""
    import numpy as np
    import PIL.Image
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection

    from mimo_b200.host import modules as M
    from mimo_b200.host.pipeline import Pose2VideoPipeline
    from mimo_b200.host.scheduler import DDIMScheduler
    from oracle import torch_oracle as O
    widths, F_, size, seed = (128, 256, 512, 512), 4, 64, 900
    den, ref = _modules(widths, seed)
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
    pipe.denoising_unet.enable_fp8()
    rng = np.random.RandomState(seed)
    img = lambda: PIL.Image.fromarray(rng.randint(0, 256, (size, size, 3), dtype=np.uint8))
    out = pipe(img(), [img() for _ in range(F_)], [img() for _ in range(F_)], size, size, F_, 2, 3.5,
               generator=torch.manual_seed(42))
    assert pipe.denoising_unet.fp8_enabled and pipe.denoising_unet.engine().fp8
    assert out.videos.shape == (1, 3, F_, size, size) and torch.isfinite(out.videos).all()
