"""eta > 0 (stochastic DDIM) and interpolation_factor >= 2 (latent frame interpolation) on the H100: the two kernels
against PyTorch's expressions (bit-exact where PyTorch's rounding is reproduced, fp64 for slerp), graph capture, the
chunked VAE decode, and the public __call__ with both options against the oracle (oracle/sampler_options_oracle.py)."""
import importlib.util
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _any_size():
    """Helpers of test_any_size_gpu.py (pipeline builder, images, relative error), loaded by path."""
    spec = importlib.util.spec_from_file_location("_any_size_helpers", Path(__file__).with_name("test_any_size_gpu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture
def registry(monkeypatch):
    """The interpolation registry, reset for this test (another test may have left a method registered)."""
    from mimo_b200.host import interpolation as I
    monkeypatch.setattr(I, "_method", None)
    return I


# ------------------------------------------------------------------------------------------------
# stochastic DDIM step
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("with_counter", [False, True])
def test_noise_step_matches_torch_expression(dtype, with_counter):
    """DDIMScheduler.step with eta = 1 in the storage dtype vs the fused kernel, at the bound of the eta = 0 tests
    (2e-3 in fp16, scaled by the unit-roundoff ratio 8 in bf16). t = 999 is the step whose direction term is 0, t = 49
    the last step, where sigma = 0."""
    from mimo_b200 import ops
    from mimo_b200.host.scheduler import DDIMScheduler
    from oracle import sampler_options_oracle as SO
    from oracle import torch_oracle as O
    torch.manual_seed(21)
    F_, h, w = 5, 8, 8
    lat = torch.randn(1, 4, F_, h, w, device=DEV).to(dtype)
    pred = torch.randn(2, 4, F_, h, w, device=DEV).to(dtype)
    noise = torch.randn(1, 4, F_, h, w, device=DEV).to(dtype)
    counter = torch.tensor([1, 2, 1, 3, 2], device=DEV).to(dtype)
    d = O.DDIM()
    d.set_timesteps(20)
    s = DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
                      steps_offset=1, prediction_type="v_prediction", rescale_betas_zero_snr=True,
                      timestep_spacing="trailing")
    s.set_timesteps(20)
    bound = 2e-3 * (8 if dtype == torch.bfloat16 else 1)
    for t in (999, 499, 49):
        co = d.coefficients(t)
        dir_c, sigma = s.noise_coefficients(t, 1.0)
        assert (sigma == 0) == (t == 49)  # 49: the last step (abar_prev = 1)
        if with_counter:
            cv = counter.view(1, F_, 1, 1)
            got = ops.cfg_ddim_step_noise(pred[0] * cv, pred[1] * cv, lat.clone(), 3.5, *co[:3], dir_c, noise, sigma,
                                          counter=counter, frame_stride=h * w)
            u, c = ((pred * counter.view(1, 1, F_, 1, 1)) / counter.view(1, 1, F_, 1, 1)).chunk(2)
        else:
            got = ops.cfg_ddim_step_noise(pred[0].contiguous(), pred[1].contiguous(), lat.clone(), 3.5, *co[:3], dir_c,
                                          noise, sigma)
            u, c = pred.chunk(2)
        want = s.step(u + 3.5 * (c - u), t, lat, eta=1.0, variance_noise=noise).prev_sample
        assert want.dtype == dtype
        diff = float((got.float() - want.float()).abs().max())
        assert diff <= bound, (t, diff)
        # sigma = 0 with zero noise: the eta = 0 kernel's bytes
        zero = torch.zeros_like(noise)
        a = ops.cfg_ddim_step_noise(pred[0].contiguous(), pred[1].contiguous(), lat.clone(), 3.5, *co, zero, 0.0)
        b = ops.cfg_ddim_step(pred[0].contiguous(), pred[1].contiguous(), lat.clone(), 3.5, *co)
        assert torch.equal(a.view(torch.int16), b.view(torch.int16)), t


# ------------------------------------------------------------------------------------------------
# latent frame interpolation
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("hw", [(64, 64), (98, 98), (13, 7)])
def test_interpolate_linear_bit_exact(dtype, hw, registry):
    """linear: the torch expression (1 - t) * v1 + t * v2 on CUDA in the storage dtype, bit for bit, through the
    reference's interpolate_latents (oracle restatement)."""
    from mimo_b200 import ops
    from oracle import sampler_options_oracle as SO
    from oracle import torch_oracle as O
    h, w = hw
    g = torch.Generator(device=DEV).manual_seed(h * w)
    for F_ in (2, 24, 25):
        lat = torch.randn(1, 4, F_, h, w, device=DEV, generator=g).to(dtype)
        for k in (2, 3, 4):
            got = ops.interpolate_frames(lat, k, ops.INTERP_LINEAR)
            want = SO.interpolate_latents(lat, k, registry.linear)
            assert got.shape == want.shape == (1, 4, (F_ - 1) * k + 1, h, w)
            assert torch.equal(got.view(torch.int16), want.view(torch.int16)), (F_, k)


def _slerp64(v0, v1, t):
    """slerp in fp64 (with the fp32 cosine test of the kernel, so both take the same branch)."""
    a, b = v0.double(), v1.double()
    cos = float((a * b).sum() / (a.norm() * b.norm()))
    if abs(cos) > 0.9995:
        return (1.0 - t) * a + t * b, False
    th = torch.tensor(cos, dtype=torch.float64).acos()
    return (torch.sin((1.0 - t) * th) * a + torch.sin(t * th) * b) / torch.sin(th), True


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_interpolate_slerp(dtype):
    """slerp against fp64, <= 1 ulp of the storage type + 1e-6 (|v0| + |v1|) per element. Pairs: near-parallel
    (1.0001 v0) and antiparallel (both must equal the linear kernel bit for bit), orthogonal, random. Repeated runs and
    a CUDA-graph replay equal the eager result bit for bit."""
    from mimo_b200 import ops
    h, w, k = 40, 24, 4
    g = torch.Generator(device=DEV).manual_seed(5)
    f0 = torch.randn(4, h, w, device=DEV, generator=g)
    f1 = f0 * 1.0001
    f2 = -f1
    r = torch.randn(4, h, w, device=DEV, generator=g)
    f3 = r - (r * f2).sum() / (f2 * f2).sum() * f2  # orthogonal to f2 (to fp32 rounding)
    f4, f5 = (torch.randn(4, h, w, device=DEV, generator=g) for _ in range(2))
    lat = torch.stack([f0, f1, f2, f3, f4, f5], dim=1).unsqueeze(0).to(dtype).contiguous()
    got = ops.interpolate_frames(lat, k, ops.INTERP_SLERP)
    lin = ops.interpolate_frames(lat, k, ops.INTERP_LINEAR)
    ulp = 2.0 ** (-10 if dtype == torch.float16 else -7)
    worst = 0.0
    for i in range(5):
        v0, v1 = lat[0, :, i], lat[0, :, i + 1]
        for j in range(1, k):
            want, curved = _slerp64(v0, v1, j / k)
            out = got[0, :, i * k + j]
            if i in (0, 1):  # near-parallel / antiparallel: the linear branch
                assert not curved
                assert torch.equal(out.view(torch.int16), lin[0, :, i * k + j].view(torch.int16)), (i, j)
                continue
            assert curved, i
            tol = ulp * want.abs() + 1e-6 * (v0.double().abs() + v1.double().abs()) + 2.0 ** -24
            excess = float(((out.double() - want).abs() - tol).max())
            worst = max(worst, float(((out.double() - want).abs() / tol).max()))
            assert excess <= 0, (i, j, excess)
        assert torch.equal(got[0, :, i * k], lat[0, :, i])
    assert torch.equal(got[0, :, 5 * k], lat[0, :, 5])
    print(f"slerp {dtype}: worst error / bound = {worst:.3f}")
    for _ in range(3):
        assert torch.equal(ops.interpolate_frames(lat, k, ops.INTERP_SLERP).view(torch.int16), got.view(torch.int16))
    static = torch.empty_like(got)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.interpolate_frames(lat, k, ops.INTERP_SLERP, out=static)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.interpolate_frames(lat, k, ops.INTERP_SLERP, out=static)
    static.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(static.view(torch.int16), got.view(torch.int16))


# ------------------------------------------------------------------------------------------------
# chunked VAE decode
# ------------------------------------------------------------------------------------------------
def test_chunked_decode_is_byte_identical():
    from mimo_b200.host import modules as M
    from mimo_b200.host.pipeline import Pose2VideoPipeline
    torch.manual_seed(3)
    pipe = Pose2VideoPipeline.__new__(Pose2VideoPipeline)
    pipe.vae = M.AutoencoderKL().to(DEV, dtype=torch.float16)
    pipe.vae_scale_factor, pipe._vae_engines = 8, None
    lat = torch.randn(1, 4, 7, 40, 24, device=DEV).half()
    one = pipe.decode_latents_device(lat)
    assert one.shape == (1, 3, 7, 320, 192)
    for per in (1, 3, 6):
        assert torch.equal(pipe.decode_latents_device(lat, frames_per_pass=per).view(torch.int16),
                           one.view(torch.int16)), per


# ------------------------------------------------------------------------------------------------
# the public __call__
# ------------------------------------------------------------------------------------------------
def test_call_with_eta_and_slerp_interpolation_vs_oracle(registry):
    """__call__ at 200 x 136 (latents 17 x 25), 26 frames = two context windows, 2 DDIM steps, CFG 3.5, eta = 1,
    interpolation_factor 2 with slerp, against oracle/sampler_options_oracle.sample_clip in fp32 fed the same draws (latents, then one noise
    tensor per step, all from the caller's generator in fp16); PyTorch-fp16 on the same graph sets the bar."""
    from mimo_b200.host.pipeline import pil_to_tensor
    from oracle import sampler_options_oracle as SO
    from oracle import torch_oracle as O
    from scripts.oracle_any_size import forwarded_upsample_size
    A = _any_size()
    F_, width, height, steps, seed, k = 26, 200, 136, 2, 930, 2
    cfg, vcfg = O.UNetConfig(block_out_channels=A.WIDTHS), O.VAEConfig()
    sds = dict(den=O.make_denoising_unet_sd(cfg, seed), ref=O.make_reference_unet_sd(cfg, seed + 1),
               pg=O.make_pose_guider_sd(seed + 2, A.WIDTHS[0]), vae=O.make_vae_sd(vcfg, seed + 3))
    pipe = A._build_pipe(A.WIDTHS, sds, A._small_clip(seed + 4))
    ref_img, poses, bks = A._images(F_, width, height, seed)
    registry.set_tensor_interpolation_method(True)
    out = pipe(ref_img, poses, bks, width, height, F_, steps, 3.5, eta=1.0, generator=torch.manual_seed(42),
               interpolation_factor=k)
    Fo = (F_ - 1) * k + 1
    assert out.videos.shape == (1, 3, Fo, height, width) and out.videos.dtype == torch.float32
    dev = torch.device(DEV)
    with torch.no_grad(), forwarded_upsample_size():
        emb = pipe._clip_embeds(ref_img).float()
        gen = torch.manual_seed(42)
        shape = (1, 4, F_, height // 8, width // 8)
        lat0 = torch.randn(shape, generator=gen, dtype=torch.float16)
        noise = [torch.randn(shape, generator=gen, dtype=torch.float16).to(dev) for _ in range(steps)]
        args = lambda cast: (cast(pil_to_tensor(ref_img, height, width, True).to(dev)),
                             cast(pil_to_tensor(poses, height, width, False).permute(1, 0, 2, 3).unsqueeze(0).to(dev)),
                             cast(pil_to_tensor(bks[:1], height, width, True).to(dev)).expand(F_, -1, -1, -1))
        r32 = lambda sd: {kk: v.half().float().to(dev) for kk, v in sd.items()}
        h16 = lambda sd: {kk: v.half().to(dev) for kk, v in sd.items()}
        opts = dict(eta=1.0, interpolation_factor=k, interpolation=registry.slerp)
        W = O.Weights(r32(sds["den"]), r32(sds["ref"]), r32(sds["pg"]), r32(sds["vae"]), cfg, vcfg)
        want = SO.sample_clip(W, *args(lambda t: t), emb.half().float(), lat0.float().to(dev), steps, 3.5,
                             step_noise=[n.float() for n in noise], **opts)
        del W
        W16 = O.Weights(h16(sds["den"]), h16(sds["ref"]), h16(sds["pg"]), h16(sds["vae"]), cfg, vcfg)
        t16 = SO.sample_clip(W16, *args(lambda t: t.half()), emb.half(), lat0.to(dev), steps, 3.5, step_noise=noise,
                            **opts)
    le, ve = A._rel(pipe.last_latents, want["latents"]), A._rel(out.videos, want["videos"])
    le16, ve16 = A._rel(t16["latents"], want["latents"]), A._rel(t16["videos"], want["videos"])
    print(f"clip 200x136x26f eta=1 k=2 slerp: latents {le:.3e} videos {ve:.3e}   "
          f"torch-fp16: latents {le16:.3e} videos {ve16:.3e}")
    assert pipe.last_latents.shape == shape
    assert le <= max(1e-3, le16) and ve <= max(1e-3, ve16), (le, ve, le16, ve16)


def test_call_at_784x784_with_eta_and_interpolation_is_finite_and_deterministic(registry):
    """The reference's default size with full-size modules, 24 frames, 2 steps, eta = 1, k = 2 (slerp): 47 finite
    frames (decoded in two passes: 47 x 784^2 pixels exceed one pass), and two calls with the same seed give the same
    bytes."""
    A = _any_size()
    F_, size, steps = 24, 784, 2
    torch.manual_seed(42)
    pipe = A._build_pipe(A.WIDTHS, None, A._small_clip(5))
    ref_img, poses, bks = A._images(F_, size, size, 11)
    registry.set_tensor_interpolation_method(True)
    assert 47 * size * size > pipe.DECODE_PIXELS_PER_PASS
    vids = []
    for _ in range(2):
        out = pipe(ref_img, poses, bks, size, size, F_, steps, 3.5, eta=1.0, generator=torch.manual_seed(7),
                   interpolation_factor=2)
        assert out.videos.shape == (1, 3, 47, size, size)
        assert bool(torch.isfinite(out.videos).all())
        vids.append(out.videos.clone())
    assert pipe.last_latents.shape == (1, 4, F_, 98, 98)
    assert torch.equal(vids[0], vids[1])
