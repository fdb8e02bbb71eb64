"""The sampler options eta > 0 (stochastic DDIM) and interpolation_factor >= 2 (latent frame interpolation) on the CPU:
the scheduler's eta step against the oracle and against the generator's draw order, this repo's sampler (preprocess +
sample_tensors, engine calls replaced by oracle-backed stand-ins as in test_pipeline_plumbing_cpu.py) against the clips
the reference's own pipeline file produced with both options (tests/golden/pipeline_sampler_options.pt, written by
oracle/gen_sampler_options_golden.py), the early refusals, and the two new C entry points' argument checks."""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch

SCHED_KW = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False, steps_offset=1,
                prediction_type="v_prediction", rescale_betas_zero_snr=True, timestep_spacing="trailing")


def _sched(n):
    from mimo_b200.host.scheduler import DDIMScheduler
    s = DDIMScheduler(**SCHED_KW)
    s.set_timesteps(n)
    return s


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("eta", [1.0, 0.3])
def test_scheduler_eta_step_matches_oracle_and_draws_like_randn(dtype, eta):
    from oracle import sampler_options_oracle as SO
    from oracle import torch_oracle as O
    s, d = _sched(4), O.DDIM()
    d.set_timesteps(4)
    g0 = torch.Generator().manual_seed(3)
    x = torch.randn(1, 4, 3, 5, 6, generator=g0).to(dtype)
    v = torch.randn(1, 4, 3, 5, 6, generator=g0).to(dtype)
    g, g_ref = torch.Generator().manual_seed(7), torch.Generator().manual_seed(7)
    for t in [int(t) for t in s.timesteps]:  # the last step has sigma = 0 and still draws
        got = s.step(v, t, x, eta=eta, generator=g).prev_sample
        noise = torch.randn(x.shape, generator=g_ref, dtype=dtype)
        want = SO.ddim_step(d, v, t, x, eta, noise)
        assert got.dtype == dtype and torch.equal(got, want.to(dtype)), t
        assert torch.equal(g.get_state(), g_ref.get_state()), t  # consumed exactly one draw of the sample's shape
        assert torch.equal(s.step(v, t, x, eta=eta, variance_noise=noise).prev_sample, got)
        dir_c, sigma = s.noise_coefficients(t, eta)
        assert sigma >= 0 and dir_c >= 0
        assert s.step_coefficients(t) == d.coefficients(t)  # unchanged by the eta path
    assert s.noise_coefficients(int(s.timesteps[-1]), eta) == (0.0, 0.0)
    with pytest.raises(ValueError, match="generator and variance_noise"):
        s.step(v, int(s.timesteps[0]), x, eta=eta, generator=g, variance_noise=noise)
    with pytest.raises(NotImplementedError):
        s.step(v, int(s.timesteps[0]), x, eta=eta, use_clipped_model_output=True)


def test_scheduler_noise_coefficients_are_diffusers_fp32_arithmetic():
    s = _sched(20)
    for t in [int(t) for t in s.timesteps[:-1]]:
        prev_t = t - 1000 // 20
        a_t, a_p = s.alphas_cumprod[t], s.alphas_cumprod[prev_t]
        var = ((1 - a_p) / (1 - a_t)) * (1 - a_t / a_p)
        std = 0.7 * var ** 0.5
        assert s.noise_coefficients(t, 0.7) == (float((1 - a_p - std ** 2) ** 0.5), float(std))


def test_zero_snr_first_step_at_eta_1_is_finite():
    """At eta = 1 on the reference's zero-terminal-SNR schedule, 1 - abar_prev - sigma^2 is 0 in real arithmetic at
    t = 999 and -1 ulp in fp32 at 20 and 25 steps, where diffusers' step (restated by the oracle) returns NaN. The
    scheduler takes sqrt(0); every other step equals the oracle to the bit."""
    from oracle import sampler_options_oracle as SO
    from oracle import torch_oracle as O
    for n in (20, 25):
        s, d = _sched(n), O.DDIM()
        d.set_timesteps(n)
        x, v, noise = (torch.randn(1, 4, 2, 3, 3, generator=torch.Generator().manual_seed(i)) for i in range(3))
        for t in [int(t) for t in s.timesteps]:
            got = s.step(v, t, x, eta=1.0, variance_noise=noise).prev_sample
            want = SO.ddim_step(d, v, t, x, 1.0, noise)
            if t == 999:
                assert bool(torch.isnan(want).all()) and bool(torch.isfinite(got).all())
                assert s.noise_coefficients(t, 1.0)[0] == 0.0
            else:
                assert torch.equal(got, want), (n, t)


def _pipeline(O, seed, widths, vcfg):
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection

    from mimo_b200.host import modules as M
    from mimo_b200.host.pipeline import Pose2VideoPipeline
    from mimo_b200.host.scheduler import DDIMScheduler
    cfg = O.UNetConfig(block_out_channels=widths)
    mk = dict(num_attention_heads=8, num_transformer_block=1, attention_block_types=["Temporal_Self", "Temporal_Self"],
              temporal_position_encoding=True, temporal_position_encoding_max_len=32, temporal_attention_dim_div=1)
    den = M.UNet3DConditionModel(block_out_channels=widths, cross_attention_dim=768, use_inflated_groupnorm=True,
                                 use_motion_module=True, motion_module_mid_block=True, motion_module_type="Vanilla",
                                 motion_module_kwargs=mk)
    ref = M.UNet2DConditionModel(block_out_channels=widths, cross_attention_dim=768)
    pg = M.PoseGuider(widths[0], 3, (16, 32, 96, 256))
    vae = M.AutoencoderKL(block_out_channels=vcfg.block_out_channels)
    sds = dict(den=O.make_denoising_unet_sd(cfg, seed), ref=O.make_reference_unet_sd(cfg, seed + 1),
               pg=O.make_pose_guider_sd(seed + 2, widths[0]), vae=O.make_vae_sd(vcfg, seed + 3))
    for m, k in ((den, "den"), (ref, "ref"), (pg, "pg"), (vae, "vae")):
        m.load_state_dict(sds[k], strict=True)
    torch.manual_seed(seed + 4)
    clip = CLIPVisionModelWithProjection(CLIPVisionConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=2,
                                                          num_attention_heads=4, image_size=224, patch_size=32,
                                                          projection_dim=cfg.cross_attention_dim)).eval()
    pipe = Pose2VideoPipeline(vae=vae, image_encoder=clip, reference_unet=ref, denoising_unet=den, pose_guider=pg,
                              scheduler=DDIMScheduler(**SCHED_KW))
    return pipe, clip


def _plumbing():
    """The oracle-backed engine stand-ins of test_pipeline_plumbing_cpu.py (loaded by path: tests/ is not a package)."""
    import importlib.util
    from pathlib import Path
    spec = importlib.util.spec_from_file_location("_plumbing_standins",
                                                  Path(__file__).with_name("test_pipeline_plumbing_cpu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod._Event, mod._oracle_engines


def _inputs(seed, size, frames):
    import PIL.Image
    rng = np.random.RandomState(seed)
    ref_img = PIL.Image.fromarray(rng.randint(0, 256, (size, size, 3), dtype=np.uint8))
    poses, bks = [], []
    for i in range(frames):
        a = np.zeros((size, size, 3), np.uint8)
        a[size // 4: size // 2 + i % 8, size // 3: size // 3 + 40] = rng.randint(11, 256, 3)
        poses.append(PIL.Image.fromarray(a))
        bks.append(PIL.Image.fromarray(rng.randint(0, 256, (size, size, 3), dtype=np.uint8)))
    return ref_img, poses, bks


@pytest.mark.parametrize("case", [0, 1])
def test_own_sampler_with_eta_and_interpolation_matches_reference_clip(monkeypatch, golden_dir, case):
    from mimo_b200 import ops
    from mimo_b200.host import interpolation as I
    from mimo_b200.host.pipeline import Pose2VideoPipeline
    from oracle import sampler_options_oracle as SO
    from oracle import torch_oracle as O
    _Event, _oracle_engines = _plumbing()
    g = torch.load(golden_dir / "pipeline_sampler_options.pt")
    c = g["cases"][case]
    seed, size, F_, steps = g["seed"], g["size"], g["F"], g["steps"]
    widths, vcfg = tuple(g["widths"]), O.VAEConfig(block_out_channels=tuple(g["vae_widths"]))
    _oracle_engines(monkeypatch, O, O.UNetConfig(block_out_channels=widths), vcfg)
    monkeypatch.setattr(torch.cuda, "Event", _Event)
    monkeypatch.setattr(I, "_method", None)
    I.set_tensor_interpolation_method(c["slerp"])
    calls = []

    def cfg_ddim_noise(pu, pc, latents, guidance, sa_t, s1a_t, sa_p, dir_c, noise, sigma, *, counter=None,
                       frame_stride=0):
        calls.append(sigma)
        v = pu + guidance * (pc - pu)
        x = latents[0]
        x0 = sa_t * x - s1a_t * v
        eps = sa_t * v + s1a_t * x
        latents[0] = sa_p * x0 + dir_c * eps + sigma * noise[0]
        return latents

    def no_plain_step(*a, **k):
        raise AssertionError("eta > 0 must not run the eta = 0 kernel")

    def interpolate(latents, k, method):
        return SO.interpolate_latents(latents, k, (I.linear, I.slerp)[method])

    monkeypatch.setattr(ops, "cfg_ddim_step", no_plain_step)
    monkeypatch.setattr(ops, "cfg_ddim_step_noise", cfg_ddim_noise)
    monkeypatch.setattr(ops, "interpolate_frames", interpolate)
    pipe, clip = _pipeline(O, seed, widths, vcfg)
    monkeypatch.setattr(Pose2VideoPipeline, "_clip", lambda self: type("C", (), {
        "image_embeds": staticmethod(lambda px: clip(px).image_embeds)})())
    eng = pipe.denoising_unet.engine()
    eng.xchg, eng._graphs = None, {}
    ref_img, poses, bks = _inputs(seed, size, F_)
    with torch.no_grad():
        host = pipe.preprocess(ref_img, poses, bks, size, size, F_, torch.manual_seed(g["generator_seed"]), torch.float32,
                               steps, c["eta"])
        assert tuple(host["step_noise"].shape) == (steps, 1, 4, F_, size // 8, size // 8)
        out = pipe.sample_tensors(host, steps, g["guidance"], eta=c["eta"], interpolation_factor=c["k"])
    assert len(calls) == steps and calls[-1] == 0.0
    lat, want_lat = out["latents"], c["latents"].float()
    assert lat.shape == (1, 4, F_, size // 8, size // 8)
    assert float((lat - want_lat).norm() / want_lat.norm()) < 2e-3  # the fixture is stored in fp16
    vid, want = out["videos"], c["videos"].float()
    assert vid.shape == (1, 3, (F_ - 1) * c["k"] + 1, size, size)
    assert float((vid[:, :, :, ::4, ::4] - want).norm() / want.norm()) < 2e-3


def _call_stub(monkeypatch, F_=4):
    """A Pose2VideoPipeline whose models claim a CUDA device and whose preprocess must never run: __call__'s checks."""
    from mimo_b200.host.pipeline import Pose2VideoPipeline
    pipe = Pose2VideoPipeline.__new__(Pose2VideoPipeline)
    pipe.denoising_unet = SimpleNamespace(device=torch.device("cuda"), dtype=torch.float16)

    def no_work(*a, **k):
        raise AssertionError("work started before the arguments were checked")

    monkeypatch.setattr(pipe, "preprocess", no_work, raising=False)
    monkeypatch.setattr(pipe, "latent_levels", no_work, raising=False)
    return lambda **kw: pipe(None, [None] * F_, [None] * F_, 64, 64, F_, 2, 3.5, **kw)


def test_refusals_come_before_any_work(monkeypatch):
    from mimo_b200.host import interpolation as I
    monkeypatch.setattr(I, "_method", None)
    call = _call_stub(monkeypatch)
    with pytest.raises(TypeError, match="set_tensor_interpolation_method"):
        call(interpolation_factor=2)
    monkeypatch.setattr(I, "_method", I.linear)
    with pytest.raises(ValueError, match="at least 2 frames"):
        _call_stub(monkeypatch, F_=1)(interpolation_factor=3)
    monkeypatch.setattr(I, "_method", lambda a, b, t: a)
    with pytest.raises(NotImplementedError, match="linear and slerp"):
        call(interpolation_factor=2)
    with pytest.raises(ValueError, match="eta"):
        call(eta=-0.5)
    with pytest.raises(NotImplementedError):
        call(context_batch_size=2)
    with pytest.raises(NotImplementedError):
        call(num_images_per_prompt=2)
    # k <= 1 is a no-op, as in the reference, whatever the registry holds: the call gets as far as the work
    for k in (0, 1, -3):
        with pytest.raises(AssertionError, match="before the arguments"):
            call(interpolation_factor=k, eta=1.0)


def test_overlay_utils_reexports_the_host_registry(monkeypatch):
    import src.pipelines.utils as U
    from mimo_b200.host import interpolation as I
    monkeypatch.setattr(I, "_method", None)
    assert U.get_tensor_interpolation_method() is None
    U.set_tensor_interpolation_method(True)
    assert I.get_tensor_interpolation_method() is I.slerp and I.kernel_method(U.slerp) == 1
    U.set_tensor_interpolation_method(False)
    assert I.get_tensor_interpolation_method() is I.linear and I.kernel_method(U.linear) == 0


def test_new_entry_points_are_bound_and_check_arguments_before_the_device_probe():
    from mimo_b200 import lib as L
    lib = L.load()
    err = lambda: lib.mimo_last_error().decode()
    P, N = ctypes.c_void_p(16), None
    for name in ("mimo_cfg_ddim_step_noise", "mimo_interpolate_frames"):
        assert name in L.SYMBOLS
    step = lambda **kw: lib.mimo_cfg_ddim_step_noise(*[kw.get(k, v) for k, v in dict(
        pu=P, pc=P, cnt=N, fs=0, lat=P, count=64, g=3.5, a=0.5, b=0.5, c=0.5, d=0.5, noise=P, sigma=0.1, dt=0,
        st=N).items()])
    for bad, needle in ((dict(noise=N), "null"), (dict(lat=N), "null"), (dict(count=0), "count"), (dict(dt=7), "dtype"),
                        (dict(sigma=-1.0), "sigma"), (dict(d=float("nan")), "dir_coef"),
                        (dict(cnt=P, fs=5), "frame_stride")):
        assert step(**bad) == -1 and needle in err(), (bad, err())
    interp = lambda **kw: lib.mimo_interpolate_frames(*[kw.get(k, v) for k, v in dict(
        src=P, dst=ctypes.c_void_p(4096), f=3, hw=64, k=2, m=1, dt=1, st=N).items()])
    for bad, needle in ((dict(src=N), "null"), (dict(dst=P), "aliased"), (dict(f=1), "frames >= 2"),
                        (dict(k=1), "k >= 2"), (dict(m=2), "method"), (dict(hw=0), "hw > 0"), (dict(dt=3), "dtype")):
        assert interp(**bad) == -1 and needle in err(), (bad, err())
