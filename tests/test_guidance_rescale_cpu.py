"""Rescaled classifier-free guidance (guidance_rescale) on the CPU: the oracle's rescale_noise_cfg against a second plain
statement of diffusers' expression, the oracle sampling loop with guidance_rescale = 0 against torch_oracle.sample_clip
and schedulers_oracle.sample_clip bit for bit, the pipeline's refusals before any work, the sampler's host logic with the
kernels replaced by torch stand-ins, and the argument checks of mimo_cfg_rescale."""
import ctypes
import importlib.util
import math
from pathlib import Path

import pytest
import torch

SCHED_KW = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False, steps_offset=1,
                prediction_type="v_prediction", rescale_betas_zero_snr=True, timestep_spacing="trailing")


def _plain_rescale(cfg, text, phi):
    """diffusers' rescale_noise_cfg written out without torch.std: unbiased variance over every element of the one
    batch entry, evaluated in fp64 and rounded to the tensors' dtype, then the same mix."""
    def std(x):
        d = x.double()
        return ((d - d.mean()) ** 2).sum().div(d.numel() - 1).sqrt().to(x.dtype)
    return phi * (cfg * (std(text) / std(cfg))) + (1 - phi) * cfg


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("phi", [0.0, 0.3, 0.7, 1.0])
def test_oracle_rescale_matches_a_plain_statement(dtype, phi):
    from oracle import guidance_rescale_oracle as GR
    g = torch.Generator().manual_seed(7)
    text = (torch.randn(1, 4, 6, 8, 8, generator=g) * 0.8 + 0.1).to(dtype)
    uncond = torch.randn(1, 4, 6, 8, 8, generator=g).to(dtype)
    cfg = uncond + 3.5 * (text - uncond)
    got = GR.rescale_noise_cfg(cfg, text, phi)
    want = _plain_rescale(cfg, text, phi)
    assert got.dtype == dtype and got.shape == cfg.shape
    if phi == 0.0:
        assert torch.equal(got, cfg)  # 0 * x + 1 * cfg
    if dtype == torch.float32:
        torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-6)
    else:  # torch.std on fp16 accumulates in a wider type than fp16 but not fp64: at most one ulp per element apart
        ulp = torch.finfo(torch.float16).eps * want.float().abs().clamp_min(2.0 ** -14)
        assert bool(((got.float() - want.float()).abs() <= ulp).all())
    std_after = float(got.double().std())
    if phi == 1.0:  # the point of the rescale: the guided prediction gets the text prediction's std
        assert abs(std_after - float(text.double().std())) < 2e-2 * std_after


def _weights(seed):
    from oracle import torch_oracle as O
    widths = (128, 256, 512, 512)
    cfg, vcfg = O.UNetConfig(block_out_channels=widths), O.VAEConfig(block_out_channels=(32, 64, 128, 128))
    return O.Weights(O.make_denoising_unet_sd(cfg, seed), O.make_reference_unet_sd(cfg, seed + 1),
                     O.make_pose_guider_sd(seed + 2, widths[0]), O.make_vae_sd(vcfg, seed + 3), cfg, vcfg)


def _clip_inputs(seed, F_, size=64):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(1, 3, size, size, generator=g) * 2 - 1, torch.rand(1, 3, F_, size, size, generator=g),
            torch.rand(F_, 3, size, size, generator=g) * 2 - 1, torch.randn(1, 768, generator=g),
            torch.randn(1, 4, F_, size // 8, size // 8, generator=g))


def test_oracle_sample_clip_at_zero_is_the_existing_oracles_bit_for_bit():
    """guidance_rescale = 0 (and omitted) computes exactly what torch_oracle.sample_clip (DDIM, here over two
    overlapping windows so the counter divides) and schedulers_oracle.sample_clip (DPM-Solver++ 2M) compute; 0.7
    changes the clip."""
    from oracle import guidance_rescale_oracle as GR
    from oracle import schedulers_oracle as SC
    from oracle import torch_oracle as O
    W, F_, steps = _weights(610), 6, 2
    args = _clip_inputs(611, F_)
    win = dict(context_frames=4, context_overlap=2, decode=False)
    with torch.no_grad():
        ddim = O.sample_clip(W, *args, steps, 3.5, **win)["latents"]
        assert torch.equal(GR.sample_clip(W, *args, steps, 3.5, guidance_rescale=0.0, **win)["latents"], ddim)
        assert torch.equal(GR.sample_clip(W, *args, steps, 3.5, **win)["latents"], ddim)
        resc = GR.sample_clip(W, *args, steps, 3.5, guidance_rescale=0.7, **win)["latents"]
        assert bool(torch.isfinite(resc).all()) and not torch.equal(resc, ddim)
        dpm = SC.sample_clip(W, *args, steps, 3.5, SC.DPMSolverPP(2), decode=False)["latents"]
        assert torch.equal(GR.sample_clip(W, *args, steps, 3.5, SC.DPMSolverPP(2), guidance_rescale=0.0,
                                          decode=False)["latents"], dpm)


def _call_stub(monkeypatch, F_=4):
    """A Pose2VideoPipeline whose models claim a CUDA device and whose preprocess must never run."""
    from types import SimpleNamespace

    from mimo_b200.host.pipeline import Pose2VideoPipeline
    pipe = Pose2VideoPipeline.__new__(Pose2VideoPipeline)
    pipe.denoising_unet = SimpleNamespace(device=torch.device("cuda"), dtype=torch.float16)
    pipe.scheduler = None  # engine_scheduler() would refuse it: the check under test must come first

    def no_work(*a, **k):
        raise AssertionError("work started before the arguments were checked")

    monkeypatch.setattr(pipe, "preprocess", no_work, raising=False)
    monkeypatch.setattr(pipe, "latent_levels", lambda *a: None, raising=False)
    return pipe


@pytest.mark.parametrize("phi", [-0.1, 1.5, float("nan"), float("inf"), -float("inf")])
def test_out_of_range_guidance_rescale_is_refused_before_any_work(monkeypatch, phi):
    pipe = _call_stub(monkeypatch)
    with pytest.raises(ValueError, match="guidance_rescale"):
        pipe(None, [None] * 4, [None] * 4, 64, 64, 4, 2, 3.5, guidance_rescale=phi)
    with pytest.raises(ValueError, match="guidance_rescale"):
        pipe.sample_tensors({"latents": torch.zeros(1, 4, 4, 8, 8)}, 2, 3.5, guidance_rescale=phi)


@pytest.mark.parametrize("phi", [0.0, 0.7, 1.0])
def test_in_range_guidance_rescale_passes_the_check(monkeypatch, phi):
    from mimo_b200.host.scheduler import DDIMScheduler
    pipe = _call_stub(monkeypatch)
    pipe.scheduler = DDIMScheduler(**SCHED_KW)
    with pytest.raises(AssertionError, match="before the arguments"):  # got as far as the work
        pipe(None, [None] * 4, [None] * 4, 64, 64, 4, 2, 3.5, guidance_rescale=phi)


def _helpers():
    """_pipeline / _plumbing / _inputs of test_sampler_options_cpu.py (loaded by path: tests/ is not a package)."""
    spec = importlib.util.spec_from_file_location("_sampler_options_helpers",
                                                  Path(__file__).with_name("test_sampler_options_cpu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _guide(pu, pc, guidance, counter):
    if counter is not None:
        cv = counter.view(1, -1, 1, 1)
        pu, pc = pu / cv, pc / cv
    return pc, pu + guidance * (pc - pu)


def _standins(calls):
    from oracle import guidance_rescale_oracle as GR

    def cfg_rescale(pu, pc, guidance, phi, out=None, counter=None, frame_stride=0):
        text, cfg = _guide(pu, pc, guidance, counter)
        out.view_as(cfg).copy_(GR.rescale_noise_cfg(cfg[None], text[None], phi)[0])
        calls.append(("rescale", out, guidance, phi, counter is not None))
        return out

    def cfg_ddim_step(pu, pc, latents, guidance, sa_t, s1a_t, sa_p, s1a_p, *, counter=None, frame_stride=0):
        calls.append(("ddim", pu, pc, guidance, counter))
        v = _guide(pu, pc, guidance, counter)[1]
        x = latents[0]
        latents[0] = sa_p * (sa_t * x - s1a_t * v) + s1a_p * (sa_t * v + s1a_t * x)
        return latents

    def cfg_multistep(pu, pc, latents, guidance, co, hist_out, *, h1=None, h2=None, noise=None, counter=None,
                      frame_stride=0):
        calls.append(("multistep", pu, pc, guidance, counter))
        a, b, cx, cm, c1, c2, cn = co
        v = _guide(pu, pc, guidance, counter)[1]
        x = latents[0]
        m = a * x + b * v
        acc = cx * x + cm * m
        for coef, t in ((c1, h1), (c2, h2), (cn, noise)):
            if t is not None:
                acc = acc + coef * t[0]
        hist_out[0] = m
        latents[0] = acc
        return latents

    return cfg_rescale, cfg_ddim_step, cfg_multistep


@pytest.mark.parametrize("scheduler", ["DDIMScheduler", "DPMSolverMultistepScheduler"])
def test_sampler_runs_the_rescale_only_with_cfg_and_feeds_its_output_to_the_step(monkeypatch, golden_dir, scheduler):
    """With CFG and phi > 0 every step calls cfg_rescale (with the counter when several windows overlap) and then the
    scheduler's step with (out, out, 1.0, counter=None); phi = 0 or guidance 1 never calls it and the step gets what it
    got before."""
    from mimo_b200 import ops
    from mimo_b200.host import scheduler as S
    from mimo_b200.host.pipeline import Pose2VideoPipeline
    from oracle import torch_oracle as O
    H = _helpers()
    _Event, _oracle_engines = H._plumbing()
    g = torch.load(golden_dir / "pipeline_schedulers.pt")
    seed, size, F_, steps = g["seed"], g["size"], g["F"], 2
    widths, vcfg = tuple(g["widths"]), O.VAEConfig(block_out_channels=tuple(g["vae_widths"]))
    _oracle_engines(monkeypatch, O, O.UNetConfig(block_out_channels=widths), vcfg)
    monkeypatch.setattr(torch.cuda, "Event", _Event)
    calls = []
    rescale, ddim, multistep = _standins(calls)
    monkeypatch.setattr(ops, "cfg_rescale", rescale)
    monkeypatch.setattr(ops, "cfg_ddim_step", ddim)
    monkeypatch.setattr(ops, "cfg_multistep", multistep)
    pipe, clip = H._pipeline(O, seed, widths, vcfg)
    pipe.scheduler = getattr(S, scheduler)(**SCHED_KW)
    monkeypatch.setattr(Pose2VideoPipeline, "_clip", lambda self: type("C", (), {
        "image_embeds": staticmethod(lambda px: clip(px).image_embeds)})())
    eng = pipe.denoising_unet.engine()
    eng.xchg, eng._graphs = None, {}
    ref_img, poses, bks = H._inputs(seed, size, F_)
    step_kind = "ddim" if scheduler == "DDIMScheduler" else "multistep"
    lat = {}
    with torch.no_grad():
        host = pipe.preprocess(ref_img, poses, bks, size, size, F_, torch.manual_seed(g["generator_seed"]), torch.float32,
                               steps)
        for guidance, phi, windows in ((3.5, 0.0, 1), (3.5, 0.7, 1), (3.5, 0.7, 2), (1.0, 0.7, 1)):
            calls.clear()
            win = dict(context_frames=4, context_overlap=2) if windows > 1 else {}
            kw = {} if phi == 0.0 else dict(guidance_rescale=phi)
            out = pipe.sample_tensors(dict(host), steps, guidance, decode=False, **win, **kw)
            lat[(guidance, phi, windows)] = out["latents"].clone()
            resc = [c for c in calls if c[0] == "rescale"]
            step = [c for c in calls if c[0] == step_kind]
            assert len(step) == steps and len(calls) == len(step) + len(resc)
            if guidance > 1.0 and phi > 0.0:
                assert len(resc) == steps
                for (_, o, g_, p_, has_cnt), (_, pu, pc, gs, cnt) in zip(resc, step):
                    assert g_ == guidance and p_ == phi and has_cnt == (windows > 1)
                    assert pu is o and pc is o and gs == 1.0 and cnt is None
            else:
                assert not resc
                assert all(gs == guidance for _, _, _, gs, _ in step)
    assert not torch.equal(lat[(3.5, 0.7, 1)], lat[(3.5, 0.0, 1)])


def test_cfg_rescale_is_bound_and_checks_arguments_before_the_device_probe():
    from mimo_b200 import lib as L
    lib = L.load()
    for name in ("mimo_cfg_rescale", "mimo_cfg_rescale_workspace_bytes"):
        assert name in L.SYMBOLS
    assert lib.mimo_abi_sizeof(14) == ctypes.sizeof(L.CfgRescaleParams)
    err = lambda: lib.mimo_last_error().decode()
    big = 300 * 4096
    assert lib.mimo_cfg_rescale_workspace_bytes(ctypes.byref(L.CfgRescaleParams(count=big))) == 256 * 32
    assert lib.mimo_cfg_rescale_workspace_bytes(ctypes.byref(L.CfgRescaleParams(count=4097))) == 2 * 32
    assert lib.mimo_cfg_rescale_workspace_bytes(ctypes.byref(L.CfgRescaleParams(count=1))) < 0
    base = dict(pred_uncond=16, pred_cond=32, counter=None, frame_stride=0, out=48, count=64, workspace=4096,
                workspace_bytes=32, phi=0.7, guidance=3.5, dtype=0)
    call = lambda **kw: lib.mimo_cfg_rescale(ctypes.byref(L.CfgRescaleParams(**{**base, **kw})), None)
    assert lib.mimo_cfg_rescale(None, None) == -1 and "null" in err()
    for bad, needle in ((dict(pred_uncond=None), "null"), (dict(pred_cond=None), "null"), (dict(out=None), "null"),
                        (dict(workspace=None), "null"), (dict(count=0), "count"), (dict(count=-5), "count"),
                        (dict(count=1), "count"), (dict(dtype=2), "dtype"), (dict(guidance=math.nan), "guidance"),
                        (dict(guidance=math.inf), "guidance"), (dict(phi=-0.1), "phi"), (dict(phi=1.5), "phi"),
                        (dict(phi=math.nan), "phi"), (dict(phi=math.inf), "phi"),
                        (dict(counter=128, frame_stride=5), "frame_stride"),
                        (dict(counter=128, frame_stride=0), "frame_stride"),
                        (dict(workspace_bytes=31), "workspace"), (dict(workspace=4104), "workspace"),
                        (dict(out=16), "aliases"), (dict(out=32), "aliases"), (dict(out=4096), "aliases"),
                        (dict(counter=48, frame_stride=4), "aliases")):
        assert call(**bad) == -1 and needle in err(), (bad, err())
