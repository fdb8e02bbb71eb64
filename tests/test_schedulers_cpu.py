"""DPM-Solver++ (multistep), Euler and Euler-ancestral on the CPU: the host schedulers' tables and tensor step()
against the oracle (oracle/schedulers_oracle.py), the affine coefficient form the fused kernel runs against step() in
float64, the generator's draw order, engine_scheduler()'s mapping of diffusers-named schedulers, the refusals, this
repo's sampler (engine calls replaced by oracle-backed stand-ins) against the clips the reference's own pipeline file
produced over these schedulers (tests/golden/pipeline_schedulers.pt, written by oracle/gen_scheduler_golden.py), and
the argument checks of mimo_cfg_multistep."""
import ctypes
import importlib.util
from pathlib import Path
from types import SimpleNamespace

import pytest
import torch

SCHED_KW = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False, steps_offset=1,
                prediction_type="v_prediction", rescale_betas_zero_snr=True, timestep_spacing="trailing")
STEPS = (4, 10, 20, 25)


def _S():
    from mimo_b200.host import scheduler as S
    return S


def _engine(kind: str, order: int = 2, **kw):
    S = _S()
    if kind == "dpm":
        return S.DPMSolverMultistepScheduler(solver_order=order, **{**SCHED_KW, **kw})
    return (S.EulerAncestralDiscreteScheduler if kind == "euler_a" else S.EulerDiscreteScheduler)(**{**SCHED_KW, **kw})


def _oracle(kind: str, order: int = 2):
    from oracle import schedulers_oracle as SC
    return SC.DPMSolverPP(order) if kind == "dpm" else (SC.EulerAncestral if kind == "euler_a" else SC.Euler)()


KINDS = [("dpm", 1), ("dpm", 2), ("dpm", 3), ("euler", 0), ("euler_a", 0)]


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


@pytest.mark.parametrize("kind,order", KINDS)
def test_tables_and_init_noise_sigma_match_oracle(kind, order):
    S = _S()
    for n in STEPS:
        s, o = _engine(kind, order), _oracle(kind, order)
        s.set_timesteps(n)
        o.set_timesteps(n)
        assert s.timesteps.dtype == o.timesteps.dtype and torch.equal(s.timesteps, o.timesteps), n
        assert torch.equal(s.sigmas, o.sigmas), n
        assert torch.equal(torch.as_tensor(s.init_noise_sigma), torch.as_tensor(o.init_noise_sigma)), n
        assert float(s.alphas_cumprod[-1]) == 2.0 ** -24
        if kind == "dpm":  # trailing spacing: DDIM's table
            d = S.DDIMScheduler(**SCHED_KW)
            d.set_timesteps(n)
            assert torch.equal(s.timesteps, d.timesteps) and s.init_noise_sigma == 1.0
        else:
            assert abs(float(s.init_noise_sigma) - 4096.0) < 1.0
    # the DDIM scheduler keeps its abar[-1] = 0
    assert float(S.DDIMScheduler(**SCHED_KW).alphas_cumprod[-1]) == 0.0


@pytest.mark.parametrize("kind,order", KINDS)
def test_step_matches_oracle(kind, order):
    """The engine's tensor step() (VP form from abar for DPM-Solver++, float64 scalars) against diffusers' arithmetic
    (sigma form, fp32 scalars) in fp32: equal to ~1e-6."""
    for n in (4, 10):
        s, o = _engine(kind, order), _oracle(kind, order)
        s.set_timesteps(n)
        o.set_timesteps(n)
        g = torch.Generator().manual_seed(n)
        x = torch.randn(1, 4, 3, 5, 6, generator=g) * float(s.init_noise_sigma)
        xo = x.clone()
        for i, t in enumerate(s.timesteps):
            v = torch.randn(x.shape, generator=g)
            noise = torch.randn(x.shape, generator=g)
            want_in = x if kind == "dpm" else o.scale_model_input(x, o.timesteps[i])
            assert torch.equal(s.scale_model_input(x, t), want_in)
            kw = dict(variance_noise=noise) if kind == "euler_a" else {}
            x = s.step(v, t, x, **kw).prev_sample
            xo = o.step(v, o.timesteps[i], xo, noise=noise if kind == "euler_a" else None).prev_sample
            assert x.dtype == torch.float32 and _rel(x, xo) < 2e-6, (n, i, _rel(x, xo))


def _affine(s, kind, n, dtype=torch.float64, seed=0):
    """Run step() and the coefficient form side by side over every step of an n-step schedule; yield the relative
    difference per step."""
    s.set_timesteps(n)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(2, 3, 4, generator=g, dtype=dtype) * float(s.init_noise_sigma)
    y = x.clone()
    hist = [None, None]
    for i, t in enumerate(s.timesteps):
        v = torch.randn(x.shape, generator=g, dtype=dtype)
        noise = torch.randn(x.shape, generator=g, dtype=dtype)
        x = s.step(v, t, x, **(dict(variance_noise=noise) if kind == "euler_a" else {})).prev_sample
        a, b, cx, cm, c1, c2, cn = s.multistep_coefficients(i)
        m = a * y + b * v
        nxt = cx * y + cm * m + cn * noise
        if c1:
            nxt = nxt + c1 * hist[(i - 1) % 2]
        if c2:
            nxt = nxt + c2 * hist[i % 2]
        hist[i % 2] = m
        y = nxt
        yield i, _rel(y, x)


@pytest.mark.parametrize("kind,order", KINDS)
@pytest.mark.parametrize("n", STEPS)
def test_coefficient_form_reproduces_step_in_float64(kind, order, n):
    s = _engine(kind, order)
    worst = max(e for _, e in _affine(s, kind, n))
    assert worst < 1e-12, worst


def test_dpm_orders_warm_up_and_lower_order_final():
    s = _engine("dpm", 3)
    s.set_timesteps(5)
    assert [s.solver_order_at(i) for i in range(5)] == [1, 2, 3, 2, 1]
    s.set_timesteps(20)
    assert [s.solver_order_at(i) for i in range(20)] == [1, 2] + [3] * 17 + [1]
    s = _engine("dpm", 2)
    s.set_timesteps(4)
    assert [s.solver_order_at(i) for i in range(4)] == [1, 2, 2, 1]
    # the last step lands on sigma = 0 and returns the x0 prediction: x' = m
    a, b, cx, cm, c1, c2, cn = s.multistep_coefficients(3)
    assert (cx, cm, c1, c2, cn) == (0.0, 1.0, 0.0, 0.0, 0.0)


def test_euler_ancestral_consumes_one_draw_per_step_and_euler_none():
    for kind, draws in (("euler_a", 1), ("euler", 0)):
        s = _engine(kind)
        s.set_timesteps(4)
        x = torch.randn(1, 4, 3, 5, 6, generator=torch.Generator().manual_seed(1)).half()
        v = torch.randn(1, 4, 3, 5, 6, generator=torch.Generator().manual_seed(2)).half()
        g, g_ref = torch.Generator().manual_seed(7), torch.Generator().manual_seed(7)
        for t in s.timesteps:  # also the last step, where sigma_up = 0
            x = s.step(v, t, x, generator=g).prev_sample
            for _ in range(draws):
                torch.randn(x.shape, generator=g_ref, dtype=torch.float16)
            assert x.dtype == torch.float16
            assert torch.equal(g.get_state(), g_ref.get_state()), (kind, t)
        assert s.draws_noise == bool(draws)


def test_engine_scheduler_maps_diffusers_named_standins():
    S = _S()
    cfg = {"_class_name": "DDIMScheduler", "_diffusers_version": "0.24.0", "num_train_timesteps": 1000, **SCHED_KW}
    for name, cls in (("DDIMScheduler", S.DDIMScheduler), ("DPMSolverMultistepScheduler", S.DPMSolverMultistepScheduler),
                      ("EulerDiscreteScheduler", S.EulerDiscreteScheduler),
                      ("EulerAncestralDiscreteScheduler", S.EulerAncestralDiscreteScheduler)):
        standin = type(name, (), {})()
        standin.config = dict(cfg)
        got = S.engine_scheduler(standin)
        assert type(got) is cls and got.config.timestep_spacing == "trailing", name
    own = S.DDIMScheduler(**SCHED_KW)
    assert S.engine_scheduler(own) is own
    standin = type("DDIMScheduler", (), {"config": cfg})()
    mapped = S.engine_scheduler(standin)
    own.set_timesteps(20)
    mapped.set_timesteps(20)
    assert torch.equal(own.timesteps, mapped.timesteps)
    for t in own.timesteps.tolist():
        assert mapped.step_coefficients(t) == own.step_coefficients(t)
    # X.from_config(pipe.scheduler.config): the DDIM config carries every constructor argument
    dpm = S.DPMSolverMultistepScheduler.from_config(own.config, solver_order=3)
    assert dpm.config.solver_order == 3 and torch.equal(dpm.alphas_cumprod[:-1], own.alphas_cumprod[:-1])
    assert S.DDIMScheduler.from_config(own.config).config == own.config
    with pytest.raises(NotImplementedError, match="DPMSolverMultistepScheduler"):
        S.engine_scheduler(type("UniPCMultistepScheduler", (), {"config": cfg})())


def test_refusals():
    S = _S()
    for cls in (S.LMSDiscreteScheduler, S.PNDMScheduler):
        with pytest.raises(NotImplementedError, match="DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler"):
            cls(**SCHED_KW)
        with pytest.raises(NotImplementedError, match="not run by the engine"):
            S.engine_scheduler(type(cls.__name__, (), {"config": SCHED_KW})())
    for kw in (dict(algorithm_type="dpmsolver"), dict(algorithm_type="sde-dpmsolver++"), dict(solver_type="heun"),
               dict(use_karras_sigmas=True), dict(thresholding=True), dict(final_sigmas_type="sigma_min"),
               dict(prediction_type="epsilon")):
        with pytest.raises(NotImplementedError):
            _engine("dpm", **kw)
    with pytest.raises(ValueError):
        _engine("dpm", 4)
    for kind in ("euler", "euler_a"):
        for kw in (dict(use_karras_sigmas=True), dict(prediction_type="epsilon")):
            with pytest.raises(NotImplementedError):
                _engine(kind, **kw)
        s = _engine(kind)
        s.set_timesteps(4)
        x = torch.zeros(2, 3)
        with pytest.raises(NotImplementedError, match="s_churn"):
            s.step(x, s.timesteps[0], x, s_churn=0.5)


def test_pipeline_refuses_lms_pndm_before_any_work(monkeypatch):
    from mimo_b200.host.pipeline import Pose2VideoPipeline
    for name in ("LMSDiscreteScheduler", "PNDMScheduler", "KDPM2DiscreteScheduler"):
        pipe = Pose2VideoPipeline.__new__(Pose2VideoPipeline)
        pipe.denoising_unet = SimpleNamespace(device=torch.device("cuda"), dtype=torch.float16)
        pipe.scheduler = type(name, (), {"config": SCHED_KW})()

        def no_work(*a, **k):
            raise AssertionError("work started before the arguments were checked")

        monkeypatch.setattr(pipe, "preprocess", no_work, raising=False)
        monkeypatch.setattr(pipe, "latent_levels", lambda *a: None, raising=False)
        with pytest.raises(NotImplementedError, match="EulerDiscreteScheduler"):
            pipe(None, [None] * 4, [None] * 4, 64, 64, 4, 2, 3.5)
        with pytest.raises(NotImplementedError, match="EulerDiscreteScheduler"):
            pipe.sample_tensors({"latents": torch.zeros(1, 4, 4, 8, 8)}, 2, 3.5)


def _helpers():
    """_pipeline / _plumbing / _inputs of test_sampler_options_cpu.py (loaded by path: tests/ is not a package)."""
    spec = importlib.util.spec_from_file_location("_sampler_options_helpers",
                                                  Path(__file__).with_name("test_sampler_options_cpu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _cfg_multistep_standin(calls):
    def cfg_multistep(pu, pc, latents, guidance, co, hist_out, *, h1=None, h2=None, noise=None, counter=None,
                      frame_stride=0):
        assert counter is None
        a, b, cx, cm, c1, c2, cn = co
        calls.append(co)
        v = pu + guidance * (pc - pu)
        x = latents[0]
        m = a * x + b * v
        acc = cx * x + cm * m
        for coef, t in ((c1, h1), (c2, h2), (cn, noise)):
            if t is not None:
                acc = acc + coef * t[0]
        hist_out[0] = m
        latents[0] = acc
        return latents
    return cfg_multistep


@pytest.mark.parametrize("case", [0, 1, 2, 3])
def test_own_sampler_matches_reference_clip(monkeypatch, golden_dir, case):
    from mimo_b200 import ops
    from mimo_b200.host import scheduler as S
    from mimo_b200.host.pipeline import Pose2VideoPipeline
    from oracle import torch_oracle as O
    H = _helpers()
    _Event, _oracle_engines = H._plumbing()
    g = torch.load(golden_dir / "pipeline_schedulers.pt")
    c = g["cases"][case]
    seed, size, F_, steps = g["seed"], g["size"], g["F"], c["steps"]
    widths, vcfg = tuple(g["widths"]), O.VAEConfig(block_out_channels=tuple(g["vae_widths"]))
    _oracle_engines(monkeypatch, O, O.UNetConfig(block_out_channels=widths), vcfg)
    monkeypatch.setattr(torch.cuda, "Event", _Event)
    calls = []

    def no_ddim(*a, **k):
        raise AssertionError("a non-DDIM scheduler must not run the DDIM kernels")

    monkeypatch.setattr(ops, "cfg_ddim_step", no_ddim)
    monkeypatch.setattr(ops, "cfg_ddim_step_noise", no_ddim)
    monkeypatch.setattr(ops, "cfg_multistep", _cfg_multistep_standin(calls))
    pipe, clip = H._pipeline(O, seed, widths, vcfg)
    cls = getattr(S, c["scheduler"])
    pipe.scheduler = cls(**SCHED_KW, **({"solver_order": c["solver_order"]} if "solver_order" in c else {}))
    monkeypatch.setattr(Pose2VideoPipeline, "_clip", lambda self: type("C", (), {
        "image_embeds": staticmethod(lambda px: clip(px).image_embeds)})())
    eng = pipe.denoising_unet.engine()
    eng.xchg, eng._graphs = None, {}
    ref_img, poses, bks = H._inputs(seed, size, F_)
    with torch.no_grad():
        host = pipe.preprocess(ref_img, poses, bks, size, size, F_, torch.manual_seed(g["generator_seed"]), torch.float32,
                               steps)
        if c["scheduler"] == "EulerAncestralDiscreteScheduler":
            assert tuple(host["step_noise"].shape) == (steps, 1, 4, F_, size // 8, size // 8)
        else:
            assert "step_noise" not in host
        out = pipe.sample_tensors(host, steps, g["guidance"], eta=0.7)  # eta reaches DDIM only
    assert len(calls) == steps
    lat, want_lat = out["latents"], c["latents"].float()
    assert float((lat - want_lat).norm() / want_lat.norm()) < 2e-3  # the fixture is stored in fp16
    vid, want = out["videos"], c["videos"].float()
    assert vid.shape == (1, 3, F_, size, size)
    assert float((vid[:, :, :, ::4, ::4] - want).norm() / want.norm()) < 2e-3


def test_cfg_multistep_is_bound_and_checks_arguments_before_the_device_probe():
    from mimo_b200 import lib as L
    lib = L.load()
    assert "mimo_cfg_multistep" in L.SYMBOLS
    assert lib.mimo_abi_sizeof(7) == ctypes.sizeof(L.CfgMultistepParams)
    err = lambda: lib.mimo_last_error().decode()
    base = dict(pred_uncond=16, pred_cond=32, latents=48, hist_out=64, h1=80, h2=96, noise=112, count=64,
                guidance=3.5, a=0.5, b=-0.5, c_x=0.5, c_m=0.5, c_1=0.1, c_2=0.1, c_n=0.1, dtype=0)
    step = lambda **kw: lib.mimo_cfg_multistep(ctypes.byref(L.CfgMultistepParams(**{**base, **kw})), None)
    assert lib.mimo_cfg_multistep(None, None) == -1 and "null" in err()
    for bad, needle in ((dict(latents=None), "null"), (dict(hist_out=None), "null"), (dict(pred_cond=None), "null"),
                        (dict(count=0), "count"), (dict(dtype=2), "dtype"), (dict(c_m=float("nan")), "non-finite"),
                        (dict(a=float("inf")), "non-finite"), (dict(h1=None), "non-zero coefficient"),
                        (dict(noise=None), "non-zero coefficient"), (dict(h2=None), "non-zero coefficient"),
                        (dict(hist_out=48), "aliases"), (dict(hist_out=16), "aliases"), (dict(hist_out=80), "aliases"),
                        (dict(hist_out=112), "aliases"), (dict(counter=128, frame_stride=5), "frame_stride")):
        assert step(**bad) == -1 and needle in err(), (bad, err())
    # hist_out may alias h2 and nulls with zero coefficients are allowed: without a device the call gets as far as the
    # device probe
    if not torch.cuda.is_available():
        assert step(hist_out=96, h1=None, c_1=0.0, noise=None, c_n=0.0) != 0
        assert "null" not in err() and "alias" not in err()
