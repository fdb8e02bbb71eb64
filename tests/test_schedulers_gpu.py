"""DPM-Solver++ (multistep), Euler and Euler-ancestral on the H100: the fused mimo_cfg_multistep kernel against an fp64
evaluation of the same expression, graph capture, a DDIM clip through engine_scheduler() with a diffusers-named
scheduler, and the public __call__ with the new schedulers against the oracle (oracle/schedulers_oracle.py)."""
import importlib.util
from pathlib import Path

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
SCHED_KW = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False, steps_offset=1,
                prediction_type="v_prediction", rescale_betas_zero_snr=True, timestep_spacing="trailing")


def _any_size():
    """Helpers of test_any_size_gpu.py (pipeline builder, images, relative error), loaded by path."""
    spec = importlib.util.spec_from_file_location("_any_size_helpers", Path(__file__).with_name("test_any_size_gpu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _coefficient_sets():
    """Real per-step scalars: a third-order DPM-Solver++ step (h1 and h2), a second-order one, Euler-ancestral's first
    step (sigma ~ 4096 and noise), each cast to fp32 once as the sampler does."""
    from mimo_b200.host import scheduler as S
    dpm = S.DPMSolverMultistepScheduler(solver_order=3, **SCHED_KW)
    dpm.set_timesteps(20)
    ea = S.EulerAncestralDiscreteScheduler(**SCHED_KW)
    ea.set_timesteps(20)
    f32 = lambda co: tuple(float(np.float32(c)) for c in co)
    return {"dpm3": f32(dpm.multistep_coefficients(7)), "dpm2": f32(dpm.multistep_coefficients(1)),
            "euler_a": f32(ea.multistep_coefficients(0)), "euler_a_mid": f32(ea.multistep_coefficients(9))}


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("with_counter", [False, True])
@pytest.mark.parametrize("terms", ["none", "history", "history_noise"])
def test_cfg_multistep_matches_fp64(dtype, with_counter, terms):
    """v is the guided prediction in the storage dtype (PyTorch's own roundings, as cfg_ddim_step); m must be
    a x + b v in fp64 rounded once to the storage type, and x' the fp64 affine update of the kernel's own m rounded once
    at the store (bound: the type's unit roundoff on each, plus fp32 arithmetic)."""
    from mimo_b200 import ops
    torch.manual_seed(31)
    F_, h, w = 5, 8, 12
    pred = torch.randn(2, 4, F_, h, w, device=DEV).to(dtype)
    counter = torch.tensor([1, 2, 1, 3, 2], device=DEV).to(dtype)
    u_roff = 2.0 ** (-11 if dtype == torch.float16 else -8)
    for name, co in _coefficient_sets().items():
        a, b, cx, cm, c1, c2, cn = co
        lat = (torch.randn(1, 4, F_, h, w, device=DEV) * (4096.0 if name == "euler_a" else 1.0)).to(dtype)
        h1, h2, noise = (torch.randn(1, 4, F_, h, w, device=DEV).to(dtype) for _ in range(3))
        use_h = terms != "none"
        use_n = terms == "history_noise"
        co = (a, b, cx, cm, c1 if use_h else 0.0, c2 if use_h else 0.0, cn if use_n else 0.0)
        hist = torch.empty_like(lat)
        kw = dict(h1=h1 if use_h else None, h2=h2 if use_h else None, noise=noise if use_n else None)
        if with_counter:
            cv = counter.view(1, F_, 1, 1)
            got = ops.cfg_multistep(pred[0] * cv, pred[1] * cv, lat.clone(), 3.5, co, hist, counter=counter,
                                    frame_stride=h * w, **kw)
            u, c = ((pred * counter.view(1, 1, F_, 1, 1)) / counter.view(1, 1, F_, 1, 1)).chunk(2)
        else:
            got = ops.cfg_multistep(pred[0].contiguous(), pred[1].contiguous(), lat.clone(), 3.5, co, hist, **kw)
            u, c = pred.chunk(2)
        v = (u + 3.5 * (c - u)).double()
        x = lat.double()
        m64 = a * x + b * v
        tol_m = u_roff * m64.abs() + 1e-6 * (abs(a) * x.abs() + abs(b) * v.abs()) + 2.0 ** -24
        assert float(((hist.double() - m64).abs() - tol_m).max()) <= 0, (name, "m")
        terms64 = [cx * x, cm * hist.double()]
        if use_h:
            terms64 += [c1 * h1.double(), c2 * h2.double()]
        if use_n:
            terms64 += [cn * noise.double()]
        want = sum(terms64)
        tol = u_roff * want.abs() + 1e-6 * sum(t.abs() for t in terms64) + 2.0 ** -24
        excess = float(((got.double() - want).abs() - tol).max())
        assert excess <= 0, (name, excess)


def test_cfg_multistep_ring_alias_and_graph_replay_are_bit_identical():
    """hist_out aliasing h2 (the two-slot ring at order 3) equals separate buffers, and a CUDA-graph replay equals the
    eager call bit for bit."""
    from mimo_b200 import ops
    torch.manual_seed(5)
    F_, h, w = 6, 16, 16
    pred = torch.randn(2, 4, F_, h, w, device=DEV).half()
    lat = torch.randn(1, 4, F_, h, w, device=DEV).half()
    noise = torch.randn(1, 4, F_, h, w, device=DEV).half()
    ring = torch.randn(2, 1, 4, F_, h, w, device=DEV).half()
    co = _coefficient_sets()["dpm3"][:6] + (0.25,)
    pu, pc = pred[0].contiguous(), pred[1].contiguous()
    sep_hist = torch.empty_like(lat)
    ref = ops.cfg_multistep(pu, pc, lat.clone(), 3.5, co, sep_hist, h1=ring[1].clone(), h2=ring[0].clone(), noise=noise)
    r = ring.clone()
    eager = ops.cfg_multistep(pu, pc, lat.clone(), 3.5, co, r[0], h1=r[1], h2=r[0], noise=noise)
    assert torch.equal(eager.view(torch.int16), ref.view(torch.int16))
    assert torch.equal(r[0].view(torch.int16), sep_hist.view(torch.int16))
    static_lat, static_ring = lat.clone(), ring.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):  # warm-up outside the capture
        rc = ring.clone()
        ops.cfg_multistep(pu, pc, lat.clone(), 3.5, co, rc[0], h1=rc[1], h2=rc[0], noise=noise)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.cfg_multistep(pu, pc, static_lat, 3.5, co, static_ring[0], h1=static_ring[1], h2=static_ring[0],
                          noise=noise)
    static_lat.copy_(lat)
    static_ring.copy_(ring)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(static_lat.view(torch.int16), ref.view(torch.int16))
    assert torch.equal(static_ring[0].view(torch.int16), sep_hist.view(torch.int16))


def test_ddim_through_a_diffusers_named_scheduler_is_byte_identical():
    """engine_scheduler() builds the engine's DDIMScheduler from a diffusers-named scheduler's config: the clip equals
    the one the engine's own DDIMScheduler makes, byte for byte."""
    A = _any_size()
    F_, size, steps = 8, 128, 3
    torch.manual_seed(42)
    pipe = A._build_pipe(A.WIDTHS, None, A._small_clip(5))
    ref_img, poses, bks = A._images(F_, size, size, 11)
    own = pipe(ref_img, poses, bks, size, size, F_, steps, 3.5, generator=torch.manual_seed(3)).videos
    own_lat = pipe.last_latents.clone()
    standin = type("DDIMScheduler", (), {})()
    standin.config = {"_class_name": "DDIMScheduler", "num_train_timesteps": 1000, "set_alpha_to_one": True, **SCHED_KW}
    pipe.scheduler = standin
    got = pipe(ref_img, poses, bks, size, size, F_, steps, 3.5, generator=torch.manual_seed(3)).videos
    assert torch.equal(pipe.last_latents.view(torch.int16), own_lat.view(torch.int16))
    assert torch.equal(got, own)


@pytest.mark.parametrize("kind,steps", [("dpmpp_2m", 10), ("euler_a", 4)])
def test_call_vs_oracle(kind, steps):
    """__call__ at 160 x 128 (latents 20 x 16), 10 frames (one window), CFG 3.5, with DPM-Solver++ 2M (10 steps) or
    Euler-ancestral (4 steps, seeded generator: initial latents then one draw per step), against
    oracle/schedulers_oracle.sample_clip in fp32 fed the same draws; PyTorch-fp16 on the same graph sets the bar."""
    from mimo_b200.host import scheduler as S
    from mimo_b200.host.pipeline import pil_to_tensor
    from oracle import schedulers_oracle as SC
    from oracle import torch_oracle as O
    from scripts.oracle_any_size import forwarded_upsample_size
    A = _any_size()
    F_, width, height, seed = 10, 160, 128, 940
    cfg, vcfg = O.UNetConfig(block_out_channels=A.WIDTHS), O.VAEConfig()
    sds = dict(den=O.make_denoising_unet_sd(cfg, seed), ref=O.make_reference_unet_sd(cfg, seed + 1),
               pg=O.make_pose_guider_sd(seed + 2, A.WIDTHS[0]), vae=O.make_vae_sd(vcfg, seed + 3))
    pipe = A._build_pipe(A.WIDTHS, sds, A._small_clip(seed + 4))
    if kind == "dpmpp_2m":
        pipe.scheduler = S.DPMSolverMultistepScheduler(solver_order=2, **SCHED_KW)
        mk = lambda: SC.DPMSolverPP(2)
    else:
        pipe.scheduler = S.EulerAncestralDiscreteScheduler(**SCHED_KW)
        mk = SC.EulerAncestral
    ref_img, poses, bks = A._images(F_, width, height, seed)
    out = pipe(ref_img, poses, bks, width, height, F_, steps, 3.5, generator=torch.manual_seed(42))
    assert out.videos.shape == (1, 3, F_, height, width) and bool(torch.isfinite(out.videos).all())
    dev = torch.device(DEV)
    with torch.no_grad(), forwarded_upsample_size():
        emb = pipe._clip_embeds(ref_img).float()
        gen = torch.manual_seed(42)
        shape = (1, 4, F_, height // 8, width // 8)
        lat0 = torch.randn(shape, generator=gen, dtype=torch.float16)
        noise = ([torch.randn(shape, generator=gen, dtype=torch.float16).to(dev) for _ in range(steps)]
                 if kind == "euler_a" else None)
        args = lambda cast: (cast(pil_to_tensor(ref_img, height, width, True).to(dev)),
                             cast(pil_to_tensor(poses, height, width, False).permute(1, 0, 2, 3).unsqueeze(0).to(dev)),
                             cast(pil_to_tensor(bks[:1], height, width, True).to(dev)).expand(F_, -1, -1, -1))
        r32 = lambda sd: {k: v.half().float().to(dev) for k, v in sd.items()}
        h16 = lambda sd: {k: v.half().to(dev) for k, v in sd.items()}
        W = O.Weights(r32(sds["den"]), r32(sds["ref"]), r32(sds["pg"]), r32(sds["vae"]), cfg, vcfg)
        want = SC.sample_clip(W, *args(lambda t: t), emb.half().float(), lat0.float().to(dev), steps, 3.5, mk(),
                              step_noise=[n.float() for n in noise] if noise else None)
        del W
        W16 = O.Weights(h16(sds["den"]), h16(sds["ref"]), h16(sds["pg"]), h16(sds["vae"]), cfg, vcfg)
        t16 = SC.sample_clip(W16, *args(lambda t: t.half()), emb.half(), lat0.to(dev), steps, 3.5, mk(),
                             step_noise=noise)
    le, ve = A._rel(pipe.last_latents, want["latents"]), A._rel(out.videos, want["videos"])
    le16, ve16 = A._rel(t16["latents"], want["latents"]), A._rel(t16["videos"], want["videos"])
    print(f"clip {width}x{height}x{F_}f {kind} {steps} steps: latents {le:.3e} videos {ve:.3e}   "
          f"torch-fp16: latents {le16:.3e} videos {ve16:.3e}")
    assert le <= max(1e-3, le16) and ve <= max(1e-3, ve16), (le, ve, le16, ve16)


def test_call_at_784x784_with_dpm_solver_is_finite_and_deterministic():
    """The reference's default size, 24 frames, DPM-Solver++ 2M at 3 steps (first, second and final first-order
    step): finite frames, and two calls with the same seed give the same bytes."""
    from mimo_b200.host import scheduler as S
    A = _any_size()
    F_, size, steps = 24, 784, 3
    torch.manual_seed(42)
    pipe = A._build_pipe(A.WIDTHS, None, A._small_clip(5))
    pipe.scheduler = S.DPMSolverMultistepScheduler(solver_order=2, **SCHED_KW)
    ref_img, poses, bks = A._images(F_, size, size, 11)
    vids = []
    for _ in range(2):
        out = pipe(ref_img, poses, bks, size, size, F_, steps, 3.5, generator=torch.manual_seed(7))
        assert out.videos.shape == (1, 3, F_, size, size)
        assert bool(torch.isfinite(out.videos).all())
        vids.append(out.videos.clone())
    assert pipe.last_latents.shape == (1, 4, F_, 98, 98)
    assert torch.equal(vids[0], vids[1])
