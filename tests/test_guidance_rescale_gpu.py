"""Rescaled classifier-free guidance on the H100: mimo_cfg_rescale against an fp64 statement of its rounding sequence and
against PyTorch's own fp16 diffusers expression, determinism (repeats, graph capture and replay, two devices), the
step kernels passing (out, out, 1.0) through, and whole clips through __call__ against the fp32 oracle
(oracle/guidance_rescale_oracle.py)."""
import importlib.util
from fractions import Fraction
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
SCHED_KW = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False, steps_offset=1,
                prediction_type="v_prediction", rescale_betas_zero_snr=True, timestep_spacing="trailing")


def _any_size():
    spec = importlib.util.spec_from_file_location("_any_size_helpers", Path(__file__).with_name("test_any_size_gpu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _inputs(dtype, F_, h, w, seed, counter):
    g = torch.Generator(device=DEV).manual_seed(seed)
    pred = (torch.randn(2, 4, F_, h, w, device=DEV, generator=g) * 0.9 + 0.05).to(dtype)
    cnt = None
    if counter:
        cnt = (torch.arange(F_, device=DEV) % 3 + 1).to(dtype)
        pred = (pred * cnt.view(1, 1, F_, 1, 1)).to(dtype)  # window sums: the kernel divides them back
    return pred[0].contiguous(), pred[1].contiguous(), cnt


def _torch_guided(pu, pc, g, cnt):
    """The reference's guidance line in PyTorch on the storage dtype (what cfg_ddim_step reproduces bit for bit)."""
    if cnt is not None:
        cv = cnt.view(1, -1, 1, 1)
        pu, pc = pu / cv, pc / cv
    return pc, pu + g * (pc - pu)


def _ulp(x, dtype):
    fi = torch.finfo(dtype)
    return fi.eps * x.float().abs().clamp_min(fi.tiny)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("counter", [False, True])
@pytest.mark.parametrize("shape", [(5, 7, 9), (16, 32, 33)])  # counts 1260 and 67584: neither a multiple of 8 x 256
def test_kernel_matches_fp64_statement(dtype, counter, shape):
    from mimo_b200 import ops
    F_, h, w = shape
    pu, pc, cnt = _inputs(dtype, F_, h, w, 11 + F_, counter)
    g = 3.5
    text, cfg = _torch_guided(pu, pc, g, cnt)
    s_t, s_g = text.double().std(), cfg.double().std()
    r64 = s_t.float().to(dtype).double() / s_g.float().to(dtype).double()
    r_near = r64.float().to(dtype)
    # phi = 1 exposes the ratio: out = rnd(cfg * r). The kernel's fp64 sums are added in another order than torch's, so
    # its std may differ in the last fp64 bits; that moves the rounded ratio only when r64 sits at a rounding boundary
    # of the storage type, and then by one ulp.
    out1 = ops.cfg_rescale(pu, pc, g, 1.0, counter=cnt, frame_stride=h * w)
    cands = [r_near]
    step = float(_ulp(r_near, dtype))
    if abs(float(r64) - float(r_near)) > 0.499 * step:
        cands += [(r_near.float() + step).to(dtype), (r_near.float() - step).to(dtype)]
    hit = [r for r in cands if torch.equal((cfg * r).view(torch.int16), out1.view(torch.int16))]
    assert hit, (float(r64), [float(r) for r in cands])
    r = hit[0]
    for phi in (0.0, 0.3, 0.7, 1.0):
        out = ops.cfg_rescale(pu, pc, g, phi, counter=cnt, frame_stride=h * w)
        want_t = phi * (cfg * r) + (1 - phi) * cfg  # PyTorch's roundings on the storage dtype, with the kernel's ratio
        assert torch.equal(out.view(torch.int16), want_t.view(torch.int16)), phi
        # the same rounding points evaluated in fp64 and rounded straight to the storage type, with the fp64 ratio
        w1, w0 = float(torch.tensor(phi, dtype=torch.float32)), float(torch.tensor(1 - phi, dtype=torch.float32))
        x = (cfg.double() * float(r64.float().to(dtype))).to(dtype).double()
        want64 = ((w1 * x).to(dtype).double() + (w0 * cfg.double()).to(dtype).double()).to(dtype)
        assert bool(((out.float() - want64.float()).abs() <= _ulp(want64, dtype)).all()), phi


@pytest.mark.parametrize("counter", [False, True])
def test_kernel_vs_pytorch_fp16_diffusers_expression(counter):
    """oracle rescale_noise_cfg run by PyTorch on the same fp16 device tensors: within one fp16 ulp per element."""
    from mimo_b200 import ops
    from oracle import guidance_rescale_oracle as GR
    F_, h, w = 24, 64, 64
    pu, pc, cnt = _inputs(torch.float16, F_, h, w, 3, counter)
    text, cfg = _torch_guided(pu, pc, 3.5, cnt)
    for phi in (0.3, 0.7):
        want = GR.rescale_noise_cfg(cfg[None], text[None], phi)[0]
        got = ops.cfg_rescale(pu, pc, 3.5, phi, counter=cnt, frame_stride=h * w)
        d = (got.float() - want.float()).abs()
        assert bool((d <= _ulp(want, torch.float16)).all()), float(d.max())


def test_repeats_graph_replay_and_devices_are_bit_identical():
    from mimo_b200 import ops
    F_, h, w = 64, 64, 64
    pu, pc, cnt = _inputs(torch.float16, F_, h, w, 5, True)
    a = ops.cfg_rescale(pu, pc, 3.5, 0.7, counter=cnt, frame_stride=h * w)
    b = ops.cfg_rescale(pu, pc, 3.5, 0.7, counter=cnt, frame_stride=h * w)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    out = torch.empty_like(pu)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.cfg_rescale(pu, pc, 3.5, 0.7, out=out, counter=cnt, frame_stride=h * w)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.cfg_rescale(pu, pc, 3.5, 0.7, out=out, counter=cnt, frame_stride=h * w)
    for _ in range(2):
        out.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int16), a.view(torch.int16))
    if torch.cuda.device_count() >= 2:  # what the ranks of a sharded run rely on: the same bits on another device
        with torch.cuda.device(1):
            o1 = ops.cfg_rescale(pu.to("cuda:1"), pc.to("cuda:1"), 3.5, 0.7, counter=cnt.to("cuda:1"),
                                 frame_stride=h * w)
        assert torch.equal(o1.cpu().view(torch.int16), a.cpu().view(torch.int16))


def _round(fr: Fraction, mant: int, emin: int) -> Fraction:
    """fr rounded to nearest-even in a binary format with `mant` significand bits and minimum exponent emin."""
    if fr == 0:
        return Fraction(0)
    sgn, a = (-1 if fr < 0 else 1), abs(fr)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    e = max(e, emin)
    q = a / Fraction(2) ** (e - mant + 1)
    n = q.numerator // q.denominator
    rem = q - n
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and n % 2):
        n += 1
    return sgn * n * Fraction(2) ** (e - mant + 1)


def test_step_kernels_pass_the_rescaled_prediction_through():
    """mimo_cfg_ddim_step and mimo_cfg_multistep fed (out, out, 1.0) without a counter give exactly the latents of
    their update applied on the host to v = out: DDIM by PyTorch's own fp16 expression, the multistep update by exact
    rational arithmetic with its fp32 fma and rounding points."""
    from mimo_b200 import ops
    from mimo_b200.host import scheduler as S
    F_, h, w = 3, 4, 5
    pu, pc, cnt = _inputs(torch.float16, F_, h, w, 9, True)
    out = ops.cfg_rescale(pu, pc, 3.5, 0.7, counter=cnt, frame_stride=h * w)
    lat = torch.randn(1, 4, F_, h, w, device=DEV).half()
    ddim = S.DDIMScheduler(**SCHED_KW)
    ddim.set_timesteps(20, device="cpu")
    sa_t, s1a_t, sa_p, s1a_p = (float(torch.tensor(c, dtype=torch.float32))
                                for c in ddim.step_coefficients(int(ddim.timesteps[5])))
    got = ops.cfg_ddim_step(out, out, lat.clone(), 1.0, sa_t, s1a_t, sa_p, s1a_p)
    v, x = out.view_as(lat), lat
    want = sa_p * (sa_t * x - s1a_t * v) + s1a_p * (sa_t * v + s1a_t * x)
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))

    dpm = S.DPMSolverMultistepScheduler(solver_order=3, **SCHED_KW)
    dpm.set_timesteps(20)
    a, b, cx, cm, c1, c2, cn = (float(torch.tensor(c, dtype=torch.float32)) for c in dpm.multistep_coefficients(7))
    h1, h2 = torch.randn(2, 1, 4, F_, h, w, device=DEV).half()
    hist = torch.empty_like(lat)
    got = ops.cfg_multistep(out, out, lat.clone(), 1.0, (a, b, cx, cm, c1, c2, 0.0), hist, h1=h1, h2=h2)
    f32 = lambda q: _round(q, 24, -126)
    f16 = lambda q: _round(q, 11, -14)
    F = lambda t: [Fraction(float(e)) for e in t.flatten().tolist()]
    A, B, CX, CM, C1, C2 = map(Fraction, (a, b, cx, cm, c1, c2))
    for vi, xi, h1i, h2i, mi, li in zip(F(out), F(lat), F(h1), F(h2), F(hist), F(got)):
        m = f16(f32(A * xi + f32(B * vi)))
        acc = f32(CX * xi + f32(CM * m))
        acc = f32(C1 * h1i + acc)
        acc = f32(C2 * h2i + acc)
        assert (mi, li) == (m, f16(acc))


def _clip_case(kind, steps, F_, context_frames, phi_list):
    """__call__ at 160 x 128 with CFG 3.5 for each phi; returns (pipe outputs, oracle fp32, PyTorch-fp16) per phi."""
    from mimo_b200.host import scheduler as S
    from mimo_b200.host.pipeline import pil_to_tensor
    from oracle import guidance_rescale_oracle as GR
    from oracle import schedulers_oracle as SC
    from oracle import torch_oracle as O
    from scripts.oracle_any_size import forwarded_upsample_size
    A = _any_size()
    width, height, seed = 160, 128, 950
    cfg, vcfg = O.UNetConfig(block_out_channels=A.WIDTHS), O.VAEConfig()
    sds = dict(den=O.make_denoising_unet_sd(cfg, seed), ref=O.make_reference_unet_sd(cfg, seed + 1),
               pg=O.make_pose_guider_sd(seed + 2, A.WIDTHS[0]), vae=O.make_vae_sd(vcfg, seed + 3))
    pipe = A._build_pipe(A.WIDTHS, sds, A._small_clip(seed + 4))
    mk = lambda: None
    if kind == "dpmpp_2m":
        pipe.scheduler = S.DPMSolverMultistepScheduler(solver_order=2, **SCHED_KW)
        mk = lambda: SC.DPMSolverPP(2)
    ref_img, poses, bks = A._images(F_, width, height, seed)
    win = dict(context_frames=context_frames, context_overlap=4)
    res = {}
    for phi in phi_list:
        out = pipe(ref_img, poses, bks, width, height, F_, steps, 3.5, generator=torch.manual_seed(42),
                   guidance_rescale=phi, **win)
        res[phi] = (pipe.last_latents.clone(), out.videos)
    dev = torch.device(DEV)
    with torch.no_grad(), forwarded_upsample_size():
        emb = pipe._clip_embeds(ref_img).float()
        lat0 = torch.randn((1, 4, F_, height // 8, width // 8), generator=torch.manual_seed(42), dtype=torch.float16)
        args = lambda cast: (cast(pil_to_tensor(ref_img, height, width, True).to(dev)),
                             cast(pil_to_tensor(poses, height, width, False).permute(1, 0, 2, 3).unsqueeze(0).to(dev)),
                             cast(pil_to_tensor(bks[:1], height, width, True).to(dev)).expand(F_, -1, -1, -1))
        r32 = lambda sd: {k: v.half().float().to(dev) for k, v in sd.items()}
        h16 = lambda sd: {k: v.half().to(dev) for k, v in sd.items()}
        phi = max(phi_list)
        W = O.Weights(r32(sds["den"]), r32(sds["ref"]), r32(sds["pg"]), r32(sds["vae"]), cfg, vcfg)
        want = GR.sample_clip(W, *args(lambda t: t), emb.half().float(), lat0.float().to(dev), steps, 3.5, mk(),
                              guidance_rescale=phi, **win)
        del W
        W16 = O.Weights(h16(sds["den"]), h16(sds["ref"]), h16(sds["pg"]), h16(sds["vae"]), cfg, vcfg)
        t16 = GR.sample_clip(W16, *args(lambda t: t.half()), emb.half(), lat0.to(dev), steps, 3.5, mk(),
                             guidance_rescale=phi, **win)
    return A, res, want, t16


@pytest.mark.parametrize("kind,steps,F_,context_frames", [("ddim", 20, 10, 24), ("dpmpp_2m", 10, 10, 24),
                                                          ("ddim", 4, 14, 8)])
def test_call_vs_oracle(kind, steps, F_, context_frames):
    """phi = 0.7, CFG 3.5: DDIM at 20 steps and DPM-Solver++ 2M at 10 on one window, and DDIM over two overlapping
    windows (14 frames, windows of 8, overlap 4: the counter path), against the fp32 oracle; PyTorch-fp16 on the same
    graph sets the bar. The phi = 0.7 clip must differ from the phi = 0 clip."""
    A, res, want, t16 = _clip_case(kind, steps, F_, context_frames, (0.0, 0.7))
    lat, vid = res[0.7]
    le, ve = A._rel(lat, want["latents"]), A._rel(vid, want["videos"])
    le16, ve16 = A._rel(t16["latents"], want["latents"]), A._rel(t16["videos"], want["videos"])
    moved = A._rel(res[0.0][0], lat)
    print(f"{kind} {steps} steps {F_}f windows of {context_frames}, phi 0.7: latents {le:.3e} videos {ve:.3e}   "
          f"torch-fp16: latents {le16:.3e} videos {ve16:.3e}   phi 0 vs 0.7 latents {moved:.3e}")
    assert bool(torch.isfinite(vid).all())
    assert le <= max(1e-3, le16) and ve <= max(1e-3, ve16), (le, ve, le16, ve16)
    assert moved > 10 * max(le, 1e-3), moved


def test_zero_and_omitted_give_byte_identical_clips():
    """guidance_rescale = 0.0 takes the default path: the same bytes as a call without the keyword (which is the parent
    commit's path, pinned by test_parity_gpu)."""
    A = _any_size()
    F_, size, steps = 8, 128, 3
    torch.manual_seed(42)
    pipe = A._build_pipe(A.WIDTHS, None, A._small_clip(5))
    ref_img, poses, bks = A._images(F_, size, size, 11)
    base = pipe(ref_img, poses, bks, size, size, F_, steps, 3.5, generator=torch.manual_seed(3)).videos
    base_lat = pipe.last_latents.clone()
    zero = pipe(ref_img, poses, bks, size, size, F_, steps, 3.5, generator=torch.manual_seed(3),
                guidance_rescale=0.0).videos
    assert torch.equal(pipe.last_latents.view(torch.int16), base_lat.view(torch.int16)) and torch.equal(zero, base)
    nocfg = pipe(ref_img, poses, bks, size, size, F_, steps, 1.0, generator=torch.manual_seed(3)).videos
    nocfg_r = pipe(ref_img, poses, bks, size, size, F_, steps, 1.0, generator=torch.manual_seed(3),
                   guidance_rescale=0.7).videos
    assert torch.equal(nocfg, nocfg_r)  # no CFG: the rescale does not run
