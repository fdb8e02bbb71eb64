"""Engine parity on an H100: whole networks through the C ABI against the oracle (fp32 torch, same fp16-rounded
weights) and against the golden vectors the reference produced (tests/golden, oracle/pin_against_reference.py).

Stated tolerance (fp16 storage, fp32 accumulate): rel-L2 of a whole UNet forward <= 3e-3 against the fp32 oracle,
and no worse than 1.5x the error of the same graph run by PyTorch itself in fp16 on this GPU (the reference's own
execution mode), whichever is larger."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def probe():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device: the product path has no CPU fallback")
    from scripts import gpu_probe
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return gpu_probe


def test_unet_small_blockwise(probe):
    assert probe._unet_parity((128, 256, 512, 512), f=4, hw=16, seed=100, tol=3e-3)


def test_unet_full_width(probe):
    assert probe._unet_parity((320, 640, 1280, 1280), f=3, hw=32, seed=400, tol=3e-3)


def test_vae_decode(probe):
    assert probe.vae_parity()


def _golden_case(golden_dir, name, widths):
    from mimo_b200 import engine as E
    from oracle import torch_oracle as O
    g = torch.load(golden_dir / name)
    cfg = O.UNetConfig(block_out_channels=widths)
    seed, f, hw = g["seed"], g["f"], g["hw"]
    sd_den = O.make_denoising_unet_sd(cfg, seed=seed)
    sd_ref = O.make_reference_unet_sd(cfg, seed=seed + 1)
    sd_pg = O.make_pose_guider_sd(seed=seed + 2, out_channels=widths[0])
    gen = torch.Generator().manual_seed(seed + 10)
    ref_lat = torch.randn(1, 4, hw, hw, generator=gen)
    emb = torch.randn(1, 1, cfg.cross_attention_dim, generator=gen)
    ehs = torch.cat([torch.zeros_like(emb), emb])
    x = torch.randn(1, 8, f, hw, hw, generator=gen).repeat(2, 1, 1, 1, 1)
    pose_img = torch.rand(1, 3, f, hw * 8, hw * 8, generator=gen)
    dev = torch.device("cuda")
    den = E.UNetEngine(sd_den, E.UNetSpec(block_out_channels=widths), dev)
    ref = E.UNetEngine(sd_ref, E.UNetSpec(block_out_channels=widths, in_channels=4, motion=False, out_head=False), dev)
    pg = E.PoseGuiderEngine(sd_pg, dev)
    banks = ref.write_banks(ref_lat.repeat(2, 1, 1, 1).half().to(dev), ehs.half().to(dev), den)
    den.begin_clip(ehs.half().to(dev), banks, cfg=True, frames=f)
    pose = pg.forward(pose_img.half().to(dev))
    pose2 = pose.reshape(1, f * hw * hw, -1).repeat(2, 1, 1).reshape(2 * f * hw * hw, -1).contiguous()
    got = den.forward(x.half().to(dev), 499, pose2).float().cpu()
    want = g["out"].float()
    return float((got - want).norm() / want.norm())


def test_reference_golden_small(golden_dir):
    # fixture written by the reference's own UNet3DConditionModel / UNet2DConditionModel / PoseGuider (fp32, CPU)
    assert _golden_case(golden_dir, "unet_small_read.pt", (128, 256, 512, 512)) < 4e-3


def test_reference_golden_full_width(golden_dir):
    assert _golden_case(golden_dir, "unet_full_read.pt", (320, 640, 1280, 1280)) < 4e-3


def _pil_inputs(F_, size, seed):
    import PIL.Image
    rng = np.random.RandomState(seed)
    ref_img = PIL.Image.fromarray(rng.randint(0, 256, (size, size, 3), dtype=np.uint8))
    poses, bks = [], []
    for i in range(F_):
        a = np.zeros((size, size, 3), np.uint8)
        a[size // 4: size // 2 + i % 8, size // 3: size // 3 + 20] = rng.randint(11, 256, 3)
        poses.append(PIL.Image.fromarray(a))
        bks.append(PIL.Image.fromarray(rng.randint(0, 256, (size, size, 3), dtype=np.uint8)))
    return ref_img, poses, bks


@pytest.mark.parametrize("F_,size,steps", [(1, 128, 2), (26, 128, 2)])
def test_pipeline_end_to_end_vs_oracle(F_, size, steps):
    """Pose2VideoPipeline.__call__ (public API, PIL in, video tensor out) against oracle.sample_clip on the same
    inputs and seed; F = 26 exercises two overlapping context windows + the counter average."""
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection

    from mimo_b200.host import modules as M
    from mimo_b200.host.pipeline import Pose2VideoPipeline, pil_to_tensor
    from mimo_b200.host.scheduler import DDIMScheduler
    from oracle import torch_oracle as O
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    widths = (128, 256, 512, 512)
    cfg, vcfg = O.UNetConfig(block_out_channels=widths), O.VAEConfig()
    seed = 500 + F_
    sds = dict(den=O.make_denoising_unet_sd(cfg, seed), ref=O.make_reference_unet_sd(cfg, seed + 1),
               pg=O.make_pose_guider_sd(seed + 2, widths[0]), vae=O.make_vae_sd(vcfg, seed + 3))
    mk = dict(num_attention_heads=8, num_transformer_block=1, attention_block_types=["Temporal_Self", "Temporal_Self"],
              temporal_position_encoding=True, temporal_position_encoding_max_len=32, temporal_attention_dim_div=1)
    den = M.UNet3DConditionModel(block_out_channels=widths, cross_attention_dim=768, use_inflated_groupnorm=True,
                                 use_motion_module=True, motion_module_mid_block=True, motion_module_type="Vanilla",
                                 motion_module_kwargs=mk, unet_use_cross_frame_attention=False,
                                 unet_use_temporal_attention=False)
    ref = M.UNet2DConditionModel(block_out_channels=widths, cross_attention_dim=768)
    pg = M.PoseGuider(widths[0], 3, (16, 32, 96, 256))
    vae = M.AutoencoderKL()
    den.load_state_dict(sds["den"], strict=True)
    ref.load_state_dict(sds["ref"], strict=True)
    pg.load_state_dict(sds["pg"], strict=True)
    vae.load_state_dict(sds["vae"], strict=True)
    torch.manual_seed(seed + 4)
    clip = CLIPVisionModelWithProjection(CLIPVisionConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=2,
                                                          num_attention_heads=4, image_size=224, patch_size=32,
                                                          projection_dim=768)).eval()
    sched = DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
                          steps_offset=1, prediction_type="v_prediction", rescale_betas_zero_snr=True,
                          timestep_spacing="trailing")
    pipe = Pose2VideoPipeline(vae=vae, image_encoder=clip, reference_unet=ref, denoising_unet=den, pose_guider=pg,
                              scheduler=sched).to("cuda", dtype=torch.float16)
    ref_img, poses, bks = _pil_inputs(F_, size, seed)
    out = pipe(ref_img, poses, bks, size, size, F_, steps, 3.5, generator=torch.manual_seed(42))
    assert out.videos.shape == (1, 3, F_, size, size) and out.videos.dtype == torch.float32
    assert float(out.videos.min()) >= 0.0 and float(out.videos.max()) <= 1.0

    # oracle: fp32 on the GPU, weights rounded to fp16 like the engine's, same CLIP embedding and the same noise
    dev = torch.device("cuda")
    r16 = lambda sd: {k: v.half().float().to(dev) for k, v in sd.items()}
    W = O.Weights(r16(sds["den"]), r16(sds["ref"]), r16(sds["pg"]), r16(sds["vae"]), cfg, vcfg)
    with torch.no_grad():
        emb = pipe._clip_embeds(ref_img).float()
        lat0 = torch.randn((1, 4, F_, size // 8, size // 8), generator=torch.manual_seed(42), dtype=torch.float16)
        got = O.sample_clip(W, pil_to_tensor(ref_img, size, size, True).to(dev),
                            pil_to_tensor(poses, size, size, False).permute(1, 0, 2, 3).unsqueeze(0).to(dev),
                            pil_to_tensor(bks, size, size, True).to(dev), emb.half().float(), lat0.float().to(dev), steps,
                            3.5)
    lat_err = float((pipe.last_latents.float() - got["latents"]).norm() / got["latents"].norm())
    vid_err = float((out.videos - got["videos"]).norm() / got["videos"].norm())
    print(f"pipeline F={F_}: latents rel_l2={lat_err:.3e} videos rel_l2={vid_err:.3e}")
    assert lat_err < 6e-3 and vid_err < 6e-3
