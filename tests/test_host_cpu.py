"""Host-side logic of the drop-in surface (no GPU): state-dict schema, context windows, scheduler tables,
constructor validation — each against the oracle / the reference-generated golden tables."""
import json

import pytest
import torch

from mimo_b200.host import context, schema
from mimo_b200.host.scheduler import DDIMScheduler
from oracle import torch_oracle as O

SCHED_KW = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False, steps_offset=1,
                prediction_type="v_prediction", rescale_betas_zero_snr=True, timestep_spacing="trailing")


def _same(sch, sd, name):
    assert set(sch) == set(sd), (name, sorted(set(sch) ^ set(sd))[:8])
    for k, shp in sch.items():
        assert tuple(shp) == tuple(sd[k].shape), (name, k)


def test_state_dict_schema_matches_reference_layout():
    cfg = O.UNetConfig(block_out_channels=(64, 128, 256, 256))
    w = cfg.block_out_channels
    _same(schema.unet_schema(w), O.make_denoising_unet_sd(cfg), "denoising unet")
    _same(schema.unet_schema(w, in_channels=4, motion=False, out_head=False), O.make_reference_unet_sd(cfg), "reference unet")
    _same(schema.pose_guider_schema(320), O.make_pose_guider_sd(), "pose guider")
    vcfg = O.VAEConfig(block_out_channels=(32, 64, 128, 128))
    _same(schema.vae_schema(vcfg.block_out_channels), O.make_vae_sd(vcfg), "vae")
    # full-size parameter counts quoted by SURVEY.md (1 312.7 M / 859.5 M / 1.09 M)
    n = lambda s: sum(int(torch.tensor(v).prod()) for k, v in s.items() if not k.endswith(".pe"))
    assert abs(n(schema.unet_schema()) / 1e6 - 1312.7) < 0.5
    assert abs(n(schema.unet_schema(in_channels=4, motion=False, out_head=False)) / 1e6 - 859.5) < 0.5
    assert abs(n(schema.pose_guider_schema(320)) / 1e6 - 1.09) < 0.02


def test_facade_modules_round_trip_state_dict():
    from mimo_b200.host.modules import PoseGuider, UNet2DConditionModel
    cfg = O.UNetConfig(block_out_channels=(32, 64, 64, 64))
    sd = O.make_reference_unet_sd(cfg)
    m = UNet2DConditionModel(block_out_channels=cfg.block_out_channels, cross_attention_dim=768, attention_head_dim=8)
    m.load_state_dict(sd, strict=True)
    back = m.state_dict()
    assert list(back) != [] and all(torch.equal(back[k], sd[k]) for k in sd)
    assert m.half().dtype == torch.float16
    pg = PoseGuider(320, 3, (16, 32, 96, 256))
    pg.load_state_dict(O.make_pose_guider_sd(), strict=True)
    with pytest.raises(RuntimeError):
        pg.load_state_dict({"conv_in.weight": torch.zeros(1)}, strict=True)


def test_context_windows_match_reference(golden_dir):
    tables = json.loads((golden_dir / "integer_tables.json").read_text())
    for F, want in tables["windows"].items():
        assert list(context.uniform(0, 20, int(F), 24, 1, 4)) == want
    with pytest.raises(ValueError):
        context.get_context_scheduler("nope")
    for v in (0, 1, 2, 3, 12345, 2 ** 63):
        assert context.ordered_halving(v) == O.ordered_halving(v)


def test_scheduler_tables_match_reference(golden_dir):
    tables = json.loads((golden_dir / "integer_tables.json").read_text())
    for N, want in tables["timesteps"].items():
        s = DDIMScheduler(**SCHED_KW)
        s.set_timesteps(int(N))
        assert [int(t) for t in s.timesteps] == want
        d = O.DDIM()
        d.set_timesteps(int(N))
        for t in want:
            assert s.step_coefficients(t) == d.coefficients(t)
    with pytest.raises(NotImplementedError):
        DDIMScheduler(clip_sample=True)


def test_unsupported_configurations_fail_loudly():
    from mimo_b200.host.modules import ReferenceAttentionControl, UNet3DConditionModel
    with pytest.raises(NotImplementedError):
        UNet3DConditionModel(block_out_channels=(32, 64, 64, 64), use_motion_module=False)
    kw = dict(use_motion_module=True, motion_module_mid_block=True, motion_module_type="Vanilla",
              motion_module_kwargs=dict(num_attention_heads=8, num_transformer_block=1,
                                        attention_block_types=["Temporal_Self", "Temporal_Self"],
                                        temporal_position_encoding=True, temporal_position_encoding_max_len=32))
    m = UNet3DConditionModel(block_out_channels=(32, 64, 64, 64), cross_attention_dim=768, **kw)
    assert m.state_dict()["conv_in.weight"].shape[1] == 8  # forced 8 input channels
    with pytest.raises(NotImplementedError):
        ReferenceAttentionControl(m, mode="read", fusion_blocks="midup")


def test_sizes_the_fused_upsampler_cannot_serve_are_refused():
    """The reference runs any size through `forward_upsample_size` (unet_3d_edit_bkfill.py:430-435; run_animate.py's
    default is 784 x 784 -> 98 x 98 latents); this engine's nearest-x2 + 3x3 kernel doubles exactly, so sizes that are
    not multiples of 64 pixels (8 latent pixels) must fail before any work is done, not read past a skip tensor."""
    from types import SimpleNamespace

    from mimo_b200 import engine as E
    from mimo_b200.host import pipeline as P
    from mimo_b200.lib import MimoError
    eng = SimpleNamespace(spec=E.UNetSpec())
    for ok in ((64, 64), (96, 64), (8, 16)):
        E.UNetEngine.check_latent_size(eng, *ok)
    for bad in ((98, 98), (64, 100), (0, 64), (4, 8)):
        with pytest.raises(MimoError, match="forward_upsample_size"):
            E.UNetEngine.check_latent_size(eng, *bad)
    E.UNetEngine.check_latent_size(SimpleNamespace(spec=E.UNetSpec(block_out_channels=(32, 64))), 6, 10)  # 2 levels: x2
    pipe = P.Pose2VideoPipeline.__new__(P.Pose2VideoPipeline)
    pipe.vae_scale_factor = 8
    pipe.denoising_unet = SimpleNamespace(config=SimpleNamespace(block_out_channels=(320, 640, 1280, 1280)))
    pipe.check_size(512, 512)
    pipe.check_size(768, 512)
    for bad in ((784, 784), (512, 520)):
        with pytest.raises(NotImplementedError, match="multiples of 64"):
            pipe.check_size(*bad)


def test_image_preprocessing_is_the_vae_image_processor_bit_for_bit():
    """pipeline :73-80 / :424-453: the byte-level host path + device-side normalisation must reproduce
    VaeImageProcessor.preprocess (RGB, LANCZOS to multiples of 8, /255, NCHW, optional 2x-1) exactly."""
    import numpy as np
    import PIL.Image

    from mimo_b200.host import pipeline as P
    rng = np.random.RandomState(3)
    imgs = [PIL.Image.fromarray(rng.randint(0, 256, (70, 90, 3), dtype=np.uint8)) for _ in range(3)]
    imgs.append(PIL.Image.fromarray(rng.randint(0, 256, (64, 64), dtype=np.uint8)))  # grayscale -> RGB
    for size in (64, 61):  # 61 -> floored to 56
        w = h = size - size % 8
        arr = np.stack([np.asarray(i.convert("RGB").resize((w, h), resample=PIL.Image.LANCZOS), dtype=np.float32) / 255.0
                        for i in imgs])
        want = torch.from_numpy(arr).permute(0, 3, 1, 2).contiguous()
        assert torch.equal(P.pil_to_tensor(imgs, size, size, False), want)
        assert torch.equal(P.pil_to_tensor(imgs, size, size, True), 2.0 * want - 1.0)
        u8 = P.pil_to_uint8(imgs, size, size)
        assert u8.dtype == torch.uint8 and tuple(u8.shape) == (len(imgs), h, w, 3)


def test_identical_background_frames_are_deduplicated():
    import numpy as np
    import PIL.Image

    from mimo_b200.host import pipeline as P
    white = lambda: PIL.Image.fromarray(np.full((32, 32, 3), 255, np.uint8))
    other = PIL.Image.fromarray(np.zeros((32, 32, 3), np.uint8))
    first, inverse = P._dedupe_images([white(), white(), other, white(), other])
    assert first == [0, 2] and inverse.tolist() == [0, 0, 1, 0, 1]
    first, inverse = P._dedupe_images([other])
    assert first == [0] and inverse.tolist() == [0]


def test_staged_preprocess_equals_the_simple_functions():
    """Pose2VideoPipeline.preprocess() writes frames straight into staging tensors, resizes on host threads, buckets the
    dedupe by a sampled CRC and draws the noise on a worker thread: every output must equal what the plain functions
    (pil_to_uint8, _dedupe_images, prepare_latents on the calling thread) give, for frames that need nothing, a mode
    conversion, a LANCZOS resize, or both."""
    import numpy as np
    import PIL.Image

    from mimo_b200.host import pipeline as P
    from mimo_b200.host.scheduler import DDIMScheduler
    rng = np.random.RandomState(5)
    rgb = lambda hh, ww: PIL.Image.fromarray(rng.randint(0, 256, (hh, ww, 3), dtype=np.uint8))
    F_, size = 6, 64
    white = lambda: PIL.Image.fromarray(np.full((size, size, 3), 255, np.uint8))
    near_white = np.full((size, size, 3), 255, np.uint8)
    near_white[17, 23, 1] = 254  # one byte off, at an offset the 1021-byte sampling stride does not visit
    assert (17 * size * 3 + 23 * 3 + 1) % 1021 != 0
    cases = {
        "as_is": ([rgb(size, size) for _ in range(F_)], [white() for _ in range(F_)]),
        "resize": ([rgb(90, 70) for _ in range(F_)], [rgb(size, size), white(), white(), rgb(size, size), white(),
                                                      PIL.Image.fromarray(near_white)]),
        "modes": ([rgb(size, size).convert("L"), rgb(size, size).convert("RGBA"), rgb(100, 50).convert("L")] +
                  [rgb(size, size) for _ in range(3)], [rgb(80, 80).convert("RGBA") for _ in range(F_)]),
    }
    pipe = P.Pose2VideoPipeline.__new__(P.Pose2VideoPipeline)
    pipe.scheduler, pipe.vae_scale_factor = DDIMScheduler(prediction_type="v_prediction", clip_sample=False), 8
    pipe._clip_pixels = lambda im: torch.zeros(1, 3, 2, 2)  # transformers' processor is not under test here
    for name, (poses, bks) in cases.items():
        for target in (size, 61):  # 61 -> floored to 56: every frame is resized
            ref = rgb(size, size)
            for dtype in (torch.float16, torch.float32):
                got = pipe.preprocess(ref, poses, bks, target, target, F_, torch.Generator().manual_seed(9), dtype)
                first, inverse = P._dedupe_images(bks)
                assert torch.equal(got["bk_inverse"], inverse), name
                assert torch.equal(got["ref_u8"], P.pil_to_uint8(ref, target, target)), name
                assert torch.equal(got["pose_u8"], P.pil_to_uint8(poses, target, target)), name
                assert torch.equal(got["bk_unique_u8"], P.pil_to_uint8([bks[i] for i in first], target, target)), name
                want = pipe.prepare_latents(1, 4, target, target, F_, dtype, "cpu", torch.Generator().manual_seed(9))
                assert got["latents"].dtype == dtype and torch.equal(got["latents"], want), name
    assert P._dedupe_raws(cases["resize"][1])[0] == [0, 1, 3, 5]  # the near-white frame is its own representative
    with pytest.raises(ValueError):
        pipe.preprocess(ref, poses[:-1], bks, size, size, F_, torch.Generator().manual_seed(9), torch.float16)
    # a failing noise draw (generator list of the wrong length) surfaces as the reference's ValueError
    with pytest.raises(ValueError, match="list of generators"):
        pipe.preprocess(ref, poses, bks, size, size, F_, [torch.Generator(), torch.Generator()], torch.float16)


def test_weight_packers_lay_out_what_the_kernels_index():
    """Host-side packing only (no device): conv weights become [cout, 9 * cin] with K = (ky*3+kx) * cin + ch (the order
    the implicit-GEMM producer walks taps and channel blocks in), GEGLU projections interleave value / gate rows per
    output tile so that one accumulator tile holds both halves of the same columns."""
    from mimo_b200 import lib as L
    from mimo_b200 import ops
    w = torch.arange(5 * 3 * 3 * 3, dtype=torch.float32).reshape(5, 3, 3, 3)
    p = ops.pack_conv3x3_weight(w)
    assert tuple(p.shape) == (8, 9 * 8)
    for co, ky, kx, ch in [(0, 0, 0, 0), (4, 2, 1, 2), (3, 1, 2, 1)]:
        assert p[co, (ky * 3 + kx) * 8 + ch] == w[co, ch, ky, kx]
    assert float(p[5:].abs().sum()) == 0.0 and float(p[:, 3:8].abs().sum()) == 0.0  # channel / row padding is zero

    n2, dim = 2560, 16
    g = L.load().mimo_gemm_geglu_granule(n2)
    assert g in (32, 64, 128) and (n2 // 2) % g == 0
    wg = torch.arange(n2 * dim, dtype=torch.float32).reshape(n2, dim)
    b = torch.arange(n2, dtype=torch.float32)
    wp, bp = ops.pack_geglu_weight(wg, b)
    inner = n2 // 2
    for j in (0, g - 1, g, 3 * g + 5, inner - 1):  # value row j and gate row j land in the same 2g-row tile
        tile, off = divmod(j, g)
        assert torch.equal(wp[tile * 2 * g + off], wg[j]) and torch.equal(wp[tile * 2 * g + g + off], wg[inner + j])
        assert bp[tile * 2 * g + off] == b[j] and bp[tile * 2 * g + g + off] == b[inner + j]


def test_conv_up2x_weight_packing_equals_interpolate_plus_conv():
    """The parity-class weights of mimo_conv_up2x (ops.pack_conv_up2x_weight) restate nearest-x2 + 3x3 conv exactly:
    evaluated with torch on the CPU against F.interpolate + conv2d (src/models/resnet.py:70-90)."""
    import torch.nn.functional as F

    from mimo_b200 import ops
    torch.manual_seed(0)
    cin, cout, n, h, w = 8, 16, 2, 5, 7
    W = torch.randn(cout, cin, 3, 3)
    x = torch.randn(n, cin, h, w)
    ref = F.conv2d(F.interpolate(x, scale_factor=2.0, mode="nearest"), W, padding=1)
    w4 = ops.pack_conv_up2x_weight(W).reshape(4, cout, 4, cin)
    out = torch.zeros(n, cout, 2 * h, 2 * w)
    xp = F.pad(x, (1, 1, 1, 1))
    for a in range(2):
        for b in range(2):
            for iy in range(2):
                for ix in range(2):
                    dy, dx = a - 1 + iy, b - 1 + ix  # the offsets csrc/gemm_wgmma.cu: mimo_conv_up2x uses
                    src = xp[:, :, 1 + dy:1 + dy + h, 1 + dx:1 + dx + w]
                    out[:, :, a::2, b::2] += torch.einsum("oc,nchw->nohw", w4[2 * a + b, :, 2 * iy + ix], src)
    assert float((out - ref).abs().max()) < 1e-4


def test_composite_oracle_and_mask_modes():
    """The numpy restatement of run_edit.py:282-300 on a hand-checked pixel, and the 16-way feather-mask selection
    (tools/util.py:393-437) of the host-side compositing helper."""
    import numpy as np

    from mimo_b200.host.composite import MASK_MODES, mask_mode
    from oracle.composite_oracle import composite_frame
    canvas = np.full((1, 1, 3), 200, np.uint8)
    bk = np.full((1, 1, 3), 100, np.uint8)
    m = np.full((1, 1), 0.25, np.float32)
    assert composite_frame(canvas, bk, m)[0, 0, 0] == 125            # 200 * .25 + 100 * .75
    occ = np.full((1, 1), 255, np.uint8)
    vid = np.full((1, 1, 3), 7, np.uint8)
    assert composite_frame(canvas, bk, m, occ, vid)[0, 0, 0] == 7    # fully occluded: the original frame wins
    prev = np.full((1, 1, 3), 25, np.uint8)
    assert composite_frame(canvas, bk, m, None, None, prev, 0.2)[0, 0, 0] == 45  # 25 * .8 + 125 * .2, truncated
    W, H = 100, 50
    assert MASK_MODES[mask_mode((0, 100, 0, 50), W, H)] == "up_down_left_right"
    assert MASK_MODES[mask_mode((0, 100, 0, 40), W, H)] == "left_right_up"
    assert MASK_MODES[mask_mode((10, 100, 0, 50), W, H)] == "up_down_right"
    assert MASK_MODES[mask_mode((0, 60, 5, 50), W, H)] == "left_down"
    assert MASK_MODES[mask_mode((10, 60, 5, 50), W, H)] == "down"
    assert MASK_MODES[mask_mode((10, 60, 5, 45), W, H)] == "inner"


def test_packed_weight_cache_container_round_trip(tmp_path):
    from mimo_b200.host import weight_cache as WC
    obj = {"w": {"a": (torch.randn(3, 4).half(), None), "b": {"C": 320, "l": [torch.ones(2), torch.zeros(1)]}},
           "names": ["x", "y"], "off": {"p": [0, 5]}}
    f = tmp_path / "t.safetensors"
    WC.save(f, obj)
    back = WC.load(f, "cpu")
    assert torch.equal(back["w"]["a"][0], obj["w"]["a"][0]) and back["w"]["a"][1] is None
    assert isinstance(back["w"]["a"], tuple) and back["w"]["b"]["C"] == 320 and back["names"] == ["x", "y"]
    a = {"k": torch.arange(10000.0)}
    b = {"k": torch.arange(10000.0)}
    b["k"][5000] += 1  # one element in the middle of a tensor: the default (full) hash must see it
    assert WC.fingerprint(a) == WC.fingerprint({"k": torch.arange(10000.0)})
    assert WC.fingerprint(a) != WC.fingerprint(b)
    assert WC.fingerprint(a, "x") != WC.fingerprint(a, "y")


def test_bank_routing_rows():
    """Which bank each frame-sample row reads (engine.bank_index_rows): unconditional rows never read the bank, the
    conditional bank is the last map the writer handed over, a CFG-sharded GPU holds one branch only."""
    from mimo_b200.engine import bank_index_rows
    assert bank_index_rows((0, 1), 3, True, 2) == ([-1, -1, -1, 1, 1, 1], 1)      # both halves written (direct engine use)
    assert bank_index_rows((0, 1), 2, True, 1) == ([-1, -1, 0, 0], 0)             # conditional half only (the pipeline)
    assert bank_index_rows((1,), 2, True, 1) == ([0, 0], 0)                       # CFG-sharded, conditional GPU
    assert bank_index_rows((0,), 2, True, 1) == ([-1, -1], 0)                     # CFG-sharded, unconditional GPU
    assert bank_index_rows((0,), 4, False, 1) == ([0, 0, 0, 0], 0)                # guidance <= 1: every row reads bank 0


def test_context_windows_sweep_against_the_reference_generated_fixture(golden_dir):
    """tests/golden/context_sweep.json was written by oracle/gen_context_golden.py from the reference's own
    src/pipelines/context.py: 2 600 (step, frames, size, stride, overlap, closed_loop) cases as window count + CRC-32 of
    the JSON text, 16 full window lists, ordered_halving fractions and get_total_steps - pure integer logic, bit-exact."""
    import zlib
    g = json.loads((golden_dir / "context_sweep.json").read_text())
    assert len(g["cases"]) >= 2000
    for step, frames, size, stride, overlap, closed, n, crc in g["cases"]:
        w = list(context.uniform(step, 20, frames, size, stride, overlap, bool(closed)))
        assert len(w) == n and zlib.crc32(json.dumps(w, separators=(",", ":")).encode()) == crc, \
            (step, frames, size, stride, overlap, closed)
        assert O.uniform_windows(step, frames, size, stride, overlap, bool(closed)) == w  # the oracle's restatement too
    for key, want in g["full"].items():
        step, frames, size, stride, overlap, closed = map(int, key.split(","))
        assert list(context.uniform(step, 20, frames, size, stride, overlap, bool(closed))) == want, key
    for v, want in g["ordered_halving"].items():
        assert context.ordered_halving(int(v)) == want
    sched = context.get_context_scheduler("uniform")
    for n, frames, size, stride, overlap, want in g["total_steps"]:
        assert context.get_total_steps(sched, list(range(n)), 20, frames, size, stride, overlap) == want
    import src.pipelines.context as overlay  # the reference's import path resolves to the same functions
    assert overlay.get_total_steps is context.get_total_steps and overlay.uniform is context.uniform


def test_parameter_counts_equal_the_published_checkpoints():
    """The third-party architectures are restated (diffusers is not installable here), so their LAYER SHAPES are pinned
    against public facts: Stable Diffusion 1.5's UNet2DConditionModel has 859 520 964 parameters and sd-vae-ft-mse's
    AutoencoderKL 83 653 863 (encoder 34 163 592, decoder 49 490 179, quant + post-quant convs 92) - the schema the
    facades materialise and the oracle's generator must give exactly those numbers."""
    import math
    n = lambda s: sum(math.prod(v) for v in s.values())
    assert n(schema.unet_schema(in_channels=4, motion=False, out_head=True)) == 859_520_964
    v = schema.vae_schema()
    assert n(v) == 83_653_863
    assert n({k: s for k, s in v.items() if k.startswith("encoder.")}) == 34_163_592
    assert n({k: s for k, s in v.items() if k.startswith("decoder.")}) == 49_490_179
    assert sum(t.numel() for t in O.make_vae_sd(O.VAEConfig(), 0).values()) == 83_653_863
