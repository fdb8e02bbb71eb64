"""Image sizes whose latents are not multiples of 8 (the reference's script default 784 x 784 -> 98 x 98 latents), on the
CPU: the per-level sizes, the up step each level takes, the frame-shard token count, the oracle against the fixture the
reference's own UNets wrote at such a size, and the argument checks of mimo_upsample_nearest."""
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from mimo_b200 import engine as E
from mimo_b200 import lib as L
from mimo_b200 import ops
from mimo_b200.host import pipeline as P
from mimo_b200.host.shard import ShardPlan
from oracle import torch_oracle as O
from scripts import oracle_any_size as OA


def test_levels_match_the_stride2_conv_shapes():
    w = torch.zeros(1, 1, 3, 3)
    for s in range(1, 131):
        t = 131 - s  # every side 1..130 on both axes, each paired with a different other side
        x = torch.zeros(1, 1, s, t)
        want = [(s, t)]
        for _ in range(3):
            x = F.conv2d(x, w, stride=2, padding=1)
            want.append(tuple(x.shape[-2:]))
        assert E.latent_levels(s, t, 4) == want, (s, t)
    assert E.latent_levels(98, 98, 4) == [(98, 98), (49, 49), (25, 25), (13, 13)]
    assert E.latent_levels(5, 7, 1) == [(5, 7)]
    for bad in ((0, 8), (8, 0), (-1, 4)):
        with pytest.raises(L.MimoError, match="empty"):
            E.latent_levels(*bad, 4)


class _Rec:
    """Stand-in activation: remembers the (h, w) it was produced at."""

    def __init__(self, h, w):
        self.h, self.w = h, w


def _fake_engine(spec):
    eng = E.UNetEngine.__new__(E.UNetEngine)
    eng.spec, eng.taps, eng.xchg = spec, None, None
    calls = {"resnet": [], "up": []}

    def resnet(p, x0, x1, tembs, n, h, w, rpb):
        assert (x0.h, x0.w) == (h, w) and (x1 is None or (x1.h, x1.w) == (h, w)), (p, h, w)
        calls["resnet"].append((p, h, w))
        return _Rec(h, w)

    def up(p, x, n, h, w, th, tw):
        assert (x.h, x.w) == (h, w)
        calls["up"].append((h, w, th, tw))
        return _Rec(th, tw)

    eng._resnet = resnet
    eng._motion = lambda p, x, b, f, hw: x
    eng._down = lambda p, x, n, h, w: _Rec((h + 1) // 2, (w + 1) // 2)
    eng._up = up
    return eng, calls


@pytest.mark.parametrize("hw", [(98, 98), (14, 10), (64, 64), (25, 17), (1, 1)])
def test_body_carries_the_level_sizes(hw):
    """Every resnet sees its input and its skip at one size, and every upsampler targets the skip on top of the stack."""
    h, w = hw
    spec = E.UNetSpec()
    eng, calls = _fake_engine(spec)
    xf = lambda p, x, n, hw_, rpb: x
    x, oh, ow = eng._body(_Rec(h, w), None, 2, 3, h, w, xf)
    lv = E.latent_levels(h, w, 4)
    assert (oh, ow) == (h, w) and (x.h, x.w) == (h, w)
    assert calls["up"] == [lv[3] + lv[2], lv[2] + lv[1], lv[1] + lv[0]]
    # the reference UNet's bank pass (write_banks) stops at the last up-block attention, after all three upsamplers
    eng2, calls2 = _fake_engine(E.UNetSpec(motion=False))
    eng2._body(_Rec(h, w), None, 2, 1, h, w, xf, stop_at="up_blocks.3.attentions.2")
    assert calls2["up"] == calls["up"]


def test_up_step_takes_the_fused_kernel_only_for_exact_doubling(monkeypatch):
    seen = []
    monkeypatch.setattr(ops, "conv_up2x", lambda x, wp, n, h, w, bias=None: seen.append(("fused", h, w)) or "y")
    monkeypatch.setattr(ops, "upsample_nearest", lambda x, n, h, w, th, tw: seen.append(("resize", h, w, th, tw)) or "r")
    monkeypatch.setattr(ops, "conv3x3", lambda x, wp, n, h, w, bias=None: seen.append(("conv", x, h, w)) or "y")
    eng = SimpleNamespace(w={"u": ("w4", "b"), "u_conv": ("w9", "b")})
    for h, w, th, tw in ((13, 13, 25, 25), (25, 25, 49, 49), (49, 49, 98, 98), (2, 2, 4, 3), (4, 3, 7, 5), (7, 5, 14, 10)):
        E.UNetEngine._up(eng, "u", None, 2, h, w, th, tw)
    assert seen == [("resize", 13, 13, 25, 25), ("conv", "r", 25, 25), ("resize", 25, 25, 49, 49), ("conv", "r", 49, 49),
                    ("fused", 49, 49),
                    ("resize", 2, 2, 4, 3), ("conv", "r", 4, 3), ("resize", 4, 3, 7, 5), ("conv", "r", 7, 5),
                    ("fused", 7, 5)]


def test_size_checks_keep_their_meaning_and_call_accepts_any_size():
    """check_latent_size / check_size still answer "does the fused x2 upsampler serve every level"; __call__'s own check
    (latent_levels) only refuses images smaller than one latent pixel."""
    pipe = P.Pose2VideoPipeline.__new__(P.Pose2VideoPipeline)
    pipe.vae_scale_factor = 8
    pipe.denoising_unet = SimpleNamespace(config=SimpleNamespace(block_out_channels=(320, 640, 1280, 1280)))
    with pytest.raises(NotImplementedError, match="multiples of 64"):
        pipe.check_size(784, 784)
    assert pipe.latent_levels(784, 784) == [(98, 98), (49, 49), (25, 25), (13, 13)]
    assert pipe.latent_levels(200, 136) == [(17, 25), (9, 13), (5, 7), (3, 4)]
    assert pipe.latent_levels(15, 8) == [(1, 1)] * 4  # floored to 8 x 8 pixels, like the images (pipeline :73-80)
    with pytest.raises(L.MimoError, match="empty"):
        pipe.latent_levels(784, 7)


def test_shard_tokens_and_plans():
    for size in (512, 768):  # multiples of 64: the coarsest level's count, as before
        h = size // 8
        assert P.shard_tokens(h, h, 4) == (h >> 3) ** 2
        for world in range(1, 9):
            for n_win in (1, 3, 4, 8):
                old = new = None
                try:
                    old = ShardPlan.make(world, 0, True, n_win, 24, min_tokens=(h >> 3) ** 2)
                except NotImplementedError:
                    pass
                try:
                    new = ShardPlan.make(world, 0, True, n_win, 24, min_tokens=P.shard_tokens(h, h, 4))
                except NotImplementedError:
                    pass
                assert (old is None) == (new is None)
                if old is not None:
                    assert (old.cfg_ways, old.win_ways, old.frame_ways) == (new.cfg_ways, new.win_ways, new.frame_ways)
    # 784 x 784: 9604, 2401, 625 and 169 tokens share no factor, so clips shard by windows and CFG only
    assert P.shard_tokens(98, 98, 4) == 1
    made = 0
    for world in range(1, 9):
        for n_win in (1, 2, 8):
            try:
                plan = ShardPlan.make(world, 0, True, n_win, 24, min_tokens=P.shard_tokens(98, 98, 4))
            except NotImplementedError:
                continue
            made += 1
            assert plan.frame_ways == 1, (world, n_win)
    assert made >= 6
    assert P.shard_tokens(14, 10, 4) == 1 and P.shard_tokens(96, 64, 4) == 96


def test_oracle_matches_the_reference_at_an_odd_size(golden_dir):
    """tests/golden/unet_odd_read.pt: the reference's own UNet2D (write) -> UNet3D (read) at a 14 x 10 latent (levels
    7 x 5, 4 x 3, 2 x 2), in fp32 (scripts/oracle_any_size.py). The oracle with forwarded upsample sizes matches it; the
    plain oracle (scale_factor=2) cannot even run there."""
    g = torch.load(golden_dir / "unet_odd_read.pt")
    cfg = O.UNetConfig(block_out_channels=tuple(g["cfg"]))
    f, h, w = g["f"], g["h"], g["w"]
    assert (h % 8, w % 8) != (0, 0)
    out = OA.oracle_odd_case(cfg, f, h, w, g["seed"])
    want = g["out"].float()
    assert out.shape == want.shape == (2, 4, f, h, w)
    err = float((out - want).norm() / want.norm())
    assert err < 1e-3, err  # the fixture is stored in fp16
    with pytest.raises(RuntimeError):
        (sd_den, sd_ref, _), ref_lat, ehs, _, _ = OA.odd_case_inputs(cfg, f, h, w, g["seed"])
        with torch.no_grad():
            O.reference_unet_banks(sd_ref, ref_lat.repeat(2, 1, 1, 1), ehs, cfg)


def test_oracle_with_forwarded_sizes_still_matches_the_even_fixture(golden_dir):
    """At sizes that halve exactly, following the skip sizes is scale_factor=2: tests/golden/unet_small_read.pt still
    holds, and the two oracle bodies agree bit for bit."""
    g = torch.load(golden_dir / "unet_small_read.pt")
    cfg = O.UNetConfig(block_out_channels=tuple(g["cfg"]))
    out = OA.oracle_odd_case(cfg, g["f"], g["hw"], g["hw"], g["seed"])
    want = g["out"].float()
    assert float((out - want).norm() / want.norm()) < 1e-3
    (sd_den, sd_ref, sd_pg), ref_lat, ehs, x, pose_img = OA.odd_case_inputs(cfg, g["f"], g["hw"], g["hw"], g["seed"])
    with torch.no_grad():
        banks = O.reference_unet_banks(sd_ref, ref_lat.repeat(2, 1, 1, 1), ehs, cfg)
        plain = O.denoising_unet(sd_den, x, 499, ehs, O.pose_guider(sd_pg, pose_img).repeat(2, 1, 1, 1, 1), banks, cfg)
    assert torch.equal(out, plain)
    assert O._unet_body is not OA.unet_body  # the context manager restored the oracle


def test_upsample_nearest_refuses_bad_arguments_before_the_device_probe():
    lib = L.load()
    PTR = 1 << 20
    call = lambda x=PTR, out=PTR, n=2, h=13, w=13, oh=25, ow=25, c=64, dt=L.F16: lib.mimo_upsample_nearest(
        x, out, n, h, w, oh, ow, c, dt, None)
    for kw, needle in (({"x": None}, "null pointer"), ({"out": None}, "null pointer"), ({"n": 0}, "positive"),
                       ({"h": 0}, "positive"), ({"ow": -1}, "positive"), ({"oh": 0}, "positive"),
                       ({"c": 12}, "multiple of 8"), ({"c": 0}, "positive"), ({"x": PTR + 8}, "aligned"),
                       ({"out": PTR + 2}, "aligned"), ({"dt": 2}, "dtype")):
        assert call(**kw) == -1, kw
        assert needle in lib.mimo_last_error().decode(), (kw, lib.mimo_last_error())
    if not torch.cuda.is_available():
        assert call() == -3  # valid arguments reach the device probe


def test_upsample_nearest_is_bound_and_declared():
    assert "mimo_upsample_nearest" in L.SYMBOLS
    assert b"0.2.0" in L.load().mimo_version()  # weight caches of the previous packing (no up_conv entries) are not reused
