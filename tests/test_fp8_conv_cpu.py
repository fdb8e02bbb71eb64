"""FP8 ResBlock convolutions without a GPU: the C-ABI structs and argument checks of mimo_groupnorm_e4m3 /
mimo_conv3x3_e4m3, the per-image scale rule on hand-computed cases and as an upper bound on random data, the e4m3 conv
weight packing, and the oracle's emulation (alone and composed with the other oracle contexts)."""
import ctypes
import math

import pytest
import torch

from mimo_b200 import lib as L
from mimo_b200 import ops

PTR = 1 << 20


def test_abi_sizeof_groupnorm_and_conv_e4m3():
    lib = L.load()
    assert lib.mimo_abi_sizeof(10) == ctypes.sizeof(L.GroupNormE4m3Params) == 128
    assert lib.mimo_abi_sizeof(11) == ctypes.sizeof(L.Conv3x3E4m3Params) == 152
    assert lib.mimo_abi_sizeof(2) == ctypes.sizeof(L.Conv3x3Params)  # mimo_conv3x3_params is unchanged


def test_entry_points_refuse_bad_arguments_before_the_device_probe():
    lib = L.load()
    err = lambda: lib.mimo_last_error().decode()

    def conv(**kw):
        p = L.Conv3x3E4m3Params()
        p.x = p.w = p.out = p.x_scale = p.w_scale = PTR
        p.c_in, p.cout, p.ldo, p.n, p.h, p.w_ = 320, 320, 320, 2, 8, 8
        for k, v in kw.items():
            setattr(p.ep if k in ("residual", "ld_res", "act") else p, k, v)
        return lib.mimo_conv3x3_e4m3(ctypes.byref(p), None)

    for kw, needle in [({"x": None}, "null pointer"), ({"x_scale": None}, "null pointer"),
                       ({"w_scale": None}, "null pointer"), ({"n": 0}, "empty problem"), ({"c_in": 0}, "empty problem"),
                       ({"c_in": 328}, "multiple of 16"), ({"cout": 324}, "multiples of 8"),
                       ({"ldo": 321}, "multiples of 8"), ({"out": PTR + 8}, "16-byte aligned"),
                       ({"residual": PTR, "ld_res": 4}, "ld_res"), ({"act": L.ACT_GEGLU}, "GEGLU"),
                       ({"workspace": PTR, "workspace_bytes": 1 << 20}, "split-K")]:
        assert conv(**kw) == -1 and needle in err(), (kw, err())

    def gn(**kw):
        p = L.GroupNormE4m3Params(c0=320, samples=2, frames=4, table_frames=4, hw=64, groups=32, eps=1e-5, dtype=L.F16)
        p.x0 = p.gamma = p.beta = p.out = p.scale = p.work = p.table = PTR
        p.work_bytes = p.table_bytes = 1 << 30
        for k, v in kw.items():
            setattr(p, k, v)
        return lib.mimo_groupnorm_e4m3(ctypes.byref(p), None)

    for kw, needle in [({"mode": 7}, "unknown mode"), ({"x0": None}, "null pointer"), ({"scale": None}, "null pointer"),
                       ({"work": None}, "null pointer"), ({"mode": L.GN_E4M3_WINDOW, "table": None}, "null pointer"),
                       ({"c0": 324}, "channels"), ({"groups": 0}, "bad sizes"), ({"work_bytes": 64}, "work smaller"),
                       ({"mode": L.GN_E4M3_WINDOW, "table_bytes": 64}, "partial table"),
                       ({"mode": L.GN_E4M3_WINDOW_APPLY, "table_frames": 2}, "table_frames")]:
        assert gn(**kw) == -1 and needle in err(), (kw, err())
    # the partials mode needs neither gamma / beta nor the outputs
    assert gn(mode=L.GN_E4M3_WINDOW_PARTIALS, gamma=None, beta=None, out=None, scale=None, work_bytes=64) == -1
    assert "work smaller" in err()


def test_workspace_bytes_follow_the_mode():
    lib = L.load()
    p = L.GroupNormE4m3Params(c0=640, samples=2, frames=24, hw=4096, groups=32, eps=1e-5, dtype=L.F16)
    frame = lib.mimo_groupnorm_e4m3_workspace_bytes(ctypes.byref(p))
    p.mode = L.GN_E4M3_WINDOW
    window = lib.mimo_groupnorm_e4m3_workspace_bytes(ctypes.byref(p))
    # per image: min / max and the sums, both [images][slabs][groups][2]; window: min / max plus [samples][groups][2]
    assert frame > 0 and frame % 2 == 0 and window - frame // 2 == 2 * 32 * 2 * 4
    # the window table keeps its format: mimo_groupnorm_window_table_bytes is unchanged by the e4m3 modes
    assert ops.groupnorm_window_table_bytes(2, 24, 4096, 640, 32) > 0


def _scales(lo, hi, mean, rstd, gamma, beta):
    t = lambda v: torch.tensor(v, dtype=torch.float32)
    return ops.e4m3_image_scales(t(lo), t(hi), t(mean), t(rstd), t(gamma), t(beta))


def _silu(z):
    return z / (1 + math.exp(-z))


def test_scale_rule_on_hand_computed_cases():
    """one image, two groups of two channels; lo / hi / mean / rstd chosen so z_lo, z_hi are exact in fp32"""
    # gamma = 0: z = beta for every element, B_c = |silu(beta_c)|
    s, inv = _scales([[-3.0, 0.0]], [[5.0, 2.0]], [[1.0, 1.0]], [[0.5, 2.0]], [0.0, 0.0, 0.0, 0.0], [3.0, -0.5, 0.0, 1.0])
    assert s.item() == pytest.approx(_silu(3.0) / 448, rel=1e-6)
    # positive gamma: channel 0 of group 0: z in [(-3 - 1) * 0.5, (5 - 1) * 0.5] = [-2, 2] holds the minimum;
    # the bound is max(|silu(-2)|, |silu(2)|, 0.27846454) = silu(2)
    s, _ = _scales([[-3.0, 0.0]], [[5.0, 2.0]], [[1.0, 1.0]], [[0.5, 2.0]], [1.0, 0.0, 0.0, 0.0], [0.0] * 4)
    assert s.item() == pytest.approx(_silu(2.0) / 448, rel=1e-6)
    # negative gamma flips the interval: gamma = -0.25 on group 1: z in [(2 - 1) * 2 * -0.25, (0 - 1) * 2 * -0.25]
    # = [-0.5, 0.5]: max(|silu(-0.5)|, silu(0.5)) = silu(0.5); the minimum -1.2785 lies outside
    s, _ = _scales([[-3.0, 0.0]], [[5.0, 2.0]], [[1.0, 1.0]], [[0.5, 2.0]], [0.0, 0.0, -0.25, 0.0], [0.0] * 4)
    assert s.item() == pytest.approx(_silu(0.5) / 448, rel=1e-6)
    # an interval inside the negative half that holds the minimum: z in [-1.5, -1] -> 0.27846454 (> |silu(-1.5)| and
    # > |silu(-1)|)
    s, _ = _scales([[0.0, 0.0]], [[1.0, 0.0]], [[0.0, 0.0]], [[1.0, 1.0]], [0.5, 0.0, 0.0, 0.0], [-1.5, 0.0, 0.0, 0.0])
    assert s.item() == pytest.approx(0.27846454 / 448, rel=1e-7)
    assert max(abs(_silu(-1.5)), abs(_silu(-1.0))) < 0.27846454
    # the same interval one step left of the minimum: z in [-3, -2.5], bound |silu(-2.5)| (the value nearer the minimum)
    s, _ = _scales([[0.0, 0.0]], [[1.0, 0.0]], [[0.0, 0.0]], [[1.0, 1.0]], [0.5, 0.0, 0.0, 0.0], [-3.0, 0.0, 0.0, 0.0])
    assert s.item() == pytest.approx(abs(_silu(-2.5)) / 448, rel=1e-6)
    # an all-zero image (beta = 0, gamma = 0): scale 1, multiplier 1
    s, inv = _scales([[0.0, 0.0]], [[0.0, 0.0]], [[0.0, 0.0]], [[1.0, 1.0]], [0.0] * 4, [0.0] * 4)
    assert s.item() == 1.0 and inv.item() == 1.0
    # IEEE quotients: amax / 448 and 448 / amax as fp32 divisions
    s, inv = _scales([[0.0, 0.0]], [[0.0, 0.0]], [[0.0, 0.0]], [[1.0, 1.0]], [0.0] * 4, [20.0, 0.0, 0.0, 0.0])
    a = torch.tensor(20.0)  # silu(20) rounds to 20 in fp32
    assert s.item() == (a / torch.tensor(448.0)).item() and inv.item() == (torch.tensor(448.0) / a).item()


@pytest.mark.parametrize("frames", [1, 3])
def test_scale_bound_is_never_below_the_true_amax(frames):
    g = torch.Generator().manual_seed(9 + frames)
    for trial in range(4):
        n, hw, C, groups = 6, 49, 64, 8
        x = torch.randn(n, hw, C, generator=g) * (1 + 3 * trial) + torch.randn(1, 1, C, generator=g) * trial
        gamma = torch.randn(C, generator=g) * 2
        beta = torch.randn(C, generator=g)
        q, scale, y = ops.groupnorm_silu_e4m3_host(x, gamma, beta, groups, 1e-5, frames)
        amax = y.abs().amax(dim=(1, 2))
        assert torch.all(scale * 448 >= amax * (1 - 2e-7)), (scale * 448 / amax).min()
        # nothing saturates except by rounding, and the bound is not loose by more than the SiLU minimum it may add
        deq = q.float() * scale[:, None, None]
        assert torch.all(q.float().abs() <= 448)
        step = torch.exp2(torch.floor(torch.log2((y / scale[:, None, None]).abs().clamp(min=2.0 ** -6))) - 3)
        assert torch.all((deq - y).abs() <= step * scale[:, None, None] * 1.0001)


def test_conv_weight_pack_is_per_output_channel():
    """the e4m3 copy of a ResBlock conv is pack_e4m3_weight of the [Cout, 9 Cin] pack: row o holds tap-major channels and
    its scale is the amax over all 9 Cin weights of output channel o"""
    g = torch.Generator().manual_seed(4)
    w = (torch.randn(40, 32, 3, 3, generator=g) * torch.logspace(-2, 1, 40)[:, None, None, None]).half()
    w[3] = 0
    pk = ops.pack_conv3x3_weight(w)
    q, s = ops.pack_e4m3_weight(pk)
    rq, rs = ops.quantize_e4m3_rows(w.permute(0, 2, 3, 1).reshape(40, 9 * 32))
    assert torch.equal(q.view(torch.uint8), rq.view(torch.uint8)) and torch.equal(s, rs)
    assert s[3] == 1 and not q[3].view(torch.uint8).any()
    # tap (ky, kx), channel c of output o sits at column (3 ky + kx) * Cin + c
    o, ky, kx, c = 7, 2, 1, 5
    assert q[o, (3 * ky + kx) * 32 + c].float() * s[o] == rq[o, (3 * ky + kx) * 32 + c].float() * rs[o]


def _small_unet():
    from oracle import torch_oracle as O
    widths = (32, 64, 64, 64)
    cfg = O.UNetConfig(block_out_channels=widths, norm_num_groups=8, motion_groups=8, heads=8, cross_attention_dim=64)
    sd = O.make_denoising_unet_sd(cfg, seed=21)
    sd_ref = O.make_reference_unet_sd(cfg, seed=22)
    f, hw = 2, 8
    g = torch.Generator().manual_seed(23)
    ref_lat = torch.randn(1, 4, hw, hw, generator=g).repeat(2, 1, 1, 1)
    emb = torch.randn(1, 1, 64, generator=g)
    ehs = torch.cat([torch.zeros_like(emb), emb])
    x = torch.randn(1, 8, f, hw, hw, generator=g).repeat(2, 1, 1, 1, 1)
    banks = O.reference_unet_banks(sd_ref, ref_lat, ehs, cfg, bank_dtype=None)
    return O, cfg, sd, x, ehs, banks


def test_oracle_fp8_conv_emulation_error_is_finite_and_composes():
    from oracle import fp8_conv_oracle as F8C
    from oracle import fp8_oracle as F8
    from oracle import window_gn_oracle as WG
    O, cfg, sd, x, ehs, banks = _small_unet()
    run = lambda: O.denoising_unet(sd, x, 499, ehs, None, banks, cfg, cfg=True)
    with torch.no_grad():
        want = run()
        with F8C.fp8_conv_emulation():
            convs = run()
        with F8.fp8_emulation(), F8C.fp8_conv_emulation():
            both = run()
        with F8C.fp8_conv_emulation(), F8.fp8_emulation():
            both2 = run()
        with F8.fp8_emulation():
            proj = run()
        again = run()
        with WG.window_groupnorm():
            wwant = run()
            with F8C.fp8_conv_emulation():
                wconv = run()
            wagain = run()
    rel = lambda a, b: float((a - b).norm() / b.norm())
    print(f"rel_l2 vs fp32: convs {rel(convs, want):.3e}, convs + projections {rel(both, want):.3e}, "
          f"projections {rel(proj, want):.3e}, window convs {rel(wconv, wwant):.3e}")
    for t in (convs, both, wconv):
        assert torch.isfinite(t).all()
    assert 0 < rel(convs, want) < 0.5 and 0 < rel(both, want) < 0.5 and 0 < rel(wconv, wwant) < 0.5
    assert torch.equal(both, both2)  # the two emulations are independent of their nesting order
    assert not torch.equal(both, proj) and not torch.equal(both, convs)
    assert torch.equal(again, want) and torch.equal(wagain, wwant)  # the contexts restore the fp32 network
    assert not torch.equal(wwant, want)
