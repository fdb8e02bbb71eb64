"""FP8 feed-forward output projection without a GPU: the C-ABI structs and argument checks of
mimo_gemm_e4m3_geglu_e4m3 / mimo_gemm_e4m3_blockscaled, the per-(row, 128-column block) rule on hand-computed e4m3 bytes,
the e4m3 packing of the ff.net.2 weights, the oracle's emulation (alone and composed with the other oracle contexts) and
the FP8 switches of the module and the engine."""
import ctypes
import types

import pytest
import torch

from mimo_b200 import lib as L
from mimo_b200 import ops

PTR = 1 << 20


def test_abi_sizeof_ff_out_entry_points():
    lib = L.load()
    assert lib.mimo_abi_sizeof(12) == ctypes.sizeof(L.GemmE4m3GegluE4m3Params) == 104
    assert lib.mimo_abi_sizeof(13) == ctypes.sizeof(L.GemmE4m3BlockscaledParams) == 160
    assert lib.mimo_abi_sizeof(9) == ctypes.sizeof(L.GemmE4m3Params) == 152  # mimo_gemm_e4m3_params is unchanged


def test_entry_points_refuse_bad_arguments_before_the_device_probe():
    lib = L.load()
    err = lambda: lib.mimo_last_error().decode()

    def geglu(**kw):
        p = L.GemmE4m3GegluE4m3Params(M=300, N=2560, K=320, lda=320, ldw=320, ldo=1280, ld_scale=300, dtype=L.F16)
        p.a = p.w = p.out = p.a_scale = p.w_scale = p.out_scale = p.bias = PTR
        for k, v in kw.items():
            setattr(p, k, v)
        return lib.mimo_gemm_e4m3_geglu_e4m3(ctypes.byref(p), None)

    for kw, needle in [({"a": None}, "null pointer"), ({"a_scale": None}, "null pointer"),
                       ({"w_scale": None}, "null pointer"), ({"out_scale": None}, "null pointer"),
                       ({"M": 0}, "empty problem"), ({"K": 328}, "multiples of 16"), ({"ldo": 1288}, "multiples of 16"),
                       ({"N": 2688}, "N % 256"), ({"N": 320}, "N % 256"), ({"ld_scale": 296}, "ld_scale"),
                       ({"ld_scale": 302}, "ld_scale"), ({"out": PTR + 8}, "16-byte aligned"),
                       ({"out_scale": PTR + 4}, "16-byte aligned")]:
        assert geglu(**kw) == -1 and needle in err(), (kw, err())

    def bs(**kw):
        p = L.GemmE4m3BlockscaledParams(M=300, N=320, K=1280, lda=1280, ldw=1280, ldo=320, ld_scale=300, dtype=L.F16)
        p.a = p.w = p.out = p.a_scale = p.w_scale = PTR
        for k, v in kw.items():
            setattr(p.ep if k in ("residual", "ld_res", "act") else p, k, v)
        return lib.mimo_gemm_e4m3_blockscaled(ctypes.byref(p), None)

    for kw, needle in [({"a": None}, "null pointer"), ({"a_scale": None}, "null pointer"),
                       ({"w_scale": None}, "null pointer"), ({"N": 0}, "empty problem"),
                       ({"K": 1296, "lda": 1296, "ldw": 1296}, "multiple of 128"), ({"lda": 1288}, "multiples of 16"),
                       ({"N": 324}, "multiples of 8"), ({"ld_scale": 296}, "ld_scale"), ({"ld_scale": 301}, "ld_scale"),
                       ({"a_scale": PTR + 4}, "16-byte aligned"), ({"out": PTR + 8}, "16-byte aligned"),
                       ({"residual": PTR, "ld_res": 4}, "ld_res"), ({"act": L.ACT_GEGLU}, "GEGLU"),
                       ({"workspace": PTR, "workspace_bytes": 1 << 20}, "split-K")]:
        assert bs(**kw) == -1 and needle in err(), (kw, err())
    lib.mimo_debug_force_bn(256)
    try:
        assert bs() == -1 and "unsupported BN" in err()
    finally:
        lib.mimo_debug_force_bn(0)


def test_block_rule_against_hand_computed_bytes():
    """two rows of two 128-column blocks. Row 0, block 0: amax 896 -> scale 2, inv 0.5: 896 -> 448 (0x7E, the largest
    finite), -896 -> 0xFE, 2^-8 -> 2^-9 (0x01, the smallest subnormal), 2.125 -> 1.0625, a tie between 1 (0x38) and 1.125
    (0x39) -> even 0x38, 2.375 -> 1.1875, a tie between 1.125 and 1.25 (0x3A) -> even 0x3A. Row 0, block 1 is all zero:
    scale 1, zero bytes. Row 1: block 0 zero, block 1 amax 3 -> 3 * (448 / 3) rounds to 448 (0x7E)."""
    y = torch.zeros(2, 256)
    y[0, :6] = torch.tensor([896.0, -896.0, 2.0 ** -8, 2.125, 2.375, 0.0])
    y[1, 130] = 3.0
    y[1, 131] = -1.5
    q, s = ops.quantize_e4m3_blocks(y, 128)
    assert s.shape == (2, 2) and s.dtype == torch.float32
    assert s.tolist() == [[2.0, 1.0], [1.0, float(torch.tensor(3.0) / torch.tensor(448.0))]]
    b = q.view(torch.uint8)
    assert b[0, :6].tolist() == [0x7E, 0xFE, 0x01, 0x38, 0x3A, 0x00]
    assert not b[0, 6:].any() and not b[1, :130].any()
    assert b[1, 130] == 0x7E and b[1, 131] == 0xF6  # -1.5 * 149.33 = -224 exactly: 0xF6
    # the same bytes as the per-row rule on each block
    for r in range(2):
        for k in range(2):
            rq, rs = ops.quantize_e4m3_rows(y[r:r + 1, 128 * k:128 * k + 128])
            assert torch.equal(rq.view(torch.uint8)[0], b[r, 128 * k:128 * k + 128]) and rs[0] == s[k, r]


def test_ff_out_weight_pack_matches_the_torch_rule():
    """UNetEngine._pack_e4m3_ff_out: one e4m3 copy per spatial transformer and per motion transformer block, each
    quantize_e4m3_rows of the [C, 4C] ff.net.2 weight (one scale per output channel)"""
    from mimo_b200 import engine as E
    g = torch.Generator().manual_seed(5)
    mk = lambda c: ((torch.randn(c, 4 * c, generator=g) * torch.logspace(-2, 1, c)[:, None]).half(),
                    torch.randn(c, generator=g).half())
    w = {"down_blocks.0.attentions.0": {"ffo": mk(32)}, "mid_block.attentions.0": {"ffo": mk(64)},
         "up_blocks.1.motion_modules.2": {"blocks": [{"ffo": mk(64)}, {"ffo": mk(64)}]}}
    w["mid_block.attentions.0"]["ffo"][0][3] = 0
    stub = types.SimpleNamespace(w=w, xf_paths=["down_blocks.0.attentions.0", "mid_block.attentions.0"])
    w8 = E.UNetEngine._pack_e4m3_ff_out(stub)
    want = {"down_blocks.0.attentions.0": w["down_blocks.0.attentions.0"]["ffo"][0],
            "mid_block.attentions.0": w["mid_block.attentions.0"]["ffo"][0],
            "up_blocks.1.motion_modules.2.0": w["up_blocks.1.motion_modules.2"]["blocks"][0]["ffo"][0],
            "up_blocks.1.motion_modules.2.1": w["up_blocks.1.motion_modules.2"]["blocks"][1]["ffo"][0]}
    assert set(w8) == set(want)
    for k, wt in want.items():
        y = wt.float()
        amax = y.abs().amax(dim=1)
        inv = torch.where(amax == 0, torch.ones_like(amax), torch.full_like(amax, 448.0) / amax)
        scale = torch.where(amax == 0, torch.ones_like(amax), amax / torch.full_like(amax, 448.0))
        rq = torch.clamp(y * inv[:, None], -448, 448).to(torch.float8_e4m3fn)
        q, s = w8[k]
        assert q.shape == wt.shape and torch.equal(q.view(torch.uint8), rq.view(torch.uint8)) and torch.equal(s, scale)
    q, s = w8["mid_block.attentions.0"]
    assert s[3] == 1 and not q[3].view(torch.uint8).any()


def test_oracle_fp8_ff_out_emulation_error_is_finite_and_composes():
    from oracle import fp8_conv_oracle as F8C
    from oracle import fp8_ff_oracle as F8F
    from oracle import fp8_oracle as F8
    from oracle import torch_oracle as O
    from oracle import window_gn_oracle as WG
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
    run = lambda: O.denoising_unet(sd, x, 499, ehs, None, banks, cfg, cfg=True)
    with torch.no_grad():
        want = run()
        with F8.fp8_emulation():
            proj = run()
            with F8F.fp8_ff_out_emulation():
                ffo = run()
        with F8F.fp8_ff_out_emulation(), F8.fp8_emulation():
            ffo2 = run()
        with F8F.fp8_ff_out_emulation():
            alone = run()  # without the FP8 projections there is no FP8 feed-forward output
        with F8.fp8_emulation(), F8C.fp8_conv_emulation(), F8F.fp8_ff_out_emulation():
            all3 = run()
        with F8.fp8_emulation(), F8C.fp8_conv_emulation():
            convs = run()
        again = run()
        with WG.window_groupnorm():
            wwant = run()
            with F8.fp8_emulation(), F8C.fp8_conv_emulation(), F8F.fp8_ff_out_emulation():
                wall = run()
    rel = lambda a, b: float((a - b).norm() / b.norm())
    print(f"rel_l2 vs fp32: projections {rel(proj, want):.3e}, + ff_out {rel(ffo, want):.3e}, + convs + ff_out "
          f"{rel(all3, want):.3e}, window all {rel(wall, wwant):.3e}")
    for t in (ffo, all3, wall):
        assert torch.isfinite(t).all()
    assert 0 < rel(ffo, want) < 0.5 and 0 < rel(all3, want) < 0.5 and 0 < rel(wall, wwant) < 0.5
    assert torch.equal(ffo, ffo2)  # nesting order does not matter
    assert not torch.equal(ffo, proj) and not torch.equal(all3, convs)
    assert torch.equal(alone, want) and torch.equal(again, want)  # the contexts restore the networks they replace


def test_module_and_engine_fp8_switches_without_a_device():
    """enable_fp8 sets the whole configuration each call; fp8_ff_out_enabled follows; disable_fp8 clears all three;
    the engine refuses ff_out without the FP8 projections before touching anything"""
    from mimo_b200 import engine as E
    from mimo_b200.host import modules as M
    den = M.UNet3DConditionModel(block_out_channels=(32, 64, 64, 64), norm_num_groups=8, cross_attention_dim=64,
                                 attention_head_dim=8, use_inflated_groupnorm=True, use_motion_module=True,
                                 motion_module_mid_block=True, motion_module_type="Vanilla",
                                 motion_module_kwargs=dict(num_attention_heads=8, num_transformer_block=1,
                                                           attention_block_types=["Temporal_Self", "Temporal_Self"],
                                                           temporal_position_encoding=True,
                                                           temporal_position_encoding_max_len=32,
                                                           temporal_attention_dim_div=1),
                                 unet_use_cross_frame_attention=False, unet_use_temporal_attention=False)
    den = den.to(torch.float16)
    assert not den.fp8_ff_out_enabled
    den.enable_fp8(ff_out=True)
    assert den.fp8_enabled and den.fp8_ff_out_enabled and not den.fp8_convs_enabled
    den.enable_fp8(convs=True, ff_out=True)
    assert den.fp8_enabled and den.fp8_ff_out_enabled and den.fp8_convs_enabled
    den.enable_fp8(convs=True)
    assert den.fp8_convs_enabled and not den.fp8_ff_out_enabled
    den.enable_fp8(ff_out=True)
    den.enable_fp8()
    assert den.fp8_enabled and not den.fp8_ff_out_enabled and not den.fp8_convs_enabled
    den.enable_fp8(convs=True, ff_out=True)
    den.disable_fp8()
    assert not den.fp8_enabled and not den.fp8_convs_enabled and not den.fp8_ff_out_enabled
    with pytest.raises(AttributeError):
        den.fp8_ff_out_enabled = True
    eng = object.__new__(E.UNetEngine)  # no device: set_fp8 must refuse before it packs or drops anything
    eng.fp8 = False
    with pytest.raises(ValueError, match="ff_out"):
        eng.set_fp8(False, ff_out=True)
    with pytest.raises(ValueError, match="convs"):
        eng.set_fp8(False, convs=True, ff_out=True)
