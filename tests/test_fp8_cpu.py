"""FP8 (e4m3) path without a GPU: the C-ABI struct and argument checks of mimo_gemm_e4m3 / mimo_layernorm_e4m3, the
e4m3 weight packing against the torch rule, and the oracle's FP8 emulation on a small seeded UNet."""
import ctypes

import pytest
import torch

from mimo_b200 import lib as L
from mimo_b200 import ops

PTR = 1 << 20


def _torch_rule(y):
    y = y.float()
    amax = y.abs().amax(dim=1)
    inv = torch.where(amax == 0, torch.ones_like(amax), torch.full_like(amax, 448.0) / amax)
    scale = torch.where(amax == 0, torch.ones_like(amax), amax / torch.full_like(amax, 448.0))
    return torch.clamp(y * inv[:, None], -448, 448).to(torch.float8_e4m3fn), scale


def test_abi_sizeof_gemm_e4m3():
    lib = L.load()
    assert lib.mimo_abi_sizeof(9) == ctypes.sizeof(L.GemmE4m3Params)
    assert ctypes.sizeof(L.GemmE4m3Params) == 152
    assert lib.mimo_abi_sizeof(1) == ctypes.sizeof(L.GemmParams)  # mimo_gemm_params is unchanged


def test_entry_points_refuse_bad_arguments_before_the_device_probe():
    lib = L.load()
    err = lambda: lib.mimo_last_error().decode()

    def gemm(**kw):
        p = L.GemmE4m3Params()
        p.a = p.w = p.out = p.a_scale = p.w_scale = PTR
        p.lda = p.ldw = p.ldo = 64
        p.M, p.N, p.K = 128, 64, 64
        for k, v in kw.items():
            setattr(p.ep if k in ("residual", "ld_res", "act", "rowvec") else p, k, v)
        return lib.mimo_gemm_e4m3(ctypes.byref(p), None)

    for kw, needle in [({"a": None}, "null pointer"), ({"w_scale": None}, "null pointer"),
                       ({"a_scale": None}, "null pointer"), ({"M": 0}, "empty problem"),
                       ({"K": 72}, "multiples of 16"), ({"lda": 72}, "multiples of 16"),
                       ({"ldo": 60}, "multiples of 8"), ({"a": PTR + 8}, "16-byte aligned"),
                       ({"workspace": PTR, "workspace_bytes": 1 << 20}, "split-K"),
                       ({"act": L.ACT_GEGLU, "residual": PTR, "ld_res": 64}, "GEGLU"),
                       ({"act": L.ACT_GEGLU, "N": 320}, "GEGLU")]:
        assert gemm(**kw) == -1 and needle in err(), (kw, err())

    def ln(x=PTR, out=PTR, scale=PTR, c=320, pe=None, rpf=1):
        return lib.mimo_layernorm_e4m3(x, PTR, PTR, out, scale, 16, c, 1e-5, pe, rpf, 1, 0, L.F16, None)

    for kw, needle in [({"x": None}, "null pointer"), ({"scale": None}, "null pointer"), ({"c": 328}, "multiple of 16"),
                       ({"c": 4096}, "<= 2048"), ({"pe": PTR, "rpf": 0}, "pe args")]:
        assert ln(**kw) == -1 and needle in err(), (kw, err())


def test_weight_pack_matches_the_torch_rule():
    g = torch.Generator().manual_seed(5)
    w = (torch.randn(96, 64, generator=g) * torch.logspace(-3, 1, 96)[:, None]).half()
    w[7] = 0  # a zero row: scale 1, all-zero bytes
    q, s = ops.pack_e4m3_weight(w)
    rq, rs = _torch_rule(w)
    assert q.dtype == torch.float8_e4m3fn and s.dtype == torch.float32
    assert torch.equal(q.view(torch.uint8), rq.view(torch.uint8)) and torch.equal(s, rs)
    assert s[7] == 1 and not q[7].view(torch.uint8).any()
    # every row reaches +-448 exactly once its amax is scaled, and nothing saturates past it
    assert torch.all(q.float().abs().amax(1)[torch.arange(96) != 7] == 448)


def test_quantization_rule_against_hand_computed_bytes():
    """The rule pinned without torch's cast: OCP E4M3FN bytes (sign, 4 exponent bits with bias 7, 3 mantissa bits) worked
    out by hand. Row 0 has amax 7, so inv = 64 and the scale is 7 / 448 = 1 / 64: every value is scaled by a power of two
    and only the rounding of the mantissa is in play. Row 1 reaches 448 at its amax and must not exceed it."""
    y = torch.tensor([[7.0, -7.0, 1.0, 0.5, 0.00390625, 0.0, 3.5, 2.0 ** -15, 0.0048828125, 0.005126953125],
                      [1.0, 0.999, -0.5, 0.25, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0]])
    q, s = ops.quantize_e4m3_rows(y)
    # row 0, x 64: 448 -> 0x7E, -448 -> 0xFE, 64 = 2^6 -> 0x68, 32 -> 0x60, 0.25 -> 0x28, 0 -> 0x00, 224 -> 0x76,
    #   2^-9 (smallest subnormal) -> 0x01, 0.3125 = 1.25 * 2^-2 -> 0x2A, 0.328125 = 1.3125 * 2^-2: tie between 1.25 and
    #   1.375 -> even mantissa 010 -> 0x2A
    assert q[0].view(torch.uint8).tolist() == [0x7E, 0xFE, 0x68, 0x60, 0x28, 0x00, 0x76, 0x01, 0x2A, 0x2A]
    assert s[0].item() == 7.0 / 448.0
    # row 1: inv = 448, 0.999 * 448 = 447.55 rounds to 448 (0x7E), 0.5 -> 224 (0xF6 with the sign), 0.25 -> 112 = 1.75 * 2^6 (0x6E)
    assert q[1].view(torch.uint8).tolist()[:4] == [0x7E, 0x7E, 0xF6, 0x6E]
    assert torch.all(q.float().abs() <= 448) and s[1] == torch.tensor(1.0) / torch.tensor(448.0)  # fp32 quotient
    # an all-zero row: scale 1, zero bytes
    q, s = ops.quantize_e4m3_rows(torch.zeros(1, 16))
    assert s.item() == 1.0 and not q.view(torch.uint8).any()


def test_geglu_pack_unpermutes_to_the_per_row_quantization():
    """The e4m3 GEGLU weight is quantized from the tile-interleaved fp16 pack; un-interleaving it (bytes and scales) must
    give the per-row quantization of the original [value rows; gate rows] weight."""
    if not L.LIB_PATH.exists():
        pytest.skip("library not built")
    g = torch.Generator().manual_seed(6)
    inner, dim = 1280, 64
    w = torch.randn(2 * inner, dim, generator=g).half()
    b = torch.randn(2 * inner, generator=g).half()
    wp, _ = ops.pack_geglu_weight(w, b)
    q, s = ops.pack_e4m3_weight(wp)
    gr = L.load().mimo_gemm_geglu_granule(2 * inner)
    # packed row r of tile t: value rows [t g, t g + g) then gate rows [t g, t g + g)
    t = torch.arange(2 * inner) // (2 * gr)
    within = torch.arange(2 * inner) % (2 * gr)
    src = torch.where(within < gr, t * gr + within, inner + t * gr + within - gr)
    unq = torch.empty_like(q.view(torch.uint8))
    uns = torch.empty_like(s)
    unq[src] = q.view(torch.uint8)
    uns[src] = s
    rq, rs = _torch_rule(w)
    assert torch.equal(unq, rq.view(torch.uint8)) and torch.equal(uns, rs)


def test_oracle_fp8_emulation_error_is_finite():
    from oracle import fp8_oracle as F8
    from oracle import torch_oracle as O
    torch.manual_seed(0)
    widths = (32, 64, 64, 64)
    cfg = O.UNetConfig(block_out_channels=widths, norm_num_groups=8, motion_groups=8, heads=8, cross_attention_dim=64)
    sd = O.make_denoising_unet_sd(cfg, seed=11)
    sd_ref = O.make_reference_unet_sd(cfg, seed=12)
    f, hw = 2, 8
    g = torch.Generator().manual_seed(13)
    ref_lat = torch.randn(1, 4, hw, hw, generator=g).repeat(2, 1, 1, 1)
    emb = torch.randn(1, 1, 64, generator=g)
    ehs = torch.cat([torch.zeros_like(emb), emb])
    x = torch.randn(1, 8, f, hw, hw, generator=g).repeat(2, 1, 1, 1, 1)
    with torch.no_grad():
        banks = O.reference_unet_banks(sd_ref, ref_lat, ehs, cfg, bank_dtype=None)
        want = O.denoising_unet(sd, x, 499, ehs, None, banks, cfg, cfg=True)
        with F8.fp8_emulation():
            got = O.denoising_unet(sd, x, 499, ehs, None, banks, cfg, cfg=True)
        again = O.denoising_unet(sd, x, 499, ehs, None, banks, cfg, cfg=True)
    err = float((got - want).norm() / want.norm())
    print(f"rel_l2(oracle_fp8, oracle_fp32) = {err:.3e}")
    assert torch.isfinite(got).all() and 0 < err < 0.5
    assert torch.equal(again, want)  # the context restores the fp32 network
