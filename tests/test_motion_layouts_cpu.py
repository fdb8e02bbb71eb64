"""Motion-module layouts other than inference_v2.yaml's, on the CPU: which configs build and which are refused, the
state-dict key sets against the reference's own UNet3D (tests/golden/unet_motion_layouts.pt, written by
oracle/gen_motion_layout_golden.py), the defaults of omitted motion_module_kwargs keys, the oracle against the
reference's outputs, the engine's packing and placement, and the frame-sharding token count."""
import zlib

import pytest
import torch

from mimo_b200 import engine as E
from mimo_b200.host import modules as M
from mimo_b200.host import pipeline as P
from mimo_b200.host import schema
from oracle import gen_motion_layout_golden as GL
from oracle import motion_layout_oracle as ML
from oracle import torch_oracle as O

WIDTHS = (128, 256, 512, 512)
_SD15 = dict(block_out_channels=WIDTHS, cross_attention_dim=768, use_motion_module=True, motion_module_type="Vanilla")
_NAMES = [c["name"] for c in GL.LAYOUTS]


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(golden_dir / "unet_motion_layouts.pt")


def _case(golden, name):
    return next(c for c in golden["cases"] if c["name"] == name)


def _model(**kw):
    return M.UNet3DConditionModel(**_SD15, **kw)


# ------------------------------------------------------------------------------------------------
# construction
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [
    dict(motion_module_mid_block=False),
    dict(motion_module_mid_block=True, motion_module_decoder_only=True),
    dict(motion_module_resolutions=(1,)),
    dict(motion_module_resolutions=[2, 8], motion_module_mid_block=True),
    dict(motion_module_resolutions=(), motion_module_mid_block=False),
    dict(motion_module_kwargs=dict(num_transformer_block=3)),
    dict(motion_module_kwargs=dict(attention_block_types=["Temporal_Self"])),
    dict(motion_module_kwargs=dict(attention_block_types=("Temporal_Self",) * 4)),
    dict(motion_module_kwargs=dict(temporal_position_encoding=True, temporal_position_encoding_max_len=24)),
    dict(motion_module_kwargs=dict(temporal_position_encoding=False)),
    dict(motion_module_kwargs=dict(temporal_position_encoding=True, temporal_position_encoding_max_len=7)),
    dict(motion_module_kwargs=dict(num_attention_heads=4)),
    dict(motion_module_kwargs=dict(num_attention_heads=16)),
    dict(motion_module_kwargs=dict(num_attention_heads=2)),
    dict(motion_module_kwargs=dict(zero_initialize=False, cross_frame_attention_mode=None, temporal_attention_dim_div=1)),
], ids=str)
def test_accepted_layouts_build(kw):
    m = _model(**kw)
    assert set(m.state_dict()) == set(schema.unet_schema(WIDTHS, motion_layout=m.motion_layout))
    assert m._spec.motion_layout == m.motion_layout


@pytest.mark.parametrize("kw,names", [
    (dict(use_motion_module=False), "use_motion_module"),
    (dict(motion_module_type="Conv"), "motion_module_type"),
    (dict(motion_module_kwargs=dict(attention_block_types=["Temporal_Self", "Temporal_Cross"])), "Temporal_Cross"),
    (dict(motion_module_kwargs=dict(attention_block_types=[])), "attention_block_types"),
    (dict(motion_module_kwargs=dict(cross_frame_attention_mode="Mid")), "cross_frame_attention_mode"),
    (dict(motion_module_kwargs=dict(temporal_attention_dim_div=2)), "temporal_attention_dim_div"),
    (dict(motion_module_kwargs=dict(num_transformer_block=0)), "num_transformer_block"),
    (dict(motion_module_kwargs=dict(num_attention_heads=64)), "num_attention_heads"),
    (dict(motion_module_kwargs=dict(num_attention_heads=3)), "num_attention_heads"),
    (dict(motion_module_kwargs=dict(num_attention_heads=1)), "num_attention_heads"),  # heads of 512 > 256 channels
    (dict(motion_module_kwargs=dict(num_attention_heads=0)), "num_attention_heads"),
    (dict(motion_module_resolutions=(1, 16)), "motion_module_resolutions"),
    (dict(unet_use_cross_frame_attention=True), "unet_use_cross_frame_attention"),
    (dict(unet_use_temporal_attention=True), "unet_use_temporal_attention"),
], ids=lambda v: v if isinstance(v, str) else None)
def test_refused_options_name_themselves(kw, names):
    args = dict(_SD15, **kw)
    with pytest.raises(NotImplementedError, match=names):
        M.UNet3DConditionModel(**args)


def test_head_widths_the_kernel_cannot_run_are_refused():
    """mimo_attn_temporal runs heads of a multiple of 8 channels, at most 256. Heads above 256 channels are refused by
    the constructor (SD1.5 widths with 4 heads: 80 / 160 / 320), before any weight is made; head widths that are not a
    multiple of 8 (16 heads at SD1.5 widths: 20 / 40 / 80) when the engine is built, before the device is touched."""
    sd15 = dict(_SD15, block_out_channels=(320, 640, 1280, 1280))
    with pytest.raises(NotImplementedError, match=r"num_attention_heads=4 .*1280"):
        M.UNet3DConditionModel(**sd15, motion_module_kwargs=dict(num_attention_heads=4))
    for heads, widths, bad in ((16, (320, 640, 1280, 1280), "widths 320 get heads of 20 channels"),
                                (32, WIDTHS, "widths 128 get heads of 4 channels")):
        spec = E.UNetSpec(block_out_channels=widths, motion_layout=schema.MotionLayout(heads=heads))
        with pytest.raises(NotImplementedError, match=rf"num_attention_heads={heads}: .*{bad}"):
            E.UNetEngine({}, spec, "cpu")
    # placed widths only: without the 320-wide modules, 16 heads run (40 / 80 channels)
    spec = E.UNetSpec(motion_layout=schema.MotionLayout(heads=16, resolutions=(2, 4, 8)))
    assert all(d % 8 == 0 for d in spec.motion_layout.head_widths(spec.block_out_channels).values())
    with pytest.raises(Exception) as e:
        E.UNetEngine({}, spec, "cpu")
    assert not isinstance(e.value, NotImplementedError)


def test_unknown_motion_kwargs_are_a_type_error():
    with pytest.raises(TypeError, match="not_a_key"):
        _model(motion_module_kwargs=dict(not_a_key=1))


def test_omitted_keys_take_the_reference_defaults():
    """VanillaTemporalModule's defaults (motion_module.py:45-55): 8 heads, 2 transformer blocks, two Temporal_Self
    attentions, no positional encoding, max_len 24; a config that leaves the keys out builds that network."""
    m = _model(motion_module_kwargs={})
    assert m.motion_layout == schema.MotionLayout(resolutions=(1, 2, 4, 8), mid_block=False, decoder_only=False,
                                                  blocks=2, attn_blocks=2, pe=False, max_len=24, heads=8)
    assert _model().motion_layout == m.motion_layout  # motion_module_kwargs=None is the same
    keys = m.state_dict().keys()
    assert not any(k.endswith("pos_encoder.pe") for k in keys)
    assert any(".transformer_blocks.1." in k for k in keys)
    # and inference_v2's explicit keys still give inference_v2's network
    v2 = _model(motion_module_mid_block=True, motion_module_kwargs=dict(
        num_attention_heads=8, num_transformer_block=1, attention_block_types=["Temporal_Self", "Temporal_Self"],
        temporal_position_encoding=True, temporal_position_encoding_max_len=32, temporal_attention_dim_div=1))
    assert v2.motion_layout == schema.MotionLayout()
    assert repr(v2._spec) == repr(E.UNetSpec(block_out_channels=WIDTHS, cross_attention_dim=768))


# ------------------------------------------------------------------------------------------------
# the reference's key sets and outputs
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", _NAMES)
def test_schema_equals_the_reference_key_set(golden, name):
    c = _case(golden, name)
    want = zlib.decompress(c["keys_zlib"]).decode().split("\n")
    assert len(want) == c["n_keys"]
    m = _model(**c["kwargs"])
    assert sorted(schema.unet_schema(WIDTHS, motion_layout=m.motion_layout)) == want
    assert sorted(m.state_dict()) == want
    # the oracle's generator makes the same keys (the fixture loaded them into the reference with strict=True)
    lay = ML.Layout(**c["layout"])
    assert sorted(ML.make_denoising_unet_sd(O.UNetConfig(block_out_channels=WIDTHS), lay, c["seed"])) == want
    assert vars(m.motion_layout) == vars(lay)


@pytest.mark.parametrize("name", _NAMES)
def test_oracle_matches_the_reference_fixture(golden, name):
    c = _case(golden, name)
    cfg = O.UNetConfig(block_out_channels=tuple(golden["widths"]))
    lay = ML.Layout(**c["layout"])
    sd_den = ML.make_denoising_unet_sd(cfg, lay, c["seed"])
    sd_ref = O.make_reference_unet_sd(cfg, seed=c["seed"] + 1)
    x = c["x"].repeat(2, 1, 1, 1, 1)
    inflated = c["kwargs"]["use_inflated_groupnorm"]
    got = GL.oracle_case(cfg, lay, inflated, sd_den, sd_ref, c["ref_lat"], c["ehs"], x)
    assert got.shape == c["out"].shape == (2, 4, golden["f"], golden["h"], golden["w"])
    assert _rel(got, c["out"]) < 3e-6  # fp32 on both sides: summation order only
    # the motion modules are live: without them the network is a different one
    bare = GL.oracle_case(cfg, ML.Layout(resolutions=(), mid_block=False), inflated, sd_den, sd_ref, c["ref_lat"],
                          c["ehs"], x)
    assert _rel(bare, c["out"]) > 1e-2


def test_layout_oracle_leaves_torch_oracle_as_it_was():
    assert O.motion_module is ML._MOTION_MODULE
    with ML.motion_layout(ML.Layout()):
        assert O.motion_module is not ML._MOTION_MODULE
    assert O.motion_module is ML._MOTION_MODULE
    # inference_v2's layout through the general module is torch_oracle's module
    cfg = O.UNetConfig(block_out_channels=(64, 64, 64, 64))
    sd = O.make_denoising_unet_sd(cfg, seed=3)
    x = torch.randn(6, 64, 3, 5, generator=torch.Generator().manual_seed(4))
    p = "up_blocks.1.motion_modules.2"
    assert torch.equal(ML.motion_module(sd, p, x, 3, ML.Layout()), O.motion_module(sd, p, x, 3, cfg))


# ------------------------------------------------------------------------------------------------
# engine placement and frame sharding
# ------------------------------------------------------------------------------------------------
def test_placement_follows_the_reference_resolutions():
    lay = schema.MotionLayout(resolutions=(1, 2), decoder_only=True, mid_block=True)
    assert [lay.placed(f"down_blocks.{i}", 4) for i in range(4)] == [False] * 4
    assert [lay.placed(f"up_blocks.{i}", 4) for i in range(4)] == [False, False, True, True]
    assert lay.placed("mid_block", 4) and lay.levels(4) == [0, 1, 3]
    # the reference's up-level rule is 2^(3 - i) whatever the number of levels: a 3-level UNet's up blocks 0, 1, 2 are
    # resolutions 8, 4, 2 (unet_3d_edit_bkfill.py:188)
    lay = schema.MotionLayout(resolutions=(1, 2), mid_block=False)
    assert [lay.placed(f"up_blocks.{i}", 3) for i in range(3)] == [False, False, True]
    assert [lay.placed(f"down_blocks.{i}", 3) for i in range(3)] == [True, True, False]
    assert lay.levels(3) == [0, 1]
    lay = schema.MotionLayout(resolutions=(1, 8), mid_block=False)
    assert [lay.placed(f"down_blocks.{i}", 4) for i in range(4)] == [True, False, False, True]
    assert [lay.placed(f"up_blocks.{i}", 4) for i in range(4)] == [True, False, False, True]
    assert lay.levels(4) == [0, 3]
    for c in GL.LAYOUTS:  # the oracle's restatement of the rule agrees
        ol = c["layout"]
        sl = schema.MotionLayout(**vars(ol))
        for i in range(4):
            for kind, n in (("down_blocks", 2), ("up_blocks", 3)):
                for j in range(n):
                    assert sl.placed(f"{kind}.{i}", 4) == ol.has_module(f"{kind}.{i}.motion_modules.{j}")
        assert sl.placed("mid_block", 4) == ol.has_module("mid_block.motion_modules.0")


def test_engine_packs_the_layout():
    """_pack on the CPU (the packing is plain torch): one entry per placed module, one block per transformer block,
    one attention per attention block, a PE table only with positional encoding."""
    from types import SimpleNamespace
    m = _model(**GL.LAYOUTS[2]["kwargs"])  # stress
    eng = SimpleNamespace()
    E.UNetEngine._pack(eng, m.state_dict(), m._spec, "cpu", torch.float32)
    mms = sorted(p for p in eng.w if ".motion_modules." in p)
    assert mms == sorted([f"up_blocks.{i}.motion_modules.{j}" for i in (2, 3) for j in range(3)]
                         + ["mid_block.motion_modules.0"])
    for p in mms:
        blocks = eng.w[p]["blocks"]
        assert len(blocks) == 2 and all(len(b["attn"]) == 3 for b in blocks)
        assert all("pe" not in a for b in blocks for a in b["attn"])
    w8 = E.UNetEngine._pack_e4m3(eng)
    assert sorted(k for k in w8 if ".motion_modules." in k) == sorted(f"{p}.{k}" for p in mms for k in range(2))
    assert all(len(w8[f"{p}.{k}"]["qkv"]) == 3 for p in mms for k in range(2))
    v1 = _model(**GL.LAYOUTS[0]["kwargs"])
    eng = SimpleNamespace()
    E.UNetEngine._pack(eng, v1.state_dict(), v1._spec, "cpu", torch.float32)
    assert "mid_block.motion_modules.0" not in eng.w
    assert eng.w["down_blocks.0.motion_modules.0"]["blocks"][0]["attn"][0]["pe"].shape == (24, 128)


def test_shard_tokens_counts_only_levels_with_motion_modules():
    # 64 x 64 latent: levels 64x64, 32x32, 16x16, 8x8
    assert P.shard_tokens(64, 64, 4) == 64 == P.shard_tokens(64, 64, 4, [0, 1, 2, 3])
    stress = schema.MotionLayout(resolutions=(1, 2), decoder_only=True, mid_block=False)
    assert P.shard_tokens(64, 64, 4, stress.levels(4)) == 1024  # 32 x 32 is the coarsest level with a module
    v1 = schema.MotionLayout(mid_block=False)
    assert P.shard_tokens(64, 64, 4, v1.levels(4)) == 64  # the 8 x 8 down / up blocks still have modules
    assert P.shard_tokens(64, 64, 4, []) == 0  # no module: nothing is split, every frame-group size divides 0
    assert P.shard_tokens(98, 98, 4, [0]) == 98 * 98
    from mimo_b200.host.shard import ShardPlan
    plan = ShardPlan.make(8, 0, True, 1, 24, min_tokens=P.shard_tokens(14, 10, 4, [0]))
    assert plan.frame_ways == 4  # 140 tokens split 4 ways; with every level (gcd 1) frames could not be split
    with pytest.raises(NotImplementedError):
        ShardPlan.make(8, 0, True, 1, 24, min_tokens=P.shard_tokens(14, 10, 4))
