"""use_inflated_groupnorm=False on the CPU: the oracle against the reference's own UNet3D (tests/golden/
unet_clip_gn_read.pt, oracle/gen_clip_gn_golden.py), the argument checks of the window GroupNorm entry points (before
any device probe), the module surface, and the calls the engine makes for a ResnetBlock3D in each mode."""
import ctypes
from types import SimpleNamespace

import pytest
import torch

from mimo_b200 import engine as E
from mimo_b200 import lib as L
from mimo_b200 import ops
from oracle import gen_clip_gn_golden as GG
from oracle import torch_oracle as O
from oracle import window_gn_oracle as WG


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())


@pytest.mark.parametrize("case", [c["name"] for c in GG.CASES])
def test_oracle_matches_reference_fixture(golden_dir, case):
    g = torch.load(golden_dir / "unet_clip_gn_read.pt")
    c = next(x for x in g["cases"] if x["name"] == case)
    cfg = O.UNetConfig(block_out_channels=tuple(g["cfg"]))
    with torch.no_grad():
        got = GG.oracle_case(cfg, c["f"], c["h"], c["w"], c["seed"])
        per_frame = GG.oracle_case(cfg, c["f"], c["h"], c["w"], c["seed"], window=False)
    assert got.shape == c["out"].shape == (2, 4, c["f"], c["h"], c["w"])
    assert _rel(got, c["out"]) < 3e-6  # fp32 on both sides: summation order only
    assert _rel(per_frame, c["out"]) > 1e-2  # the fixture tells the two networks apart


def test_window_oracle_leaves_torch_oracle_as_it_was():
    """The window network is a swap-in: outside window_groupnorm() the oracle's functions are its own, and the window
    GroupNorm is nn.GroupNorm on the [b, C, f, H, W] video tensor."""
    assert O.denoising_unet is WG._DENOISING_UNET and O.resnet_block is WG._RESNET_BLOCK
    with WG.window_groupnorm():
        assert O.denoising_unet is WG.denoising_unet
    assert O.denoising_unet is WG._DENOISING_UNET
    x = torch.randn(6, 64, 3, 5)
    sd = {"n.weight": torch.rand(64) + 0.5, "n.bias": torch.randn(64)}
    want = torch.nn.functional.group_norm(x.reshape(2, 3, 64, 3, 5).transpose(1, 2), 32, sd["n.weight"], sd["n.bias"],
                                          1e-5).transpose(1, 2).reshape(6, 64, 3, 5)
    assert torch.equal(WG.group_norm_frames(sd, "n", x, 32, 1e-5, 3), want)
    # one frame per sample: the per-frame GroupNorm
    assert torch.equal(WG.group_norm_frames(sd, "n", x, 32, 1e-5, 1), O._gn(sd, "n", x, 32, 1e-5))


# ------------------------------------------------------------------------------------------------
# C entry points: argument checks (they run before the device probe, so they are testable without a GPU)
# ------------------------------------------------------------------------------------------------
L_ERR_ARG = -1
_ENTRY = ("mimo_groupnorm_window", "mimo_groupnorm_window_partials", "mimo_groupnorm_window_apply")


def _params(**kw):
    buf = ctypes.create_string_buffer(64)  # any non-null address: nothing is dereferenced on these paths
    a = ctypes.addressof(buf)
    p = L.GroupNormWindowParams(x0=a, c0=320, gamma=a, beta=a, out=a, table=a, stats=a, samples=2, frames=4,
                                table_frames=4, hw=64, groups=32, eps=1e-5, silu=1, dtype=L.F16)
    p.table_bytes = L.load().mimo_groupnorm_window_table_bytes(ctypes.byref(p))
    for k, v in kw.items():
        setattr(p, k, v)
    return p, buf


def test_abi_and_table_size():
    lib = L.load()
    assert lib.mimo_abi_sizeof(8) == ctypes.sizeof(L.GroupNormWindowParams)
    assert lib.mimo_abi_sizeof(3) == ctypes.sizeof(L.GroupNormParams)  # the per-frame struct is unchanged
    one = ops.groupnorm_window_table_bytes(2, 1, 64 * 64, 320)
    assert one > 0 and one % 16 == 0
    # frame-major records: the table of G frame slices is G times a slice's, so the slices' tables concatenate
    for G in (2, 4, 8):
        assert ops.groupnorm_window_table_bytes(2, 24, 64 * 64, 320) == G * ops.groupnorm_window_table_bytes(2, 24 // G,
                                                                                                             64 * 64, 320)
    # one record: the K_g row plus one row per slab, padded to 16 bytes
    assert one == 2 * 4 * ((2 * 32 * (43 + 1) + 3) // 4 * 4)  # 64 x 64 at 320 channels: 43 slabs


@pytest.mark.parametrize("entry", _ENTRY)
def test_entry_points_refuse_bad_arguments(entry):
    lib = L.load()
    fn = getattr(lib, entry)
    assert fn(None, None) == L_ERR_ARG
    for field in ("x0", "table"):
        p, _keep = _params(**{field: None})
        assert fn(ctypes.byref(p), None) == L_ERR_ARG, field
        assert b"null" in lib.mimo_last_error()
    if entry != "mimo_groupnorm_window_partials":
        for field in ("gamma", "beta", "out", "stats"):
            p, _keep = _params(**{field: None})
            assert fn(ctypes.byref(p), None) == L_ERR_ARG, field
    for frames in (0, -3):
        p, _keep = _params(frames=frames)
        assert fn(ctypes.byref(p), None) == L_ERR_ARG
        assert b"bad sizes" in lib.mimo_last_error()
    for bad in (dict(samples=0), dict(hw=0), dict(groups=0), dict(groups=65), dict(c0=12), dict(c0=328),
                dict(dtype=5), dict(c0=8, groups=4)):
        p, _keep = _params(**bad)
        assert fn(ctypes.byref(p), None) == L_ERR_ARG, bad
    p, _keep = _params()
    p.table_bytes -= 16  # a partial table of the wrong size
    assert fn(ctypes.byref(p), None) == L_ERR_ARG
    assert b"table" in lib.mimo_last_error()


def test_apply_checks_the_window_table():
    lib = L.load()
    p, _keep = _params(table_frames=2)  # the window cannot hold fewer frames than the slice being normalised
    assert lib.mimo_groupnorm_window_apply(ctypes.byref(p), None) == L_ERR_ARG
    p, _keep = _params(table_frames=8)  # a table sized for 4 frames does not cover a window of 8
    assert lib.mimo_groupnorm_window_apply(ctypes.byref(p), None) == L_ERR_ARG
    assert b"table" in lib.mimo_last_error()
    p.table_bytes *= 2
    # valid arguments: on a machine without an H100 it is the device probe that refuses; on one, the kernel would run on
    # these host addresses
    if not torch.cuda.is_available():
        rc = lib.mimo_groupnorm_window_apply(ctypes.byref(p), None)
        assert rc != L_ERR_ARG


def test_table_bytes_refuses_bad_sizes():
    with pytest.raises(L.MimoError, match="bad sizes"):
        ops.groupnorm_window_table_bytes(2, 0, 64, 320)
    with pytest.raises(L.MimoError, match="channels"):
        ops.groupnorm_window_table_bytes(2, 4, 64, 12)


# ------------------------------------------------------------------------------------------------
# module surface
# ------------------------------------------------------------------------------------------------
_MK = dict(num_attention_heads=8, num_transformer_block=1, attention_block_types=["Temporal_Self", "Temporal_Self"],
           temporal_position_encoding=True, temporal_position_encoding_max_len=32, temporal_attention_dim_div=1)
_KW = dict(use_motion_module=True, motion_module_mid_block=True, motion_module_type="Vanilla", motion_module_kwargs=_MK)


@pytest.mark.parametrize("flag", [None, False, True])
def test_module_stores_the_flag(flag):
    from mimo_b200.host.modules import UNet2DConditionModel, UNet3DConditionModel
    kw = {} if flag is None else {"use_inflated_groupnorm": flag}
    m = UNet3DConditionModel(block_out_channels=(32, 64, 64, 64), cross_attention_dim=768, **kw, **_KW)
    want = bool(flag)  # the reference's default is False (unet_3d_edit_bkfill.py:71)
    assert m.use_inflated_groupnorm is want and m.config.use_inflated_groupnorm is want
    assert m._spec.inflated_groupnorm is want
    assert UNet2DConditionModel(block_out_channels=(32, 64, 64, 64))._spec.inflated_groupnorm is True
    # the packed weights do not depend on the flag: it does not key the weight cache
    assert repr(m._spec) == repr(E.UNetSpec(block_out_channels=(32, 64, 64, 64), cross_attention_dim=768))


def test_from_pretrained_2d_passes_the_flag(tmp_path):
    import json

    from mimo_b200.host.modules import UNet3DConditionModel
    widths = (32, 64, 64, 64)
    src = UNet3DConditionModel(block_out_channels=widths, cross_attention_dim=768, use_inflated_groupnorm=True, **_KW)
    sd = {k: v for k, v in src.state_dict().items() if "motion_modules" not in k}
    sd["conv_in.weight"] = sd["conv_in.weight"][:, :4].contiguous()
    (tmp_path / "unet").mkdir()
    (tmp_path / "unet" / "config.json").write_text(json.dumps(dict(block_out_channels=list(widths),
                                                                   cross_attention_dim=768)))
    torch.save(sd, tmp_path / "unet" / "diffusion_pytorch_model.bin")
    for flag in (False, True):
        m = UNet3DConditionModel.from_pretrained_2d(tmp_path, tmp_path / "none.ckpt", subfolder="unet",
                                                    unet_additional_kwargs=dict(_KW, use_inflated_groupnorm=flag))
        assert m.use_inflated_groupnorm is flag and m._spec.inflated_groupnorm is flag
    m = UNet3DConditionModel.from_pretrained_2d(tmp_path, tmp_path / "none.ckpt", subfolder="unet",
                                                unet_additional_kwargs=_KW)
    assert m.use_inflated_groupnorm is False


# ------------------------------------------------------------------------------------------------
# the calls of one ResnetBlock3D and of the output norm
# ------------------------------------------------------------------------------------------------
def _recording_engine(monkeypatch, inflated: bool, xchg=None):
    calls = []

    def rec(name):
        def f(*a, **kw):
            calls.append((name, a, kw))
            return torch.zeros(3, 8) if name != "groupnorm_window_partials" else kw.get("table")
        return f

    for name in ("groupnorm", "groupnorm_window", "groupnorm_window_partials", "groupnorm_window_apply", "conv3x3",
                 "gemm"):
        monkeypatch.setattr(ops, name, rec(name))
    monkeypatch.setattr(ops, "groupnorm_window_table_bytes", lambda b, f, hw, c, g: 64 * b * f)
    eng = E.UNetEngine.__new__(E.UNetEngine)
    eng.spec = E.UNetSpec(inflated_groupnorm=inflated)
    eng.xchg = xchg
    eng.w = {"r": {"n1": ("g1", "b1"), "c1": ("w1", "cb1"), "n2": ("g2", "b2"), "c2": ("w2", "cb2"),
                   "sc": ("ws", "sb")}}
    eng.temb_off = {"r": (0, 8)}
    return eng, calls


def _resnet_call(eng, window):
    x0, x1, tembs = torch.zeros(3, 8), torch.zeros(3, 8), torch.zeros(2, 8)
    eng._window_gn = window
    eng._resnet("r", x0, x1, tembs, 2 * 3, 4, 5, 3 * 4 * 5)  # 2 CFG branches x 3 frames of 4 x 5
    return x0, x1


def test_resnet_calls_with_the_flag_on_are_unchanged(monkeypatch):
    eng, calls = _recording_engine(monkeypatch, True)
    x0, x1 = _resnet_call(eng, not eng.spec.inflated_groupnorm)
    names = [c[0] for c in calls]
    assert names == ["groupnorm", "conv3x3", "groupnorm", "gemm", "conv3x3"]
    # exactly the arguments of the per-frame block: n = b * f images of hw pixels, eps = norm_eps, SiLU fused
    n1, n2 = calls[0], calls[2]
    assert n1[1][0] is x0 and n1[1][1:] == ("g1", "b1", 6, 20) and n1[2] == dict(groups=32, eps=1e-5, silu=True, x1=x1)
    assert n2[1][1:] == ("g2", "b2", 6, 20) and n2[2] == dict(groups=32, eps=1e-5, silu=True, x1=None)


def test_resnet_calls_in_window_mode(monkeypatch):
    eng, calls = _recording_engine(monkeypatch, False)
    x0, x1 = _resnet_call(eng, True)
    names = [c[0] for c in calls]
    assert names == ["groupnorm_window", "conv3x3", "groupnorm_window", "gemm", "conv3x3"]
    n1 = calls[0]
    # samples = the CFG branches this GPU evaluates, frames = the window's frames
    assert n1[1][0] is x0 and n1[1][1:] == ("g1", "b1", 2, 3, 20)
    assert n1[2] == dict(groups=32, eps=1e-5, silu=True, x1=x1)


def test_resnet_calls_frame_sharded(monkeypatch):
    pulls = []

    class Buf:
        def __init__(self):
            self.nbytes = 4096
            self.bytes = torch.zeros(4096, dtype=torch.uint8)

    xchg = SimpleNamespace(G=4, bufs={"A": Buf(), "B": Buf(), "N0": Buf(), "N1": Buf(), "N2": Buf()},
                           pull=lambda mode, name, dst, b, fl, hw, C: pulls.append((mode, name, tuple(dst.shape), b, fl,
                                                                                    hw, C)) or dst)
    eng, calls = _recording_engine(monkeypatch, False, xchg)
    x0, x1 = _resnet_call(eng, True)
    names = [c[0] for c in calls]
    assert names == ["groupnorm_window_partials", "groupnorm_window_apply", "conv3x3", "groupnorm_window_partials",
                     "groupnorm_window_apply", "gemm", "conv3x3"]
    need = 64 * 2 * 3  # the stand-in table size of this member's 3 frames
    # this member's table goes to its peer buffer; the group gathers the 4 tables byte for byte (16 bytes a row)
    assert calls[0][2]["table"].data_ptr() == xchg.bufs["N0"].bytes.data_ptr()
    assert pulls == [(2, "N0", (4 * need // 16, 8), 1, 1, need // 16, 8), (2, "N1", (4 * need // 16, 8), 1, 1, need // 16, 8)]
    ap = calls[1]
    assert ap[1][4:] == (2, 3, 12, 20)  # samples, this member's frames, the window's 12 frames, hw
    # without its peer buffer the engine refuses instead of guessing
    del xchg.bufs["N1"]
    with pytest.raises(L.MimoError, match="N1"):
        _resnet_call(eng, True)
