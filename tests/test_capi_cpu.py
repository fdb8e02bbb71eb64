"""CPU-side checks of the drop-in boundary: the library loads without a GPU, exports every symbol the header
declares, and every compute entry point refuses to run without an sm_90 device (no CPU fallback)."""
import ctypes
import re
from pathlib import Path

import pytest
import torch

from mimo_b200 import lib as L
from mimo_b200 import ops

ROOT = Path(__file__).resolve().parents[1]


def _header_functions():
    text = (ROOT / "include" / "mimo_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(mimo_[a-z0-9_]+)\s*\(", text)))


def test_header_symbols_are_exported_and_bound():
    names = _header_functions()
    assert len(names) >= 18
    cdll = ctypes.CDLL(str(L.LIB_PATH))
    for n in names:
        assert hasattr(cdll, n), f"{n} declared in include/mimo_b200.h but not exported by the library"
        assert n in L.SYMBOLS, f"{n} declared in the header but has no ctypes binding in mimo_b200/lib.py"
    for n in L.SYMBOLS:
        assert n in names, f"{n} is bound in lib.py but not declared in the header"


def test_version_and_struct_layout():
    lib = L.load()
    assert b"sm_90a" in lib.mimo_version()
    # the ctypes mirrors must match the C structs (pointer + int64 + float layout, natural alignment)
    for which, st in enumerate((L.Epilogue, L.GemmParams, L.Conv3x3Params, L.GroupNormParams, L.AttnParams)):
        assert lib.mimo_abi_sizeof(which) == ctypes.sizeof(st), st.__name__
    assert lib.mimo_abi_sizeof(99) == -1


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU behaviour")
def test_no_cpu_fallback():
    lib = L.load()
    assert lib.mimo_device_check(0) != 0
    assert b"no CPU fallback" in lib.mimo_last_error() or b"CUDA" in lib.mimo_last_error()
    a = torch.zeros(8, 8, dtype=torch.float16)
    with pytest.raises(L.MimoError):
        ops.gemm(a, a)
    from mimo_b200.host.modules import PoseGuider
    pg = PoseGuider(320, block_out_channels=(16, 32, 96, 256)).half()
    with pytest.raises(L.MimoError):
        pg(torch.zeros(1, 3, 1, 64, 64, dtype=torch.float16))


def test_geglu_granule_and_arg_validation():
    lib = L.load()
    assert lib.mimo_gemm_geglu_granule(2560) in (32, 64, 128)
    p = L.GemmParams()
    assert lib.mimo_gemm(ctypes.byref(p), None) == -1  # MIMO_ERR_ARG: null pointers
    assert b"null" in lib.mimo_last_error()


def test_integration_md_stub_binds_the_library():
    """The ctypes stub INTEGRATION.md shows a maintainer (section 2) is executed as written up to its first GPU call: the
    struct mirror must match the C struct, the workspace query must answer on the CPU, and a launch without a device
    must come back as an error string, not a crash."""
    import os
    text = (ROOT / "INTEGRATION.md").read_text()
    block = re.search(r"```python\n(# src/models/resnet\.py.*?)```", text, flags=re.S).group(1)
    ns = {}
    cwd = os.getcwd()
    os.chdir(ROOT)  # the stub loads "mimo_b200/libmimo_b200.so" relative to the checkout
    try:
        exec(compile(block, "INTEGRATION.md:stub", "exec"), ns)
    finally:
        os.chdir(cwd)
    lib, P = ns["_lib"], ns["GroupNormParams"]
    p = P(1 << 20, 320, None, 0, 1 << 20, 1 << 20, 1 << 20, None, 2, 4096, 32, 1e-5, 1, 0)
    need = lib.mimo_groupnorm_workspace_bytes(ctypes.byref(p))
    assert need > 0 and need % 8 == 0
    bad = P(1 << 20, 321, None, 0, 1 << 20, 1 << 20, 1 << 20, None, 2, 4096, 32, 1e-5, 1, 0)
    assert lib.mimo_groupnorm_workspace_bytes(ctypes.byref(bad)) < 0 and b"multiples of 8" in lib.mimo_last_error()
    if not torch.cuda.is_available():
        p.stats = 1 << 20
        assert lib.mimo_groupnorm(ctypes.byref(p), None) < 0
        assert b"CUDA" in lib.mimo_last_error() or b"fallback" in lib.mimo_last_error()


def test_argument_errors_of_every_compute_entry_point():
    """Error behaviour of the C ABI (include/mimo_b200.h: "return 0 on success, negative on error; mimo_last_error()
    gives the thread-local message"): every entry point validates its arguments BEFORE touching the device, so the
    refusals can be checked here without a GPU. Pointers are fake non-null addresses that are never dereferenced."""
    lib = L.load()
    PTR = 1 << 20
    err = lambda: lib.mimo_last_error().decode()
    hits = []

    def refused(rc, needle):
        """rc = MIMO_ERR_ARG with the message; a few checks sit behind the device probe and answer MIMO_ERR_DEVICE (-3) on
        a machine without a GPU - also a refusal, but not the one under test."""
        assert rc == -1 and needle in err() or (rc == -3 and not torch.cuda.is_available()), (rc, err())
        hits.append(rc)

    def gemm(**kw):
        p = L.GemmParams()
        p.a = p.w = p.out = PTR
        p.lda = p.ldw = p.ldo = 64
        p.M, p.N, p.K = 128, 64, 64
        for k, v in kw.items():
            setattr(p.ep if k in ("residual", "ld_res", "act", "rowvec") else p, k, v)
        return lib.mimo_gemm(ctypes.byref(p), None)

    refused(gemm(M=0), "empty problem")
    refused(gemm(K=60), "multiples of 8")
    refused(gemm(ldo=63), "multiples of 8")
    refused(gemm(residual=PTR, ld_res=7), "ld_res")
    refused(gemm(act=L.ACT_GEGLU, residual=PTR, ld_res=64), "GEGLU")
    refused(gemm(a1=PTR, K1=12, lda1=16), "K1/lda1")
    refused(gemm(act=L.ACT_GEGLU, N=72), "N % tile")  # GEGLU tile 64 does not divide N = 72

    def conv(fn=lib.mimo_conv3x3, **kw):
        p = L.Conv3x3Params()
        p.x0 = p.w = p.out = PTR
        p.c0, p.cout, p.ldo, p.n, p.h, p.w_ = 64, 64, 64, 1, 8, 8
        for k, v in kw.items():
            setattr(p.ep if k in ("residual", "ld_res", "act", "rowvec") else p, k, v)
        return fn(ctypes.byref(p), None)

    refused(conv(x0=None), "null pointer")
    refused(conv(h=0), "empty problem")
    refused(conv(c0=60), "multiples of 8")
    refused(conv(act=L.ACT_GEGLU), "GEGLU")
    refused(conv(lib.mimo_conv_up2x, residual=PTR, ld_res=64), "epilogue only")

    gn = L.GroupNormParams()
    gn.x0 = gn.gamma = gn.beta = gn.out = gn.stats = PTR
    gn.c0, gn.n, gn.hw, gn.groups = 320, 2, 64, 32
    assert lib.mimo_groupnorm_workspace_bytes(ctypes.byref(gn)) > 0
    gn.groups = 48
    refused(lib.mimo_groupnorm(ctypes.byref(gn), None), "divisible by groups")
    gn.groups, gn.c0 = 32, 64  # 2 channels per group: an 8-channel vector would straddle four groups
    refused(lib.mimo_groupnorm(ctypes.byref(gn), None), "channels per group")
    gn.c0, gn.out = 320, None
    refused(lib.mimo_groupnorm(ctypes.byref(gn), None), "null pointer")

    ln = lambda c, pe=None, rpf=1, frames=1: lib.mimo_layernorm(PTR, PTR, PTR, PTR, 16, c, 1e-5, pe, rpf, frames, 0, L.F16, None)
    refused(ln(324), "multiple of 8")
    refused(ln(4096), "<= 2048")
    refused(ln(320, pe=PTR, rpf=0), "pe args")

    at = L.AttnParams()
    at.q = at.k = at.v = at.out = PTR
    at.ld_qkv, at.ld_out, at.n, at.lq, at.heads, at.d = 960, 320, 1, 64, 8, 40
    at.d = 44
    refused(lib.mimo_attn_spatial(ctypes.byref(at), None), "d % 8")
    at.d, at.bank_k, at.bank_v, at.bank_index, at.lb, at.nb, at.ld_bank = 40, PTR, PTR, PTR, 64, 1, 644
    refused(lib.mimo_attn_spatial(ctypes.byref(at), None), "ld_bank")

    tp = L.AttnTemporalParams()
    tp.q = tp.k = tp.v = tp.out = PTR
    tp.ld_q = tp.ld_kv = tp.ld_out = 320
    tp.batch, tp.q_frames, tp.kv_frames, tp.frames_per_chunk, tp.hw, tp.heads, tp.d = 1, 40, 40, 40, 64, 8, 40
    refused(lib.mimo_attn_temporal(ctypes.byref(tp), None), "frames <= 32")  # PE table length (motion_module.py:264)

    ex = L.ExchangeParams()
    ex.dst = ex.ctl = PTR
    ex.G, ex.r, ex.b, ex.fl, ex.hw, ex.C = 9, 0, 1, 1, 64, 320
    refused(lib.mimo_exchange(ctypes.byref(ex), None), "group size")
    ex.G, ex.mode = 2, 3
    refused(lib.mimo_exchange(ctypes.byref(ex), None), "mode")
    ex.mode, ex.hw = 0, 63
    refused(lib.mimo_exchange(ctypes.byref(ex), None), "divisible by the group size")
    ex.hw = 64
    refused(lib.mimo_exchange(ctypes.byref(ex), None), "null peer pointer")

    refused(lib.mimo_im2col3x3(PTR, PTR, 1, 8, 8, 64, 3, 0, 1, 9 * 64, L.F16, None), "im2col")  # stride 3
    refused(lib.mimo_ncfhw_to_nhwc(PTR, PTR, 1, 9, 1, 8, 8, 8, 0, L.F16, None), "ncfhw_to_nhwc")  # cpad < c
    refused(lib.mimo_nhwc_to_ncfhw(PTR, PTR, 1, 4, 1, 8, 8, 3, 0, L.F16, None), "nhwc_to_ncfhw")  # ld < c
    refused(lib.mimo_add(PTR, PTR, PTR, 12, L.F16, None), "mimo_add")
    refused(lib.mimo_composite_frame(PTR, PTR, PTR, PTR, None, None, 0.0, PTR, 64, None), "come together")
    refused(lib.mimo_cfg_ddim_step(PTR, PTR, PTR, 0, PTR, 4 * 64, 3.5, 1.0, 0.0, 1.0, 0.0, L.F16, None),
            "frame_stride")  # a per-frame counter needs the frame stride
    refused(lib.mimo_peer_alloc(0, ctypes.byref(ctypes.c_void_p()), ctypes.create_string_buffer(64)), "peer_alloc")
    assert len(hits) >= 30 and sum(1 for rc in hits if rc == -1) >= len(hits) - 3, hits  # all but a few checks precede the probe
