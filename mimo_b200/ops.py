"""Tensor-level wrappers over the C ABI. PyTorch is only the owner of device memory and of the stream here:
every function enqueues exactly the kernels of one C entry point on torch's current CUDA stream.

Activations are channels-last 2-D views: [rows, C] with rows = (frame-sample, y, x).

Optional profiling (bench.py): when PROFILE is a list, every call is bracketed by CUDA events on the launching
stream and appends (name, flops, bytes, ev_start, ev_stop) with the call's ALGORITHMIC flops / bytes.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional

import torch

from . import lib as L

_launches = 0  # number of kernels launched through the C ABI (bench.py's gpu_launches)
PROFILE: Optional[List[tuple]] = None


def launches() -> int:
    return _launches


def add_launches(k: int) -> None:
    """Account for kernels launched by a CUDA-graph replay (the graph was recorded from these same wrappers)."""
    global _launches
    _launches += k


class _Call:
    """Counts kernel launches and, when profiling, brackets the call with events."""

    __slots__ = ("name", "k", "flops", "bytes", "e0")

    def __init__(self, name: str, kernels: int = 1, flops: float = 0.0, bytes_: float = 0.0):
        self.name, self.k, self.flops, self.bytes = name, kernels, flops, bytes_

    def __enter__(self):
        global _launches
        _launches += self.k
        if PROFILE is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e0.record()
        return self

    def __exit__(self, *exc):
        if PROFILE is not None:
            e1 = torch.cuda.Event(enable_timing=True)
            e1.record()
            PROFILE.append((self.name, self.flops, self.bytes, self.e0, e1))
        return False


def _stream() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _dt(t: torch.Tensor) -> int:
    if t.dtype == torch.float16:
        return L.F16
    if t.dtype == torch.bfloat16:
        return L.BF16
    raise L.MimoError(f"unsupported dtype {t.dtype}: engine tensors are fp16 or bf16")


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    if t is None:
        return None
    if not t.is_cuda:
        raise L.MimoError("mimo_b200 ops need CUDA tensors (there is no CPU fallback)")
    return t.data_ptr()


_WORKSPACE: dict = {}
WORKSPACE_BYTES = 96 << 20


def _workspace(device: torch.device) -> torch.Tensor:
    """One persistent split-K scratch buffer per device (stable address: captured CUDA graphs keep pointing at it)."""
    key = (device.type, device.index)
    ws = _WORKSPACE.get(key)
    if ws is None:
        ws = torch.empty(WORKSPACE_BYTES, dtype=torch.uint8, device=device)
        _WORKSPACE[key] = ws
    return ws


def _epilogue(bias=None, rowvec=None, rows_per_group=1, residual=None, scale=1.0, act=L.ACT_NONE) -> L.Epilogue:
    ep = L.Epilogue()
    ep.bias = _ptr(bias)
    ep.rowvec = _ptr(rowvec)
    ep.rows_per_group = int(rows_per_group)
    ep.ld_rowvec = rowvec.stride(0) if rowvec is not None else 0
    ep.residual = _ptr(residual)
    ep.ld_res = residual.stride(0) if residual is not None else 0
    ep.scale = float(scale)
    ep.act = int(act)
    return ep


def gemm(a: torch.Tensor, w: torch.Tensor, out: Optional[torch.Tensor] = None, *, a1: Optional[torch.Tensor] = None,
         bias=None, rowvec=None, rows_per_group=1, residual=None, scale=1.0, act=L.ACT_NONE) -> torch.Tensor:
    """out[M, N(or N/2 for GEGLU)] = epilogue([a | a1][M, K + K1] @ w[N, K + K1]^T)."""
    K1 = a1.shape[1] if a1 is not None else 0
    assert a.dim() == 2 and w.dim() == 2 and a.shape[1] + K1 == w.shape[1]
    assert a.stride(1) == 1 and w.stride(1) == 1
    M, K = a.shape
    N = w.shape[0]
    n_out = N // 2 if act == L.ACT_GEGLU else N
    if out is None:
        out = torch.empty((M, n_out), dtype=a.dtype, device=a.device)
    assert out.shape == (M, n_out) and out.stride(1) == 1
    p = L.GemmParams()
    p.a, p.lda = _ptr(a), a.stride(0)
    p.a1, p.lda1, p.K1 = (_ptr(a1), a1.stride(0), K1) if a1 is not None else (None, 0, 0)
    p.w, p.ldw = _ptr(w), w.stride(0)
    p.out, p.ldo = _ptr(out), out.stride(0)
    p.M, p.N, p.K = M, N, K
    p.dtype = _dt(a)
    p.ep = _epilogue(bias, rowvec, rows_per_group, residual, scale, act)
    ws = _workspace(a.device)
    p.workspace, p.workspace_bytes = ws.data_ptr(), ws.numel()
    kt = K + K1
    with _Call("gemm", 1, 2.0 * M * N * kt, 2.0 * (M * kt + N * kt + M * n_out + (M * N if residual is not None else 0))):
        L.check(L.load().mimo_gemm(C.byref(p), _stream()), "mimo_gemm")
    return out


def gemm_e4m3(a: torch.Tensor, a_scale: torch.Tensor, w: torch.Tensor, w_scale: torch.Tensor, dtype: torch.dtype,
              out: Optional[torch.Tensor] = None, *, bias=None, rowvec=None, rows_per_group=1, residual=None, scale=1.0,
              act=L.ACT_NONE) -> torch.Tensor:
    """out[M, N(or N/2 for GEGLU)] = epilogue((a[M, K] @ w[N, K]^T) * a_scale[:, None] * w_scale[None, :]): a and w are
    torch.float8_e4m3fn, the scales fp32, out / bias / residual `dtype`."""
    assert a.dtype == torch.float8_e4m3fn and w.dtype == torch.float8_e4m3fn
    assert a.dim() == 2 and w.dim() == 2 and a.shape[1] == w.shape[1] and a.stride(1) == 1 and w.stride(1) == 1
    assert a_scale.dtype == torch.float32 and w_scale.dtype == torch.float32
    assert a_scale.shape == (a.shape[0],) and w_scale.shape == (w.shape[0],)
    M, K = a.shape
    N = w.shape[0]
    n_out = N // 2 if act == L.ACT_GEGLU else N
    if out is None:
        out = torch.empty((M, n_out), dtype=dtype, device=a.device)
    assert out.shape == (M, n_out) and out.stride(1) == 1 and out.dtype == dtype
    p = L.GemmE4m3Params()
    p.a, p.lda, p.a_scale = _ptr(a), a.stride(0), _ptr(a_scale)
    p.w, p.ldw, p.w_scale = _ptr(w), w.stride(0), _ptr(w_scale)
    p.out, p.ldo = _ptr(out), out.stride(0)
    p.M, p.N, p.K = M, N, K
    p.dtype = _dt(out)
    p.ep = _epilogue(bias, rowvec, rows_per_group, residual, scale, act)
    with _Call("gemm_e4m3", 1, 2.0 * M * N * K, M * K + N * K + 4.0 * (M + N) + 2.0 * (M * n_out + (M * N if residual is not None else 0))):
        L.check(L.load().mimo_gemm_e4m3(C.byref(p), _stream()), "mimo_gemm_e4m3")
    return out


E4M3_BLOCK = 128  # K elements per activation scale of gemm_e4m3_blockscaled (one GEGLU tile's output columns)


def gemm_e4m3_geglu_e4m3(a: torch.Tensor, a_scale: torch.Tensor, w: torch.Tensor, w_scale: torch.Tensor,
                         dtype: torch.dtype, *, bias=None):
    """gemm_e4m3(..., act=GEGLU) with an e4m3 output: returns (q [M, N/2] float8_e4m3fn, scale [N/2 / 128, M] fp32),
    q[:, 128 b:128 b + 128] * scale[b][:, None] ~ the fp32 GEGLU values, quantized per row and 128-column block by
    quantize_e4m3_blocks' rule (include/mimo_b200.h). w is the GEGLU-packed e4m3 weight (N % 256 == 0), bias `dtype`."""
    assert a.dtype == torch.float8_e4m3fn and w.dtype == torch.float8_e4m3fn
    assert a.dim() == 2 and w.dim() == 2 and a.shape[1] == w.shape[1] and a.stride(1) == 1 and w.stride(1) == 1
    assert a_scale.dtype == torch.float32 and w_scale.dtype == torch.float32
    assert a_scale.shape == (a.shape[0],) and w_scale.shape == (w.shape[0],)
    M, K = a.shape
    N = w.shape[0]
    lds = (M + 3) // 4 * 4
    out = torch.empty((M, N // 2), dtype=torch.float8_e4m3fn, device=a.device)
    sc = torch.empty((N // 2 // E4M3_BLOCK, lds), dtype=torch.float32, device=a.device)
    p = L.GemmE4m3GegluE4m3Params()
    p.a, p.lda, p.a_scale = _ptr(a), a.stride(0), _ptr(a_scale)
    p.w, p.ldw, p.w_scale = _ptr(w), w.stride(0), _ptr(w_scale)
    p.bias = _ptr(bias) if bias is not None else None
    if bias is not None:
        assert bias.dtype == dtype and bias.shape == (N,)
    p.out, p.ldo = _ptr(out), out.stride(0)
    p.out_scale, p.ld_scale = _ptr(sc), lds
    p.M, p.N, p.K = M, N, K
    p.dtype = L.BF16 if dtype == torch.bfloat16 else L.F16
    with _Call("gemm_e4m3_geglu_e4m3", 1, 2.0 * M * N * K, M * K + N * K + 4.0 * (M + N) + M * N // 2 + 4.0 * M * N / 256):
        L.check(L.load().mimo_gemm_e4m3_geglu_e4m3(C.byref(p), _stream()), "mimo_gemm_e4m3_geglu_e4m3")
    return out, sc[:, :M]


def gemm_e4m3_blockscaled(a: torch.Tensor, a_scale: torch.Tensor, w: torch.Tensor, w_scale: torch.Tensor,
                          dtype: torch.dtype, out: Optional[torch.Tensor] = None, *, bias=None, rowvec=None,
                          rows_per_group=1, residual=None, scale=1.0, act=L.ACT_NONE) -> torch.Tensor:
    """out[M, N] = epilogue((sum_b (a_b @ w_b^T) * a_scale[b][:, None]) * w_scale[None, :]) over the 128-wide K blocks b:
    a [M, K] float8_e4m3fn with a_scale [K / 128, M] fp32 (gemm_e4m3_geglu_e4m3's output), w [N, K] float8_e4m3fn with one
    fp32 scale per row (pack_e4m3_weight); out / bias / residual `dtype`."""
    assert a.dtype == torch.float8_e4m3fn and w.dtype == torch.float8_e4m3fn
    assert a.dim() == 2 and w.dim() == 2 and a.shape[1] == w.shape[1] and a.stride(1) == 1 and w.stride(1) == 1
    assert a_scale.dtype == torch.float32 and w_scale.dtype == torch.float32
    M, K = a.shape
    N = w.shape[0]
    assert a_scale.shape == (K // E4M3_BLOCK, M) and w_scale.shape == (N,)
    if a_scale.stride(1) != 1 or a_scale.stride(0) % 4 or a_scale.data_ptr() % 16:  # rows of whole 16-byte groups
        lds = (M + 3) // 4 * 4
        a_scale = torch.zeros((K // E4M3_BLOCK, lds), dtype=torch.float32, device=a.device)[:, :M].copy_(a_scale)
    if out is None:
        out = torch.empty((M, N), dtype=dtype, device=a.device)
    assert out.shape == (M, N) and out.stride(1) == 1 and out.dtype == dtype
    p = L.GemmE4m3BlockscaledParams()
    p.a, p.lda = _ptr(a), a.stride(0)
    p.a_scale, p.ld_scale = _ptr(a_scale), a_scale.stride(0) if a_scale.shape[0] > 1 else (M + 3) // 4 * 4
    p.w, p.ldw, p.w_scale = _ptr(w), w.stride(0), _ptr(w_scale)
    p.out, p.ldo = _ptr(out), out.stride(0)
    p.M, p.N, p.K = M, N, K
    p.dtype = _dt(out)
    p.ep = _epilogue(bias, rowvec, rows_per_group, residual, scale, act)
    with _Call("gemm_e4m3_blockscaled", 1, 2.0 * M * N * K,
               M * K + N * K + 4.0 * (M * K / E4M3_BLOCK + N) + 2.0 * (M * N + (M * N if residual is not None else 0))):
        L.check(L.load().mimo_gemm_e4m3_blockscaled(C.byref(p), _stream()), "mimo_gemm_e4m3_blockscaled")
    return out


def conv3x3(x0: torch.Tensor, w: torch.Tensor, n: int, h: int, wd: int, out: Optional[torch.Tensor] = None, *,
            x1: Optional[torch.Tensor] = None, bias=None, rowvec=None, rows_per_group: Optional[int] = None,
            residual=None, scale=1.0, act=L.ACT_NONE) -> torch.Tensor:
    """3x3/s1/p1 conv over channels-last x0 [n*h*wd, c0] (+ x1 [n*h*wd, c1]); w packed [cout, 9*(c0+c1)]."""
    c0 = x0.shape[1]
    c1 = x1.shape[1] if x1 is not None else 0
    cout = w.shape[0]
    assert x0.is_contiguous() and (x1 is None or x1.is_contiguous()) and w.is_contiguous()
    assert w.shape[1] == 9 * (c0 + c1) and x0.shape[0] == n * h * wd
    if out is None:
        out = torch.empty((n * h * wd, cout), dtype=x0.dtype, device=x0.device)
    p = L.Conv3x3Params()
    p.x0, p.c0 = _ptr(x0), c0
    p.x1, p.c1 = _ptr(x1), c1
    p.w = _ptr(w)
    p.out, p.ldo = _ptr(out), out.stride(0)
    p.n, p.h, p.w_, p.cout = n, h, wd, cout
    p.dtype = _dt(x0)
    p.ep = _epilogue(bias, rowvec, rows_per_group or h * wd, residual, scale, act)
    ws = _workspace(x0.device)
    p.workspace, p.workspace_bytes = ws.data_ptr(), ws.numel()
    M, cin = n * h * wd, c0 + c1
    with _Call("conv3x3", 1, 2.0 * M * cout * 9 * cin,
               2.0 * (M * cin + 9 * cin * cout + M * cout + (M * cout if residual is not None else 0))):
        L.check(L.load().mimo_conv3x3(C.byref(p), _stream()), "mimo_conv3x3")
    return out


def conv3x3_e4m3(x: torch.Tensor, x_scale: torch.Tensor, w: torch.Tensor, w_scale: torch.Tensor, n: int, h: int,
                 wd: int, dtype: torch.dtype, out: Optional[torch.Tensor] = None, *, bias=None, rowvec=None,
                 rows_per_group: Optional[int] = None, residual=None, scale=1.0, act=L.ACT_NONE) -> torch.Tensor:
    """conv3x3() from e4m3 operands: x [n*h*wd, c] float8_e4m3fn with one fp32 scale per image (groupnorm_e4m3's
    output), w [cout, 9*c] float8_e4m3fn with one fp32 scale per output channel (pack_e4m3_weight of the conv3x3 pack);
    out / bias / rowvec / residual `dtype`."""
    assert x.dtype == torch.float8_e4m3fn and w.dtype == torch.float8_e4m3fn
    assert x_scale.dtype == torch.float32 and w_scale.dtype == torch.float32
    c, cout = x.shape[1], w.shape[0]
    assert x.is_contiguous() and w.is_contiguous() and w.shape[1] == 9 * c and x.shape[0] == n * h * wd
    assert x_scale.shape == (n,) and w_scale.shape == (cout,)
    if out is None:
        out = torch.empty((n * h * wd, cout), dtype=dtype, device=x.device)
    assert out.dtype == dtype and out.stride(1) == 1
    p = L.Conv3x3E4m3Params()
    p.x, p.x_scale, p.c_in = _ptr(x), _ptr(x_scale), c
    p.w, p.w_scale = _ptr(w), _ptr(w_scale)
    p.out, p.ldo = _ptr(out), out.stride(0)
    p.n, p.h, p.w_, p.cout = n, h, wd, cout
    p.dtype = _dt(out)
    p.ep = _epilogue(bias, rowvec, rows_per_group or h * wd, residual, scale, act)
    M = n * h * wd
    with _Call("conv3x3_e4m3", 1, 2.0 * M * cout * 9 * c,
               M * c + 9 * c * cout + 4.0 * (n + cout) + 2.0 * (M * cout + (M * cout if residual is not None else 0))):
        L.check(L.load().mimo_conv3x3_e4m3(C.byref(p), _stream()), "mimo_conv3x3_e4m3")
    return out


def conv_up2x(x: torch.Tensor, w4: torch.Tensor, n: int, h: int, wd: int, *, bias=None, scale=1.0, act=L.ACT_NONE,
              out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """nearest-x2 upsample + 3x3 conv of channels-last x [n*h*wd, c] -> [n*2h*2wd, cout]; w4 from pack_conv_up2x_weight."""
    c = x.shape[1]
    cout = w4.shape[1]
    assert x.is_contiguous() and w4.is_contiguous() and w4.shape == (4, cout, 4 * c) and x.shape[0] == n * h * wd
    if out is None:
        out = torch.empty((n * 4 * h * wd, cout), dtype=x.dtype, device=x.device)
    p = L.Conv3x3Params()
    p.x0, p.c0 = _ptr(x), c
    p.x1, p.c1 = None, 0
    p.w = _ptr(w4)
    p.out, p.ldo = _ptr(out), out.stride(0)
    p.n, p.h, p.w_, p.cout = n, h, wd, cout
    p.dtype = _dt(x)
    p.ep = _epilogue(bias, None, 1, None, scale, act)
    M = n * h * wd
    # algorithmic work of the REFERENCE op (9 taps on the 4x image); the kernel executes 4/9 of it
    with _Call("conv3x3", 4, 2.0 * 4 * M * cout * 9 * c, 2.0 * (M * c + 16 * c * cout + 4 * M * cout)):
        L.check(L.load().mimo_conv_up2x(C.byref(p), _stream()), "mimo_conv_up2x")
    return out


def im2col3x3(x: torch.Tensor, n: int, h: int, wd: int, *, stride=1, upshift=0, pad_lo=1,
              out: Optional[torch.Tensor] = None) -> torch.Tensor:
    c = x.shape[1]
    uh, uw = h << upshift, wd << upshift
    oh = (uh + 2 * pad_lo - 3 + (0 if pad_lo else 1)) // stride + 1
    ow = (uw + 2 * pad_lo - 3 + (0 if pad_lo else 1)) // stride + 1
    if out is None:
        out = torch.empty((n * oh * ow, 9 * c), dtype=x.dtype, device=x.device)
    with _Call("im2col", 1, 0.0, 2.0 * (x.numel() + out.numel())):
        L.check(L.load().mimo_im2col3x3(_ptr(x), _ptr(out), n, h, wd, c, stride, upshift, pad_lo, out.stride(0),
                                        _dt(x), _stream()), "mimo_im2col3x3")
    return out


def groupnorm(x0: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, n: int, hw: int, *, groups=32,
              eps=1e-5, silu=False, x1: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
              stats: Optional[torch.Tensor] = None) -> torch.Tensor:
    c0 = x0.shape[1]
    c1 = x1.shape[1] if x1 is not None else 0
    if out is None:
        out = torch.empty((n * hw, c0 + c1), dtype=x0.dtype, device=x0.device)
    p = L.GroupNormParams()
    p.x0, p.c0 = _ptr(x0), c0
    p.x1, p.c1 = _ptr(x1), c1
    p.gamma, p.beta = _ptr(gamma), _ptr(beta)
    p.out = _ptr(out)
    p.n, p.hw, p.groups = n, hw, groups
    p.eps = float(eps)
    p.silu = int(bool(silu))
    p.dtype = _dt(x0)
    need = L.load().mimo_groupnorm_workspace_bytes(C.byref(p))
    if need < 0:
        L.check(int(need), "mimo_groupnorm_workspace_bytes")
    if stats is None:
        stats = torch.empty(((need + 3) // 4,), dtype=torch.float32, device=x0.device)
    assert x0.is_contiguous() and out.is_contiguous() and stats.numel() * 4 >= need
    p.stats = _ptr(stats)
    with _Call("groupnorm", 2, 0.0, 2.0 * 2 * out.numel()):  # algorithmic: one read + one write
        L.check(L.load().mimo_groupnorm(C.byref(p), _stream()), "mimo_groupnorm")
    return out


def _gnw_params(x0, samples, frames, hw, groups, *, x1=None, gamma=None, beta=None, out=None, table=None, stats=None,
                table_frames=0, eps=1e-5, silu=False, dtype=None) -> L.GroupNormWindowParams:
    p = L.GroupNormWindowParams()
    p.x0, p.c0 = _ptr(x0), x0.shape[1]
    p.x1, p.c1 = _ptr(x1), (x1.shape[1] if x1 is not None else 0)
    p.gamma, p.beta, p.out, p.stats = _ptr(gamma), _ptr(beta), _ptr(out), _ptr(stats)
    p.table, p.table_bytes = _ptr(table), (table.numel() * table.element_size() if table is not None else 0)
    p.samples, p.frames, p.table_frames, p.hw, p.groups = int(samples), int(frames), int(table_frames), int(hw), int(groups)
    p.eps, p.silu, p.dtype = float(eps), int(bool(silu)), _dt(x0) if dtype is None else dtype
    return p


def groupnorm_window_table_bytes(samples: int, frames: int, hw: int, channels: int, groups: int = 32) -> int:
    """Bytes of the window-mode partial table of `frames` frames of `samples` samples (no GPU needed)."""
    p = L.GroupNormWindowParams(c0=int(channels), samples=int(samples), frames=int(frames), hw=int(hw),
                                groups=int(groups), dtype=L.F16)
    need = L.load().mimo_groupnorm_window_table_bytes(C.byref(p))
    if need < 0:
        L.check(int(need), "mimo_groupnorm_window_table_bytes")
    return int(need)


def _gnw_table(table: Optional[torch.Tensor], need: int, device) -> torch.Tensor:
    if table is None:
        return torch.empty((need // 4,), dtype=torch.float32, device=device)
    assert table.dtype == torch.float32 and table.is_contiguous() and table.numel() * 4 >= need
    return table


def groupnorm_window(x0: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, samples: int, frames: int, hw: int, *,
                     groups=32, eps=1e-5, silu=False, x1: Optional[torch.Tensor] = None,
                     out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """torch.nn.GroupNorm(+SiLU) over [samples, C, frames, h, w] on channels-last x0 [samples*frames*hw, c0] (+ x1):
    one set of statistics per sample and group over all `frames` frames."""
    c = x0.shape[1] + (x1.shape[1] if x1 is not None else 0)
    assert x0.is_contiguous() and (x1 is None or x1.is_contiguous()) and x0.shape[0] == samples * frames * hw
    if out is None:
        out = torch.empty((samples * frames * hw, c), dtype=x0.dtype, device=x0.device)
    assert out.is_contiguous()
    table = _gnw_table(None, groupnorm_window_table_bytes(samples, frames, hw, c, groups), x0.device)
    stats = torch.empty((samples * groups * 2,), dtype=torch.float32, device=x0.device)
    p = _gnw_params(x0, samples, frames, hw, groups, x1=x1, gamma=gamma, beta=beta, out=out, table=table, stats=stats,
                    table_frames=frames, eps=eps, silu=silu)
    with _Call("groupnorm", 3, 0.0, 2.0 * 2 * out.numel()):
        L.check(L.load().mimo_groupnorm_window(C.byref(p), _stream()), "mimo_groupnorm_window")
    return out


def groupnorm_window_partials(x0: torch.Tensor, samples: int, frames: int, hw: int, *, groups=32,
                              x1: Optional[torch.Tensor] = None, table: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The window-mode partial table of x0's `frames` frames (fp32, frame-major: tables of consecutive frame slices
    concatenate into the whole window's). `table`: an fp32 buffer to write it to (e.g. a peer-memory source)."""
    c = x0.shape[1] + (x1.shape[1] if x1 is not None else 0)
    assert x0.is_contiguous() and (x1 is None or x1.is_contiguous()) and x0.shape[0] == samples * frames * hw
    table = _gnw_table(table, groupnorm_window_table_bytes(samples, frames, hw, c, groups), x0.device)
    p = _gnw_params(x0, samples, frames, hw, groups, x1=x1, table=table)
    with _Call("groupnorm", 1, 0.0, 2.0 * x0.shape[0] * c):
        L.check(L.load().mimo_groupnorm_window_partials(C.byref(p), _stream()), "mimo_groupnorm_window_partials")
    return table


def groupnorm_window_apply(x0: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, table: torch.Tensor, samples: int,
                           frames: int, table_frames: int, hw: int, *, groups=32, eps=1e-5, silu=False,
                           x1: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Normalise x0's `frames` frames (+ affine, SiLU) with the statistics of a partial table that covers all
    `table_frames` frames of the window."""
    c = x0.shape[1] + (x1.shape[1] if x1 is not None else 0)
    assert x0.is_contiguous() and (x1 is None or x1.is_contiguous()) and x0.shape[0] == samples * frames * hw
    if out is None:
        out = torch.empty((samples * frames * hw, c), dtype=x0.dtype, device=x0.device)
    assert out.is_contiguous()
    table = _gnw_table(table, groupnorm_window_table_bytes(samples, table_frames, hw, c, groups), x0.device)
    stats = torch.empty((samples * groups * 2,), dtype=torch.float32, device=x0.device)
    p = _gnw_params(x0, samples, frames, hw, groups, x1=x1, gamma=gamma, beta=beta, out=out, table=table, stats=stats,
                    table_frames=table_frames, eps=eps, silu=silu)
    with _Call("groupnorm", 2, 0.0, 2.0 * 2 * out.numel()):
        L.check(L.load().mimo_groupnorm_window_apply(C.byref(p), _stream()), "mimo_groupnorm_window_apply")
    return out


def _gn8(mode: int, x0, samples, frames, hw, groups, *, x1=None, gamma=None, beta=None, eps=1e-5, table=None,
         table_frames=0, work=None, out=None, scale=None):
    """one mimo_groupnorm_e4m3 call; returns `work` (allocated here when None)"""
    c = x0.shape[1] + (x1.shape[1] if x1 is not None else 0)
    assert x0.is_contiguous() and (x1 is None or x1.is_contiguous()) and x0.shape[0] == samples * frames * hw
    p = L.GroupNormE4m3Params(mode=int(mode), samples=int(samples), frames=int(frames), table_frames=int(table_frames),
                              hw=int(hw), groups=int(groups), eps=float(eps), dtype=_dt(x0))
    p.x0, p.c0 = _ptr(x0), x0.shape[1]
    p.x1, p.c1 = _ptr(x1), (x1.shape[1] if x1 is not None else 0)
    p.gamma, p.beta, p.out, p.scale = _ptr(gamma), _ptr(beta), _ptr(out), _ptr(scale)
    need = L.load().mimo_groupnorm_e4m3_workspace_bytes(C.byref(p))
    if need < 0:
        L.check(int(need), "mimo_groupnorm_e4m3_workspace_bytes")
    if work is None:
        work = torch.empty(((need + 3) // 4,), dtype=torch.float32, device=x0.device)
    assert work.dtype == torch.float32 and work.is_contiguous() and work.numel() * 4 >= need
    p.work, p.work_bytes = _ptr(work), work.numel() * 4
    p.table, p.table_bytes = _ptr(table), (table.numel() * table.element_size() if table is not None else 0)
    rows = samples * frames * hw
    kernels = {L.GN_E4M3_FRAME: 2, L.GN_E4M3_WINDOW: 3, L.GN_E4M3_WINDOW_PARTIALS: 1, L.GN_E4M3_WINDOW_APPLY: 2}[mode]
    moved = 2.0 * rows * c + (rows * c + 4.0 * samples * frames if mode != L.GN_E4M3_WINDOW_PARTIALS else 0)
    with _Call("groupnorm_e4m3", kernels, 0.0, moved):
        L.check(L.load().mimo_groupnorm_e4m3(C.byref(p), _stream()), "mimo_groupnorm_e4m3")
    return work


def _gn8_out(x0, x1, images, hw):
    c = x0.shape[1] + (x1.shape[1] if x1 is not None else 0)
    return (torch.empty((images * hw, c), dtype=torch.float8_e4m3fn, device=x0.device),
            torch.empty((images,), dtype=torch.float32, device=x0.device))


def groupnorm_e4m3(x0: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, n: int, hw: int, *, groups=32, eps=1e-5,
                   x1: Optional[torch.Tensor] = None, window_frames: Optional[int] = None):
    """SiLU(GroupNorm) of channels-last x0 (+ x1) quantized per image for conv3x3_e4m3: returns (q [n*hw, C]
    float8_e4m3fn, scale [n] fp32), q * scale ~ SiLU(GroupNorm(x)) (include/mimo_b200.h and e4m3_image_scales give
    the rule). Statistics per image, or with `window_frames` per sample over that many consecutive images."""
    q, sc = _gn8_out(x0, x1, n, hw)
    if window_frames is None:
        _gn8(L.GN_E4M3_FRAME, x0, n, 1, hw, groups, x1=x1, gamma=gamma, beta=beta, eps=eps, out=q, scale=sc)
    else:
        f = int(window_frames)
        c = q.shape[1]
        table = _gnw_table(None, groupnorm_window_table_bytes(n // f, f, hw, c, groups), x0.device)
        _gn8(L.GN_E4M3_WINDOW, x0, n // f, f, hw, groups, x1=x1, gamma=gamma, beta=beta, eps=eps, table=table,
             table_frames=f, out=q, scale=sc)
    return q, sc


def groupnorm_e4m3_partials(x0: torch.Tensor, samples: int, frames: int, hw: int, *, groups=32,
                            x1: Optional[torch.Tensor] = None, table: Optional[torch.Tensor] = None):
    """groupnorm_window_partials() for the e4m3 output: the window table of x0's frames (same bytes as the 16-bit
    call) and the per-frame min / max that groupnorm_e4m3_apply reads. Returns (table, work)."""
    c = x0.shape[1] + (x1.shape[1] if x1 is not None else 0)
    table = _gnw_table(table, groupnorm_window_table_bytes(samples, frames, hw, c, groups), x0.device)
    work = _gn8(L.GN_E4M3_WINDOW_PARTIALS, x0, samples, frames, hw, groups, x1=x1, table=table)
    return table, work


def groupnorm_e4m3_apply(x0: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, table: torch.Tensor,
                         work: torch.Tensor, samples: int, frames: int, table_frames: int, hw: int, *, groups=32,
                         eps=1e-5, x1: Optional[torch.Tensor] = None):
    """groupnorm_window_apply() for the e4m3 output, with the `work` of groupnorm_e4m3_partials on the same frames:
    returns (q, scale) as groupnorm_e4m3."""
    q, sc = _gn8_out(x0, x1, samples * frames, hw)
    _gn8(L.GN_E4M3_WINDOW_APPLY, x0, samples, frames, hw, groups, x1=x1, gamma=gamma, beta=beta, eps=eps, table=table,
         table_frames=table_frames, work=work, out=q, scale=sc)
    return q, sc


def layernorm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, *, eps=1e-5, pe: Optional[torch.Tensor] = None,
              rows_per_frame=1, frames=1, pe_frame_offset=0, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    assert x.is_contiguous() and x.dim() == 2
    if out is None:
        out = torch.empty_like(x)
    with _Call("layernorm", 1, 0.0, 2.0 * 2 * x.numel()):
        L.check(L.load().mimo_layernorm(_ptr(x), _ptr(gamma), _ptr(beta), _ptr(out), x.shape[0], x.shape[1], float(eps),
                                        _ptr(pe), int(rows_per_frame), int(frames), int(pe_frame_offset), _dt(x),
                                        _stream()), "mimo_layernorm")
    return out


def layernorm_e4m3(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, *, eps=1e-5,
                   pe: Optional[torch.Tensor] = None, rows_per_frame=1, frames=1, pe_frame_offset=0):
    """layernorm() quantized per row for gemm_e4m3: returns (q [rows, C] float8_e4m3fn, scale [rows] fp32), with
    q * scale ~ the fp32 LN(+PE) output (include/mimo_b200.h gives the exact rule)."""
    assert x.is_contiguous() and x.dim() == 2
    out = torch.empty(x.shape, dtype=torch.float8_e4m3fn, device=x.device)
    sc = torch.empty((x.shape[0],), dtype=torch.float32, device=x.device)
    with _Call("layernorm_e4m3", 1, 0.0, 2.0 * x.numel() + x.numel() + 4.0 * x.shape[0]):
        L.check(L.load().mimo_layernorm_e4m3(_ptr(x), _ptr(gamma), _ptr(beta), _ptr(out), _ptr(sc), x.shape[0], x.shape[1],
                                             float(eps), _ptr(pe), int(rows_per_frame), int(frames), int(pe_frame_offset),
                                             _dt(x), _stream()), "mimo_layernorm_e4m3")
    return out, sc


def attn_spatial(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, n: int, lq: int, heads: int, *,
                 bank_k: Optional[torch.Tensor] = None, bank_v: Optional[torch.Tensor] = None,
                 bank_index: Optional[torch.Tensor] = None, scale: Optional[float] = None,
                 out: Optional[torch.Tensor] = None, n_bank_frames: Optional[int] = None) -> torch.Tensor:
    """q/k/v: [n*lq, C] column slices (views) of one fused buffer; bank_k/v: [nb, lb, C]; bank_index int32 [n].
    n_bank_frames (profiling only): how many of the n frames attend to the bank."""
    Cdim = q.shape[1]
    d = Cdim // heads
    assert q.stride(0) == k.stride(0) == v.stride(0) and q.stride(1) == 1
    if out is None:
        out = torch.empty((n * lq, Cdim), dtype=q.dtype, device=q.device)
    p = L.AttnParams()
    p.q, p.k, p.v, p.ld_qkv = _ptr(q), _ptr(k), _ptr(v), q.stride(0)
    lb = 0
    if bank_k is not None:
        assert bank_v is not None and bank_index is not None and bank_index.dtype == torch.int32
        assert bank_k.stride(0) == bank_v.stride(0)
        nb = 1 if bank_k.dim() == 2 else bank_k.shape[0]
        p.bank_k, p.bank_v, p.ld_bank = _ptr(bank_k), _ptr(bank_v), bank_k.stride(-2)
        lb = bank_k.shape[-2]
        p.lb = lb
        p.nb = nb
        p.bank_index = _ptr(bank_index)
    else:
        p.bank_k = p.bank_v = p.bank_index = None
        p.ld_bank, p.lb, p.nb = 0, 0, 0
    p.out, p.ld_out = _ptr(out), out.stride(0)
    p.n, p.lq, p.heads, p.d = n, lq, heads, d
    p.scale = float(scale if scale is not None else d ** -0.5)
    p.dtype = _dt(q)
    nbf = (n if n_bank_frames is None else n_bank_frames) if lb else 0
    with _Call("attn_spatial", 1, 4.0 * Cdim * lq * (n * lq + nbf * lb), 2.0 * (4 * n * lq * Cdim + 2 * lb * Cdim)):
        L.check(L.load().mimo_attn_spatial(C.byref(p), _stream()), "mimo_attn_spatial")
    return out


def attn_temporal(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, batch: int, frames: int, hw: int, heads: int, *,
                  scale: Optional[float] = None, out: Optional[torch.Tensor] = None, q_frames: Optional[int] = None,
                  frames_per_chunk: Optional[int] = None, chunk_stride_rows: int = 0) -> torch.Tensor:
    """q: [batch*q_frames*hw, C]; k/v: column slices of one buffer holding all `frames` frames, possibly as
    frames/frames_per_chunk chunks chunk_stride_rows apart (frame-sharded clip, see the header)."""
    Cdim = q.shape[1]
    d = Cdim // heads
    fq = frames if q_frames is None else q_frames
    if out is None:
        out = torch.empty((batch * fq * hw, Cdim), dtype=q.dtype, device=q.device)
    p = L.AttnTemporalParams()
    p.q, p.ld_q = _ptr(q), q.stride(0)
    p.k, p.v, p.ld_kv = _ptr(k), _ptr(v), k.stride(0)
    assert k.stride(0) == v.stride(0)
    p.out, p.ld_out = _ptr(out), out.stride(0)
    p.chunk_stride_rows = int(chunk_stride_rows)
    p.batch, p.q_frames, p.kv_frames = batch, fq, frames
    p.frames_per_chunk = frames if frames_per_chunk is None else frames_per_chunk
    p.hw, p.heads, p.d = hw, heads, d
    p.scale = float(scale if scale is not None else d ** -0.5)
    p.dtype = _dt(q)
    rows = batch * fq * hw
    with _Call("attn_temporal", 1, 4.0 * rows * frames * Cdim, 2.0 * (2 * rows + 2 * batch * frames * hw) * Cdim):
        L.check(L.load().mimo_attn_temporal(C.byref(p), _stream()), "mimo_attn_temporal")
    return out


def exchange(xg, mode: int, name: str, dst: torch.Tensor, b: int, fl: int, hw: int, Cdim: int,
             residual: Optional[torch.Tensor] = None) -> torch.Tensor:
    """One mimo_exchange of frame group `xg` (host/shard.py: Exchange): pull from every member's source buffer `name`
    into the local tensor `dst` (mode 0 frames->pixels, 1 pixels->frames (+ residual), 2 all-gather)."""
    assert dst.is_contiguous() and (residual is None or (residual.is_contiguous() and residual.shape == dst.shape))
    p = L.ExchangeParams()
    src, flags = xg.bufs[name], xg.flags
    for s in range(xg.G):
        p.peer_src[s] = src.peer_ptrs[s]
        p.peer_ready[s] = flags.peer_ptrs[s]
    p.ctl, p.dst, p.residual = _ptr(xg.ctl), _ptr(dst), _ptr(residual)
    p.mode, p.G, p.r = int(mode), xg.G, xg.r
    p.b, p.fl, p.hw, p.C = int(b), int(fl), int(hw), int(Cdim)
    p.dtype = _dt(dst)
    p.max_blocks, p.timeout_ms = int(xg.max_blocks), int(xg.timeout_ms)
    rows = b * fl * hw * (xg.G if mode == 2 else 1)
    need = b * fl * hw * Cdim * dst.element_size()  # every member's source holds b*fl*hw rows in all three modes
    if need > src.nbytes or dst.numel() != rows * Cdim:
        raise L.MimoError(f"exchange: source buffer '{name}' ({src.nbytes} B) or dst ({tuple(dst.shape)}) does not fit "
                          f"b={b} fl={fl} hw={hw} C={Cdim} mode={mode}")
    with _Call("exchange", 1, 0.0, 2.0 * dst.numel() * dst.element_size() + (dst.numel() * dst.element_size() if residual is not None else 0)):
        L.check(L.load().mimo_exchange(C.byref(p), _stream()), "mimo_exchange")
    return dst


def ncfhw_to_nhwc(src: torch.Tensor, cpad: int, dtype: torch.dtype, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    b, c, f, h, w = src.shape
    assert src.is_contiguous() and src.dtype in (torch.float32, dtype)
    if out is None:
        out = torch.empty((b * f * h * w, cpad), dtype=dtype, device=src.device)
    with _Call("layout", 1, 0.0, src.numel() * src.element_size() + 2.0 * out.numel()):
        L.check(L.load().mimo_ncfhw_to_nhwc(_ptr(src), _ptr(out), b, c, f, h, w, cpad,
                                            int(src.dtype == torch.float32), _dt(out), _stream()), "mimo_ncfhw_to_nhwc")
    return out


def nhwc_to_ncfhw(src: torch.Tensor, b: int, c: int, f: int, h: int, w: int, *, out_dtype: Optional[torch.dtype] = None,
                  out: Optional[torch.Tensor] = None) -> torch.Tensor:
    out_dtype = out_dtype or src.dtype
    if out is None:
        out = torch.empty((b, c, f, h, w), dtype=out_dtype, device=src.device)
    with _Call("layout", 1, 0.0, 2.0 * b * c * f * h * w + out.numel() * out.element_size()):
        L.check(L.load().mimo_nhwc_to_ncfhw(_ptr(src), _ptr(out), b, c, f, h, w, src.stride(0),
                                            int(out.dtype == torch.float32), _dt(src), _stream()), "mimo_nhwc_to_ncfhw")
    return out


def upsample2x(x: torch.Tensor, n: int, h: int, w: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    c = x.shape[1]
    assert x.is_contiguous()
    if out is None:
        out = torch.empty((n * 4 * h * w, c), dtype=x.dtype, device=x.device)
    with _Call("upsample2x", 1, 0.0, 2.0 * 5 * x.numel()):
        L.check(L.load().mimo_upsample2x(_ptr(x), _ptr(out), n, h, w, c, _dt(x), _stream()), "mimo_upsample2x")
    return out


def upsample_nearest(x: torch.Tensor, n: int, h: int, w: int, oh: int, ow: int,
                     out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """F.interpolate(mode="nearest", size=(oh, ow)) of channels-last x [n*h*w, c] -> [n*oh*ow, c], bit-identical."""
    c = x.shape[1]
    assert x.is_contiguous() and x.shape[0] == n * h * w
    if out is None:
        out = torch.empty((n * oh * ow, c), dtype=x.dtype, device=x.device)
    assert out.is_contiguous() and out.shape == (n * oh * ow, c)
    with _Call("upsample_nearest", 1, 0.0, float(x.element_size() * (x.numel() + out.numel()))):
        L.check(L.load().mimo_upsample_nearest(_ptr(x), _ptr(out), n, h, w, oh, ow, c, _dt(x), _stream()),
                "mimo_upsample_nearest")
    return out


def softmax_rows_(x: torch.Tensor) -> torch.Tensor:
    assert x.dim() == 2 and x.stride(1) == 1
    with _Call("softmax_rows", 1, 0.0, 2.0 * 2 * x.numel()):
        L.check(L.load().mimo_softmax_rows(_ptr(x), x.shape[0], x.shape[1], x.stride(0), _dt(x), _stream()),
                "mimo_softmax_rows")
    return x


def add(a: torch.Tensor, b: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    if out is None:
        out = torch.empty_like(a)
    with _Call("elementwise", 1, 0.0, 2.0 * 3 * a.numel()):
        L.check(L.load().mimo_add(_ptr(a), _ptr(b), _ptr(out), a.numel(), _dt(a), _stream()), "mimo_add")
    return out


def silu(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    if out is None:
        out = torch.empty_like(x)
    with _Call("elementwise", 1, 0.0, 2.0 * 2 * x.numel()):
        L.check(L.load().mimo_silu(_ptr(x), _ptr(out), x.numel(), _dt(x), _stream()), "mimo_silu")
    return out


def quick_gelu(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    if out is None:
        out = torch.empty_like(x)
    with _Call("elementwise", 1, 0.0, 2.0 * 2 * x.numel()):
        L.check(L.load().mimo_quick_gelu(_ptr(x), _ptr(out), x.numel(), _dt(x), _stream()), "mimo_quick_gelu")
    return out


def composite_frame(canvas: torch.Tensor, bk: torch.Tensor, mask: torch.Tensor, *, occ: Optional[torch.Tensor] = None,
                    vid: Optional[torch.Tensor] = None, prev: Optional[torch.Tensor] = None, factor: float = 0.0,
                    out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """run_edit.py:282-300 for one frame; uint8 [H, W, 3] images, float32 [H, W] mask, uint8 [H, W] occlusion."""
    for t in (canvas, bk) + tuple(x for x in (occ, vid, prev) if x is not None):
        assert t.dtype == torch.uint8 and t.is_contiguous() and t.is_cuda
    assert mask.dtype == torch.float32 and mask.is_contiguous() and mask.shape == canvas.shape[:2]
    if out is None:
        out = torch.empty_like(canvas)
    px = canvas.shape[0] * canvas.shape[1]
    with _Call("composite", 1, 0.0, float(px * (3 * (3 + (occ is not None) + (prev is not None)) + 4 + (occ is not None)))):
        L.check(L.load().mimo_composite_frame(_ptr(canvas), _ptr(bk), _ptr(mask), _ptr(occ), _ptr(vid), _ptr(prev),
                                              float(factor), _ptr(out), px, _stream()), "mimo_composite_frame")
    return out


def cfg_ddim_step(pred_uncond: torch.Tensor, pred_cond: torch.Tensor, latents: torch.Tensor, guidance: float,
                  sqrt_a_t: float, sqrt_1ma_t: float, sqrt_a_prev: float, sqrt_1ma_prev: float, *,
                  counter: Optional[torch.Tensor] = None, frame_stride: int = 0) -> torch.Tensor:
    """In-place DDIM update of `latents` from the two CFG halves of the (window-accumulated) prediction."""
    assert pred_uncond.is_contiguous() and pred_cond.is_contiguous() and latents.is_contiguous()
    with _Call("cfg_ddim", 1, 0.0, 2.0 * 4 * latents.numel()):
        L.check(L.load().mimo_cfg_ddim_step(_ptr(pred_uncond), _ptr(pred_cond), _ptr(counter), int(frame_stride),
                                            _ptr(latents), latents.numel(), float(guidance), float(sqrt_a_t),
                                            float(sqrt_1ma_t), float(sqrt_a_prev), float(sqrt_1ma_prev), _dt(latents),
                                            _stream()), "mimo_cfg_ddim_step")
    return latents


def cfg_ddim_step_noise(pred_uncond: torch.Tensor, pred_cond: torch.Tensor, latents: torch.Tensor, guidance: float,
                        sqrt_a_t: float, sqrt_1ma_t: float, sqrt_a_prev: float, dir_coef: float, noise: torch.Tensor,
                        sigma: float, *, counter: Optional[torch.Tensor] = None, frame_stride: int = 0) -> torch.Tensor:
    """cfg_ddim_step for eta > 0: direction coefficient `dir_coef` = sqrt(1 - abar_prev - sigma^2), plus sigma * noise."""
    assert pred_uncond.is_contiguous() and pred_cond.is_contiguous() and latents.is_contiguous()
    assert noise.is_contiguous() and noise.numel() == latents.numel() and noise.dtype == latents.dtype
    with _Call("cfg_ddim", 1, 0.0, 2.0 * 5 * latents.numel()):
        L.check(L.load().mimo_cfg_ddim_step_noise(_ptr(pred_uncond), _ptr(pred_cond), _ptr(counter), int(frame_stride),
                                                  _ptr(latents), latents.numel(), float(guidance), float(sqrt_a_t),
                                                  float(sqrt_1ma_t), float(sqrt_a_prev), float(dir_coef), _ptr(noise),
                                                  float(sigma), _dt(latents), _stream()), "mimo_cfg_ddim_step_noise")
    return latents


def cfg_multistep(pred_uncond: torch.Tensor, pred_cond: torch.Tensor, latents: torch.Tensor, guidance: float,
                  coefficients, hist_out: torch.Tensor, *, h1: Optional[torch.Tensor] = None,
                  h2: Optional[torch.Tensor] = None, noise: Optional[torch.Tensor] = None,
                  counter: Optional[torch.Tensor] = None, frame_stride: int = 0) -> torch.Tensor:
    """In-place multistep solver update of `latents` (DPM-Solver++, Euler, Euler-ancestral) from the two CFG halves:
    coefficients = (a, b, c_x, c_m, c_1, c_2, c_n) of the scheduler's multistep_coefficients(i); m = a x + b v goes to
    `hist_out` (which may be `h2`). A None h1 / h2 / noise is a zero term."""
    a, b, cx, cm, c1, c2, cn = (float(c) for c in coefficients)
    for t in (pred_uncond, pred_cond, latents, hist_out) + tuple(x for x in (h1, h2, noise) if x is not None):
        assert t.is_contiguous() and t.dtype == latents.dtype
    for t in (pred_uncond, pred_cond, hist_out) + tuple(x for x in (h1, h2, noise) if x is not None):
        assert t.numel() == latents.numel()
    p = L.CfgMultistepParams(pred_uncond=_ptr(pred_uncond), pred_cond=_ptr(pred_cond), counter=_ptr(counter),
                             frame_stride=int(frame_stride), latents=_ptr(latents), count=latents.numel(),
                             hist_out=_ptr(hist_out), h1=_ptr(h1), h2=_ptr(h2), noise=_ptr(noise),
                             guidance=float(guidance), a=a, b=b, c_x=cx, c_m=cm, c_1=c1, c_2=c2, c_n=cn,
                             dtype=_dt(latents))
    n_in = 3 + sum(x is not None for x in (h1, h2, noise))
    with _Call("cfg_multistep", 1, 0.0, float(latents.element_size() * (n_in + 2) * latents.numel())):
        L.check(L.load().mimo_cfg_multistep(C.byref(p), _stream()), "mimo_cfg_multistep")
    return latents


def cfg_rescale(pred_uncond: torch.Tensor, pred_cond: torch.Tensor, guidance: float, phi: float,
                out: Optional[torch.Tensor] = None, counter: Optional[torch.Tensor] = None,
                frame_stride: int = 0) -> torch.Tensor:
    """Rescaled CFG (guidance_rescale = phi): the guided prediction of the two (window-summed) halves, as cfg_ddim_step
    forms it, rescaled by std(text) / std(cfg) over the whole tensor and mixed with weight phi, written to `out`
    (allocated when None). Feed the step kernels (out, out, guidance 1.0, no counter) afterwards."""
    assert pred_uncond.is_contiguous() and pred_cond.is_contiguous() and pred_cond.dtype == pred_uncond.dtype
    assert pred_cond.numel() == pred_uncond.numel()
    if out is None:
        out = torch.empty_like(pred_cond)
    assert out.is_contiguous() and out.dtype == pred_cond.dtype and out.numel() == pred_cond.numel()
    p = L.CfgRescaleParams(pred_uncond=_ptr(pred_uncond), pred_cond=_ptr(pred_cond), counter=_ptr(counter),
                           frame_stride=int(frame_stride), out=_ptr(out), count=out.numel(), phi=float(phi),
                           guidance=float(guidance), dtype=_dt(out))
    need = L.load().mimo_cfg_rescale_workspace_bytes(C.byref(p))
    if need < 0:
        L.check(int(need), "mimo_cfg_rescale_workspace_bytes")
    ws = torch.empty(((need + 7) // 8,), dtype=torch.float64, device=out.device)
    p.workspace, p.workspace_bytes = _ptr(ws), ws.numel() * 8
    with _Call("cfg_rescale", 2, 0.0, float(out.element_size() * 3 * out.numel())):  # algorithmic: two reads, one write
        L.check(L.load().mimo_cfg_rescale(C.byref(p), _stream()), "mimo_cfg_rescale")
    return out


INTERP_LINEAR, INTERP_SLERP = 0, 1


def interpolate_frames(latents: torch.Tensor, k: int, method: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """[1, 4, F, h, w] -> [1, 4, (F-1)*k + 1, h, w]: k-1 interpolated frames between each pair of neighbours
    (pipeline interpolate_latents); method INTERP_LINEAR or INTERP_SLERP."""
    b, c, f, h, w = latents.shape
    assert b == 1 and c == 4 and latents.is_contiguous()
    shape = (1, 4, (f - 1) * k + 1, h, w)
    if out is None:
        out = torch.empty(shape, dtype=latents.dtype, device=latents.device)
    assert out.is_contiguous() and tuple(out.shape) == shape and out.dtype == latents.dtype
    with _Call("interpolate_frames", 1, 0.0, float(latents.element_size() * (2 * latents.numel() + out.numel()))):
        L.check(L.load().mimo_interpolate_frames(_ptr(latents), _ptr(out), f, h * w, k, method, _dt(latents), _stream()),
                "mimo_interpolate_frames")
    return out


# ------------------------------------------------------------------------------------------------
# weight packing (host side, once per model load)
# ------------------------------------------------------------------------------------------------
def pack_conv3x3_weight(w: torch.Tensor, cin_pad: Optional[int] = None, cout_pad: Optional[int] = None) -> torch.Tensor:
    """OIHW [cout, cin, 3, 3] -> [cout_pad, 9 * cin_pad], K index = (ky*3+kx) * cin_pad + ch."""
    cout, cin = w.shape[:2]
    cin_pad = cin_pad or (cin + 7) // 8 * 8
    cout_pad = cout_pad or (cout + 7) // 8 * 8
    p = torch.zeros((cout_pad, 9, cin_pad), dtype=w.dtype, device=w.device)
    p[:cout, :, :cin] = w.permute(0, 2, 3, 1).reshape(cout, 9, cin)
    return p.reshape(cout_pad, 9 * cin_pad).contiguous()


def pack_conv_up2x_weight(w: torch.Tensor, b: Optional[torch.Tensor] = None) -> torch.Tensor:
    """OIHW [cout, cin, 3, 3] of the conv that FOLLOWS a nearest-x2 upsampling -> [4, cout_pad, 4 * cin_pad] for
    mimo_conv_up2x: class 2a+b holds, for tap (iy, ix), the sum (in fp32, rounded once) of the 3x3 taps (ky, kx) that read
    source pixel (y - 1 + a + iy, x - 1 + b + ix) when producing output pixel (2y + a, 2x + b)."""
    cout, cin = w.shape[:2]
    cin_pad, cout_pad = (cin + 7) // 8 * 8, (cout + 7) // 8 * 8
    sets = {0: ([0], [1, 2]), 1: ([0, 1], [2])}  # parity -> (taps landing on the first / second source row)
    wf = w.float()
    out = torch.zeros((4, cout_pad, 4, cin_pad), dtype=torch.float32, device=w.device)
    for a in range(2):
        for bb in range(2):
            for iy in range(2):
                for ix in range(2):
                    acc = sum(wf[:, :, ky, kx] for ky in sets[a][iy] for kx in sets[bb][ix])
                    out[2 * a + bb, :cout, 2 * iy + ix, :cin] = acc
    return out.reshape(4, cout_pad, 4 * cin_pad).to(w.dtype).contiguous()


def pack_geglu_weight(w: torch.Tensor, b: Optional[torch.Tensor]):
    """diffusers GEGLU proj weight [2*inner, dim] (value rows then gate rows) -> tile-interleaved rows."""
    n2 = w.shape[0]
    inner = n2 // 2
    g = L.load().mimo_gemm_geglu_granule(n2)
    assert inner % g == 0
    wv, wg = w[:inner].reshape(inner // g, g, -1), w[inner:].reshape(inner // g, g, -1)
    wp = torch.stack([wv, wg], dim=1).reshape(n2, -1).contiguous()
    bp = None
    if b is not None:
        bv, bg = b[:inner].reshape(inner // g, g), b[inner:].reshape(inner // g, g)
        bp = torch.stack([bv, bg], dim=1).reshape(n2).contiguous()
    return wp, bp


E4M3_MAX = 448.0


def quantize_e4m3_rows(y: torch.Tensor):
    """The per-row e4m3 rule of mimo_layernorm_e4m3 on the host: amax = max |y| of each row (in fp32), q = y * (448 /
    amax) rounded to nearest and saturated, scale = amax / 448; a zero row gets scale 1. Returns (q float8_e4m3fn, scale
    fp32). torch's cast does not saturate (it gives NaN past 448), hence the clamp. Both divisions are tensor / tensor:
    torch turns a division by a Python scalar into a multiplication by its reciprocal, which is not the IEEE quotient."""
    y = y.float()
    amax = y.abs().amax(dim=1)
    zero = amax == 0
    inv = torch.where(zero, torch.ones_like(amax), torch.full_like(amax, E4M3_MAX) / amax)
    scale = torch.where(zero, torch.ones_like(amax), amax / torch.full_like(amax, E4M3_MAX))
    q = torch.clamp(y * inv[:, None], -E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    return q.contiguous(), scale.contiguous()


def quantize_e4m3_blocks(y: torch.Tensor, block: int = E4M3_BLOCK):
    """The per-(row, block) e4m3 rule of mimo_gemm_e4m3_geglu_e4m3 on the host: quantize_e4m3_rows applied to each run of
    `block` consecutive columns of each row of y [M, K] (K % block == 0), with the same tensor / tensor divisions. Returns
    (q [M, K] float8_e4m3fn, scale [K / block, M] fp32, block-major as the kernel writes it)."""
    M, K = y.shape
    assert K % block == 0
    q, s = quantize_e4m3_rows(y.float().reshape(M * (K // block), block))
    return q.reshape(M, K).contiguous(), s.reshape(M, K // block).t().contiguous()


def pack_e4m3_weight(w: torch.Tensor):
    """A [N, K] weight (already in gemm's row order, e.g. pack_geglu_weight's) as (e4m3 [N, K], fp32 scale [N]): one
    scale per output channel by quantize_e4m3_rows, so the rows' order - and the GEGLU tile interleave - is kept."""
    return quantize_e4m3_rows(w)


SILU_ARGMIN, SILU_MIN_ABS = -1.2784645, 0.27846454  # SiLU's only turning point: its minimum, silu(-1.2784645)


def e4m3_image_scales(lo: torch.Tensor, hi: torch.Tensor, mean: torch.Tensor, rstd: torch.Tensor, gamma: torch.Tensor,
                      beta: torch.Tensor) -> torch.Tensor:
    """The per-image scale rule of mimo_groupnorm_e4m3 on the host. lo / hi: [n, groups] min / max of x over each image's
    elements of a group; mean / rstd: [n, groups] the statistics the normaliser uses (the image's own, or its sample's
    window statistics); gamma / beta: [C]. For each channel c of group g, z_lo = (lo - mean) * (rstd * gamma_c) + beta_c
    and z_hi likewise (one rounding after the product and sum, as the kernel's fma), B_c = max(|silu(z_lo)|,
    |silu(z_hi)|, 0.27846454 if [z_lo, z_hi] holds SiLU's minimum at -1.2784645); amax = max_c B_c and scale = amax / 448
    (an IEEE quotient), or 1 when amax is 0. Returns (scale, inv) [n] fp32: inv = 448 / amax (1 when amax is 0) is the
    multiplier of SiLU's output ahead of the rounding."""
    C_ = gamma.numel()
    g_of_c = torch.arange(C_, device=lo.device) // (C_ // lo.shape[1])
    sc = rstd.float()[:, g_of_c] * gamma.float()[None]
    z = [((v.float() - mean.float())[:, g_of_c].double() * sc.double() + beta.double()[None]).float() for v in (lo, hi)]
    bnd = torch.maximum(torch.nn.functional.silu(z[0]).abs(), torch.nn.functional.silu(z[1]).abs())
    inside = (torch.minimum(z[0], z[1]) <= SILU_ARGMIN) & (torch.maximum(z[0], z[1]) >= SILU_ARGMIN)
    bnd = torch.where(inside, torch.clamp(bnd, min=SILU_MIN_ABS), bnd)
    amax = bnd.amax(dim=1)
    zero, one, top = amax == 0, torch.ones_like(amax), torch.full_like(amax, E4M3_MAX)
    return torch.where(zero, one, amax / top), torch.where(zero, one, top / amax)


def groupnorm_silu_e4m3_host(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, groups: int, eps: float,
                             frames: int = 1):
    """SiLU(GroupNorm) of x [n, hw, C] quantized per image by e4m3_image_scales, in torch (the oracle's and the tests'
    statement of mimo_groupnorm_e4m3). Statistics per image, or with frames > 1 per sample of `frames` consecutive images
    (fp64 sums, rounded to fp32). Returns (q [n, hw, C] float8_e4m3fn, scale [n] fp32, y = the fp32 SiLU(GroupNorm(x)))."""
    n, hw, C_ = x.shape
    xf = x.float()
    xs = xf.double().reshape(n // frames, frames, hw, groups, C_ // groups)
    mean = xs.mean(dim=(1, 2, 4))
    var = xs.var(dim=(1, 2, 4), unbiased=False)
    mean = mean.float().repeat_interleave(frames, 0)
    rstd = torch.rsqrt(var.float() + eps).repeat_interleave(frames, 0)
    xg = xf.reshape(n, hw, groups, C_ // groups)
    lo, hi = xg.amin(dim=(1, 3)), xg.amax(dim=(1, 3))
    scale, inv = e4m3_image_scales(lo, hi, mean, rstd, gamma, beta)
    g_of_c = torch.arange(C_, device=x.device) // (C_ // groups)
    sc = rstd[:, g_of_c] * gamma.float()[None]
    y = ((xf - mean[:, g_of_c][:, None]).double() * sc[:, None].double() + beta.double()).float()
    y = torch.nn.functional.silu(y)
    q = torch.clamp(y * inv[:, None, None], -E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    return q, scale, y
