"""Kernel bring-up probe (GPU box only): runs one named check against a plain PyTorch fp32 reference and prints
compact diagnostics. Each check is meant to run in its own process (a trapped kernel poisons the context):

    python scripts/gpu_probe.py list
    python scripts/gpu_probe.py <name> [...]
"""
from __future__ import annotations

import math
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from mimo_b200 import lib as L  # noqa: E402
from mimo_b200 import ops  # noqa: E402

DEV = "cuda"


def rel_err(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-12))


def report(name, got, ref, tol=2e-3):
    e = rel_err(got, ref)
    mx = float((got.float() - ref.float()).abs().max())
    bad = not (e < tol) or not math.isfinite(e)
    print(f"[{'FAIL' if bad else ' ok '}] {name}: rel_l2={e:.3e} max_abs={mx:.3e} ref_rms={float(ref.float().pow(2).mean().sqrt()):.3e}")
    if bad:
        d = (got.float() - ref.float()).abs()
        thr = 1e-2 * float(ref.float().abs().max()) + 1e-6
        wrong = d > thr
        print(f"       wrong elems: {int(wrong.sum())}/{wrong.numel()}  nan={int(torch.isnan(got.float()).sum())}")
        if got.dim() == 2:
            rows = wrong.any(dim=1).nonzero().flatten()
            cols = wrong.any(dim=0).nonzero().flatten()
            print(f"       bad rows: {rows[:24].tolist()}{'...' if rows.numel() > 24 else ''} (n={rows.numel()})")
            print(f"       bad cols: {cols[:24].tolist()}{'...' if cols.numel() > 24 else ''} (n={cols.numel()})")
            print("       got[:4,:8] =", got[:4, :8].float().cpu().numpy().round(3).tolist())
            print("       ref[:4,:8] =", ref[:4, :8].float().cpu().numpy().round(3).tolist())
    return not bad


def ints(shape, lo=-3, hi=4, dtype=torch.float16):
    return torch.randint(lo, hi, shape, device=DEV).to(dtype)


# ------------------------------------------------------------------------------------------------
def gemm_case(M, N, K, bn=0, dtype=torch.float16, **kw):
    lib = L.load()
    lib.mimo_debug_force_bn(bn)
    torch.manual_seed(M * 7 + N * 3 + K)
    a = ints((M, K), dtype=dtype)
    w = ints((N, K), dtype=dtype)
    try:
        out = ops.gemm(a, w)
        torch.cuda.synchronize()
    finally:
        lib.mimo_debug_force_bn(0)
    ref = a.double() @ w.double().t()
    ok = report(f"gemm M={M} N={N} K={K} bn={bn}", out, ref, tol=1e-3)
    # integer inputs: every fp32 partial sum is exact, so the output is the exact product rounded once
    bad = int((out != ref.to(out.dtype)).sum())
    if bad:
        print(f"[FAIL] gemm M={M} N={N} K={K} bn={bn}: not bit-exact, {bad}/{out.numel()} elements differ")
    ok &= bad == 0
    return ok, a, w, out, ref


def gemm_basic():
    ok, a, w, out, ref = gemm_case(128, 64, 64, bn=64)
    if not ok:
        # decode which operand / which k-slice is broken
        lib = L.load()
        lib.mimo_debug_force_bn(64)
        for k0 in (0, 16, 32, 48):
            a2 = torch.zeros_like(a)
            a2[:, k0:k0 + 16] = 1
            o = ops.gemm(a2, w)
            torch.cuda.synchronize()
            report(f"  A=1 on k[{k0}:{k0+16}]", o, a2.float() @ w.float().t(), tol=1e-3)
        a3 = torch.zeros_like(a)
        a3[torch.arange(128), torch.arange(128) % 64] = 1  # row r selects k = r % 64
        o = ops.gemm(a3, w)
        torch.cuda.synchronize()
        report("  A one-hot(k=r%64)", o, a3.float() @ w.float().t(), tol=1e-3)
    return ok


def gemm_shapes():
    ok = True
    for (M, N, K, bn) in [(128, 64, 128, 64), (128, 64, 16, 64), (128, 64, 200, 64), (100, 64, 64, 64),
                          (256, 128, 320, 128), (384, 320, 320, 160), (256, 512, 256, 256), (300, 200, 136, 0),
                          (384, 960, 320, 192), (200, 400, 72, 192),
                          (2, 1280, 320, 0), (4096, 320, 320, 0), (4096, 2560, 320, 0), (1000, 640, 2560, 0)]:
        ok &= gemm_case(M, N, K, bn)[0]
    return ok


def gemm_persistent():
    # more tiles than SMs -> exercises the accumulator double buffering and barrier phase wrap-around
    ok = True
    for (M, N, K, bn) in [(128 * 300, 64, 64, 64), (128 * 160, 320, 192, 160), (128 * 40, 1280, 1280, 256),
                          (128 * 100, 960, 320, 192),
                          (128 * 151, 128, 64 * 13, 128)]:
        ok &= gemm_case(M, N, K, bn)[0]
    return ok


def gemm_epilogue():
    ok = True
    torch.manual_seed(1)
    M, N, K = 512, 320, 320
    a = torch.randn(M, K, device=DEV).half()
    w = (torch.randn(N, K, device=DEV) / math.sqrt(K)).half()
    bias = torch.randn(N, device=DEV).half()
    res = torch.randn(M, N, device=DEV).half()
    rv = torch.randn(M // 128, N, device=DEV).half()
    base = a.float() @ w.float().t()
    ok &= report("gemm+bias", ops.gemm(a, w, bias=bias), base + bias.float())
    ok &= report("gemm+bias+res", ops.gemm(a, w, bias=bias, residual=res), base + bias.float() + res.float())
    ok &= report("gemm+bias+rowvec+res*0.5",
                 ops.gemm(a, w, bias=bias, residual=res, rowvec=rv, rows_per_group=128, scale=0.5),
                 (base + bias.float() + res.float() + rv.float().repeat_interleave(128, 0)) * 0.5)
    ok &= report("gemm+bias+silu", ops.gemm(a, w, bias=bias, act=L.ACT_SILU), torch.nn.functional.silu(base + bias.float()))
    # GEGLU (diffusers GEGLU: proj -> chunk(2) -> h * gelu(gate))
    w2 = (torch.randn(2 * 1280, K, device=DEV) / math.sqrt(K)).half()
    b2 = torch.randn(2 * 1280, device=DEV).half()
    wp, bp = ops.pack_geglu_weight(w2, b2)
    y = a.float() @ w2.float().t() + b2.float()
    hval, gate = y.chunk(2, dim=-1)
    ok &= report("gemm+geglu", ops.gemm(a, wp, bias=bp, act=L.ACT_GEGLU), hval * torch.nn.functional.gelu(gate))
    # bf16
    ab, wb = a.bfloat16(), w.bfloat16()
    ok &= report("gemm bf16", ops.gemm(ab, wb, bias=bias.bfloat16()), ab.float() @ wb.float().t() + bias.bfloat16().float(), tol=6e-3)
    torch.cuda.synchronize()
    return ok


def conv_case(n, h, w, c0, cout, c1=0, bn=0, **ep):
    lib = L.load()
    lib.mimo_debug_force_bn(bn)
    torch.manual_seed(n + h * 3 + c0)
    x0 = torch.randn(n, c0, h, w, device=DEV).half()
    x1 = torch.randn(n, c1, h, w, device=DEV).half() if c1 else None
    wt = (torch.randn(cout, c0 + c1, 3, 3, device=DEV) / math.sqrt(9 * (c0 + c1))).half()
    bias = torch.randn(cout, device=DEV).half()
    xin = torch.cat([x0, x1], 1) if c1 else x0
    ref = torch.nn.functional.conv2d(xin.float(), wt.float(), bias.float(), padding=1)
    ref = ref.permute(0, 2, 3, 1).reshape(n * h * w, cout)
    x0l = x0.permute(0, 2, 3, 1).reshape(n * h * w, c0).contiguous()
    x1l = x1.permute(0, 2, 3, 1).reshape(n * h * w, c1).contiguous() if c1 else None
    wp = ops.pack_conv3x3_weight(wt, cin_pad=c0 + c1)
    out = ops.conv3x3(x0l, wp, n, h, w, x1=x1l, bias=bias)
    torch.cuda.synchronize()
    ok = report(f"conv3x3 n={n} {h}x{w} c={c0}+{c1}->{cout} bn={bn}", out, ref)
    lib.mimo_debug_force_bn(0)
    return ok


def conv_basic():
    ok = conv_case(1, 8, 16, 64, 64, bn=64)       # one 128-pixel tile (8 rows x 16)
    ok &= conv_case(2, 8, 8, 64, 64, bn=64)       # two images per tile
    ok &= conv_case(1, 16, 16, 64, 64, bn=64)     # two tiles along h
    return ok


def conv_shapes():
    ok = True
    for args in [(2, 64, 64, 320, 320), (3, 32, 32, 640, 640), (4, 16, 16, 1280, 1280), (6, 8, 8, 1280, 1280),
                 (2, 64, 64, 8, 320), (2, 64, 64, 320, 8), (2, 32, 32, 640, 640, 320), (1, 16, 16, 1280, 1280, 640),
                 (1, 24, 24, 64, 64), (3, 12, 12, 128, 64), (1, 256, 256, 128, 128), (5, 8, 8, 72, 64),
                 (1, 96, 96, 64, 320)]:
        ok &= conv_case(*args)
    return ok


def norms():
    ok = True
    torch.manual_seed(2)
    for (n, hw, c0, c1, eps, silu) in [(3, 4096, 320, 0, 1e-5, True), (2, 1024, 640, 0, 1e-6, False),
                                       (2, 256, 1280, 640, 1e-5, True), (2, 1024, 640, 320, 1e-5, True),
                                       (2, 64, 1280, 1280, 1e-5, True), (1, 4096, 128, 0, 1e-6, True),
                                       (1, 1024, 512, 0, 1e-6, True), (2, 16, 256, 0, 1e-6, False)]:
        C = c0 + c1
        x0 = (torch.randn(n * hw, c0, device=DEV) * 2 + 0.5).half()
        x1 = (torch.randn(n * hw, c1, device=DEV) - 1).half() if c1 else None
        g = (1 + 0.2 * torch.randn(C, device=DEV)).half()
        b = (0.2 * torch.randn(C, device=DEV)).half()
        x = torch.cat([x0, x1], 1) if c1 else x0
        xr = x.float().reshape(n, hw, C).permute(0, 2, 1)
        ref = torch.nn.functional.group_norm(xr, 32, g.float(), b.float(), eps)
        if silu:
            ref = torch.nn.functional.silu(ref)
        ref = ref.permute(0, 2, 1).reshape(n * hw, C)
        out = ops.groupnorm(x0, g, b, n, hw, eps=eps, silu=silu, x1=x1)
        ok &= report(f"groupnorm n={n} hw={hw} c={c0}+{c1} silu={silu}", out, ref)
    for (rows, C) in [(1000, 320), (513, 640), (64, 1280), (7, 2048)]:
        x = (torch.randn(rows, C, device=DEV) * 3 + 1).half()
        g = (1 + 0.2 * torch.randn(C, device=DEV)).half()
        b = (0.2 * torch.randn(C, device=DEV)).half()
        ref = torch.nn.functional.layer_norm(x.float(), (C,), g.float(), b.float(), 1e-5)
        ok &= report(f"layernorm rows={rows} c={C}", ops.layernorm(x, g, b), ref)
    # LN + positional encoding: rows ordered ((b f) hw)
    bsz, f, hw, C = 2, 5, 12, 320
    x = torch.randn(bsz * f * hw, C, device=DEV).half()
    g = torch.ones(C, device=DEV).half()
    b = torch.zeros(C, device=DEV).half()
    pe = torch.randn(32, C, device=DEV).half()
    ref = torch.nn.functional.layer_norm(x.float(), (C,)).reshape(bsz, f, hw, C) + pe[:f].float()[None, :, None, :]
    ok &= report("layernorm+pe", ops.layernorm(x, g, b, pe=pe, rows_per_frame=hw, frames=f), ref.reshape(-1, C))
    return ok


def temporal():
    ok = True
    torch.manual_seed(3)
    for (bsz, f, hw, heads, d) in [(2, 24, 64, 8, 40), (1, 24, 16, 8, 80), (2, 16, 4, 8, 160), (1, 1, 8, 8, 40),
                                   (1, 32, 8, 8, 40)]:
        C = heads * d
        qkv = torch.randn(bsz * f * hw, 3 * C, device=DEV).half()
        q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
        out = ops.attn_temporal(q, k, v, bsz, f, hw, heads)

        def tr(t):  # (b f) p (h d) -> (b p) h f d
            return t.float().reshape(bsz, f, hw, heads, d).permute(0, 2, 3, 1, 4).reshape(bsz * hw, heads, f, d)

        ref = torch.nn.functional.scaled_dot_product_attention(tr(q), tr(k), tr(v))
        ref = ref.reshape(bsz, hw, heads, f, d).permute(0, 3, 1, 2, 4).reshape(bsz * f * hw, C)
        ok &= report(f"attn_temporal b={bsz} f={f} hw={hw} d={d}", out, ref)
    # frame-sharded form: this "rank" owns frames [r*fl, (r+1)*fl); K|V of all ranks sit in rank-major chunks
    for (bsz, f, hw, heads, d, world) in [(2, 24, 8, 8, 40, 2), (2, 24, 4, 8, 80, 4), (1, 24, 4, 8, 160, 8)]:
        C = heads * d
        fl = f // world
        q_full = torch.randn(bsz, f, hw, C, device=DEV).half()
        kv_full = torch.randn(bsz, f, hw, 2 * C, device=DEV).half()
        # chunk g holds frames [g*fl, (g+1)*fl) of every batch entry: [(b, f_local, p)] rows
        kv_chunks = torch.cat([kv_full[:, gg * fl:(gg + 1) * fl].reshape(bsz * fl * hw, 2 * C) for gg in range(world)])

        def tr(t_, ff):
            return t_.float().reshape(bsz, ff, hw, heads, d).permute(0, 2, 3, 1, 4).reshape(bsz * hw, heads, ff, d)

        for rk in (0, world - 1):
            q = q_full[:, rk * fl:(rk + 1) * fl].reshape(bsz * fl * hw, C).contiguous()
            out = ops.attn_temporal(q, kv_chunks[:, :C], kv_chunks[:, C:], bsz, f, hw, heads, q_frames=fl,
                                    frames_per_chunk=fl, chunk_stride_rows=bsz * fl * hw)
            ref = torch.nn.functional.scaled_dot_product_attention(tr(q, fl), tr(kv_full[..., :C], f), tr(kv_full[..., C:], f))
            ref = ref.reshape(bsz, hw, heads, fl, d).permute(0, 3, 1, 2, 4).reshape(bsz * fl * hw, C)
            ok &= report(f"attn_temporal sharded world={world} rank={rk} d={d}", out, ref)
    return ok


def spatial_case(n, lq, heads, d, lb=0, bank_idx=None):
    torch.manual_seed(n * 5 + lq + d)
    C = heads * d
    qkv = torch.randn(n * lq, 3 * C, device=DEV).half()
    q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    bk = bv = bi = None
    if lb:
        bkv = torch.randn(2, lb, 2 * C, device=DEV).half()
        bk, bv = bkv[:, :, :C], bkv[:, :, C:]
        bi = torch.tensor(bank_idx, dtype=torch.int32, device=DEV)
    out = ops.attn_spatial(q, k, v, n, lq, heads, bank_k=bk, bank_v=bv, bank_index=bi)
    torch.cuda.synchronize()

    def hd(t, L_):
        return t.float().reshape(-1, L_, heads, d).permute(0, 2, 1, 3)

    refs = []
    for i in range(n):
        qi = hd(q[i * lq:(i + 1) * lq], lq)
        ki = hd(k[i * lq:(i + 1) * lq], lq)
        vi = hd(v[i * lq:(i + 1) * lq], lq)
        if lb and bank_idx[i] >= 0:
            ki = torch.cat([ki, hd(bk[bank_idx[i]], lb)], 2)
            vi = torch.cat([vi, hd(bv[bank_idx[i]], lb)], 2)
        o = torch.nn.functional.scaled_dot_product_attention(qi, ki, vi)
        refs.append(o.permute(0, 2, 1, 3).reshape(lq, C))
    ref = torch.cat(refs)
    return report(f"attn_spatial n={n} lq={lq} d={d} lb={lb}", out, ref)


def spatial_basic():
    ok = spatial_case(1, 128, 1, 64)
    ok &= spatial_case(1, 128, 8, 40)
    ok &= spatial_case(1, 256, 8, 40)
    return ok


def spatial_shapes():
    ok = True
    ok &= spatial_case(2, 1024, 8, 40, lb=1024, bank_idx=[-1, 1])
    ok &= spatial_case(2, 1024, 8, 80, lb=1024, bank_idx=[-1, 1])
    ok &= spatial_case(2, 256, 8, 160, lb=256, bank_idx=[0, 1])
    ok &= spatial_case(4, 64, 8, 160, lb=64, bank_idx=[-1, -1, 1, 1])
    ok &= spatial_case(2, 576, 8, 40, lb=576, bank_idx=[-1, 1])   # 24x24: ragged tiles
    ok &= spatial_case(1, 4096, 8, 40, lb=4096, bank_idx=[1])
    ok &= spatial_case(2, 320, 8, 80, lb=320, bank_idx=[1, -1])   # d=80 ping-pong kernel, ragged tiles
    ok &= spatial_case(1, 200, 4, 128)                             # dp = 128, second query tile partly out of range
    ok &= spatial_case(3, 130, 8, 16, lb=70, bank_idx=[0, -1, 1])  # tiny head dim, ragged bank
    ok &= spatial_case(2, 64, 8, 32, lb=64, bank_idx=[-1, 1])      # whole second query tile out of range
    return ok


def elementwise():
    ok = True
    torch.manual_seed(4)
    b, c, f, h, w = 2, 8, 3, 16, 16
    x = torch.randn(b, c, f, h, w, device=DEV)
    nhwc = ops.ncfhw_to_nhwc(x, 8, torch.float16)
    ref = x.permute(0, 2, 3, 4, 1).reshape(b * f * h * w, c)
    ok &= report("ncfhw_to_nhwc f32->f16", nhwc, ref)
    x4 = torch.randn(b, 4, f, h, w, device=DEV).half()
    nh = ops.ncfhw_to_nhwc(x4, 8, torch.float16)
    ref = torch.cat([x4, torch.zeros_like(x4)], 1).permute(0, 2, 3, 4, 1).reshape(b * f * h * w, 8)
    ok &= report("ncfhw_to_nhwc pad", nh, ref)
    back = ops.nhwc_to_ncfhw(nh, b, 4, f, h, w, out_dtype=torch.float32)
    ok &= report("nhwc_to_ncfhw", back, x4.float())
    a1, a2 = torch.randn(4096, device=DEV).half(), torch.randn(4096, device=DEV).half()
    ok &= report("add", ops.add(a1, a2), a1.float() + a2.float())
    ok &= report("silu", ops.silu(a1), torch.nn.functional.silu(a1.float()))
    # im2col: stride 2, and upsample x2
    n, hh, ww, cc = 2, 8, 8, 16
    xi = torch.randn(n, cc, hh, ww, device=DEV).half()
    xl = xi.permute(0, 2, 3, 1).reshape(-1, cc).contiguous()
    wt = torch.randn(24, cc, 3, 3, device=DEV).half() / 12
    wp = ops.pack_conv3x3_weight(wt)
    col = ops.im2col3x3(xl, n, hh, ww, stride=2)
    ref = torch.nn.functional.conv2d(xi.float(), wt.float(), stride=2, padding=1).permute(0, 2, 3, 1).reshape(-1, 24)
    ok &= report("im2col s2 + gemm", ops.gemm(col, wp), ref)
    col = ops.im2col3x3(xl, n, hh, ww, upshift=1)
    up = torch.nn.functional.interpolate(xi.float(), scale_factor=2.0, mode="nearest")
    ref = torch.nn.functional.conv2d(up, wt.float(), padding=1).permute(0, 2, 3, 1).reshape(-1, 24)
    ok &= report("im2col up2 + gemm", ops.gemm(col, wp), ref)
    col = ops.im2col3x3(xl, n, hh, ww, stride=2, pad_lo=0)
    ref = torch.nn.functional.conv2d(torch.nn.functional.pad(xi.float(), (0, 1, 0, 1)), wt.float(), stride=2)
    ok &= report("im2col s2 asym-pad + gemm", ops.gemm(col, wp), ref.permute(0, 2, 3, 1).reshape(-1, 24))
    return ok


def perf():
    """Rough kernel timings (CUDA events, inputs > L2 where it matters)."""
    def timeit(fn, iters=10):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters

    for (M, N, K) in [(196608, 320, 320), (196608, 2560, 320), (196608, 320, 1280), (49152, 640, 640),
                      (49152, 5120, 640), (12288, 1280, 1280), (12288, 10240, 1280), (8192, 8192, 8192)]:
        a = torch.randn(M, K, device=DEV).half()
        w = torch.randn(N, K, device=DEV).half()
        out = torch.empty(M, N, device=DEV, dtype=torch.half)
        ms = timeit(lambda: ops.gemm(a, w, out=out))
        ms_t = timeit(lambda: torch.matmul(a, w.t(), out=out))
        print(f"gemm {M}x{N}x{K}: {ms:.3f} ms = {2*M*N*K/ms/1e9:.0f} TFLOP/s   (cuBLAS {ms_t:.3f} ms = {2*M*N*K/ms_t/1e9:.0f})")
    for (n, h, c, co) in [(48, 64, 320, 320), (48, 32, 640, 640), (48, 16, 1280, 1280), (48, 8, 1280, 1280)]:
        x = torch.randn(n * h * h, c, device=DEV).half()
        w = torch.randn(co, 9 * c, device=DEV).half()
        out = torch.empty(n * h * h, co, device=DEV, dtype=torch.half)
        ms = timeit(lambda: ops.conv3x3(x, w, n, h, h, out=out))
        fl = 2 * n * h * h * co * 9 * c
        xc = x.reshape(n, h, h, c).permute(0, 3, 1, 2).contiguous(memory_format=torch.channels_last)
        wc = w.reshape(co, 3, 3, c).permute(0, 3, 1, 2).contiguous(memory_format=torch.channels_last)
        ms_t = timeit(lambda: torch.nn.functional.conv2d(xc, wc, padding=1))
        print(f"conv3x3 n={n} {h}x{h} {c}->{co}: {ms:.3f} ms = {fl/ms/1e9:.0f} TFLOP/s   (cuDNN {ms_t:.3f} ms = {fl/ms_t/1e9:.0f})")
    for (n, lq, d, lb) in [(24, 4096, 40, 4096), (24, 4096, 40, 0), (24, 1024, 80, 1024), (24, 256, 160, 256)]:
        C = 8 * d
        qkv = torch.randn(n * lq, 3 * C, device=DEV).half()
        bkv = torch.randn(2, max(lb, 1), 2 * C, device=DEV).half()
        bi = torch.ones(n, dtype=torch.int32, device=DEV)
        out = torch.empty(n * lq, C, device=DEV, dtype=torch.half)
        if lb:
            fn = lambda: ops.attn_spatial(qkv[:, :C], qkv[:, C:2*C], qkv[:, 2*C:], n, lq, 8, bank_k=bkv[:, :, :C], bank_v=bkv[:, :, C:], bank_index=bi, out=out)
        else:
            fn = lambda: ops.attn_spatial(qkv[:, :C], qkv[:, C:2*C], qkv[:, 2*C:], n, lq, 8, out=out)
        ms = timeit(fn, 5)
        fl = 4 * n * lq * (lq + lb) * C
        print(f"attn_spatial n={n} lq={lq} d={d} lb={lb}: {ms:.3f} ms = {fl/ms/1e9:.0f} TFLOP/s")
    for (n, hw, c) in [(48, 4096, 320), (48, 1024, 640), (48, 256, 1280)]:
        x = torch.randn(n * hw, c, device=DEV).half()
        g = torch.ones(c, device=DEV).half()
        b = torch.zeros(c, device=DEV).half()
        out = torch.empty_like(x)
        ms = timeit(lambda: ops.groupnorm(x, g, b, n, hw, silu=True, out=out))
        print(f"groupnorm n={n} hw={hw} c={c}: {ms:.3f} ms = {2*x.numel()*2/ms/1e6:.0f} GB/s (1R+1W algorithmic)")
        ms = timeit(lambda: ops.layernorm(x, g, b, out=out))
        print(f"layernorm rows={n*hw} c={c}: {ms:.3f} ms = {2*x.numel()*2/ms/1e6:.0f} GB/s")
    for (hw, d) in [(4096, 40), (1024, 80), (256, 160)]:
        C = 8 * d
        qkv = torch.randn(48 * hw, 3 * C, device=DEV).half()
        out = torch.empty(48 * hw, C, device=DEV, dtype=torch.half)
        ms = timeit(lambda: ops.attn_temporal(qkv[:, :C], qkv[:, C:2*C], qkv[:, 2*C:], 2, 24, hw, 8, out=out))
        print(f"attn_temporal hw={hw} d={d}: {ms:.3f} ms = {4*48*hw*C*2/ms/1e6:.0f} GB/s")
    return True


def _oracle():
    from oracle import torch_oracle as O
    return O


def _unet_parity(cfg_widths, f, hw, seed, taps=True, tol=3e-2):
    """engine (fp16 kernels) vs oracle (fp32 torch on the GPU, TF32 off) on one CFG window, block by block."""
    from mimo_b200 import engine as E
    O = _oracle()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cfg = O.UNetConfig(block_out_channels=cfg_widths)
    sd_den = O.make_denoising_unet_sd(cfg, seed=seed)
    sd_ref = O.make_reference_unet_sd(cfg, seed=seed + 1)
    sd_pg = O.make_pose_guider_sd(seed=seed + 2, out_channels=cfg.block_out_channels[0])
    g = torch.Generator().manual_seed(seed + 10)
    ref_lat = torch.randn(1, 4, hw, hw, generator=g)
    emb = torch.randn(1, 1, cfg.cross_attention_dim, generator=g)
    ehs = torch.cat([torch.zeros_like(emb), emb])
    x = torch.randn(1, 8, f, hw, hw, generator=g).repeat(2, 1, 1, 1, 1)
    pose_img = torch.rand(1, 3, f, hw * 8, hw * 8, generator=g)
    t = 499
    dev = torch.device(DEV)
    # oracle: fp32 weights rounded to fp16 first (the engine stores fp16 weights), math in fp32
    r16 = lambda sd: {k: v.half().float().to(dev) for k, v in sd.items()}
    o_den, o_ref, o_pg = r16(sd_den), r16(sd_ref), r16(sd_pg)
    with torch.no_grad():
        banks = O.reference_unet_banks(o_ref, ref_lat.repeat(2, 1, 1, 1).half().float().to(dev), ehs.half().float().to(dev), cfg)
        pose_o = O.pose_guider(o_pg, pose_img.half().float().to(dev))
        O.TAPS = {} if taps else None
        want = O.denoising_unet(o_den, x.half().float().to(dev), t, ehs.half().float().to(dev),
                                pose_o.repeat(2, 1, 1, 1, 1), banks, cfg, cfg=True)
        otaps, O.TAPS = O.TAPS, None
    spec = E.UNetSpec(block_out_channels=cfg_widths)
    den = E.UNetEngine(sd_den, spec, dev)
    ref = E.UNetEngine(sd_ref, E.UNetSpec(block_out_channels=cfg_widths, in_channels=4, motion=False, out_head=False), dev)
    pg = E.PoseGuiderEngine(sd_pg, dev)
    ok = True
    pose_e = pg.forward(pose_img.half().to(dev))
    pose_e5 = pose_e.reshape(1, f, hw, hw, -1).permute(0, 4, 1, 2, 3)
    ok &= report("pose_guider engine", pose_e5, pose_o, tol=5e-3)
    ebanks = ref.write_banks(ref_lat.repeat(2, 1, 1, 1).half().to(dev), ehs.half().to(dev), den)
    # compare one projected bank against the oracle's bank features pushed through the reader's to_k
    p0 = den.xf_paths[0]
    C0 = den.w[p0]["C"]
    wk = o_den[p0 + ".transformer_blocks.0.attn1.to_k.weight"]
    ok &= report(f"bank K {p0}", ebanks[p0][:, :, :C0], banks[p0].float() @ wk.t(), tol=5e-3)
    plast = [p for p in den.xf_paths if p.startswith("up_blocks")][-1]
    Cl = den.w[plast]["C"]
    wkl = o_den[plast + ".transformer_blocks.0.attn1.to_k.weight"]
    ok &= report(f"bank K {plast}", ebanks[plast][:, :, :Cl], banks[plast].float() @ wkl.t(), tol=3e-2)
    den.begin_clip(ehs.half().to(dev), ebanks, cfg=True, frames=f)
    den.taps = {} if taps else None
    pose_rep = pose_e.reshape(1, f * hw * hw, -1).repeat(2, 1, 1).reshape(2 * f * hw * hw, -1).contiguous()
    got = den.forward(x.half().to(dev), t, pose_rep)
    torch.cuda.synchronize()
    if taps:
        for name, ov in otaps.items():
            if name in den.taps:
                e = rel_err(den.taps[name], ov)
                flag = "" if e < tol else "   <<<<<<"
                print(f"    tap {name:40s} rel_l2={e:.3e}{flag}")
                ok &= e < tol  # every block output is held to the same bound as the network output
    ok &= report(f"denoising_unet widths={cfg_widths} f={f} latent={hw}", got, want, tol=tol)
    return ok


def unet_small():
    return _unet_parity((128, 256, 512, 512), f=4, hw=16, seed=100)


def unet_full():
    return _unet_parity((320, 640, 1280, 1280), f=4, hw=32, seed=400)


def vae_parity():
    from mimo_b200 import engine as E
    O = _oracle()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device(DEV)
    ok = True
    for widths, hw, n in [((32, 64, 128, 128), 16, 2), ((128, 256, 512, 512), 32, 2)]:
        if widths[0] < 128:
            continue  # 32 groups need >= 4 channels per group in the GN kernel
        cfg = O.VAEConfig(block_out_channels=widths)
        sd = O.make_vae_sd(cfg, seed=7)
        z = torch.randn(n, 4, hw, hw, generator=torch.Generator().manual_seed(8)) * 3
        o_sd = {k: v.half().float().to(dev) for k, v in sd.items()}
        with torch.no_grad():
            want = O.vae_decode(o_sd, z.half().float().to(dev), cfg)
        eng = E.VAEDecoderEngine(sd, dev)
        got = eng.decode(z.half().to(dev))
        torch.cuda.synchronize()
        ok &= report(f"vae_decode widths={widths} latent={hw}", got, want, tol=2e-2)
    return ok


CHECKS = {f.__name__: f for f in [unet_small, unet_full, vae_parity,gemm_basic, gemm_shapes, gemm_persistent, gemm_epilogue, conv_basic, conv_shapes,
                                  norms, temporal, spatial_basic, spatial_shapes, elementwise, perf]}

if __name__ == "__main__":
    names = sys.argv[1:]
    if names == ["list"]:
        print(" ".join(CHECKS))
        sys.exit(0)
    L.check(L.load().mimo_device_check(0), "device check")
    allok = True
    for nm in names:
        t0 = time.time()
        try:
            ok = CHECKS[nm]()
            torch.cuda.synchronize()
        except Exception as e:  # noqa: BLE001
            ok = False
            print(f"[EXC ] {nm}: {type(e).__name__}: {e}")
        print(f"== {nm}: {'PASS' if ok else 'FAIL'} ({time.time()-t0:.1f}s)")
        allok &= ok
    sys.exit(0 if allok else 1)
