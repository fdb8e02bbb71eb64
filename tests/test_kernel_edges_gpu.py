"""Kernel edges on an H100: every kernel family against a plain high-precision PyTorch reference of the same operation,
on the same rounded inputs, in fp16 and bf16, at the shapes and inputs where kernels go wrong.

Comparisons:
  exact(got, ref64)     bit-equality with the fp64 result rounded once to the output type. Used where every input is a
                        small integer, so that every fp32 partial sum is an exact integer below 2**24 and the kernel
                        rounds only once (GEMM, convolutions, their epilogues, split-K).
  close(got, ref, tol)  rel-L2 <= tol over the whole output AND <= 4 tol in every row (every 128-element chunk of a 1-D
                        output), so that one wrong row, ragged tail or tile cannot hide in a large output. Rows whose
                        reference norm is negligible must instead have an absolute error below 4 tol x the RMS row norm.
  tol_for(lo, ref64)    for results that cannot be exact: max(2e-3, 2 x rel-L2 of PyTorch computing the same operation in
                        the same storage type), the contract test_parity_gpu.py uses.
  tol_rounded(ref64, dt) for GroupNorm and LayerNorm: max(2e-3, 2 x rel-L2 of the exact result rounded to the storage
                        type). PyTorch's own fp16 / bf16 group_norm on an H100 is off by 4e-3 .. 1e-2 rel-L2 once the
                        mean is 30 .. 1000 std (measured), so its error would excuse a kernel that cancels digits.
Inputs hit the weak spots: ragged M / N / K, strided views whose margins hold a sentinel that must survive, softmax
logits with std 10-30 whose maximum arrives in the last tile, GroupNorm / LayerNorm inputs whose mean is up to 1000x
their standard deviation.
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = "cuda"
DTYPES = [torch.float16, torch.bfloat16]
FLOOR = 2e-3
SENTINEL = -77.0  # exact in fp16 and bf16, and far from every value the kernels write here


def _dn(dt):
    return "f16" if dt == torch.float16 else "bf16"


@pytest.fixture(scope="module", autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device: the product path has no CPU fallback")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


@pytest.fixture(scope="module")
def lib():
    from mimo_b200 import lib as L
    return L.load()


@pytest.fixture(scope="module")
def ops():
    from mimo_b200 import ops as O
    return O


@pytest.fixture(scope="module")
def L():
    from mimo_b200 import lib as L_
    return L_


# ------------------------------------------------------------------------------------------------
# comparison helpers
# ------------------------------------------------------------------------------------------------
def _rows(t):
    t = t.double()
    if t.dim() == 1:
        t = F.pad(t, (0, (-t.numel()) % 128)).reshape(-1, 128)
    return t.reshape(t.shape[0], -1)


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _worst(name, g, r):
    d = (g - r).abs()
    rn = r.norm(dim=1).clamp_min(1e-30)
    row_err = (g - r).norm(dim=1) / rn
    cn = r.norm(dim=0).clamp_min(1e-30)
    col_err = (g - r).norm(dim=0) / cn
    rows = torch.argsort(row_err, descending=True)[:8]
    cols = torch.argsort(col_err, descending=True)[:8]
    print(f"       {name}: max_abs={float(d.max()):.3e} nan={int(torch.isnan(g).sum())}")
    print(f"       worst rows: {[(int(i), round(float(row_err[i]), 5)) for i in rows]}")
    print(f"       worst cols: {[(int(i), round(float(col_err[i]), 5)) for i in cols]}")
    i = int(rows[0])
    print(f"       got[{i}, :8] = {g[i, :8].tolist()}")
    print(f"       ref[{i}, :8] = {r[i, :8].tolist()}")


def exact(got, ref64, name=""):
    """Bit-equality with the fp64 reference rounded once to got's type."""
    want = ref64.to(got.dtype)
    ok = torch.equal(got, want)
    if not ok:
        bad = got.double() != want.double()
        print(f"[FAIL] {name}: not bit-exact, {int(bad.sum())}/{bad.numel()} elements differ")
        _worst(name, _rows(got), _rows(want))
    return ok


def close(got, ref, tol, name=""):
    """Global rel-L2 <= tol and per-row rel-L2 <= 4 tol (rows with a non-negligible reference norm)."""
    g, r = _rows(got), _rows(ref)
    diff = (g - r).norm(dim=1)
    rn = r.norm(dim=1)
    rms = float(rn.pow(2).mean().sqrt())
    keep = rn > 1e-3 * rms
    e = float((g - r).norm() / (r.norm() + 1e-30))
    per = torch.where(keep, diff / rn.clamp_min(1e-30), torch.zeros_like(diff))
    worst = float(per.max())
    small_ok = bool((diff[~keep] <= 4 * tol * rms).all())
    ok = math.isfinite(e) and bool(torch.isfinite(g).all()) and e <= tol and worst <= 4 * tol and small_ok
    print(f"[{' ok ' if ok else 'FAIL'}] {name}: rel_l2={e:.3e} worst_row={worst:.3e} tol={tol:.2e}")
    if not ok:
        _worst(name, g, r)
    return ok


def tol_for(lo, ref64):
    """max(floor, 2 x the error of PyTorch computing the same operation in the same storage type)."""
    return max(FLOOR, 2.0 * _rel(lo, ref64))


def tol_rounded(ref64, dtype):
    """max(floor, 2 x the error of rounding the exact result to the storage type)."""
    return max(FLOOR, 2.0 * _rel(ref64.to(dtype), ref64))


def padded(rows, cols, dtype, lpad=8, rpad=24):
    """A sentinel-filled [rows, lpad + cols + rpad] buffer and its [rows, cols] column view (ld > cols)."""
    buf = torch.full((rows, lpad + cols + rpad), SENTINEL, dtype=dtype, device=DEV)
    return buf, buf[:, lpad:lpad + cols]


def margins_intact(buf, cols, lpad=8):
    ok = bool((buf[:, :lpad] == SENTINEL).all()) and bool((buf[:, lpad + cols:] == SENTINEL).all())
    if not ok:
        print("[FAIL] a kernel wrote outside its output view")
    return ok


def ints(shape, dtype, lo=-3, hi=4):
    return torch.randint(lo, hi, shape, device=DEV).to(dtype)


def col_slice(rows, cols, dtype, off, extra):
    """Integer [rows, cols] view at column `off` of a [rows, cols + extra] tensor (ld > cols)."""
    return ints((rows, cols + extra), dtype)[:, off:off + cols]


# ------------------------------------------------------------------------------------------------
# GEMM (gemm_wgmma.cu): bit-exact on integer inputs
# ------------------------------------------------------------------------------------------------
BNS = [0, 64, 128, 160, 192, 256]  # 0: the automatic choice


def _gemm_ref(a, w, a1=None, bias=None, rv=None, rpg=1, res=None, scale=1.0):
    aa = a.double() if a1 is None else torch.cat([a.double(), a1.double()], 1)
    y = aa @ w.double().t()
    if bias is not None:
        y = y + bias.double()
    if rv is not None:
        y = y + rv.double()[torch.arange(a.shape[0], device=DEV) // rpg]
    if res is not None:
        y = y + res.double()
    return y * scale


@pytest.mark.parametrize("dtype", DTYPES, ids=_dn)
@pytest.mark.parametrize("bn", BNS)
def test_gemm_ragged_exact(lib, ops, bn, dtype):
    """M not a multiple of 128, N not a multiple of BN, K not a multiple of 64; accumulators stored as they are."""
    torch.manual_seed(10 + bn)
    ok = True
    lib.mimo_debug_force_bn(bn)
    try:
        for M, N, K in [(300, 328, 200), (1, 8, 8), (129, 136, 72), (77, 264, 584)]:
            a, w = ints((M, K), dtype), ints((N, K), dtype)
            ok &= exact(ops.gemm(a, w), _gemm_ref(a, w), f"gemm {M}x{N}x{K} bn={bn} {_dn(dtype)}")
    finally:
        lib.mimo_debug_force_bn(0)
    assert ok


@pytest.mark.parametrize("dtype", DTYPES, ids=_dn)
@pytest.mark.parametrize("scale", [1.0, 0.5])
@pytest.mark.parametrize("bn", BNS)
def test_gemm_epilogue_strided_exact(lib, ops, bn, scale, dtype):
    """bias + row vector (rows_per_group 100, ld_rowvec > N as engine.py passes tembs[:, off:off + cout]) + residual
    (ld_res > N), a as a column slice (lda > K), out as a column slice of a sentinel-filled buffer."""
    torch.manual_seed(20 + bn)
    M, N, K, rpg = 300, 328, 200, 100
    a = col_slice(M, K, dtype, 8, 24)
    w = ints((N, K), dtype)
    bias = ints((N,), dtype)
    rv = col_slice(3, N, dtype, 32, 64)
    res = col_slice(M, N, dtype, 16, 40)
    buf, out = padded(M, N, dtype)
    lib.mimo_debug_force_bn(bn)
    try:
        ops.gemm(a, w, out=out, bias=bias, rowvec=rv, rows_per_group=rpg, residual=res, scale=scale)
    finally:
        lib.mimo_debug_force_bn(0)
    ok = exact(out, _gemm_ref(a, w, bias=bias, rv=rv, rpg=rpg, res=res, scale=scale), f"gemm epilogue bn={bn} s={scale}")
    assert margins_intact(buf, N) and ok


@pytest.mark.parametrize("dtype", DTYPES, ids=_dn)
@pytest.mark.parametrize("k0", [8, 56, 64, 72, 120])
def test_gemm_two_sources_exact(lib, ops, k0, dtype):
    """[a0 | a1] with the split at K0: the first source's K tail must not leak into the second's K blocks."""
    torch.manual_seed(30 + k0)
    M, N, K1 = 260, 200, 136
    a0 = ints((M, k0), dtype)
    a1 = col_slice(M, K1, dtype, 8, 16)
    w = ints((N, k0 + K1), dtype)
    bias = ints((N,), dtype)
    res = ints((M, N), dtype)
    ok = True
    for bn in (0, 64, 192):
        lib.mimo_debug_force_bn(bn)
        try:
            got = ops.gemm(a0, w, a1=a1, bias=bias, residual=res)
        finally:
            lib.mimo_debug_force_bn(0)
        ok &= exact(got, _gemm_ref(a0, w, a1=a1, bias=bias, res=res), f"gemm [{k0}|{K1}] bn={bn}")
    assert ok


@pytest.mark.parametrize("dtype", DTYPES, ids=_dn)
def test_gemm_persistent_wrap_exact(ops, dtype):
    """Several times more output tiles than SMs: every persistent CTA runs many tiles, so the operand / residual rings
    and the accumulator hand-off wrap their barrier phases many times."""
    torch.manual_seed(40)
    M, N, K = 128 * 150 + 37, 264, 200
    a, w = ints((M, K), dtype), ints((N, K), dtype)
    bias, res = ints((N,), dtype), ints((M, N), dtype)
    rv = ints((7, N), dtype)
    ok = exact(ops.gemm(a, w), _gemm_ref(a, w), "gemm persistent plain")
    ok &= exact(ops.gemm(a, w, bias=bias, rowvec=rv, rows_per_group=3000, residual=res, scale=0.5),
                _gemm_ref(a, w, bias=bias, rv=rv, rpg=3000, res=res, scale=0.5), "gemm persistent epilogue")
    assert ok


@pytest.mark.parametrize("dtype", DTYPES, ids=_dn)
def test_gemm_split_k_exact(lib, ops, dtype):
    """Split-K (fp32 partials in the workspace, then the reduce kernel applies the epilogue): bit-exact with the whole
    strided epilogue, bit-identical run to run."""
    torch.manual_seed(50)
    M, N, K, rpg = 200, 328, 2056, 75  # 2 x 2 tiles, 33 K blocks: two splits
    a = col_slice(M, K, dtype, 8, 24)
    w = ints((N, K), dtype)
    bias = ints((N,), dtype)
    rv = col_slice(3, N, dtype, 32, 64)
    res = col_slice(M, N, dtype, 16, 40)
    buf, out = padded(M, N, dtype)
    ws = ops._workspace(a.device)
    ws.zero_()
    lib.mimo_debug_splitk(1)
    try:
        ops.gemm(a, w, out=out, bias=bias, rowvec=rv, rows_per_group=rpg, residual=res, scale=0.5)
        again = ops.gemm(a, w, bias=bias, rowvec=rv, rows_per_group=rpg, residual=res, scale=0.5)
    finally:
        lib.mimo_debug_splitk(0)
    torch.cuda.synchronize()
    assert bool(ws.any()), "split-K was not taken: the workspace holds no partials"
    ok = exact(out, _gemm_ref(a, w, bias=bias, rv=rv, rpg=rpg, res=res, scale=0.5), "split-K gemm")
    assert margins_intact(buf, N) and ok and torch.equal(out, again)


@pytest.mark.parametrize("dtype", DTYPES, ids=_dn)
def test_conv_split_k_exact(lib, ops, dtype):
    torch.manual_seed(51)
    n, h, w, c0, c1, co = 2, 8, 8, 160, 160, 320  # 1 x 2 tiles, 45 K blocks: two splits
    x0, x1 = ints((n, c0, h, w), dtype), ints((n, c1, h, w), dtype)
    W = ints((co, c0 + c1, 3, 3), dtype)
    bias, tv, res = ints((co,), dtype), col_slice(n, co, dtype, 8, 16), col_slice(n * h * w, co, dtype, 8, 8)
    ws = ops._workspace(x0.device)
    ws.zero_()
    lib.mimo_debug_splitk(1)
    try:
        got = ops.conv3x3(_nhwc(x0), ops.pack_conv3x3_weight(W, cin_pad=c0 + c1), n, h, w, x1=_nhwc(x1), bias=bias,
                          rowvec=tv, rows_per_group=h * w, residual=res)
    finally:
        lib.mimo_debug_splitk(0)
    torch.cuda.synchronize()
    assert bool(ws.any()), "split-K was not taken: the workspace holds no partials"
    assert exact(got, _conv_ref(torch.cat([x0, x1], 1), W, bias, tv, h * w, res), "split-K conv")


@pytest.mark.parametrize("dtype", DTYPES, ids=_dn)
def test_gemm_silu_geglu(L, ops, dtype):
    """SiLU and GEGLU epilogues are not exact: rel-L2 against fp64 within twice PyTorch's own error in the same type."""
    torch.manual_seed(60)
    M, K = 300, 320
    a = torch.randn(M, K, device=DEV).to(dtype)
    w = (torch.randn(1280, K, device=DEV) / math.sqrt(K)).to(dtype)
    b = torch.randn(1280, device=DEV).to(dtype)
    ref = F.silu(a.double() @ w.double().t() + b.double())
    lo = F.silu(a @ w.t() + b)
    ok = close(ops.gemm(a, w, bias=b, act=L.ACT_SILU), ref, tol_for(lo, ref), f"gemm+silu {_dn(dtype)}")
    w2 = (torch.randn(2 * 1280, K, device=DEV) / math.sqrt(K)).to(dtype)
    b2 = torch.randn(2 * 1280, device=DEV).to(dtype)
    wp, bp = ops.pack_geglu_weight(w2, b2)
    hv, gate = (a.double() @ w2.double().t() + b2.double()).chunk(2, dim=-1)
    ref = hv * F.gelu(gate)
    hl, gl = (a @ w2.t() + b2).chunk(2, dim=-1)
    lo = hl * F.gelu(gl)
    ok &= close(ops.gemm(a, wp, bias=bp, act=L.ACT_GEGLU), ref, tol_for(lo, ref), f"gemm+geglu {_dn(dtype)}")
    assert ok


# ------------------------------------------------------------------------------------------------
# 3x3 convolution and the fused nearest-x2 upsample + conv: bit-exact on integer inputs
# ------------------------------------------------------------------------------------------------
def _nhwc(x):
    n, c, h, w = x.shape
    return x.permute(0, 2, 3, 1).reshape(n * h * w, c).contiguous()


def _conv_ref(x, W, bias=None, rv=None, rpg=1, res=None):
    n, _, h, w = x.shape
    y = _nhwc(F.conv2d(x.double(), W.double(), None if bias is None else bias.double(), padding=1))
    if rv is not None:
        y = y + rv.double()[torch.arange(n * h * w, device=DEV) // rpg]
    if res is not None:
        y = y + res.double()
    return y


CONV_CASES = [  # n, h, w, c0, c1, cout
    (5, 1, 1, 64, 0, 64),      # 1x1 images: 8 of 9 taps are padding, 5 images share a tile
    (3, 1, 3, 64, 0, 72),
    (3, 3, 1, 64, 0, 72),
    (4, 2, 2, 72, 0, 64),
    (1, 3, 130, 64, 0, 64),    # w > 128: a tile row is 128 pixels, the second is ragged
    (3, 5, 7, 64, 0, 136),     # n*h*w = 105, not a multiple of 128
    (2, 9, 11, 64, 72, 200),   # two sources, the second one's K ragged
]


@pytest.mark.parametrize("dtype", DTYPES, ids=_dn)
@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: "n{}_{}x{}_c{}+{}_o{}".format(*c))
def test_conv3x3_edges_exact(lib, ops, case, dtype):
    """Degenerate and ragged images, two sources, bias + per-image row vector (ld_rowvec > cout) + residual
    (ld_res > cout), out as a column slice of a sentinel-filled buffer; three tile widths."""
    n, h, w, c0, c1, co = case
    torch.manual_seed(n * 1000 + h * 31 + w)
    x0 = ints((n, c0, h, w), dtype)
    x1 = ints((n, c1, h, w), dtype) if c1 else None
    W = ints((co, c0 + c1, 3, 3), dtype)
    bias = ints((co,), dtype)
    tv = col_slice(n, co, dtype, 8, 16)
    res = col_slice(n * h * w, co, dtype, 8, 8)
    wp = ops.pack_conv3x3_weight(W, cin_pad=c0 + c1)
    x = x0 if x1 is None else torch.cat([x0, x1], 1)
    ref_plain = _conv_ref(x, W)
    ref = _conv_ref(x, W, bias, tv, h * w, res)
    ok = True
    for bn in (0, 64, 160):
        lib.mimo_debug_force_bn(bn)
        try:
            plain = ops.conv3x3(_nhwc(x0), wp, n, h, w, x1=None if x1 is None else _nhwc(x1))
            buf, out = padded(n * h * w, co, dtype)
            ops.conv3x3(_nhwc(x0), wp, n, h, w, out=out, x1=None if x1 is None else _nhwc(x1), bias=bias, rowvec=tv,
                        rows_per_group=h * w, residual=res)
        finally:
            lib.mimo_debug_force_bn(0)
        ok &= exact(plain, ref_plain, f"conv3x3 {case} bn={bn}") and exact(out, ref, f"conv3x3+epilogue {case} bn={bn}")
        ok &= margins_intact(buf, co)
    assert ok


@pytest.mark.parametrize("dtype", DTYPES, ids=_dn)
@pytest.mark.parametrize("hw", [(1, 1), (1, 5), (3, 2)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_conv_up2x_small_exact(ops, hw, dtype):
    """Nearest-x2 upsample + 3x3 conv on tiny sources; the pre-summed parity-class weights are exact on integers."""
    h, w = hw
    n, cin, co = 2, 64, 72
    torch.manual_seed(70 + h * 10 + w)
    x = ints((n, cin, h, w), dtype)
    W = ints((co, cin, 3, 3), dtype)
    b = ints((co,), dtype)
    ref = _nhwc(F.conv2d(F.interpolate(x.double(), scale_factor=2.0, mode="nearest"), W.double(), b.double(), padding=1))
    got = ops.conv_up2x(_nhwc(x), ops.pack_conv_up2x_weight(W), n, h, w, bias=b)
    assert exact(got, ref, f"conv_up2x {h}x{w}")


# ------------------------------------------------------------------------------------------------
# spatial attention (attn_spatial.cu): fp64 reference, checked per query row
# ------------------------------------------------------------------------------------------------
SHARP_S, SHARP_MU = 3.0, 3.0  # q = 3 randn + 3, k = 3 randn: logits (default scale) have std ~ 12.7
PLANT_GAP = 40.0               # a planted key's logit exceeds the others' mean by ~40


def _spatial_inputs(n, lq, heads, d, dtype, lb=0, nb=0, sharp=True, plant=None, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    C = heads * d
    s, mu = (SHARP_S, SHARP_MU) if sharp else (1.0, 0.0)
    qkv = torch.randn(n * lq, 3 * C, device=DEV, generator=g)
    qkv[:, :C] = qkv[:, :C] * s + mu
    qkv[:, C:2 * C] *= s
    bkv = None
    if lb:
        bkv = torch.randn(nb, lb, 2 * C, device=DEV, generator=g)
        bkv[..., :C] *= s
    if plant is not None:
        kappa = PLANT_GAP / (mu * math.sqrt(d))
        if plant == "bank_last":
            bkv[:, lb - 1, :C] += kappa
        else:  # a key of the last self tile, or the last (ragged tail) key
            j = lq - 1 if plant == "tail" else min((lq - 1) // 128 * 128 + 3, lq - 1)
            qkv.view(n, lq, 3 * C)[:, j, C:2 * C] += kappa
    qkv = qkv.to(dtype)
    return qkv, (bkv.to(dtype) if bkv is not None else None)


def _spatial_ref(qkv, bkv, bidx, n, lq, heads, d, scale, fp64):
    C = heads * d
    q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    outs = []
    hd = lambda t: t.reshape(1, -1, heads, d).transpose(1, 2)  # [1, heads, L, d]
    for i in range(n):
        sl = slice(i * lq, (i + 1) * lq)
        qi, ki, vi = hd(q[sl]), hd(k[sl]), hd(v[sl])
        if bkv is not None and bidx[i] >= 0:
            ki = torch.cat([ki, hd(bkv[bidx[i], :, :C])], 2)
            vi = torch.cat([vi, hd(bkv[bidx[i], :, C:])], 2)
        if fp64:
            p = torch.softmax((qi.double() @ ki.double().transpose(-1, -2)) * scale, -1)
            o = p @ vi.double()
        else:
            o = F.scaled_dot_product_attention(qi, ki, vi, scale=scale)
        outs.append(o.transpose(1, 2).reshape(lq, C))
    return torch.cat(outs)


def _spatial_check(ops, n, lq, heads, d, dtype, lb=0, nb=0, bidx=None, scale=None, plant=None, sharp=True, seed=0):
    C = heads * d
    qkv, bkv = _spatial_inputs(n, lq, heads, d, dtype, lb, nb, sharp, plant, seed)
    bank = {}
    if lb:
        bank = dict(bank_k=bkv[:, :, :C], bank_v=bkv[:, :, C:],
                    bank_index=torch.tensor(bidx, dtype=torch.int32, device=DEV))
    buf, out = padded(n * lq, C, dtype, lpad=8, rpad=32)  # ld_out = C + 40
    ops.attn_spatial(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], n, lq, heads, scale=scale, out=out, **bank)
    sc = scale if scale is not None else d ** -0.5
    ref = _spatial_ref(qkv, bkv, bidx, n, lq, heads, d, sc, True)
    lo = _spatial_ref(qkv, bkv, bidx, n, lq, heads, d, sc, False)
    name = f"attn_spatial n={n} lq={lq} h={heads} d={d} lb={lb} plant={plant} scale={scale} {_dn(dtype)}"
    ok = close(out, ref, tol_for(lo, ref), name)
    return margins_intact(buf, C) and ok


# one head dim per instantiation DP = round_up(d, 16) = 16 ... 192, non-multiples of 16 included; 152 | 168 straddle
# the switch from two MMA warpgroups to one at DP = 160
SPATIAL_DS = [8, 24, 40, 56, 72, 88, 104, 120, 136, 152, 168, 184, 192]


@pytest.mark.parametrize("dtype", DTYPES, ids=_dn)
@pytest.mark.parametrize("d", SPATIAL_DS)
def test_attn_spatial_head_dims(ops, d, dtype):
    """Sharp logits, 3 banks with a permuted bank_index holding -1, ragged self / bank tiles, ld_out > C."""
    assert _spatial_check(ops, 4, 200, 2, d, dtype, lb=150, nb=3, bidx=[2, -1, 0, 1], seed=d)


@pytest.mark.parametrize("dtype", DTYPES, ids=_dn)
@pytest.mark.parametrize("d", [40, 160])
@pytest.mark.parametrize("plant", ["self_last", "tail", "bank_last"])
def test_attn_spatial_late_max(ops, plant, d, dtype):
    """Each row's largest logit sits in the last self tile, on the ragged tail key, or in the last bank tile, so the
    running max rises late and the earlier tiles' O and l must be rescaled by alpha."""
    assert _spatial_check(ops, 3, 300, 2, d, dtype, lb=200, nb=2, bidx=[1, 0, -1], plant=plant, seed=7)


@pytest.mark.parametrize("dtype", DTYPES, ids=_dn)
def test_attn_spatial_scale(ops, dtype):
    assert _spatial_check(ops, 2, 260, 2, 64, dtype, lb=130, nb=2, bidx=[1, 0], scale=0.3, seed=8)
    assert _spatial_check(ops, 2, 260, 2, 64, dtype, lb=130, nb=2, bidx=[1, 0], scale=0.05, sharp=False, seed=9)


@pytest.mark.parametrize("dtype", DTYPES, ids=_dn)
@pytest.mark.parametrize("lb", [1, 127, 129])
def test_attn_spatial_bank_lengths(ops, lb, dtype):
    assert _spatial_check(ops, 3, 130, 2, 40, dtype, lb=lb, nb=2, bidx=[1, -1, 0], plant="bank_last", seed=lb)


@pytest.mark.parametrize("dtype", DTYPES, ids=_dn)
@pytest.mark.parametrize("d", [40, 160])
@pytest.mark.parametrize("lq", [1, 65, 129])
def test_attn_spatial_query_lengths(ops, lq, d, dtype):
    assert _spatial_check(ops, 2, lq, 2, d, dtype, lb=100, nb=2, bidx=[1, 0], plant="tail", seed=lq)


# ------------------------------------------------------------------------------------------------
# temporal attention (attn_temporal.cu)
# ------------------------------------------------------------------------------------------------
def _temporal_ref(q, k, v, b, fq, fk, hw, heads, d, scale, fp64):
    def tr(t, f):  # (b f) p (h d) -> b p h f d
        return t.reshape(b, f, hw, heads, d).permute(0, 2, 3, 1, 4)
    qt, kt, vt = tr(q, fq), tr(k, fk), tr(v, fk)
    if fp64:
        o = torch.softmax((qt.double() @ kt.double().transpose(-1, -2)) * scale, -1) @ vt.double()
    else:
        o = F.scaled_dot_product_attention(qt, kt, vt, scale=scale)
    return o.permute(0, 3, 1, 2, 4).reshape(b * fq * hw, heads * d)


def _sharp_qkv(rows, C, dtype, seed, frames_view=None, plant_frame=None, d=None):
    g = torch.Generator(device=DEV).manual_seed(seed)
    qkv = torch.randn(rows, 3 * C, device=DEV, generator=g)
    qkv[:, :C] = qkv[:, :C] * SHARP_S + SHARP_MU
    qkv[:, C:2 * C] *= SHARP_S
    if plant_frame is not None:
        b, f, hw = frames_view
        qkv.view(b, f, hw, 3 * C)[:, plant_frame, :, C:2 * C] += 20.0 / (SHARP_MU * math.sqrt(d))
    return qkv.to(dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=_dn)
@pytest.mark.parametrize("hd", [(8, 40), (8, 80), (8, 160), (32, 256)], ids=lambda t: f"h{t[0]}d{t[1]}")
@pytest.mark.parametrize("frames", [2, 31, 32])
def test_attn_temporal_edges(ops, frames, hd, dtype):
    """Sharp logits, the last frame's keys raised; up to the 32-frame / 32-head / d = 256 limits; ld_out > C."""
    heads, d = hd
    b, hw = 2, 6
    C = heads * d
    qkv = _sharp_qkv(b * frames * hw, C, dtype, seed=frames + d, frames_view=(b, frames, hw), plant_frame=frames - 1, d=d)
    q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    buf, out = padded(b * frames * hw, C, dtype)
    ops.attn_temporal(q, k, v, b, frames, hw, heads, out=out)
    sc = d ** -0.5
    ref = _temporal_ref(q, k, v, b, frames, frames, hw, heads, d, sc, True)
    lo = _temporal_ref(q, k, v, b, frames, frames, hw, heads, d, sc, False)
    ok = close(out, ref, tol_for(lo, ref), f"attn_temporal F={frames} h={heads} d={d} {_dn(dtype)}")
    assert margins_intact(buf, C) and ok


@pytest.mark.parametrize("dtype", DTYPES, ids=_dn)
def test_attn_temporal_sharded(ops, dtype):
    """Frame-sharded form: this rank's q_frames queries against all kv_frames frames held in rank-major chunks."""
    b, f, hw, heads, d, world = 2, 24, 8, 8, 40, 4
    C, fl = heads * d, f // world
    q_full = _sharp_qkv(b * f * hw, C, dtype, seed=90)[:, :C].reshape(b, f, hw, C)
    kv_full = _sharp_qkv(b * f * hw, C, dtype, seed=91)[:, C:].reshape(b, f, hw, 2 * C)
    kv_chunks = torch.cat([kv_full[:, r * fl:(r + 1) * fl].reshape(b * fl * hw, 2 * C) for r in range(world)])
    ok = True
    for rk in (0, 2, world - 1):
        q = q_full[:, rk * fl:(rk + 1) * fl].reshape(b * fl * hw, C).contiguous()
        out = ops.attn_temporal(q, kv_chunks[:, :C], kv_chunks[:, C:], b, f, hw, heads, q_frames=fl,
                                frames_per_chunk=fl, chunk_stride_rows=b * fl * hw)
        k = kv_full[..., :C].reshape(b * f * hw, C)
        v = kv_full[..., C:].reshape(b * f * hw, C)
        sc = d ** -0.5
        ref = _temporal_ref(q, k, v, b, fl, f, hw, heads, d, sc, True)
        lo = _temporal_ref(q, k, v, b, fl, f, hw, heads, d, sc, False)
        ok &= close(out, ref, tol_for(lo, ref), f"attn_temporal sharded rank={rk} {_dn(dtype)}")
    assert ok


def test_attn_temporal_rejects_33_frames(L, ops):
    """33 frames exceed the kernel's limit; the entry point refuses before launching anything."""
    C = 8 * 40
    qkv = torch.zeros(33 * 4, 3 * C, dtype=torch.float16, device=DEV)
    with pytest.raises(L.MimoError, match="frames <= 32"):
        ops.attn_temporal(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], 1, 33, 4, 8)


# ------------------------------------------------------------------------------------------------
# GroupNorm / LayerNorm (norm.cu)
# ------------------------------------------------------------------------------------------------
def _gn_inputs(n, hw, C, ratio, dtype, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = (torch.randn(n * hw, C, device=DEV, generator=g) + ratio).to(dtype)  # std 1, mean = ratio
    gamma = (1 + 0.2 * torch.randn(C, device=DEV, generator=g)).to(dtype)
    beta = (0.2 * torch.randn(C, device=DEV, generator=g)).to(dtype)
    return x, gamma, beta


def _gn_ref(x, gamma, beta, n, hw, groups, eps, silu):
    C = x.shape[1]
    xt = x.double().reshape(n, hw, C).permute(0, 2, 1)
    y = F.group_norm(xt, groups, gamma.double(), beta.double(), eps)
    if silu:
        y = F.silu(y)
    return y.permute(0, 2, 1).reshape(n * hw, C)


def _gn_check(ops, n, hw, c0, c1, groups, ratio, dtype, silu=False, eps=1e-6):
    C = c0 + c1
    x, gamma, beta = _gn_inputs(n, hw, C, ratio, dtype, seed=hw + C + int(ratio))
    x0 = x[:, :c0].contiguous()
    x1 = x[:, c0:].contiguous() if c1 else None
    got = ops.groupnorm(x0, gamma, beta, n, hw, groups=groups, eps=eps, silu=silu, x1=x1)
    again = ops.groupnorm(x0, gamma, beta, n, hw, groups=groups, eps=eps, silu=silu, x1=x1)
    ref = _gn_ref(x, gamma, beta, n, hw, groups, eps, silu)
    name = f"groupnorm n={n} hw={hw} c={c0}+{c1} g={groups} mean/std={ratio} {_dn(dtype)}"
    ok = close(got, ref, tol_rounded(ref, dtype), name)
    same = torch.equal(got, again)
    if not same:
        print(f"[FAIL] {name}: two runs differ")
    return ok and same


GN_CASES = [  # n, hw, c0, c1, groups
    (2, 1024, 320, 0, 32),
    (2, 256, 128, 0, 32),      # 4 channels per group: an 8-channel vector spans two groups
    (2, 256, 512, 0, 64),      # 64 groups
    (2, 256, 328, 312, 32),    # the x0 | x1 split falls inside group 16 (channels 320..339)
    (3, 1, 320, 0, 32),        # fewer pixels than the P pixel lanes of a block
    (3, 3, 320, 0, 32),
    (1, 4096, 320, 0, 32),     # 43 slabs per image: the four-part slab reduction
]


@pytest.mark.parametrize("dtype", DTYPES, ids=_dn)
@pytest.mark.parametrize("ratio", [0, 30, 300, 1000])
@pytest.mark.parametrize("case", GN_CASES, ids=lambda c: "n{}_hw{}_c{}+{}_g{}".format(*c))
def test_groupnorm_offset(ops, case, ratio, dtype):
    """Inputs whose mean is up to 1000x their std: the statistics must not cancel; two runs bit-identical."""
    assert _gn_check(ops, *case, ratio, dtype, silu=case[0] == 2)


@pytest.mark.parametrize("dtype", DTYPES, ids=_dn)
def test_groupnorm_vae_size(ops, dtype):
    """The VAE decoder's largest GroupNorm at 768x768: 128 channels, 589 824 pixels, 4096-pixel runs per thread."""
    assert _gn_check(ops, 1, 768 * 768, 128, 0, 32, 300, dtype, silu=True)


LN_CS = [320, 640, 1280, 8, 328, 2048]  # layernorm5 (320 / 640 / 1280) and the generic kernel


@pytest.mark.parametrize("dtype", DTYPES, ids=_dn)
@pytest.mark.parametrize("ratio", [0, 1000])
@pytest.mark.parametrize("C", LN_CS)
def test_layernorm_offset(ops, C, ratio, dtype):
    """Row counts that fill no block exactly, inputs with mean/std up to 1000."""
    rows = 1001
    g = torch.Generator(device=DEV).manual_seed(C + ratio)
    x = (torch.randn(rows, C, device=DEV, generator=g) + ratio).to(dtype)
    gamma = (1 + 0.2 * torch.randn(C, device=DEV, generator=g)).to(dtype)
    beta = (0.2 * torch.randn(C, device=DEV, generator=g)).to(dtype)
    ref = F.layer_norm(x.double(), (C,), gamma.double(), beta.double(), 1e-5)
    got = ops.layernorm(x, gamma, beta)
    assert close(got, ref, tol_rounded(ref, dtype), f"layernorm C={C} mean/std={ratio} {_dn(dtype)}")


@pytest.mark.parametrize("dtype", DTYPES, ids=_dn)
@pytest.mark.parametrize("C", [320, 328])
def test_layernorm_pe_frame_offset(ops, C, dtype):
    """LN + positional encoding with pe_frame_offset != 0 (the frame-sharded temporal path): frame f of the local rows
    takes encoding row offset + f. The reference rounds LN's output to the storage type before adding it."""
    b, f, hw, off = 2, 4, 12, 5
    g = torch.Generator(device=DEV).manual_seed(C)
    x = (3 * torch.randn(b * f * hw, C, device=DEV, generator=g) + 1).to(dtype)
    gamma = (1 + 0.2 * torch.randn(C, device=DEV, generator=g)).to(dtype)
    beta = (0.2 * torch.randn(C, device=DEV, generator=g)).to(dtype)
    pe = torch.randn(32, C, device=DEV, generator=g).to(dtype)
    pe_rows = pe[off:off + f].repeat_interleave(hw, 0).repeat(b, 1)
    ref = F.layer_norm(x.double(), (C,), gamma.double(), beta.double(), 1e-5).to(dtype).double() + pe_rows.double()
    got = ops.layernorm(x, gamma, beta, pe=pe, rows_per_frame=hw, frames=f, pe_frame_offset=off)
    assert close(got, ref, tol_rounded(ref, dtype), f"layernorm+pe offset={off} C={C} {_dn(dtype)}")


# ------------------------------------------------------------------------------------------------
# small kernels (elementwise.cu)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=_dn)
@pytest.mark.parametrize("cols", [8, 4096, 9216])
def test_softmax_rows_sharp_strided(ops, cols, dtype):
    """Logits with std 25, rows of a wider buffer (ld > cols) whose margins must survive; 9216 is the VAE mid-block
    attention at 768x768."""
    rows = 37
    g = torch.Generator(device=DEV).manual_seed(cols)
    buf, x = padded(rows, cols, dtype)
    x.copy_(25 * torch.randn(rows, cols, device=DEV, generator=g))
    ref = torch.softmax(x.double(), -1)
    lo = torch.softmax(x, -1)
    ops.softmax_rows_(x)
    ok = close(x, ref, tol_for(lo, ref), f"softmax_rows cols={cols} {_dn(dtype)}")
    assert margins_intact(buf, cols) and ok


@pytest.mark.parametrize("with_counter", [False, True], ids=["plain", "counter"])
def test_cfg_ddim_step_bf16(ops, with_counter):
    """bf16 CFG + DDIM update against the same torch expression in bf16. The fp16 test's bound (2e-3) is scaled by the
    ratio of the two types' unit roundoff (2^-8 / 2^-11 = 8)."""
    from oracle import torch_oracle as O
    dt = torch.bfloat16
    torch.manual_seed(11)
    F_, h, w = 5, 8, 8
    lat = torch.randn(1, 4, F_, h, w, device=DEV).to(dt)
    pred = torch.randn(2, 4, F_, h, w, device=DEV).to(dt)
    counter = torch.tensor([1, 2, 1, 3, 2], device=DEV).to(dt)
    d = O.DDIM()
    d.set_timesteps(20)
    for t in (999, 499, 49):
        co = d.coefficients(t)
        if with_counter:
            cv = counter.view(1, F_, 1, 1)
            got = ops.cfg_ddim_step(pred[0] * cv, pred[1] * cv, lat.clone(), 3.5, *co, counter=counter,
                                    frame_stride=h * w)
            u, c = ((pred * counter.view(1, 1, F_, 1, 1)) / counter.view(1, 1, F_, 1, 1)).chunk(2)
        else:
            got = ops.cfg_ddim_step(pred[0].contiguous(), pred[1].contiguous(), lat.clone(), 3.5, *co)
            u, c = pred.chunk(2)
        want = d.step(u + 3.5 * (c - u), t, lat)
        assert want.dtype == dt
        diff = float((got.float() - want.float()).abs().max())
        assert diff <= 8 * 2e-3, (t, diff)


@pytest.mark.parametrize("numel", [1, 7, 4097])
def test_elementwise_rejects_partial_vectors(L, ops, numel):
    """add / silu / quick_gelu work on whole 8-element vectors; other counts are refused before any launch."""
    x = torch.zeros(numel, dtype=torch.bfloat16, device=DEV)
    for fn in (lambda: ops.add(x, x), lambda: ops.silu(x), lambda: ops.quick_gelu(x)):
        with pytest.raises(L.MimoError, match="bad arguments"):
            fn()


@pytest.mark.parametrize("numel", [8, 4104, 132 * 16 * 256 * 8 + 8])  # the last one wraps the grid-stride loop
def test_elementwise_bf16(ops, numel):
    dt = torch.bfloat16
    g = torch.Generator(device=DEV).manual_seed(numel)
    a = (torch.randint(-64, 64, (numel,), device=DEV, generator=g) / 8).to(dt)  # sums exact in bf16
    b = (torch.randint(-64, 64, (numel,), device=DEV, generator=g) / 8).to(dt)
    ok = exact(ops.add(a, b), a.double() + b.double(), f"add n={numel}")
    x = (3 * torch.randn(numel, device=DEV, generator=g)).to(dt)
    ref = F.silu(x.double())
    ok &= close(ops.silu(x), ref, tol_for(F.silu(x), ref), f"silu n={numel}")
    ref = x.double() * torch.sigmoid(1.702 * x.double())
    lo = x * torch.sigmoid(1.702 * x)
    ok &= close(ops.quick_gelu(x), ref, tol_for(lo, ref), f"quick_gelu n={numel}")
    assert ok
