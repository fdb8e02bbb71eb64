"""Launch each hot kernel a few times at hot-path shapes so that `ncu -k regex:<name>` can capture it in isolation
(GPU box only):   ncu --set full --clock-control none --import-source on -k regex:attn_spatial -s 2 -c 1 \
                      -o attn python scripts/ncu_kernels.py attn
"""
from __future__ import annotations

import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from mimo_b200 import lib as L  # noqa: E402
from mimo_b200 import ops  # noqa: E402

dev = "cuda"


def attn(n=12, lq=4096, d=40, lb=4096):
    C = 8 * d
    qkv = torch.randn(n * lq, 3 * C, device=dev).half()
    bkv = torch.randn(2, lb, 2 * C, device=dev).half()
    bi = torch.ones(n, dtype=torch.int32, device=dev)
    for _ in range(4):
        ops.attn_spatial(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], n, lq, 8, bank_k=bkv[:, :, :C], bank_v=bkv[:, :, C:],
                         bank_index=bi)


def attn80():
    attn(n=8, lq=1024, d=80, lb=1024)


def gemm(M=196608, N=320, K=320):
    a = torch.randn(M, K, device=dev).half()
    w = torch.randn(N, K, device=dev).half()
    b = torch.randn(N, device=dev).half()
    r = torch.randn(M, N, device=dev).half()
    for _ in range(4):
        ops.gemm(a, w, bias=b, residual=r)


def qkv(M=196608, N=960, K=320):
    a = torch.randn(M, K, device=dev).half()
    w = torch.randn(N, K, device=dev).half()
    for _ in range(4):
        ops.gemm(a, w)


def geglu(M=196608, N=2560, K=320):
    a = torch.randn(M, K, device=dev).half()
    w = torch.randn(N, K, device=dev).half()
    b = torch.randn(N, device=dev).half()
    for _ in range(4):
        ops.gemm(a, w, bias=b, act=L.ACT_GEGLU)


def conv(n=48, h=64, c=320, co=320):
    x = torch.randn(n * h * h, c, device=dev).half()
    w = torch.randn(co, 9 * c, device=dev).half()
    b = torch.randn(co, device=dev).half()
    for _ in range(4):
        ops.conv3x3(x, w, n, h, h, bias=b)


def conv1280():
    conv(48, 16, 1280, 1280)


def norm(n=48, hw=4096, c=320):
    x = torch.randn(n * hw, c, device=dev).half()
    g = torch.ones(c, device=dev).half()
    b = torch.zeros(c, device=dev).half()
    for _ in range(4):
        ops.groupnorm(x, g, b, n, hw, silu=True)
        ops.layernorm(x, g, b)


def convup(n=48, h=32, c=640):
    x = torch.randn(n * h * h, c, device=dev).half()
    w4 = ops.pack_conv_up2x_weight(torch.randn(c, c, 3, 3, device=dev).half() / 70)
    b = torch.randn(c, device=dev).half()
    for _ in range(2):
        ops.conv_up2x(x, w4, n, h, h, bias=b)


def ffo(M=49152, N=640, K=2560):
    gemm(M, N, K)


def temporal(hw=4096, d=40):
    C = 8 * d
    qkv = torch.randn(48 * hw, 3 * C, device=dev).half()
    for _ in range(4):
        ops.attn_temporal(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], 2, 24, hw, 8)


if __name__ == "__main__":
    for name in sys.argv[1:]:
        globals()[name]()
    torch.cuda.synchronize()
