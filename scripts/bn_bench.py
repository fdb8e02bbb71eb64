"""Debug aid (GPU box): MMA-bound GEMM throughput per forced tile width (is every UMMA N equally efficient?)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from mimo_b200 import lib as L, ops

def timeit(fn, n=10):
    for _ in range(3): fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); a.record()
    for _ in range(n): fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / n

lib = L.load()
for (M, N, K) in [(128 * 132 * 2, 3840, 4096), (196608, 960, 320), (196608, 320, 320), (49152, 640, 640)]:
    a = torch.randn(M, K, device="cuda").half(); w = torch.randn(N, K, device="cuda").half()
    out = torch.empty(M, N, device="cuda", dtype=torch.half)
    for bn in (64, 128, 160, 192, 256):
        lib.mimo_debug_force_bn(bn)
        ms = timeit(lambda: ops.gemm(a, w, out=out))
        print(f"gemm {M}x{N}x{K} bn={bn}: {ms:.3f} ms = {2*M*N*K/ms/1e9:.0f} TFLOP/s", flush=True)
    lib.mimo_debug_force_bn(0)
