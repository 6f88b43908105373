"""rp_gemm throughput on the mid-size / large shapes of configs 3 and 5 next to torch.matmul (cuBLAS) on the same operands."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from replay_b200 import ops


def t(fn, n=10):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


shapes = [(25600, 1024, 256, False, "bert ffn1 fwd"), (25600, 256, 1024, False, "bert ffn2 fwd"), (25600, 768, 256, False, "bert qkv"),
          (25600, 256, 1024, True, "bert ffn1 dgrad (B MN-major)"), (51200, 128, 128, False, "c2 proj"),
          (16384, 512, 512, False, "c5 proj"), (1408, 200_000, 512, False, "c5 G gemm slice (N=200K)"),
          (819200, 256, 128, False, "predict K|V projection (4096 x 200)")]
for M, N, K, b_mn, name in shapes:
    A = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    W = (torch.randn(N, K, device="cuda") * 0.1).to(torch.bfloat16)
    Bop = W.T.contiguous() if b_mn else W
    C = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    ms = t(lambda: ops.gemm(A, Bop, C, M, N, K, b_mn=b_mn))
    ms_ref = t(lambda: torch.matmul(A, W.T, out=C))
    fl = 2.0 * M * N * K
    print(f"{name:32s} M={M:6d} N={N:7d} K={K:5d}: rp_gemm {ms * 1e3:8.1f} us {fl / ms / 1e9:7.0f} TFLOP/s | cuBLAS {ms_ref * 1e3:8.1f} us "
          f"{fl / ms_ref / 1e9:7.0f} TFLOP/s", flush=True)
