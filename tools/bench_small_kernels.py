"""Fixed cost of the small body kernels: time rp_gemm at several sizes inside a CUDA graph (100 launches per replay)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from replay_b200 import ops
dev = "cuda"
def bench(fn, n=100):
    fn(); torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(n): fn()
    g.replay(); torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); g.replay(); g.replay(); g.replay(); b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / (3 * n) * 1e3
for M in (128, 1024, 12800, 51200, 204800):
    A = torch.randn(M, 128, device=dev).bfloat16(); W = torch.randn(128, 128, device=dev).bfloat16()
    C = torch.empty(M, 128, device=dev, dtype=torch.bfloat16); bias = torch.randn(128, device=dev)
    R = torch.randn(M, 128, device=dev).bfloat16()
    t0 = bench(lambda: ops.gemm(A, W, C, M, 128, 128))
    t1 = bench(lambda: ops.gemm(A, W, C, M, 128, 128, bias=bias, act=1, residual=R))
    t2 = bench(lambda: ops.gemm(A, W, C, M, 128, 128, b_mn=True))
    print(f"gemm M={M:7d} N=K=128: plain {t0:6.1f} us | bias+relu+residual {t1:6.1f} us | B MN-major {t2:6.1f} us | data-sheet HBM time {(M*128*2*2)/3.35e6:5.1f} us")
T = 51200
dY = torch.randn(T, 128, device=dev).bfloat16(); X = torch.randn(T, 128, device=dev).bfloat16()
dW = torch.zeros(128, 128, device=dev)
for split in (1, 8, 33, 66, 132):
    t = bench(lambda: ops.gemm(dY, X, dW, 128, 128, T, a_mn=True, b_mn=True, out_mode=1, split_k=split))
    print(f"wgrad T={T} split={split:3d}: {t:6.1f} us")
x = torch.randn(T, 128, device=dev).bfloat16()
t = bench(lambda: x.add_(1.0))
print(f"torch elementwise add_ on [51200,128] bf16: {t:6.1f} us")
