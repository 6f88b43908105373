"""wgmma issue-rate probe: SM cycles per 64xNx16 bf16 MMA of one warpgroup for the operand forms the kernels use."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from replay_b200._lib import check, lib

L = lib()
st = torch.cuda.current_stream().cuda_stream
names = {0: "SS  A K-major  B K-major ", 1: "SS  A K-major  B MN-major", 2: "RS  A regs     B K-major ", 3: "RS  A regs     B MN-major",
         4: "SS  A MN-major B K-major ", 5: "SS  A MN-major B MN-major"}
names.update({8 + 0: "SS  N=256  B K-major      ", 8 + 2: "RS  N=256  B K-major      ", 16 + 0: "SS  N=64   B K-major      ",
              16 + 2: "RS  N=64   B K-major      "})
for grid in (torch.cuda.get_device_properties(0).multi_processor_count,):   # one CTA per SM
    for mode, nm in names.items():
        out = torch.zeros(grid, dtype=torch.int64, device="cuda")
        iters = 2000
        check(L.rp_selftest_mma_probe(mode, iters, grid, out.data_ptr(), st), "probe")
        torch.cuda.synchronize()
        c = out.float().mean().item() / (iters * 8)
        n = 256 if (mode >> 3) == 1 else (64 if (mode >> 3) == 2 else 128)
        print(f"grid {grid:3d}  {nm}: {c:6.1f} clk per 64x{n}x16 MMA (ideal {n // 2}: 4096 dense bf16 FLOP/clk/SM) -> {100 * (n / 2) / c:5.1f} % of peak", flush=True)
