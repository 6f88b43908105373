"""TMA feed-rate probe: bytes per clock one SM can pull from L2 with [box_rows x 64] bf16 boxes (the B-operand pattern of the
score / CE kernels) when nothing consumes them.  Prints GB/s per SM and chip-wide for several box shapes and table sizes."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from replay_b200._lib import check, lib

L = lib()
st = torch.cuda.current_stream().cuda_stream
for rows, d, name in ((50_000, 128, "50K x 128 (12.8 MB, L2-resident)"), (500_000, 128, "500K x 128 (128 MB)")):
    tab = torch.randn(rows, d, device="cuda").to(torch.bfloat16)
    for box_rows in (128, 256):
        for grid in (1, torch.cuda.get_device_properties(0).multi_processor_count):
            for same in (0, 1):
                tiles = 2000
                f = lambda: check(L.rp_selftest_tma_probe(tab.data_ptr(), rows, d, box_rows, tiles, same, grid, st), "probe")
                f()
                torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                f()
                b.record()
                torch.cuda.synchronize()
                ms = a.elapsed_time(b)
                byt = grid * tiles * box_rows * d * 2
                print(f"{name:36s} box {box_rows:3d}x64 grid {grid:3d} same_tile {same}: {byt / ms / 1e6:8.1f} GB/s total, "
                      f"{byt / ms / 1e6 / grid:7.1f} GB/s per SM ({byt / grid / (ms * 1e-3 * 1.965e9):5.1f} B/clk)", flush=True)
