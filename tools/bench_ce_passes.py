"""Per-launch times of the full-catalog CE head at config 2 (SASRec L 200, d 128, |I| 50 000, 512 sequences).

    python tools/bench_ce_passes.py [--iters 50] [--warmup 5] [--out DIR]

Builds the engine as bench.py does, runs one training step, then times the head alone on that step's operands (hc,
labels_c, n_valid, the item table):
  * CUDA events around rp_ce_head_fwd and rp_ce_head_bwd, each `--iters` launches back to back;
  * torch.profiler (CUDA activities, a separate run of `--iters` forward + backward pairs) for the kernels inside them:
    ce_bound_kernel, the fused pass (ce_bwd_kernel MODE 2), its completion (ce_loss_reduce_kernel or
    ce_fused_finalize_kernel), the dE pass (ce_bwd_kernel MODE 1) and ce_label_scatter_kernel.
The two GEMM passes each execute 2 x (2 T_v |I| d) FLOP (S, then dH or dE); their executed TFLOP/s is that over the kernel
time.  The GPU name, power limit and the SM clocks sampled over the timed windows are printed with the numbers.  Another
build of the library is timed with RP_B200_LIB=<path to librp_b200.so>.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the config-2 engine and batches exactly as the benchmark builds them)


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        row = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, check=True).stdout.strip().split(", ")
        return {"name": row[0], "power_limit_w": float(row[1]), "clocks_max_sm_mhz": float(row[2])}
    except (OSError, subprocess.CalledProcessError, ValueError, IndexError):
        return {"name": torch.cuda.get_device_name(0), "power_limit_w": None, "clocks_max_sm_mhz": None}


def kernel_label(name: str):
    m = re.search(r"ce_bwd_kernel<(\d+), (\d+), (\d+), (\d+), (\w+)>", name)
    if m:
        mode = int(m.group(4))
        return {1: "dE pass (ce_bwd_kernel MODE 1)", 2: "fused pass (ce_bwd_kernel MODE 2)"}.get(mode, f"ce_bwd_kernel MODE {mode}")
    m = re.search(r"(ce_\w+_kernel)", name)
    return m.group(1) if m else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for the profiler's kernel table (optional)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ce_passes.py needs a GPU")
    from replay_b200 import _lib, ops
    from replay_b200.trainer import Trainer

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    c = dict(bench.CONFIGS[2])
    B, L, d, I = c["per_gpu_batch"], c["seq_len"], c["d"], c["n_items"]
    _mod, core, _ = bench.build_module(c, dev)
    eng = core.ensure_engine(B, L, with_grad=True)
    tr = Trainer(eng, use_graph=False)
    data = bench.make_batches(c, B, seed=1234)
    eng.n_valid_hint = int(bench.valid_targets(c, data) * B)
    tr.step(*(t.to(dev) for t in data))
    torch.cuda.synchronize()
    T_v = int(eng.n_valid.item())
    table, dW = eng.params16["item_emb"][:I], eng.grads["item_emb"]

    def fwd():
        ops.ce_head_fwd(eng.ce, eng.hc, table, eng.labels_c, eng.n_valid, d_hc=eng.s["dhc"], n_valid_hint=eng.n_valid_hint)

    def bwd():
        ops.ce_head_bwd(eng.ce, eng.hc, table, eng.labels_c, eng.n_valid, eng.s["dhc"], dW, n_valid_hint=eng.n_valid_hint)

    def events(fn):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for _ in range(args.iters):
            fn()
        ev[1].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]) / args.iters

    for _ in range(args.warmup):
        fwd()
        bwd()
    torch.cuda.synchronize()
    fused_taken = bool(ops.ce_head_fused_taken(eng.ce))
    sampler = bench.ClockSampler(0)
    sampler.start()
    fwd_ms, bwd_ms = events(fwd), events(bwd)

    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.iters):
            fwd()
            bwd()
        torch.cuda.synchronize()
    clocks = sampler.stop()
    per = {}
    for e in prof.events():
        lab = kernel_label(e.name) if e.device_type == torch.autograd.DeviceType.CUDA else None
        if lab is not None:
            per.setdefault(lab, []).append(e.time_range.elapsed_us() / 1e3)   # us -> ms
    gemm_pair = 2 * (2.0 * T_v * I * d)
    kernels = {}
    for lab, ts in sorted(per.items(), key=lambda kv: -sum(kv[1])):
        # a kernel launched twice per call (the fused pass behind the two-pass forward exits at once while the bound
        # holds): the working launch is the longer one of each pair
        work = sorted(ts)[-args.iters:]
        ms = work[len(work) // 2]
        row = {"ms": ms, "ms_per_call": sum(ts) / args.iters, "launches_per_call": len(ts) / args.iters}
        if lab.startswith(("fused pass", "dE pass")):
            row["executed_tflops"] = gemm_pair / (ms * 1e-3) / 1e12
        kernels[lab] = row
    line = {"tool": "bench_ce_passes", "lib": _lib.LIB_PATH, "gpu": gpu_info(), "clocks": clocks,
            "shape": {"T_v": T_v, "capacity": int(eng.hc.shape[0]), "n_items": I, "d": d}, "fused_path_taken": fused_taken,
            "events_ms": {"rp_ce_head_fwd": fwd_ms, "rp_ce_head_bwd": bwd_ms}, "iters": args.iters, "kernels": kernels}
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "ce_passes_kernels.txt"), "w") as fh:
            fh.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=30))
    print(json.dumps(line))


if __name__ == "__main__":
    main()
