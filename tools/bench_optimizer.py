"""Cost of the fused optimizer step (rp_optimizer_step): the step alone over flat buffers of the config-2 size (the
new-path SASRec of bench.py, about 6.5 M parameters) and of config 5 (L 512, d 512, a million items, about 513 M), for
Adam with weight decay 0 / 1e-2 and SGD with momentum 0 / 0.9; then the whole captured config-2 training step (512
sequences, bench.py's seeded batches) with each optimizer.

    python tools/bench_optimizer.py [--iters 50] [--rounds 5] [--out DIR]

The step alone is timed with CUDA events over ``--iters`` launches after a warm-up (at least 30 at config 5).  The whole
config-2 step runs one module per optimizer, built up front, and times ``--rounds`` windows of 100 steps for each,
alternating the optimizers from window to window; it reports the median and the range.  The step-alone rate counts the bytes the
algorithm must move per parameter: Adam reads p, g, m, v and writes p, m, v (28 B), SGD with momentum reads p, g, buf
and writes p, buf (20 B), SGD without reads p, g and writes p (12 B); every kind also zeroes g (4 B) and writes the bf16
shadow (2 B).  The share of peak is that rate over the H100 SXM data sheet's 3.35 TB/s.  The card's name, power limit and
maximum SM clock are printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM = 3.35e12
OPTS = {"adam": dict(kind="adam"), "adam_wd1e-2": dict(kind="adam", weight_decay=1e-2),
        "sgd": dict(kind="sgd"), "sgd_mom0.9": dict(kind="sgd", momentum=0.9)}


def bytes_per_param(o) -> int:
    state = {"adam": 28, "sgd": 20 if o.momentum else 12}[o.kind]
    return state + 4 + 2


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def time_alone(n, opt, iters, dev):
    from replay_b200._lib import check, lib
    from replay_b200.engine import _OPT_KINDS

    L = lib()
    f32 = dict(device=dev, dtype=torch.float32)
    p, g, m, v = torch.randn(n, **f32), torch.zeros(n, **f32), torch.zeros(n, **f32), torch.zeros(n, **f32)
    p16 = torch.empty(n, device=dev, dtype=torch.bfloat16)
    lr, step = torch.full((1,), 1e-3, **f32), torch.zeros(1, device=dev, dtype=torch.int32)
    st = torch.cuda.current_stream(dev).cuda_stream

    def run():
        check(L.rp_optimizer_step(_OPT_KINDS[opt.kind], p.data_ptr(), g.data_ptr(), m.data_ptr(),
                                  v.data_ptr() if opt.kind == "adam" else None, p16.data_ptr(), n, lr.data_ptr(),
                                  step.data_ptr(), opt.betas[0], opt.betas[1], opt.eps, opt.weight_decay, opt.momentum,
                                  1.0, None, 1, st), "rp_optimizer_step")

    for _ in range(5):
        run()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        run()
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / iters
    del p, g, m, v, p16
    torch.cuda.empty_cache()
    return ms


def config2_trainers(dev):
    """one captured config-2 training step per optimizer, on bench.py's seeded batches"""
    import bench
    from replay_b200.engine import OptimizerConfig
    from replay_b200.trainer import Trainer

    c = dict(bench.CONFIGS[2])
    B, L = 512, c["seq_len"]
    n_batches = 6
    data = bench.make_batches(c, B * n_batches, seed=1234)
    devb = [t.reshape(n_batches, B, L).to(dev) for t in data]
    out = {}
    for name, kw in OPTS.items():
        _, core, _ = bench.build_module(c, dev)
        eng = core.ensure_engine(B, L, with_grad=True)
        eng.n_valid_hint = int(bench.valid_targets(c, data) * B)
        tr = Trainer(eng, use_graph=True, opt=OptimizerConfig(**kw))
        for i in range(5):
            tr.step(*(t[i % n_batches] for t in devb))
        out[name] = (tr, eng)
    torch.cuda.synchronize()
    return out, devb


def time_window(tr, devb, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(steps):
        tr.step(*(t[i % len(devb[0])] for t in devb))
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for a JSON copy of the results")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_optimizer.py needs a GPU")
    from replay_b200.engine import OptimizerConfig

    dev = torch.device("cuda", 0)
    res = {"card": card(), "alone": [], "config2_step": []}
    print(f"# {res['card']}")
    trainers, devb = config2_trainers(dev)
    n2 = next(iter(trainers.values()))[1].n_flat
    windows = {name: [] for name in OPTS}
    for _ in range(args.rounds):
        for name, (tr, _) in trainers.items():
            windows[name].append(time_window(tr, devb, 100))
    for name, ms in windows.items():
        ms = sorted(ms)
        res["config2_step"].append(dict(optimizer=name, median_ms=ms[len(ms) // 2], min_ms=ms[0], max_ms=ms[-1]))
        print(f"config 2 step  {name:12s} median {ms[len(ms) // 2]:7.3f} ms  range {ms[0]:.3f}-{ms[-1]:.3f} ms "
              f"({args.rounds} alternated windows of 100 steps)")
    del trainers, devb
    torch.cuda.empty_cache()
    for label, n in (("config 2", n2), ("config 5", 513_000_000)):
        for name, kw in OPTS.items():
            opt = OptimizerConfig(**kw)
            ms = time_alone(n, opt, args.iters if n < 1e8 else max(30, args.iters // 5), dev)
            rate = bytes_per_param(opt) * n / (ms * 1e-3)
            res["alone"].append(dict(size=label, n=n, optimizer=name, ms=ms, bytes_per_s=rate, share_of_hbm=rate / HBM))
            print(f"{label} alone  n {n:>11,d}  {name:12s} {ms:8.3f} ms  {rate / 1e9:7.0f} GB/s  {100 * rate / HBM:5.1f} % of 3.35 TB/s")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_optimizer.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
