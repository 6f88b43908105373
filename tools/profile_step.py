"""Per-kernel GPU time of one captured config-2 training step (new-path SASRec, L 200, d 128, 2 heads, |I| 50 000, 512
sequences, dropout 0.2, bench.py's seeded batches), from torch.profiler over replays of the step graph.

    python tools/profile_step.py [--steps 20] [--batch 512] [--out DIR]

Run it on its own: tracing slows the host, so the end-to-end step time comes from bench.py, not from here.  Prints one line
per kernel (mean microseconds per step, share of the summed kernel time, launches per step) and the split between the CE
head, the body and the rest.  RP_PACKED_BODY=0 profiles the padded body for comparison.
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HEAD = ("ce_",)
BODY = ("attn_", "ln_qkv", "post_attn", "pre_attn", "wgrad", "embed", "row_plan", "layernorm")


def _group(name: str) -> str:
    if any(k in name for k in HEAD):
        return "ce head"
    if any(k in name for k in BODY):
        return "body"
    return "other"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--out", default=None, help="directory for a JSON copy of the table")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("profile_step.py needs a GPU")

    import bench
    from replay_b200.trainer import Trainer

    dev = torch.device("cuda", 0)
    c = dict(bench.CONFIGS[2])
    B, L = args.batch, c["seq_len"]
    _, core, _ = bench.build_module(c, dev)
    eng = core.ensure_engine(B, L, with_grad=True)
    tr = Trainer(eng, use_graph=True)
    n_batches = 6
    data = bench.make_batches(c, B * n_batches, seed=1234)
    devb = [t.reshape(n_batches, B, L).to(dev) for t in data]
    eng.n_valid_hint = int(bench.valid_targets(c, data) * B)
    for i in range(5):   # warm-up and graph capture
        tr.step(*(t[i % n_batches] for t in devb))
    torch.cuda.synchronize()

    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(args.steps):
            tr.step(*(t[i % n_batches] for t in devb))
        torch.cuda.synchronize()
    per = collections.defaultdict(lambda: [0.0, 0])
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and not ev.name.startswith(("Memcpy", "Memset")):
            per[ev.name][0] += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            per[ev.name][1] += 1
    total = sum(v[0] for v in per.values())
    groups = collections.defaultdict(float)
    rows = []
    for name, (us, n) in sorted(per.items(), key=lambda kv: -kv[1][0]):
        groups[_group(name)] += us / args.steps
        rows.append(dict(kernel=name[:110], us_per_step=us / args.steps, share=us / total, launches_per_step=n / args.steps))
    props = torch.cuda.get_device_properties(dev)
    print(f"# {props.name}; packed body: {eng.packed_eligible()}; {args.steps} steps of {B} sequences")
    for r in rows:
        print(f"{r['us_per_step']:10.1f} us  {100 * r['share']:5.1f} %  x{r['launches_per_step']:4.1f}  {r['kernel']}")
    print("# per step: " + ", ".join(f"{k} {v / 1000:.3f} ms" for k, v in sorted(groups.items())) + f", kernels {total / args.steps / 1000:.3f} ms")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        tag = "packed" if eng.packed_eligible() else "padded"
        with open(os.path.join(args.out, f"profile_step_{tag}.json"), "w") as fh:
            json.dump(dict(gpu=props.name, packed=eng.packed_eligible(), groups_ms={k: v / 1000 for k, v in groups.items()},
                           kernels=rows), fh, indent=1)


if __name__ == "__main__":
    main()
