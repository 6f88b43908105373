"""Training-step time of the legacy SASRec with the scalable cross-entropy head (loss_type="SCE") next to the full-catalog CE
head, at config 2 (L=200 d=128 H=2 |I|=50K, B=256) and config 5 (L=512 d=512 H=8 |I|=1M, B=32), in one process.  Eager
launches, CUDA events, median of repeats.  The SCE head's time is split into the bucket draw, the row selection, the item
selection, the bucket CE forward and the bucket CE backward (each timed alone on the step's own inputs).

    python tools/bench_sce.py [--repeats 5] [--steps 10]
"""
import argparse
import ctypes
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from replay_b200._lib import SCE_BUCKET_CE, SCE_DRAW, SCE_SELECT_X, SCE_SELECT_Y, check
from replay_b200.engine import EncoderConfig, SasRecEngine
from replay_b200.synthetic import make_sequences

CONFIGS = {2: dict(B=256, L=200, d=128, H=2, I=50_000), 5: dict(B=32, L=512, d=512, H=8, I=1_000_000)}
SCE = [(256, 256, 256), (256, 512, 512)]   # (n_buckets, bucket_size_x, bucket_size_y)


def _time(fn, steps, repeats):
    out = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(steps):
            fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b) / steps)
    return statistics.median(out)


def card():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                             str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--configs", default="2,5")
    args = ap.parse_args()
    name, pl = card()
    print(f"card: {name}, power limit {pl}", flush=True)
    for c in (int(v) for v in args.configs.split(",")):
        cf = CONFIGS[c]
        B, L, d, H, I = cf["B"], cf["L"], cf["d"], cf["H"], cf["I"]
        ids, pm, lab, tm = make_sequences(B, I, L, seed=1234)
        lab = lab.clamp(max=I - 1)
        for sce in [None] + SCE:
            eng = SasRecEngine(EncoderConfig(n_items=I, d=d, n_heads=H, n_blocks=2, max_len=L, dropout=0.2, variant="legacy"),
                               B, L, "cuda", seed=1)
            if sce is not None:
                eng.set_loss("sce", n_buckets=sce[0], bucket_size_x=sce[1], bucket_size_y=sce[2])
            eng.set_batch(ids.cuda(), pm.cuda(), lab.cuda(), tm.cuda())
            eng.n_valid_hint = int(tm.sum())
            losses = [float(eng.train_step()[0]) for _ in range(3)]
            ms = _time(eng.train_step, args.steps, args.repeats)
            label = "full CE" if sce is None else f"SCE n_b={sce[0]} bs_x={sce[1]} bs_y={sce[2]}"
            line = (f"config {c} {label:34s} {ms:8.2f} ms/step -> {B / ms * 1e3:9.0f} seq/s  loss {losses[0]:.3f} -> "
                    f"{losses[-1]:.3f}")
            if sce is not None:
                eng.forward_train()
                st = eng._stream()
                desc = ctypes.byref(eng.sce["desc"])
                parts = {}
                for part, bits in (("draw", SCE_DRAW), ("select rows", SCE_SELECT_X), ("select items", SCE_SELECT_Y),
                                   ("bucket CE fwd", SCE_BUCKET_CE)):
                    parts[part] = _time(lambda b=bits: check(eng.lib.rp_sce_head_fwd(desc, b, st), "rp_sce_head_fwd"),
                                        args.steps, args.repeats)
                dhc = eng.s["dhc"].data_ptr()
                parts["bucket CE bwd"] = _time(lambda: check(eng.lib.rp_sce_head_bwd(desc, dhc, st), "rp_sce_head_bwd"),
                                               args.steps, args.repeats)
                line += "  |  head: " + ", ".join(f"{k} {v:.3f} ms" for k, v in parts.items())
            print(line, flush=True)
            del eng
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
