"""Time the new-path SASRec training step on multi-positive targets at the config-2 shape (L 200, d 128, 2 heads, 2 blocks,
50 000 items, dropout 0.2, batch 512): P in {1, 4} for full-catalog BCE, CESampled with 256 shared negatives and CESampled
with 128 per-position negatives.  Prints one JSON line per case: ms / step and seq / s of the graph-replayed fused step
(forward + backward + Adam), ms of the loss head alone (forward + backward), and the card's name and power limit.

    python tools/bench_multi_positive.py [--batch 512] [--steps 30] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from replay_b200.engine import EncoderConfig, SasRecEngine  # noqa: E402
from replay_b200.trainer import Trainer  # noqa: E402

L, D, N_ITEMS = 200, 128, 50_000
CASES = [("bce", None, 0), ("ce_sampled", "shared", 256), ("ce_sampled", "perpos", 128)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in q.split(",")]
    except Exception as e:  # noqa: BLE001
        return [torch.cuda.get_device_name(), f"unknown ({e})", "unknown"]


def batch(B, P, g):
    lens = torch.randint(L // 4, L + 1, (B,), generator=g)
    pm = torch.arange(L).unsqueeze(0) >= (L - lens).unsqueeze(1)
    ids = torch.where(pm, torch.randint(0, N_ITEMS, (B, L), generator=g), torch.full((B, L), N_ITEMS))
    lab = torch.randint(0, N_ITEMS, (B, L, P), generator=g)
    m = pm.unsqueeze(-1) & (torch.rand(B, L, P, generator=g) < 0.75)
    m[..., 0] = pm
    return ids.cuda(), pm.cuda(), lab.cuda(), m.cuda()


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    name, power, sm_clock = card()
    cfg = EncoderConfig(n_items=N_ITEMS, d=D, n_heads=2, n_blocks=2, max_len=L, dropout=0.2, variant="new")
    eng = SasRecEngine(cfg, args.batch, L, "cuda")
    g = torch.Generator().manual_seed(0)
    for kind, shape, n_neg in CASES:
        for P in (1, 4):
            ids, pm, lab, m = batch(args.batch, P, g)
            if P == 1:
                lab, m = lab[..., 0], m[..., 0]
            if kind == "bce":
                eng.set_loss("bce")
            else:
                eng.set_loss(kind, n_neg=n_neg, neg_shape=shape)
            eng.set_batch(ids, pm, lab, m)
            if kind != "bce":
                rows = 1 if shape == "shared" else args.batch * L
                eng.set_negatives(torch.randint(0, N_ITEMS, (rows, n_neg), generator=g).cuda())
            tr = Trainer(eng, use_graph=True)
            step_ms = timed(lambda: tr.run(), args.steps, args.warmup)
            eng.forward_train()
            G = eng.grads["item_emb"]
            table = eng.params16["item_emb"][:N_ITEMS]

            def head():
                if kind == "bce":
                    eng._catalog_head_fwd(table)
                    eng._catalog_head_bwd(table, G)
                else:
                    import ctypes
                    sd = eng._sampled_desc()
                    eng.lib.rp_sampled_head_fwd(ctypes.byref(sd), eng._stream())
                    eng.lib.rp_sampled_head_bwd(ctypes.byref(sd), eng.s["dhc"].data_ptr(), G.data_ptr(), eng._stream())

            head_ms = timed(head, args.steps, args.warmup)
            print(json.dumps(dict(loss=kind, negatives=shape, n_neg=n_neg, P=P, batch=args.batch, ms_per_step=round(step_ms, 3),
                                  seq_per_s=round(args.batch / step_ms * 1e3), head_ms=round(head_ms, 3), gpu=name,
                                  power_limit=power, max_sm_clock=sm_clock, n_pairs=int(m.sum()))), flush=True)


if __name__ == "__main__":
    main()
