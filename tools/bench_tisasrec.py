#!/usr/bin/env python
"""TiSASRec (the legacy SasRec with ti_modification=True) against the non-Ti legacy SasRec on the H100.

    python tools/bench_tisasrec.py [--steps 20] [--warmup 5] [--batch 256] [--users 4096]

Shape: hidden 128, 2 heads, 2 blocks, L 200, |I| 50 000, dropout 0.2, full-catalog CE, time_span 256, MovieLens-shaped
synthetic sequences (replay_b200.synthetic) with timestamps a few minutes apart.  Reports, as one JSON line:
- training sequences / s of the Lightning module's fused, graph-replayed training_step, both models;
- predict_topk(k=10) with the seen filter at --users users per call, both models;
- the time-interval attention's forward and backward (rp_ti_attn_fwd / rp_ti_attn_bwd with the rp_gemm products around
  them) per block, from CUDA events;
- the reference's formulation in eager torch (oracle/tisasrec.py materialises the [B, L, L, d] time embeddings as the
  reference does): one forward + backward at the largest batch of 256 / 128 / ... that fits;
- the card's name, power limit and SM clock, read in the same run.
Writes nothing to disk."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), (v.strip() for v in out.splitlines()[0].split(",")))) if out else {}


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(steps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / steps   # ms


def batch(B, L, n_items, dev, seed):
    from replay_b200.synthetic import make_sequences

    ids, pm, lab, tm = make_sequences(B, n_items, L, seed=seed)
    g = torch.Generator().manual_seed(seed)
    ts = (1_700_000_000 + torch.randint(0, 600, (B, L), generator=g).cumsum(1)) * pm
    return {"feature_tensor": {"item_id": ids.to(dev), "timestamp": ts.to(dev)}, "padding_mask": pm.to(dev),
            "positive_labels": lab.to(dev), "target_padding_mask": tm.to(dev)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--users", type=int, default=4096)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tisasrec.py measures on a GPU; none is visible")
    from replay_b200.models.nn.sequential import SasRec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    dev = torch.device("cuda")
    d, H, L, n_items, span, drop = 128, 2, 200, 50_000, 256, 0.2
    schema = TensorSchema(TensorFeatureInfo("item_id", n_items, n_items, d), timestamp_feature_name="timestamp")
    res = dict(shape=dict(hidden=d, heads=H, blocks=2, L=L, n_items=n_items, dropout=drop, time_span=span, batch=a.batch,
                          users=a.users), card=card())
    train = batch(a.batch, L, n_items, dev, 1)
    users = batch(a.users, L, n_items, dev, 2)
    seen = users["feature_tensor"]["item_id"]
    for ti in (False, True):
        m = SasRec(schema, block_count=2, head_count=H, hidden_size=d, max_seq_len=L, dropout_rate=drop, ti_modification=ti,
                   time_span=span, device=dev)
        ms = timed(lambda: m.training_step(train), a.steps, a.warmup)
        if ti:   # on the training batch the engine holds now, before predict re-sizes it
            eng = m._model.core.engine
            fwd = timed(lambda: eng._ti_attention_forward(0, True, drop), a.steps, a.warmup)
            bwd = timed(lambda: eng._ti_attention_backward(0, drop), a.steps, a.warmup)
            res["attention_ms_per_block"] = dict(forward=fwd, backward=bwd)
        pm = timed(lambda: m.predict_topk(users, 10, seen_ids=seen), a.steps, a.warmup)
        res["tisasrec" if ti else "sasrec"] = dict(train_seq_per_s=a.batch / ms * 1e3, train_step_ms=ms, predict_ms=pm,
                                                   predict_users_per_s=a.users / pm * 1e3)
        del m
        torch.cuda.empty_cache()
    res["eager_reference_formulation"] = eager(train, d, H, L, n_items, span, drop, a)
    print(json.dumps(res))


def eager(train, d, H, L, n_items, span, drop, a):
    """oracle/tisasrec.py in fp32 eager torch with dropout on every term the reference drops."""
    import oracle.tisasrec as oti

    P = oti.random_params(n_items, d, L, 2, span, seed=0)
    P = {k: ([{kk: vv.cuda().requires_grad_(True) for kk, vv in b.items()} for b in v] if k == "blocks"
             else v.cuda().requires_grad_(True)) for k, v in P.items()}
    B = a.batch
    while B >= 1:
        f = {k: v[:B] for k, v in train["feature_tensor"].items()}
        pm, lab, tm = train["padding_mask"][:B], train["positive_labels"][:B], train["target_padding_mask"][:B]
        ks = 1.0 / (1.0 - drop)
        keep = lambda *s: (torch.rand(*s, device="cuda") >= drop).float() * ks  # noqa: E731

        def step():
            kp = {"item": keep(B, L, d), "pos_k": keep(B, L, d), "pos_v": keep(B, L, d), "time_k": keep(B, L, L, d),
                  "time_v": keep(B, L, L, d),
                  "blocks": [{"att": keep(B, H, L, L), "ffn1": keep(B, L, d), "ffn2": keep(B, L, d)} for _ in range(2)]}
            oti.train_loss(P, f["item_id"], pm, f["timestamp"], lab, tm, H, span, kp).backward()

        try:
            torch.cuda.reset_peak_memory_stats()
            ms = timed(step, max(1, a.steps // 4), 1)
            return dict(batch=B, train_seq_per_s=B / ms * 1e3, step_ms=ms,
                        peak_gib=torch.cuda.max_memory_allocated() / 2**30)
        except torch.OutOfMemoryError:
            torch.cuda.empty_cache()
            B //= 2
    return dict(batch=0)


if __name__ == "__main__":
    main()
