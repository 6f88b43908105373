"""Throughput of SasRec with the DiffTransformer encoder at the config-2 shape (L 200, d 128, 2 heads, 50K items, 512
sequences per training step), next to the SASRec encoder and the reference module run eagerly in torch on the same GPU.

    python tools/bench_diff.py [--steps 20] [--warmup 5]

Prints one JSON line: the card name and power limit (read in the same call), training sequences/s of the DiffTransformer
and SASRec encoders (fused step, CUDA graph, full-catalog CE), of the eager torch restatement of the reference
(oracle/diff.py, fp32 autograd + torch.optim.Adam, the same sizes) and predict users/s at 4096 users (seen-filtered top-10).
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_ITEMS, D, H, L, B, N_BLOCKS = 50_000, 128, 2, 200, 512, 2


def _model(encoder):
    from replay_b200.nn.agg import SumAggregator
    from replay_b200.nn.embedding import SequenceEmbedding
    from replay_b200.nn.loss import CE
    from replay_b200.nn.mask import DefaultAttentionMask
    from replay_b200.nn.sequential import (DiffTransformerLayer, PositionAwareAggregator, SasRec, SasRecBody,
                                           SasRecTransformerLayer)
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    sch = TensorSchema(TensorFeatureInfo("item_id", N_ITEMS, N_ITEMS, D))
    enc = DiffTransformerLayer(D, H, N_BLOCKS) if encoder == "diff" else SasRecTransformerLayer(D, H, N_BLOCKS, 0.0, "relu")
    body = SasRecBody(SequenceEmbedding(sch), PositionAwareAggregator(SumAggregator(D), L, 0.0), DefaultAttentionMask("item_id", H),
                      enc, torch.nn.LayerNorm(D))
    return SasRec(body, loss=CE(ignore_index=N_ITEMS))


def _batch(n, dev):
    g = torch.Generator().manual_seed(0)
    lens = torch.randint(20, L + 1, (n,), generator=g)
    pm = torch.arange(L).unsqueeze(0) >= (L - lens).unsqueeze(1)
    ids = torch.where(pm, torch.randint(0, N_ITEMS, (n, L), generator=g), torch.full((n, L), N_ITEMS))
    labels = torch.where(pm, torch.randint(0, N_ITEMS, (n, L), generator=g), torch.full((n, L), N_ITEMS))
    return ids.to(dev), pm.to(dev), labels.to(dev), pm.to(dev)


def _timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(steps):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / 1e3 / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_diff needs a GPU")
    dev = torch.device("cuda")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    ids, pm, labels, tm = _batch(B, dev)
    out = {"card": card, "shape": dict(n_items=N_ITEMS, d=D, heads=H, L=L, batch=B, blocks=N_BLOCKS)}
    for enc in ("diff", "sasrec"):
        m = _model(enc)
        s = _timed(lambda: m.core.fused_step(ids, pm, labels, tm), a.steps, a.warmup)
        out[f"train_seq_per_s_{enc}"] = round(B / s, 1)
        if enc == "diff":
            users = _batch(4096, dev)
            m.eval()
            s = _timed(lambda: m.predict_topk({"item_id": users[0]}, users[1], 10, seen_ids=users[0]), a.steps, a.warmup)
            out["predict_users_per_s_diff_4096"] = round(4096 / s, 1)
    # the reference module's computation, eager torch fp32 on the same GPU (oracle/diff.py restates it line by line)
    from oracle import diff as od
    from oracle.sasrec import ce_loss

    sd = {k: v.detach().float().to(dev) for k, v in _model("diff").state_dict().items()}
    P = {k: v.clone().requires_grad_(True) for k, v in od.params_of(sd).items()}
    opt = torch.optim.Adam(P.values(), lr=1e-3, betas=(0.9, 0.98))
    table_key = "body.embedder.feature_embedders.item_id.emb.weight"

    def ref_step():
        opt.zero_grad(set_to_none=True)
        h = od.diff_body(dict(sd, **P), ids, pm, H)
        ce_loss(h, P[table_key][:N_ITEMS], labels, tm).backward()
        opt.step()

    s = _timed(ref_step, max(3, a.steps // 4), 2)
    out["train_seq_per_s_reference_eager"] = round(B / s, 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
