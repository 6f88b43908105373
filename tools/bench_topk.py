"""Fused scores -> seen filter -> top-K (rp_score_topk) at the config-4 predict shape, for K up to 1024.

    python tools/bench_topk.py [--iters 10] [--warmup 3]

Shape: 500 000 items, d = 128, 200 seen ids per user, seeded random inputs.  Reports, with CUDA events:
  fused      ops.score_topk for K in {10, 32, 100, 256, 1024} x {512, 4096, 32 768} users per call
  dense      the path it replaces: bf16 logits GEMM -> fp32 [B, |I|] -> clone + seen scatter -> torch.topk, where it fits
  e2e        K = 100 through TorchTopItemsCallback + SeenItemsFilter on a new-path SasRec (2 blocks, L = 200), 4096 users
  ascending  the worst case for admission: scores strictly increasing with the column over the whole catalog (the last
             item split admits every item), same K x users grid as fused
Prints the card name and power limit it read, then one JSON line per measurement."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

I, D, S = 500_000, 128, 200
KS, USERS = (10, 32, 100, 256, 1024), (512, 4096, 32768)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        out = ""
    return out or torch.cuda.get_device_name(0) + ", power limit unknown"


def elapsed_ms(fn, n, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def emit(**kw):
    print(json.dumps(kw), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_topk.py needs a GPU")
    from replay_b200 import ops

    print(f"card: {card()}", flush=True)
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(0)
    table = (torch.randn(I, D, device=dev, generator=g) * 0.05).to(torch.bfloat16)
    hq_all = (torch.randn(max(USERS), D, device=dev, generator=g) * 0.3).to(torch.bfloat16)
    seen_all = torch.randint(0, I + 50, (max(USERS), S), device=dev, generator=g)
    gemm_tflop = lambda B: 2.0 * B * I * D / 1e12  # noqa: E731
    for B in USERS:
        hq, seen = hq_all[:B].contiguous(), seen_all[:B].contiguous()
        ss = ops.seen_prepare(seen, I)
        for K in KS:
            ms = elapsed_ms(lambda: ops.score_topk(hq, table, K, ss), args.iters, args.warmup)
            emit(kind="fused", users=B, K=K, ms=round(ms, 4), users_per_s=round(B / ms * 1e3),
                 tflops=round(gemm_tflop(B) / ms * 1e3, 1))
        for K in (10, 100, 1024):
            need = 2 * B * I * 4 + B * I * 2
            if need > torch.cuda.mem_get_info()[0] * 0.9:
                emit(kind="dense", users=B, K=K, ms=None, note=f"does not fit: needs {need / 1e9:.1f} GB of logits")
                continue
            ok = (seen >= 0) & (seen < I)
            rows = torch.arange(B, device=dev)[:, None].expand_as(seen)[ok]
            cols = seen[ok]

            def dense():
                logits = torch.mm(hq, table.T).float()
                filt = logits.clone()
                filt[rows, cols] = float("-inf")
                return torch.topk(filt, K, dim=1)

            ms = elapsed_ms(dense, args.iters, args.warmup)
            emit(kind="dense", users=B, K=K, ms=round(ms, 4), users_per_s=round(B / ms * 1e3))
            torch.cuda.empty_cache()
    # worst case for the wide kernel: every item beats all earlier ones.  Rows are the base-256 digits of the column + 1 and
    # hq = (1, 2^-8, 2^-16): the score (j + 1) / 65536 is exact in bf16 x fp32 and strictly increasing over all I items,
    # so the last item split admits every item and no other split can raise its threshold
    j = torch.arange(I, device=dev) + 1
    asc = torch.zeros(I, D, device=dev)
    asc[:, 0], asc[:, 1], asc[:, 2] = (j // 65536).float(), ((j // 256) % 256).float(), (j % 256).float()
    asc = asc.to(torch.bfloat16)
    hq_asc = torch.zeros(max(USERS), D, device=dev)
    hq_asc[:, 0], hq_asc[:, 1], hq_asc[:, 2] = 1.0, 2.0 ** -8, 2.0 ** -16
    hq_asc = hq_asc.to(torch.bfloat16)
    s = (hq_asc[:1].float() @ asc.float().T)[0]  # fp32, as the kernel accumulates
    assert bool((s[1:] > s[:-1]).all()), "the ascending catalog is not strictly increasing"
    for B in USERS:
        hq = hq_asc[:B].contiguous()
        ss = ops.seen_prepare(seen_all[:B].contiguous(), I)
        for K in KS:
            ms = elapsed_ms(lambda: ops.score_topk(hq, asc, K, ss), args.iters, args.warmup)
            emit(kind="ascending", users=B, K=K, ms=round(ms, 4), users_per_s=round(B / ms * 1e3))
    del asc, hq_asc
    # end to end through the new-path predict callback
    from replay_b200.nn.lightning import LightningModule, SeenItemsFilter, TorchTopItemsCallback
    from replay_b200.nn.sequential import SasRec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema
    from replay_b200.synthetic import make_sequences

    B, L = 4096, 200
    model = SasRec.from_params(TensorSchema(TensorFeatureInfo("item_id", I, I, D)), embedding_dim=D, num_heads=2,
                               num_blocks=2, max_sequence_length=L, dropout=0.0, seed=1)
    model.eval()
    lm = LightningModule(model)
    ids, pm, _, _ = (t.to(dev) for t in make_sequences(B, I, L, seed=2))
    batch = {"query_id": torch.arange(B, device=dev), "feature_tensors": {"item_id": ids}, "padding_mask": pm, "seen_ids": ids}
    for K in (10, 100):
        cb = TorchTopItemsCallback(top_k=K, query_column="query_id", item_column="item_id",
                                   postprocessors=[SeenItemsFilter(item_count=I, seen_items_column="seen_ids")])
        cb.on_predict_epoch_start(None, lm)

        def step():
            cb.on_predict_batch_end(None, lm, lm.predict_step(batch, 0), batch, 0)
            cb._query_batches.clear(); cb._item_batches.clear(); cb._item_scores.clear()

        ms = elapsed_ms(step, args.iters, args.warmup)
        emit(kind="e2e_callback", users=B, K=K, ms=round(ms, 4), users_per_s=round(B / ms * 1e3))


if __name__ == "__main__":
    main()
