"""BERT4Rec training throughput at shapes the kernels see padded, and the share of the full-catalog head in the step.

    python tools/bench_bert_shapes.py [--steps 30] [--warmup 5] [--shape NAME ...] [--passes P] [--no-positional]
                                      [--kernels FILE]

Shapes (|I| = 100 K, untied biased head, uniform 15 % masking, 2 blocks):
  tutorial  hidden 300 / 4 heads (head_dim 75 -> 4 x 128 = 512 columns, FFN 1200 -> 1280), L = 100, batch 512, dropout 0.5
            (the reference's examples/10_bert4rec_example.ipynb)
  d512      hidden 512 / 8 heads, L = 200, batch 512, dropout 0.1
  c3        hidden 256 / 4 heads, L = 200, batch 256, dropout 0.1 (bench.py's BERT4Rec configuration)
``--passes`` applies every block P times in a row (num_passes_over_block, default 1) and ``--no-positional`` drops the
positional embedding (enable_positional_embedding=False).
The step is Trainer's CUDA-graph step (forward + backward + Adam).  The head share is the CE head's forward + backward
(replay_b200.ops.ce_head_fwd / ce_head_bwd, biased, d = 512 chunked backward) on the step's own rows, timed alone with CUDA
events.  Prints the card name and power limit it read, then one JSON line per shape.  ``--kernels FILE`` also writes, per
shape, the ordered CUDA kernel names of one eager training step recorded with torch.profiler (the launches the captured
step replays), as JSON."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

SHAPES = {"tutorial": dict(d=300, heads=4, L=100, batch=512, dropout=0.5),
          "d512": dict(d=512, heads=8, L=200, batch=512, dropout=0.1),
          "c3": dict(d=256, heads=4, L=200, batch=256, dropout=0.1)}
N_ITEMS, BLOCKS = 100_000, 2


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        out = ""
    return out or torch.cuda.get_device_name(0) + ", power limit unknown"


def elapsed_ms(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def kernel_sequence(eng, ids, pm, tok):
    """ordered CUDA kernel names of one eager training step (forward + backward + Adam)"""
    from torch.profiler import ProfilerActivity, profile

    eng.set_batch(ids, pm, tok, ids)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.train_step()
        torch.cuda.synchronize()
    evs = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "memset" not in e.name.lower()
           and "memcpy" not in e.name.lower()]
    return [e.name for e in sorted(evs, key=lambda e: e.time_range.start)]


def run(name, c, steps, warmup, passes=1, positional=True, kernels=None):
    from replay_b200 import ops
    from replay_b200.engine_bert import Bert4RecEngine, BertConfig
    from replay_b200.models.nn.sequential import uniform_masker
    from replay_b200.synthetic import make_sequences
    from replay_b200.trainer import Trainer

    B, L = c["batch"], c["L"]
    cfg = BertConfig(n_items=N_ITEMS, d=c["d"], n_heads=c["heads"], n_blocks=BLOCKS, max_len=L, dropout=c["dropout"],
                     passes=passes, positional=positional)
    eng = Bert4RecEngine(cfg, B, L, "cuda", seed=1)
    ids, pm, _, _ = make_sequences(B, N_ITEMS, L, seed=3, pad_value=0)
    tok = uniform_masker(pm, 0.15, torch.Generator().manual_seed(0))
    ids, pm, tok = ids.cuda(), pm.cuda(), tok.cuda()
    if kernels is not None:
        kernels[name] = kernel_sequence(eng, ids, pm, tok)
    tr = Trainer(eng)
    for _ in range(warmup):
        loss = tr.step(ids, pm, tok, ids)
    torch.cuda.synchronize()
    ms = elapsed_ms(lambda: tr.step(ids, pm, tok, ids), steps)
    loss = float(tr.step(ids, pm, tok, ids)[0])
    torch.cuda.synchronize()
    W16, bias = eng._head()
    dW = torch.empty(N_ITEMS, cfg.dp, device="cuda")
    db = torch.empty(eng.I128, device="cuda")

    def head():
        ops.ce_head_fwd(eng.ce, eng.hc, W16, eng.labels_c, eng.n_valid, bias=bias, d_hc=eng.s["dhc"])
        ops.ce_head_bwd(eng.ce, eng.hc, W16, eng.labels_c, eng.n_valid, eng.s["dhc"], dW, bias=bias, d_bias=db)

    head()
    torch.cuda.synchronize()
    head_ms = elapsed_ms(head, max(3, steps // 3))
    return dict(shape=name, hidden=c["d"], heads=c["heads"], passes=passes, positional=positional, padded_columns=cfg.dp,
                ffn_columns=cfg.ffn_p, L=L, batch=B, n_items=N_ITEMS, dropout=c["dropout"], n_valid=int(eng.n_valid.item()),
                ms_per_step=round(ms, 3), train_seq_per_s=round(B / ms * 1e3, 1), head_ms=round(head_ms, 3), head_share=round(head_ms / ms, 3),
                loss=round(loss, 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--shape", choices=sorted(SHAPES), action="append")
    ap.add_argument("--passes", type=int, default=1)
    ap.add_argument("--no-positional", action="store_true")
    ap.add_argument("--kernels", help="write the kernel sequence of one eager step per shape to this JSON file")
    args = ap.parse_args()
    print("card:", card())
    kernels = {} if args.kernels else None
    for name in args.shape or ["tutorial", "d512"]:
        print(json.dumps(run(name, SHAPES[name], args.steps, args.warmup, args.passes, not args.no_positional, kernels)),
              flush=True)
    if kernels is not None:
        with open(args.kernels, "w") as fh:
            json.dump(kernels, fh)


if __name__ == "__main__":
    main()
