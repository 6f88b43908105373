"""TwoTower training and predict rates (CUDA events, eager launches), next to the new-path SasRec on the same inputs.

    python tools/bench_twotower.py [--shape c2|c5|all]

c2: L 200, d 128, 2 heads, |I| 50 K, 512 sequences per step.  c5: L 512, d 512, 8 heads, |I| 1 M, 32 sequences.
Per shape: training ms/step and seq/s with CE and with CESampled (256 shared negatives) for TwoTower and SasRec; the item
tower's own forward + backward time over the rows each loss gives it (the catalog for CE, the compacted candidates'
capacity for CESampled); whether the CE head's single-pass path ran (ops.ce_head_fused_taken: its device bound on
max|h| * max|e| decides); the peak device memory of each training engine; predict users/s for a seen-filtered top-10.  The card's name, power limit and max SM clock are
printed first."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from replay_b200 import ops
from replay_b200.engine import EncoderConfig, SasRecEngine
from replay_b200.engine_twotower import TwoTowerConfig, TwoTowerEngine
from replay_b200.synthetic import make_sequences

SHAPES = {"c2": dict(B=512, L=200, d=128, H=2, I=50_000, predict_B=4096), "c5": dict(B=32, L=512, d=512, H=8, I=1_000_000, predict_B=256)}


def timed(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def run(name, s, steps):
    B, L, d, H, I = s["B"], s["L"], s["d"], s["H"], s["I"]
    ids, pm, lab, tm = (t.cuda() for t in make_sequences(B, I, L, seed=1234))
    neg = torch.randint(0, I, (256,), generator=torch.Generator().manual_seed(0)).cuda()
    for model in ("twotower", "sasrec"):
        for kind in ("ce", "ce_sampled"):
            torch.cuda.reset_peak_memory_stats()
            if model == "twotower":
                eng = TwoTowerEngine(TwoTowerConfig(n_items=I, d=d, n_heads=H, n_blocks=2, max_len=L, dropout=0.2), B, L, "cuda", seed=1)
            else:
                eng = SasRecEngine(EncoderConfig(n_items=I, d=d, n_heads=H, n_blocks=2, max_len=L, dropout=0.2, variant="new"), B, L,
                                   "cuda", seed=1)
            eng.packed_body = True
            if kind != "ce":
                eng.set_loss(kind, n_neg=256, neg_shape="shared")
                eng.set_negatives(neg)
            eng.set_batch(ids, pm, lab, tm)
            eng.n_valid_hint = int(tm.sum())
            losses = [float(eng.train_step()[0]) for _ in range(3)]
            ms = timed(eng.train_step, steps)
            line = f"{name} {model:8s} {kind:10s}: {ms:7.2f} ms/step -> {B / ms * 1e3:9.0f} seq/s  loss {losses[0]:.3f} -> {losses[-1]:.3f}"
            line += f"  peak memory {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB"
            if kind == "ce":
                line += f"  CE single-pass path: {ops.ce_head_fused_taken(eng.ce)}"
            if model == "twotower":
                rows = I if kind == "ce" else eng.sampled["cap"]
                x0 = eng.params16["item_emb"] if kind == "ce" else eng.tw["x0"]
                out = eng.tw["cache"] if kind == "ce" else eng.tw["out"]

                def tower():
                    eng.tower_forward(x0, rows, out)
                    eng.tower_backward(x0, rows)

                tower()
                line += f"  tower fwd+bwd over {rows} rows: {timed(tower, steps):.2f} ms"
                if kind == "ce_sampled":
                    line += f" ({int(eng.tw['n_slots'])} distinct candidates)"
            print(line, flush=True)
            if model == "twotower" and kind == "ce":
                P = s["predict_B"]
                pids, ppm, _, _ = (t.cuda() for t in make_sequences(P, I, L, seed=99))
                inf = TwoTowerEngine(TwoTowerConfig(n_items=I, d=d, n_heads=H, n_blocks=2, max_len=L), P, L, "cuda", seed=1,
                                     with_grad=False)
                inf.p32.copy_(eng.p32)
                inf.refresh_shadow()
                table = inf.tower_table()
                seen = ops.seen_prepare(pids.masked_fill(~ppm, I), I)

                def predict():
                    inf.set_batch(pids, ppm)
                    ops.score_topk(inf.forward_last_hidden(), table, 10, seen)

                predict()
                ms_p = timed(predict, max(3, steps // 2))

                def recompute():
                    inf.tower_valid = False
                    inf.tower_table()

                tower_ms = timed(recompute, 3)
                print(f"{name} twotower predict top-10: {P} users in {ms_p:.2f} ms -> {P / ms_p * 1e3:9.0f} users/s "
                      f"(tower over the catalog once: {tower_ms:.2f} ms)",
                      flush=True)
                del inf, table
            del eng
            torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="all", choices=["c2", "c5", "all"])
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    print(torch.cuda.get_device_name(), "power limit, max SM clock:",
          os.popen("nvidia-smi --query-gpu=power.limit,clocks.max.sm --format=csv,noheader").read().strip(), flush=True)
    for name in (["c2", "c5"] if args.shape == "all" else [args.shape]):
        run(name, SHAPES[name], args.steps)


if __name__ == "__main__":
    main()
