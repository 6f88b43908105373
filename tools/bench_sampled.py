"""Training-step time of config 2 (SASRec L=200 d=128 H=2 |I|=50K, B=256, dropout 0.2) with the sampled heads next to the
full-catalog CE head (eager launches, CUDA events).  LogInCESampled and CESampledWeighted run beside CESampled in each
negative layout; the card's name, power limit and max SM clock are printed first."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from replay_b200.engine import EncoderConfig, SasRecEngine
from replay_b200.synthetic import make_sequences

B, L, d, I = 256, 200, 128, 50_000
ids, pm, lab, tm = make_sequences(B, I, L, seed=1234)
cases = [("ce", None, 0), ("ce_sampled", "shared", 1000), ("login_ce_sampled", "shared", 1000),
         ("ce_sampled_weighted", "shared", 1000), ("ce_sampled", "shared", 4096), ("bce_sampled", "shared", 1000),
         ("ce_sampled", "perseq", 100), ("login_ce_sampled", "perseq", 100), ("ce_sampled_weighted", "perseq", 100),
         ("ce_sampled", "perpos", 100), ("login_ce_sampled", "perpos", 100), ("ce_sampled_weighted", "perpos", 100),
         ("legacy_ce_sampled", "perpos", 100)]
print(torch.cuda.get_device_name(), "power limit",
      os.popen("nvidia-smi --query-gpu=power.limit,clocks.max.sm --format=csv,noheader").read().strip(), flush=True)
for kind, shape, N in cases:
    eng = SasRecEngine(EncoderConfig(n_items=I, d=d, n_heads=2, n_blocks=2, max_len=L, dropout=0.2, variant="new"), B, L, "cuda", seed=1)
    if kind != "ce":
        eng.set_loss(kind, n_neg=N, neg_shape=shape)
        g = torch.Generator().manual_seed(0)
        neg = {"shared": (N,), "perseq": (B, N), "perpos": (B, L, N)}[shape]
        eng.set_negatives(torch.randint(0, I, neg, generator=g).cuda())
    eng.set_batch(ids.cuda(), pm.cuda(), lab.cuda(), tm.cuda())
    if kind == "ce_sampled_weighted":
        eng.set_row_weights(torch.rand(B, L, generator=torch.Generator().manual_seed(1)).cuda() + 0.5)
    eng.n_valid_hint = int(tm.sum())
    losses = [float(eng.train_step()[0]) for _ in range(5)]
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(20):
        eng.train_step()
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / 20
    print(f"{kind:18s} {str(shape):7s} N={N:5d}: {ms:6.2f} ms/step eager -> {B / ms * 1e3:8.0f} seq/s  loss {losses[0]:.3f} -> {losses[-1]:.3f}", flush=True)
    del eng
    torch.cuda.empty_cache()
