"""One predict() call at the scoring leg's shape (4096 users, L=200, d=128, |I|=500K), e.g. to trace with torch.profiler."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from replay_b200 import ops
from replay_b200.engine import EncoderConfig, SasRecEngine
from replay_b200.synthetic import make_sequences

Bu, L, d, I = 4096, 200, 128, 500_000
es = SasRecEngine(EncoderConfig(n_items=I, d=d, n_heads=2, n_blocks=2, max_len=L, variant="new"), Bu, L, "cuda", seed=7, with_grad=False)
uid, upm, _, _ = make_sequences(Bu, I, L, seed=7)
uid, upm = uid.cuda(), upm.cuda()
tab = es.params16["item_emb"][:I]
for _ in range(3):
    es.set_batch(uid, upm)
    hq = es.forward_last_hidden()
    ops.score_topk(hq, tab, 10, ops.seen_prepare(uid, I))
torch.cuda.synchronize()
