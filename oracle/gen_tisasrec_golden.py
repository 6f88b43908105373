"""Generate tests/golden/sasrec_ti_*.npz FROM THE REAL REFERENCE's SasRecModel(ti_modification=True) (run in the build
container only; the reference is not on the GPU box).  TEST INFRASTRUCTURE.

    PYTHONPATH=oracle/shim:/root/reference python oracle/gen_tisasrec_golden.py

Each file holds the weights (sd::<key>), the batch (ids, pad, times, labels, tmask), the hidden states of forward_step,
the full-catalog CE loss over the valid targets (legacy lightning.py:335-355) and its gradients (grad::<key>), all at
dropout 0.  Cases: tiny (d 50, 1 head, L 12, time_span 8: clipping, ties and zero gaps), d 64 / 2 heads / L 50 /
time_span 256 with int64 timestamps and left padding at timestamp 0, and float32 timestamps whose differences round."""
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "shim"))
sys.path.insert(1, "/root/reference")
warnings.filterwarnings("ignore")

from replay.data import FeatureHint, FeatureSource, FeatureType  # noqa: E402
from replay.data.nn import TensorFeatureInfo, TensorFeatureSource, TensorSchema  # noqa: E402
from replay.models.nn.sequential.sasrec.model import SasRecModel  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")


def schema(n_items, d):
    return TensorSchema([
        TensorFeatureInfo(name="item_id", is_seq=True, cardinality=n_items, padding_value=n_items, embedding_dim=d,
                          feature_type=FeatureType.CATEGORICAL,
                          feature_sources=[TensorFeatureSource(FeatureSource.INTERACTIONS, "item_id")],
                          feature_hint=FeatureHint.ITEM_ID),
        TensorFeatureInfo(name="timestamp", is_seq=True, feature_type=FeatureType.NUMERICAL,
                          feature_sources=[TensorFeatureSource(FeatureSource.INTERACTIONS, "timestamp")],
                          feature_hint=FeatureHint.TIMESTAMP)])


def make_batch(g, B, L, n_items, times_kind):
    lens = torch.randint(1, L + 2, (B,), generator=g)
    lens[0], lens[1] = L + 1, 2
    ids = torch.full((B, L + 1), n_items, dtype=torch.int64)
    msk = torch.zeros(B, L + 1, dtype=torch.bool)
    times = torch.zeros(B, L + 1, dtype=torch.float64)
    for b in range(B):
        n = int(lens[b])
        ids[b, L + 1 - n:] = torch.randint(0, n_items, (n,), generator=g)
        msk[b, L + 1 - n:] = True
        if times_kind == "tiny":     # steps of 0 (ties), 1 .. 4 and 9 .. 12 (beyond time_span 8)
            steps = torch.randint(0, 3, (n,), generator=g) * 4 + torch.randint(0, 2, (n,), generator=g) * 5
        elif times_kind == "int":
            steps = torch.randint(0, 200, (n,), generator=g) * torch.randint(0, 2, (n,), generator=g)
        else:                        # seconds around 1.7e9: float32 holds them to 128 s, so the differences round
            steps = torch.rand(n, generator=g, dtype=torch.float64) * 600
        times[b, L + 1 - n:] = (1.7e9 if times_kind == "float" else 1000) + steps.double().cumsum(0)
    times = times.float() if times_kind == "float" else times.long()
    return ids[:, :-1], msk[:, :-1], times[:, :-1], ids[:, 1:], msk[:, 1:]


def gen(tag, B, L, d, H, n_items, span, times_kind, seed):
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    model = SasRecModel(schema(n_items, d), num_blocks=2, num_heads=H, hidden_size=d, max_len=L, dropout=0.0,
                        ti_modification=True, time_span=span).double()
    with torch.no_grad():
        for _, p in model.named_parameters():
            if p.dim() == 1:
                p.add_(torch.randn(p.shape, generator=g, dtype=torch.float64) * 0.05)
    model.eval()
    ids, pad, times, labels, tmask = make_batch(g, B, L, n_items, times_kind)
    feats = {"item_id": ids, "timestamp": times}
    hidden = model.forward_step(feats, pad)
    logits = model.get_logits(hidden)
    loss = torch.nn.functional.cross_entropy(logits[tmask], labels[tmask])
    model.zero_grad()
    loss.backward()
    out = {"sd::" + k: v.detach().float().numpy().copy() for k, v in model.state_dict().items()}
    out.update({"grad::" + k: (p.grad if p.grad is not None else torch.zeros_like(p)).float().numpy().copy()
                for k, p in model.named_parameters()})
    out.update(ids=ids.numpy(), pad=pad.numpy(), times=times.numpy(), labels=labels.numpy(), tmask=tmask.numpy(),
               hidden=hidden.detach().float().numpy(), loss=np.float64(loss.item()), n_heads=H, time_span=span)
    np.savez_compressed(os.path.join(OUT, f"sasrec_ti_{tag}.npz"), **out)
    print(tag, float(loss))


if __name__ == "__main__":
    gen("tiny", 6, 12, 50, 1, 40, 8, "tiny", 1)
    gen("d64h2", 8, 50, 64, 2, 300, 256, "int", 2)
    gen("fp32_times", 8, 40, 64, 2, 200, 64, "float", 3)
