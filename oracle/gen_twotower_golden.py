"""Generate the TwoTower golden vectors FROM THE REAL REFERENCE (run in the build container only).  TEST INFRASTRUCTURE.

    python oracle/gen_twotower_golden.py

Writes tests/golden/twotower_*.npz from ``replay.nn.sequential.twotower.TwoTower.from_params`` with an item-id reader:
seeded inputs, the weights as a seed (oracle.twotower.seeded_state_dict) with a checksum of every tensor, the train loss
and every gradient for CE (bf16 bits; the sum and norm of each for the others), BCE, CESampled (shared, per-sequence and per-position negatives with duplicates,
ignored entries and negatives equal to the positive), LogInCESampled and CESampledWeighted, the state after one Adam
step, the eval logits, candidate logits, a seen-filtered top-10 and the full key list (with and without the cache).  All
with dropout 0.  tests/test_twotower_cpu.py checks oracle/twotower.py against them; tests/test_gpu_twotower.py the CUDA path.
"""
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "shim"))
sys.path.insert(1, "/root/reference")
sys.path.insert(2, HERE)
sys.path.insert(3, os.path.dirname(HERE))
warnings.filterwarnings("ignore")

from gen_golden import make_batch, schema  # noqa: E402
from oracle.diff import checksum, to_bf16_bits  # noqa: E402
from oracle.twotower import seeded_state_dict  # noqa: E402
from replay.nn.loss import BCE, CE, CESampled, CESampledWeighted, LogInCESampled  # noqa: E402
from replay.nn.sequential.twotower import TwoTower  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")


class ItemIdReader:
    def __init__(self, n):
        self.ids = torch.arange(n)

    def __getitem__(self, key):
        return self.ids

    @property
    def feature_names(self):
        return ["item_id"]


IGNORE = 5   # the reference's item tower indexes the candidates before any masking: an ignored id must be an item


def negatives(g, B, L, n_items, N, shape, ignore):
    """negatives with duplicates, ignored entries and (per position) entries equal to the positive"""
    dims = {"shared": (N,), "perseq": (B, N), "perpos": (B, L, N)}[shape]
    neg = torch.randint(0, n_items, dims, generator=g)
    flat = neg.view(-1)
    flat[1] = flat[0]                                  # a duplicate
    flat[2] = ignore                                   # an ignored entry
    return neg


def run_loss(model, loss, ids, pm, labels, tm, neg=None, weights=None):
    model.loss = loss
    loss.logits_callback = model.get_logits   # TwoTower.__init__ wires the loss it is built with only
    model.train()
    model.zero_grad(set_to_none=True)
    ft = {"item_id": ids}
    if weights is not None:
        ft["sample_weight"] = weights
    out = model(feature_tensors=ft, padding_mask=pm, positive_labels=labels.unsqueeze(-1), negative_labels=neg,
                target_padding_mask=tm.unsqueeze(-1))
    out["loss"].backward()
    grads = {}
    for k, p in model.named_parameters():
        if p.grad is not None:
            grads[k] = p.grad.detach().clone()
    return float(out["loss"]), grads


def gen(tag, B, L, d, H, n_items, n_blocks, seed, N=7):
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    sch = schema(n_items, d, n_items)
    model = TwoTower.from_params(sch, ItemIdReader(n_items), embedding_dim=d, num_heads=H, num_blocks=n_blocks,
                                 max_sequence_length=L, dropout=0.0)
    sd = seeded_state_dict(n_items, d, H, L, n_blocks, seed)
    model.load_state_dict(sd, strict=True)
    ids, pm, labels, tm = make_batch(g, B, L, n_items, n_items)
    keys = list(model.state_dict())
    out = dict(ignore_index=IGNORE, sd_keys=np.array(keys), sd_sums=np.array([checksum(model.state_dict()[k]) for k in keys]), seed=seed,
               ids=ids.numpy(), pad_mask=pm.numpy(), labels=labels.numpy(), target_mask=tm.numpy(), n_items=n_items, d=d,
               H=H, L=L, n_blocks=n_blocks, N=N)
    cases = {"ce": (CE(ignore_index=n_items), None, None), "bce": (BCE(), None, None)}
    for shape in ("shared", "perseq", "perpos"):
        neg = negatives(g, B, L, n_items, N, shape, IGNORE)
        if shape == "perpos":   # a negative equal to its positive
            neg[0, -1, 3] = labels[0, -1]
        out[f"neg_{shape}"] = neg.numpy()
        cases[f"ce_sampled_{shape}"] = (CESampled(negative_labels_ignore_index=IGNORE), neg, None)
    cases["login_ce_sampled_perseq"] = (LogInCESampled(negative_labels_ignore_index=IGNORE), torch.as_tensor(out["neg_perseq"]), None)
    w = torch.rand(B, L, generator=g) * 2
    out["weights"] = w.numpy()
    cases["ce_sampled_weighted_shared"] = (CESampledWeighted(feature_name="sample_weight",
                                                             negative_labels_ignore_index=IGNORE),
                                           torch.as_tensor(out["neg_shared"]), w.unsqueeze(-1))
    for name, (loss, neg, wt) in cases.items():
        val, grads = run_loss(model, loss, ids, pm, labels, tm, neg, wt)
        out[f"{name}::loss"] = val
        for k, v in grads.items():   # every gradient of CE in full; of the other losses its sum and norm (size)
            if name == "ce":
                out[f"{name}::grad::{k}"] = to_bf16_bits(v)
            else:
                out[f"{name}::gsum::{k}"] = np.array([float(v.double().sum()), float(v.double().norm())])
    # one Adam step of the CE loss (betas of the reference's optimizer factory)
    model.loss = CE(ignore_index=n_items)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3, betas=(0.9, 0.98))
    run_loss(model, model.loss, ids, pm, labels, tm)
    opt.step()
    out["adam_sums"] = np.array([checksum(v) for k, v in model.state_dict().items() if v.is_floating_point()])
    model.load_state_dict(sd, strict=True)
    model.eval()
    with torch.no_grad():
        lo = model(feature_tensors={"item_id": ids}, padding_mask=pm)["logits"]
        out["eval_logits"] = lo.numpy()
        out["cache_keys"] = np.array(list(model.state_dict()))
        cand = torch.tensor([3, 0, n_items - 1, 7, 11])
        out["candidates"] = cand.numpy()
        out["cand_logits"] = model(feature_tensors={"item_id": ids}, padding_mask=pm, candidates_to_score=cand)["logits"].numpy()
        seen = lo.clone()
        for b in range(B):
            seen[b, ids[b][pm[b]]] = -torch.inf
        out["top10"] = torch.topk(seen, 10, dim=-1).indices.numpy()
    path = os.path.join(OUT, f"twotower_{tag}.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path))


if __name__ == "__main__":
    gen("d64h2", B=6, L=12, d=64, H=2, n_items=40, n_blocks=2, seed=11)
    gen("d50h1", B=5, L=10, d=50, H=1, n_items=33, n_blocks=1, seed=12)
    gen("d128h2", B=4, L=9, d=128, H=2, n_items=29, n_blocks=1, seed=13)
