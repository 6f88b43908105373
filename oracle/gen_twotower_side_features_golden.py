"""Generate the side-feature TwoTower golden vectors FROM THE REAL REFERENCE (run in the build container only; the reference
checkout is not on the GPU box).  TEST INFRASTRUCTURE.

    python oracle/gen_twotower_side_features_golden.py

Writes tests/golden/twotower_side_{d64h2,d50h1}.npz from ``replay.nn.sequential.twotower.TwoTower.from_params`` on a
schema with the item id, a categorical of cardinality 20 ("genre"), one of cardinality 1000 ("brand"), a categorical list
of width 4 ("tags"), a numerical feature of tensor_dim 3 ("stats"), an identity numerical ("vec", tensor_dim = d) and a
sequence-only categorical ("ctx").  The item features reader holds every feature but "ctx" (left-padded lists with
all-padding bags, padding values and ids of the item table).  The query tower takes every feature per token (random,
left-padded as in oracle/gen_side_features_golden.py).  Each file holds the batch, the reader, the weights as a seed with
a checksum (oracle.side_features.seeded_state_dict over the model's distinct parameters), the train loss and gradients
for CE (every gradient in full), BCE, CESampled (shared, per-sequence and per-position negatives), LogInCESampled and
CESampledWeighted (the embedder's tables in full, the sum and norm of every gradient), checksums of the state after one
Adam step, the eval logits, candidate logits, a seen-filtered top-10, the full key list and shapes (with and without the
cache).  All with dropout 0.  tests/test_twotower_side_features_cpu.py checks oracle/twotower_side_features.py against
them; tests/test_gpu_twotower_side_features.py the CUDA path.
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

from gen_golden import make_batch  # noqa: E402
from gen_side_features_golden import schema, side_batch  # noqa: E402
from gen_twotower_golden import IGNORE, negatives  # noqa: E402
from oracle.side_features import seeded_state_dict, state_dict_checksum  # noqa: E402
from replay.nn.loss import BCE, CE, CESampled, CESampledWeighted, LogInCESampled  # noqa: E402
from replay.nn.sequential.twotower import TwoTower  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")


def specs(d):
    return [dict(name="genre", kind="cat", cardinality=20, padding_value=20, width=1),
            dict(name="brand", kind="cat", cardinality=1000, padding_value=1000, width=1),
            dict(name="tags", kind="bag", cardinality=30, padding_value=30, width=4),
            dict(name="stats", kind="num", cardinality=0, padding_value=0, width=3),
            dict(name="vec", kind="ident", cardinality=0, padding_value=0, width=d),
            dict(name="ctx", kind="cat", cardinality=7, padding_value=7, width=1)]


READER = ("item_id", "genre", "brand", "tags", "stats", "vec")


def item_columns(g, fs, n_items):
    """The reader's columns over the catalog: padding values, left-padded lists with all-padding bags, ids up to the
    cardinality (the brand table is larger than the catalog)."""
    out = {"item_id": torch.arange(n_items)}
    for f in fs:
        if f["name"] not in READER:
            continue
        if f["kind"] == "cat":
            v = torch.randint(0, f["cardinality"], (n_items,), generator=g)
            v[torch.rand(n_items, generator=g) < 0.1] = f["padding_value"]
        elif f["kind"] == "bag":
            K = f["width"]
            v = torch.randint(0, f["cardinality"], (n_items, K), generator=g)
            n_live = torch.randint(0, K + 1, (n_items,), generator=g)
            n_live[0] = 0                                 # an all-padding bag
            v[torch.arange(K)[None, :] < (K - n_live)[:, None]] = f["padding_value"]
            v[1, -1] = v[1, -2]                           # a repeated id inside one bag
        else:
            v = torch.randn(n_items, f["width"], generator=g)
        out[f["name"]] = v
    return out


class Reader:
    def __init__(self, cols):
        self.cols = cols

    def __getitem__(self, key):
        return self.cols[key]

    @property
    def feature_names(self):
        return list(self.cols)


def run_loss(model, loss, ft, pm, labels, tm, neg=None):
    model.loss = loss
    loss.logits_callback = model.get_logits
    model.train()
    model.zero_grad(set_to_none=True)
    out = model(feature_tensors=ft, padding_mask=pm, positive_labels=labels.unsqueeze(-1), negative_labels=neg,
                target_padding_mask=tm.unsqueeze(-1))
    out["loss"].backward()
    return float(out["loss"]), {k: p.grad.detach().clone() for k, p in model.named_parameters() if p.grad is not None}


def gen(tag, B, L, d, H, n_items, n_blocks, seed, method, N=7):
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    fs = specs(d)
    cols = item_columns(g, fs, n_items)
    sch = schema(n_items, d, fs)
    model = TwoTower.from_params(sch, Reader(cols), embedding_dim=d, num_heads=H, num_blocks=n_blocks, max_sequence_length=L,
                                 dropout=0.0, categorical_list_feature_aggregation_method=method)
    pkeys = [k for k, _ in model.named_parameters()]   # the shared embedder once, under body.embedder
    pshapes = [tuple(p.shape) for _, p in model.named_parameters()]
    pads = {f"body.embedder.feature_embedders.{f['name']}.emb.weight": f["padding_value"] for f in fs if f["kind"] in ("cat", "bag")}
    pads["body.embedder.feature_embedders.item_id.emb.weight"] = n_items
    sd = seeded_state_dict(pkeys, pshapes, seed, pads)
    model.load_state_dict(sd, strict=False)
    ids, pm, labels, tm = make_batch(g, B, L, n_items, n_items)
    feats = side_batch(g, fs, pm)
    ft = {"item_id": ids, **feats}
    full = model.state_dict()
    keys = list(full)
    out = dict(sd_seed=seed, sd_keys=np.array(pkeys), sd_shapes=np.array(["x".join(map(str, t)) for t in pshapes]),
               sd_checksum=state_dict_checksum(sd, pkeys), pad_keys=np.array(list(pads)), pad_rows=np.array(list(pads.values())),
               keys=np.array(keys), key_shapes=np.array(["x".join(map(str, full[k].shape)) for k in keys]),
               key_dtypes=np.array([str(full[k].dtype) for k in keys]), ignore_index=IGNORE, seed=seed, ids=ids.numpy(),
               pad_mask=pm.numpy(), labels=labels.numpy(), target_mask=tm.numpy(), n_items=n_items, d=d, H=H, L=L,
               n_blocks=n_blocks, N=N, method=method, reader=np.array(READER))
    out.update({f"f_{k}": np.array([f[k] for f in fs]) for k in ("name", "kind", "padding_value", "width", "cardinality")})
    out.update({"feat::" + k: v.numpy() for k, v in feats.items()})
    out.update({"item::" + k: v.numpy() for k, v in cols.items()})
    cases = {"ce": (CE(ignore_index=n_items), None, None), "bce": (BCE(), None, None)}
    for shape in ("shared", "perseq", "perpos"):
        neg = negatives(g, B, L, n_items, N, shape, IGNORE)
        if shape == "perpos":
            neg[0, -1, 3] = labels[0, -1]
        out[f"neg_{shape}"] = neg.numpy()
        cases[f"ce_sampled_{shape}"] = (CESampled(negative_labels_ignore_index=IGNORE), neg, None)
    cases["login_ce_sampled_perseq"] = (LogInCESampled(negative_labels_ignore_index=IGNORE), torch.as_tensor(out["neg_perseq"]), None)
    w = torch.rand(B, L, generator=g) * 2
    out["weights"] = w.numpy()
    cases["ce_sampled_weighted_shared"] = (CESampledWeighted(feature_name="sample_weight", negative_labels_ignore_index=IGNORE),
                                           torch.as_tensor(out["neg_shared"]), w.unsqueeze(-1))
    for name, (loss, neg, wt) in cases.items():
        f2 = dict(ft, sample_weight=wt) if wt is not None else ft
        val, grads = run_loss(model, loss, f2, pm, labels, tm, neg)
        out[f"{name}::loss"] = val
        for k, v in grads.items():
            if name == "ce" or ".feature_embedders." in k:
                out[f"{name}::grad::{k}"] = v.numpy().copy()
            out[f"{name}::gsum::{k}"] = np.array([float(v.double().sum()), float(v.double().norm())])
    model.loss = CE(ignore_index=n_items)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3, betas=(0.9, 0.98))
    run_loss(model, model.loss, ft, pm, labels, tm)
    opt.step()
    adam = {k: p.detach() for k, p in model.named_parameters()}
    out["adam_checksum"] = state_dict_checksum(adam, pkeys)
    model.load_state_dict(sd, strict=False)
    model.eval()
    with torch.no_grad():
        lo = model(feature_tensors=ft, padding_mask=pm)["logits"]
        out["eval_logits"] = lo.numpy()
        out["cache_keys"] = np.array(list(model.state_dict()))
        cand = torch.tensor([3, 0, n_items - 1, 7, 11])
        out["candidates"] = cand.numpy()
        out["cand_logits"] = model(feature_tensors=ft, padding_mask=pm, candidates_to_score=cand)["logits"].numpy()
        model.body.item_tower.cache = None   # candidates without the cache: the tower over the candidates' features
        out["cand_logits_nocache"] = model(feature_tensors=ft, padding_mask=pm, candidates_to_score=cand)["logits"].numpy()
        seen = lo.clone()
        for b in range(B):
            seen[b, ids[b][pm[b]]] = -torch.inf
        out["top10"] = torch.topk(seen, 10, dim=-1).indices.numpy()
    path = os.path.join(OUT, f"twotower_side_{tag}.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, "loss", out["ce::loss"], "bytes", os.path.getsize(path))


if __name__ == "__main__":
    gen("d64h2", B=6, L=12, d=64, H=2, n_items=60, n_blocks=2, seed=61, method="sum")
    gen("d50h1", B=5, L=10, d=50, H=1, n_items=45, n_blocks=1, seed=62, method="mean")
