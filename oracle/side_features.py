"""Plain-torch CPU restatement of the new-path SASRec's input stage with side features (TEST INFRASTRUCTURE - see
oracle/__init__.py): ``SequenceEmbedding`` over every schema feature, summed by ``SumAggregator``, then the SASRec body of
oracle/sasrec.py.

Reference files restated (under /root/reference/replay): nn/embedding.py (CategoricalEmbedding: Embedding / EmbeddingBag
with ``padding_idx``; NumericalEmbedding: Linear(tensor_dim, d), values [B, L] when tensor_dim == 1; IdentityEmbedding),
nn/agg.py:44-53 (SumAggregator), nn/sequential/sasrec/agg.py:37-53 (x = s * sqrt(d) + pe[-L:], dropout).

A feature spec is a dict ``name, kind ("cat" | "bag" | "num" | "ident"), cardinality, padding_value, width`` (bag width K
or numerical tensor_dim).  Side parameters of the canonical dict ``P["side"]``: ``<name>`` = table [cardinality + 1, d] for
"cat" / "bag", ``<name>.w`` [d, tensor_dim] and ``<name>.b`` [d] for "num".
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import sasrec as osr

PREFIX = "body.embedder.feature_embedders."


def side_from_state_dict(sd, specs):
    out = {}
    for f in specs:
        if f["kind"] in ("cat", "bag"):
            out[f["name"]] = sd[f"{PREFIX}{f['name']}.emb.weight"]
        elif f["kind"] == "num":
            out[f["name"] + ".w"] = sd[f"{PREFIX}{f['name']}.linear.weight"]
            out[f["name"] + ".b"] = sd[f"{PREFIX}{f['name']}.linear.bias"]
    return out


def seeded_state_dict(keys, shapes, seed, pad_rows):
    """Weights drawn from ``seed`` in the given key order (2-D xavier-normal, norm weights 1 + 0.05 N, other 1-D 0.05 N).
    ``pad_rows``: key -> padding row, zeroed as ``torch.nn.Embedding(padding_idx=...)`` initialises it."""
    g = torch.Generator().manual_seed(int(seed))
    sd = {}
    for k, shp in zip(keys, shapes):
        shp = tuple(int(n) for n in shp)
        v = torch.randn(shp, generator=g, dtype=torch.float32)
        if len(shp) == 2:
            v = v * math.sqrt(2.0 / (shp[0] + shp[1]))
        else:
            v = v * 0.05 + (1.0 if "norm" in k and k.endswith(".weight") else 0.0)
        if k in pad_rows:
            v[pad_rows[k]] = 0.0
        sd[k] = v
    return sd


def state_dict_checksum(sd, keys):
    return np.array([[float(sd[k].double().sum()), float((sd[k].double() ** 2).sum())] for k in keys])


def golden_state_dict(z):
    """The reference weights of a golden file: regenerated from ``sd_seed`` and checked against ``sd_checksum``."""
    keys = [str(k) for k in z["sd_keys"]]
    shapes = [tuple(int(n) for n in str(s).split("x")) for s in z["sd_shapes"]]
    pads = {str(k): int(r) for k, r in zip(z["pad_keys"], z["pad_rows"])}
    sd = seeded_state_dict(keys, shapes, int(z["sd_seed"]), pads)
    if not np.allclose(state_dict_checksum(sd, keys), z["sd_checksum"], rtol=1e-6, atol=1e-6):
        raise AssertionError("regenerated weights do not match the golden checksum")
    return sd


def golden_specs(z):
    return [dict(name=str(n), kind=str(k), cardinality=int(c), padding_value=int(p), width=int(w))
            for n, k, c, p, w in zip(z["f_name"], z["f_kind"], z["f_card"], z["f_pad"], z["f_width"])]


def embed_sum(P, specs, ids, feats, method="sum"):
    """s [B, L, d]: the item row plus every side term (nn/embedding.py + nn/agg.py SumAggregator)."""
    s = P["item_emb"][ids]
    side = P["side"]
    for f in specs:
        v = feats[f["name"]]
        if f["kind"] == "cat":
            tab = side[f["name"]]
            s = s + torch.where((v == f["padding_value"]).unsqueeze(-1), torch.zeros_like(tab[0]), tab[v])
        elif f["kind"] == "bag":
            tab = side[f["name"]]
            keep = (v != f["padding_value"]).to(tab.dtype)
            tot = (tab[v] * keep.unsqueeze(-1)).sum(-2)
            if method == "mean":
                tot = tot / keep.sum(-1, keepdim=True).clamp_min(1.0)
            s = s + tot
        elif f["kind"] == "num":
            x = v.to(s.dtype)
            if f["width"] == 1 and x.dim() == 2:
                x = x.unsqueeze(-1)
            s = s + x @ side[f["name"] + ".w"].T + side[f["name"] + ".b"]
        else:
            s = s + v.to(s.dtype)
    return s


def body(P, specs, ids, feats, pad_mask, n_heads, method="sum", lnf_eps=1e-5):
    """Train-mode hidden states [B, L, d] (dropout off) of oracle.sasrec.sasrec_body's new path on the summed input."""
    B, L = ids.shape
    d = P["item_emb"].shape[1]
    pad_id = P["item_emb"].shape[0] - 1
    ids = ids.masked_fill(~pad_mask, pad_id)
    x = embed_sum(P, specs, ids, feats, method) * (d ** 0.5) + P["pos_emb"][P["pos_emb"].shape[0] - L:].unsqueeze(0)
    causal = torch.tril(torch.ones(L, L, dtype=torch.bool))
    visible = causal.unsqueeze(0) & pad_mask.unsqueeze(1)
    for blk in P["blocks"]:
        q = osr.layer_norm(x, blk["ln1_w"], blk["ln1_b"], 1e-8)
        x = q + osr.mha(q, x, blk, n_heads, visible)
        x = osr.layer_norm(x, blk["ln2_w"], blk["ln2_b"], 1e-8)
        x = x + (torch.relu(x @ blk["w1"].T + blk["b1"]) @ blk["w2"].T + blk["b2"])
    return osr.layer_norm(x, P["lnf_w"], P["lnf_b"], lnf_eps)


def loss_and_grads(P, specs, ids, feats, pad_mask, labels, target_mask, n_heads, method="sum"):
    """CE loss and autograd gradients of every parameter (pad rows of the categorical tables frozen)."""
    def leaf(v):
        return v.detach().clone().requires_grad_(True)

    Pg = {k: ([{kk: leaf(vv) for kk, vv in b.items()} for b in v] if k == "blocks" else
              {kk: leaf(vv) for kk, vv in v.items()} if k == "side" else leaf(v)) for k, v in P.items()}
    h = body(Pg, specs, ids, feats, pad_mask, n_heads, method)
    n_items = Pg["item_emb"].shape[0] - 1
    loss = osr.ce_loss(h, Pg["item_emb"][:n_items], labels, target_mask)
    loss.backward()

    def grad(v):
        return v.grad if v.grad is not None else torch.zeros_like(v)

    G = {k: ([{kk: grad(vv) for kk, vv in b.items()} for b in v] if k == "blocks" else
             {kk: grad(vv) for kk, vv in v.items()} if k == "side" else grad(v)) for k, v in Pg.items()}
    G["item_emb"][-1].zero_()
    for f in specs:
        if f["kind"] in ("cat", "bag"):
            G["side"][f["name"]][f["padding_value"]].zero_()
    return loss.detach(), G
