"""Plain-torch CPU restatement of the new-path SASRec's input stage through ConcatAggregator (TEST INFRASTRUCTURE - see
oracle/__init__.py): ``SequenceEmbedding`` over every schema feature, each at its own embedding_dim, concatenated in
ascending order of feature name and projected by ``feat_projection``, then the SASRec body of oracle/sasrec.py.

Reference files restated (under /root/reference/replay): nn/embedding.py (every feature kind, as oracle/side_features.py
restates it), nn/agg.py:56-109 (ConcatAggregator: sorted names, torch.cat, Linear(sum of widths, d) with more than one
input), nn/sequential/sasrec/agg.py:37-53 (x = agg * sqrt(d) + pe[-L:], dropout).

Feature specs are oracle/side_features.py's with one more key, ``dim`` (the feature's embedding width).  Side parameters
are ``P["side"]`` as there, at width ``dim``; ``P["proj_w"]`` [d, sum of widths] and ``P["proj_b"]`` [d] are the projection
(absent with the item alone).
"""
from __future__ import annotations

import numpy as np
import torch

from . import sasrec as osr
from . import side_features as osf

PROJ = "body.embedding_aggregator.embedding_aggregator.feat_projection."


def golden_specs(z):
    specs = osf.golden_specs(z)
    for f, dim in zip(specs, z["f_dim"]):
        f["dim"] = int(dim)
    return specs


def params_from_state_dict(sd, specs):
    P = osr.params_from_new_state_dict(sd)
    P["side"] = osf.side_from_state_dict(sd, specs)
    if PROJ + "weight" in sd:
        P["proj_w"], P["proj_b"] = sd[PROJ + "weight"], sd[PROJ + "bias"]
    return P


def feature_embedding(P, f, feats, shape, method):
    """One side feature's embedding [B, L, dim], from oracle/side_features.py's term of that feature alone."""
    zero = {"item_emb": torch.zeros(1, f["dim"], dtype=P["item_emb"].dtype), "side": P["side"]}
    return osf.embed_sum(zero, [f], torch.zeros(shape, dtype=torch.long), feats, method)


def embed_concat(P, specs, ids, feats, item_name="item_id", method="sum"):
    """The aggregated input [B, L, d] before the sqrt(d) scale: sorted concatenation, projected with more than one input."""
    parts = {item_name: P["item_emb"][ids]}
    for f in specs:
        parts[f["name"]] = feature_embedding(P, f, feats, ids.shape, method)
    x = torch.cat([parts[k] for k in sorted(parts)], dim=-1)
    if len(parts) > 1:
        x = x @ P["proj_w"].T + P["proj_b"]
    return x


def body(P, specs, ids, feats, pad_mask, n_heads, item_name="item_id", method="sum", lnf_eps=1e-5):
    """Train-mode hidden states [B, L, d] (dropout off) of the new-path body on the concatenated input."""
    B, L = ids.shape
    d = P["item_emb"].shape[1]
    pad_id = P["item_emb"].shape[0] - 1
    ids = ids.masked_fill(~pad_mask, pad_id)
    x = embed_concat(P, specs, ids, feats, item_name, method) * (d ** 0.5) + P["pos_emb"][P["pos_emb"].shape[0] - L:].unsqueeze(0)
    causal = torch.tril(torch.ones(L, L, dtype=torch.bool))
    visible = causal.unsqueeze(0) & pad_mask.unsqueeze(1)
    for blk in P["blocks"]:
        q = osr.layer_norm(x, blk["ln1_w"], blk["ln1_b"], 1e-8)
        x = q + osr.mha(q, x, blk, n_heads, visible)
        x = osr.layer_norm(x, blk["ln2_w"], blk["ln2_b"], 1e-8)
        x = x + (torch.relu(x @ blk["w1"].T + blk["b1"]) @ blk["w2"].T + blk["b2"])
    return osr.layer_norm(x, P["lnf_w"], P["lnf_b"], lnf_eps)


def loss_and_grads(P, specs, ids, feats, pad_mask, labels, target_mask, n_heads, item_name="item_id", method="sum"):
    """CE loss and autograd gradients of every parameter (pad rows of the item and categorical tables frozen)."""
    def leaf(v):
        return v.detach().clone().requires_grad_(True)

    Pg = {k: ([{kk: leaf(vv) for kk, vv in b.items()} for b in v] if k == "blocks" else
              {kk: leaf(vv) for kk, vv in v.items()} if k == "side" else leaf(v)) for k, v in P.items()}
    h = body(Pg, specs, ids, feats, pad_mask, n_heads, item_name, method)
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


def batch_of(z, specs):
    """(ids, pad_mask, labels, target_mask, feats) of a golden file, as CPU tensors"""
    t = lambda k: torch.from_numpy(np.asarray(z[k]))  # noqa: E731
    return t("ids"), t("pad_mask"), t("labels"), t("target_mask"), {f["name"]: t("feat::" + f["name"]) for f in specs}
