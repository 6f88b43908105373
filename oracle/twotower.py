"""Plain-torch restatement of RePlay's TwoTower with the from_params towers (TEST INFRASTRUCTURE - see oracle/__init__.py).

Parameters are the reference's own ``state_dict`` (keys of ``TwoTower.from_params``); everything is computed in their dtype
(fp64 to adjudicate).  The query tower is oracle/sasrec.py's new-path body; the item tower is SwiGLUEncoder(d, 2d).

Reference files restated (under replay/ of the reference project):
  nn/sequential/twotower/model.py (QueryTower, ItemTower, TwoTower.get_logits / forward_*) ; nn/ffn.py:60-135 (SwiGLU,
  SwiGLUEncoder) ; nn/loss/{ce,bce,login_ce}.py through oracle/sampled.py and oracle/sampled_ext.py
"""
from __future__ import annotations

import math

import torch

from . import sampled as osm
from . import sampled_ext as osx
from . import sasrec as osr

RMS_EPS = float(torch.finfo(torch.float32).eps)   # torch.nn.RMSNorm(eps=None) on the reference's fp32 activations
ITEM_KEYS = tuple(f"body.{p}embedder.feature_embedders.item_id.emb.weight" for p in ("", "query_tower.", "item_tower."))


def n_blocks_of(sd) -> int:
    n = 0
    while f"body.query_tower.encoder.attention_layers.{n}.in_proj_weight" in sd:
        n += 1
    return n


def query_params(sd) -> dict:
    """oracle/sasrec.py's canonical parameters of the query tower (the shared item table under the main key)"""
    q = {k.replace("body.query_tower.", "body."): v for k, v in sd.items() if k.startswith("body.query_tower.")}
    q[ITEM_KEYS[0]] = sd[ITEM_KEYS[0]]
    n = osr._count_blocks(q, "body.encoder.")
    return {"item_emb": q[ITEM_KEYS[0]], "pos_emb": q["body.embedding_aggregator.pe.weight"],
            "blocks": osr._blocks_from_sd(q, "body.encoder.", n), "lnf_w": q["body.output_normalization.weight"],
            "lnf_b": q["body.output_normalization.bias"]}


def rms_norm(x, w, eps=RMS_EPS):
    return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps) * w


def swiglu_encoder(sd, x):
    """SwiGLUEncoder.forward: x = norm1(sw1(x) + x); x = norm2(sw2(x) + x)"""
    for layer in (1, 2):
        p = f"body.item_tower.encoder.sw{layer}."
        g = x @ sd[p + "WG.weight"].T + sd[p + "WG.bias"]
        lin = x @ sd[p + "W1.weight"].T + sd[p + "W1.bias"]
        y = (torch.nn.functional.silu(g) * lin) @ sd[p + "W2.weight"].T + sd[p + "W2.bias"]
        x = rms_norm(y + x, sd[f"body.item_tower.encoder.norm{layer}.weight"])
    return x


def item_tower(sd, candidates=None):
    """ItemTower.forward: the encoder over the item table's rows of the catalog (or of the candidates)"""
    n = sd["body.item_tower.item_reference_item_id"].numel()
    ids = torch.arange(n) if candidates is None else candidates
    return swiglu_encoder(sd, sd[ITEM_KEYS[0]][ids])


def query_hidden(sd, ids, pad_mask, n_heads):
    return osr.sasrec_body(query_params(sd), ids, pad_mask, n_heads, "new")


def bce_full(hidden, table, labels, target_mask):
    """replay/nn/loss/bce.py:10-95: BCEWithLogits(sum) against the one-hot positive over the catalog / number of targets"""
    h, y = hidden[target_mask], labels[target_mask]
    z = h @ table.T
    onehot = torch.zeros_like(z)
    onehot[torch.arange(len(y)), y] = 1
    return torch.nn.functional.binary_cross_entropy_with_logits(z, onehot, reduction="sum") / len(y)


def train_loss(sd, ids, pad_mask, labels, target_mask, n_heads, kind="ce", negatives=None, weights=None, ignore_index=-100,
               log_eps=1e-6, clamp=100.0):
    """TwoTower.forward_train's loss.  The item tower is row-wise, so the sampled losses' item_tower(candidates) rows equal
    the catalog tower's rows at those ids: the sampled heads score the catalog tower directly."""
    h = query_hidden(sd, ids, pad_mask, n_heads)
    Y = item_tower(sd)
    if kind == "ce":
        return osr.ce_loss(h, Y, labels, target_mask)
    if kind == "bce":
        return bce_full(h, Y, labels, target_mask)
    if kind == "ce_sampled":
        return osm.ce_sampled(h, Y, labels, negatives, target_mask, ignore_index=ignore_index)
    if kind == "bce_sampled":
        return osm.bce_sampled(h, Y, labels, negatives, target_mask, log_eps, clamp, ignore_index=ignore_index)
    if kind == "login_ce_sampled":
        return osx.login_ce_sampled(h, Y, labels, negatives, target_mask, log_eps, clamp, ignore_index=ignore_index)
    if kind == "ce_sampled_weighted":
        return osx.ce_sampled_weighted(h, Y, labels, negatives, target_mask, weights, ignore_index=ignore_index)
    raise ValueError(kind)


def loss_and_grads(sd, *args, **kwargs):
    """Loss and d(loss)/d(every parameter), keyed like ``sd``.  The shared item table's gradient is under the main key
    (``body.embedder...``); its padding row is frozen (torch.nn.Embedding(padding_idx))."""
    leaves = {k: v.detach().clone().requires_grad_(v.is_floating_point()) for k, v in sd.items() if k not in ITEM_KEYS[1:]}
    view = dict(leaves)
    for k in ITEM_KEYS[1:]:
        view[k] = leaves[ITEM_KEYS[0]]
    loss = train_loss(view, *args, **kwargs)
    loss.backward()
    G = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in leaves.items() if v.is_floating_point()}
    G[ITEM_KEYS[0]][-1].zero_()
    return loss.detach(), G


def eval_logits(sd, ids, pad_mask, n_heads, candidates=None):
    """TwoTower.forward_inference's logits: the last position's query state against the item tower"""
    h = query_hidden(sd, ids, pad_mask, n_heads)[:, -1]
    return h @ item_tower(sd, candidates).T


def seeded_state_dict(n_items, d, n_heads, L, n_blocks, seed, dtype=torch.float32) -> dict:
    """A TwoTower state_dict drawn from ``seed`` (keys in the reference's order): xavier-scaled matrices, 1-D parameters
    around their initial values so every term of the model is exercised; the padding row of the item table zero."""
    from replay_b200.nn.sequential.twotower import twotower_keys

    g = torch.Generator().manual_seed(seed)
    shapes = _shapes(n_items, d, L, n_blocks)
    sd = {}
    for k in twotower_keys(n_blocks):
        if k.endswith("item_reference_item_id"):
            sd[k] = torch.arange(n_items)
            continue
        if k in ITEM_KEYS[1:]:
            sd[k] = sd[ITEM_KEYS[0]]
            continue
        shp = shapes(k)
        if len(shp) >= 2:
            v = torch.randn(shp, generator=g) * math.sqrt(2.0 / (shp[0] + shp[1]))
            if k == ITEM_KEYS[0]:
                v = v * 4
                v[n_items].zero_()
        elif k.endswith(("norm1.weight", "norm2.weight", "layernorms.0.weight", "output_normalization.weight")) or \
                "layernorms" in k and k.endswith("weight"):
            v = 1 + 0.1 * torch.randn(shp, generator=g)
        else:
            v = 0.05 * torch.randn(shp, generator=g)
        sd[k] = v.to(dtype)
    return sd


def _shapes(n_items, d, L, n_blocks):
    def shape(k):
        if k in ITEM_KEYS:
            return (n_items + 1, d)
        if k.endswith("pe.weight"):
            return (L, d)
        if k.endswith("in_proj_weight"):
            return (3 * d, d)
        if k.endswith("in_proj_bias"):
            return (3 * d,)
        if k.endswith("out_proj.weight"):
            return (d, d)
        if k.endswith(("conv1.weight", "conv2.weight")):
            return (d, d, 1)
        if k.endswith(("WG.weight", "W1.weight")):
            return (2 * d, d)
        if k.endswith(("WG.bias", "W1.bias")):
            return (2 * d,)
        if k.endswith("W2.weight"):
            return (d, 2 * d)
        return (d,)
    return shape


def to_dtype(sd, dtype):
    out = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in sd.items()}
    for k in ITEM_KEYS[1:]:
        out[k] = out[ITEM_KEYS[0]]
    return out
