"""Plain-torch CPU restatement of RePlay's BERT4Rec with its two body options (TEST INFRASTRUCTURE - see oracle/__init__.py):
``num_passes_over_block`` (bert4rec/model.py:139-141: every block applied that many times in a row with its own weights)
and ``enable_positional_embedding=False`` (model.py:236-237, 289-291: no position table, no positional term).

Built on oracle/bert4rec.py: a model without the position table is evaluated with an all-zero one, which adds exactly
nothing.  The canonical parameter dict is oracle/bert4rec.py's, with ``pos_emb`` absent when the embedding is off.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import bert4rec as ob

POS_KEY = "item_embedder.position.pe.weight"


def params_from_state_dict(sd, item_feature="item_id"):
    """oracle.bert4rec.params_from_state_dict for a state dict with or without the position table."""
    if POS_KEY in sd:
        return ob.params_from_state_dict(sd, item_feature)
    item = sd[f"item_embedder.cat_embeddings.{item_feature}.weight"]
    P = ob.params_from_state_dict({**sd, POS_KEY: item.new_zeros(1, item.shape[1])}, item_feature)
    del P["pos_emb"]
    return P


def seeded_state_dict(keys, shapes, seed):
    """Weights drawn from ``seed`` in the given key order, so a golden file can store the seed instead of the tensors:
    2-D tensors xavier-normal (the reference's init, model.py:167-170), LayerNorm weights 1 + 0.05 N(0, 1), every other
    1-D tensor 0.05 N(0, 1) (perturbed, so the goldens exercise the biases).  The tied head's ``_head._item_embedder.*``
    keys alias the embedder's tensors (model.py:398-409) and repeat them."""
    g = torch.Generator().manual_seed(int(seed))
    sd = {}
    for k, shp in zip(keys, shapes):
        if k.startswith("_head._item_embedder."):
            sd[k] = sd["item_embedder." + k[len("_head._item_embedder."):]]
            continue
        shp = tuple(int(n) for n in shp)
        v = torch.randn(shp, generator=g, dtype=torch.float32)
        if len(shp) == 2:
            v = v * math.sqrt(2.0 / (shp[0] + shp[1]))
        else:
            v = v * 0.05 + (1.0 if k.endswith("norm.weight") else 0.0)
        sd[k] = v
    return sd


def state_dict_checksum(sd, keys):
    """float64 [n_keys, 2]: sum and sum of squares of every tensor (guards a seeded state dict against a changed generator)"""
    return np.array([[float(sd[k].double().sum()), float((sd[k].double() ** 2).sum())] for k in keys])


def golden_state_dict(z):
    """The reference weights of a golden file written by gen_bert4rec_passes_golden.py: regenerated from ``sd_seed`` in the
    order of ``sd_keys`` (shapes ``sd_shapes``, "AxB" strings) and checked against the stored checksums."""
    keys = [str(k) for k in z["sd_keys"]]
    shapes = [tuple(int(n) for n in str(s).split("x")) for s in z["sd_shapes"]]
    sd = seeded_state_dict(keys, shapes, int(z["sd_seed"]))
    np.testing.assert_allclose(state_dict_checksum(sd, keys), z["sd_checksum"], rtol=1e-9, atol=1e-9)
    return sd


def _with_pos(P, L):
    if "pos_emb" in P:
        return P
    return {**P, "pos_emb": P["item_emb"].new_zeros(L, P["item_emb"].shape[1])}


def body(P, ids, pad_mask, token_mask, n_heads, num_passes=1):
    """Hidden states [B, L, d], dropout off."""
    return ob.bert4rec_body(_with_pos(P, ids.shape[1]), ids, pad_mask, token_mask, n_heads, num_passes)


def train_loss(P, ids, pad_mask, token_mask, labels, n_heads, num_passes=1):
    """CE over positions that are real and masked (lightning.py:344-351)."""
    h = body(P, ids, pad_mask, token_mask, n_heads, num_passes)
    w, b = ob.head_weights(P)
    sel = pad_mask & ~token_mask
    logits = h[sel] @ w.T + b
    y = labels[sel]
    return (torch.logsumexp(logits, -1) - logits.gather(1, y[:, None])[:, 0]).mean()


def logits(P, h, item_ids=None):
    """The biased head (BaseHead.forward, model.py:363-382) over hidden states h [..., d]."""
    w, b = ob.head_weights(P)
    if item_ids is not None:
        w, b = w[item_ids], b[item_ids]
    return h @ w.T + b
