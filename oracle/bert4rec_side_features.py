"""Plain-torch CPU restatement of RePlay's legacy BERT4Rec with side features (TEST INFRASTRUCTURE - see oracle/__init__.py).

BertEmbedding.forward (bert4rec/model.py:239-296) with sum aggregation: every categorical feature's ``nn.Embedding`` row
(no padding row: every id in [0, cardinality) is a trainable row) and every numerical feature's values, summed, then
``where(token_mask, sum, mask_embedding) + position``.  The body, the heads and the seeded golden weights are
oracle/bert4rec_passes.py's: the summed inputs enter it as a per-token "item table", so the body is not restated again.

Side features are given as ``specs``: a list of (name, kind) with kind "cat" or "ident", in the order of the reference's
sum (categoricals, then numericals, each in schema order).  The canonical parameter dict is oracle/bert4rec_passes.py's
plus ``feat`` = {name: table [cardinality, d]} for the categoricals.
"""
from __future__ import annotations

import torch

from . import bert4rec as ob
from . import bert4rec_passes as op


def params_from_state_dict(sd, specs, item_feature="item_id"):
    P = op.params_from_state_dict(sd, item_feature)
    P["feat"] = {n: sd[f"item_embedder.cat_embeddings.{n}.weight"].detach().clone() for n, k in specs if k == "cat"}
    return P


def summed_input(P, ids, feats, specs):
    """s [B, L, d] = item_emb[ids] + sum of the categorical rows + sum of the numerical values (before <MASK> and position)"""
    s = P["item_emb"][ids]
    for n, k in specs:
        s = s + (P["feat"][n][feats[n]] if k == "cat" else feats[n].to(s.dtype))
    return s


def body(P, ids, pad_mask, token_mask, feats, specs, n_heads, num_passes=1):
    """Hidden states [B, L, d], dropout off.  Token (b, t) reads row b * L + t of a table holding the summed inputs."""
    B, L = ids.shape
    s = summed_input(P, ids, feats, specs)
    Q = {k: v for k, v in P.items() if k != "feat"}
    Q["item_emb"] = s.reshape(B * L, -1)
    return op.body(Q, torch.arange(B * L).view(B, L), pad_mask, token_mask, n_heads, num_passes)


def logits(P, h, item_ids=None):
    return op.logits(P, h, item_ids)


def train_loss(P, ids, pad_mask, token_mask, labels, feats, specs, n_heads, num_passes=1, loss="ce"):
    """CE (lightning.py:332-351) or BCE (lightning.py:273-305, summed over items and averaged over rows) over the positions
    that are real and masked."""
    h = body(P, ids, pad_mask, token_mask, feats, specs, n_heads, num_passes)
    w, b = ob.head_weights(P)
    sel = pad_mask & ~token_mask
    lg = h[sel] @ w.T + b
    y = labels[sel]
    if loss == "ce":
        return (torch.logsumexp(lg, -1) - lg.gather(1, y[:, None])[:, 0]).mean()
    t = torch.zeros_like(lg).scatter_(1, y[:, None], 1.0)
    return torch.nn.functional.binary_cross_entropy_with_logits(lg, t, reduction="sum") / lg.shape[0]
