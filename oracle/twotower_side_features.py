"""Plain-torch restatement of RePlay's TwoTower with side features (TEST INFRASTRUCTURE - see oracle/__init__.py): the
``from_params`` towers over one ``SequenceEmbedding`` both towers share, summed by ``SumAggregator``.

* Query tower: oracle/side_features.py's input stage (item row plus every side term, sqrt(d) scale, positions) and the
  new-path SASRec body, then the output LayerNorm.
* Item tower: for each catalog item (or candidate) the item row plus the term of every feature the item features reader
  holds, taken from the reader's column at that item; no scale, position or dropout; then oracle/twotower.py's
  SwiGLUEncoder.

Parameters are the reference's ``state_dict`` under its main keys (``body.embedder...`` for the shared tables, as
``named_parameters`` lists them).  A feature spec is oracle/side_features.py's dict; ``reader`` maps feature name to the
reader's column over the catalog (the item id's column is arange and is not used).

Reference files restated (under replay/ of the reference project): nn/sequential/twotower/model.py (QueryTower, ItemTower,
TwoTower.get_logits / forward_*), nn/embedding.py, nn/agg.py:44-53, nn/ffn.py:60-135.
"""
from __future__ import annotations

import torch

from . import sampled as osm
from . import sampled_ext as osx
from . import sasrec as osr
from . import side_features as osf
from . import twotower as ott

ITEM_KEY = ott.ITEM_KEYS[0]


def golden_specs(z):
    """the feature specs of a tests/golden/twotower_side_*.npz file"""
    return [dict(name=str(n), kind=str(k), cardinality=int(c), padding_value=int(p), width=int(w))
            for n, k, c, p, w in zip(z["f_name"], z["f_kind"], z["f_cardinality"], z["f_padding_value"], z["f_width"])]


def _params(sd, specs):
    P = ott.query_params({**sd, **{k: sd[ITEM_KEY] for k in ott.ITEM_KEYS[1:]}})
    P["side"] = osf.side_from_state_dict(sd, specs)
    return P


def item_input(sd, specs, reader, method="sum", candidates=None):
    """X0 [n, d]: the item rows plus the reader features' terms, at the catalog or the candidates"""
    n = sd[ITEM_KEY].shape[0] - 1
    ids = torch.arange(n) if candidates is None else candidates
    fs = [f for f in specs if f["name"] in reader]
    P = {"item_emb": sd[ITEM_KEY], "side": osf.side_from_state_dict(sd, fs)}
    return osf.embed_sum(P, fs, ids, {f["name"]: reader[f["name"]][ids] for f in fs}, method)


def item_tower(sd, specs, reader, method="sum", candidates=None):
    return ott.swiglu_encoder(sd, item_input(sd, specs, reader, method, candidates))


def query_hidden(sd, specs, ids, feats, pad_mask, n_heads, method="sum"):
    return osf.body(_params(sd, specs), specs, ids, feats, pad_mask, n_heads, method)


def train_loss(sd, specs, reader, ids, feats, pad_mask, labels, target_mask, n_heads, method="sum", kind="ce",
               negatives=None, weights=None, ignore_index=-100, log_eps=1e-6, clamp=100.0):
    """TwoTower.forward_train's loss.  The item tower is row-wise, so the sampled losses' item_tower(candidates) rows equal
    the catalog tower's rows at those ids."""
    h = query_hidden(sd, specs, ids, feats, pad_mask, n_heads, method)
    Y = item_tower(sd, specs, reader, method)
    if kind == "ce":
        return osr.ce_loss(h, Y, labels, target_mask)
    if kind == "bce":
        return ott.bce_full(h, Y, labels, target_mask)
    if kind == "ce_sampled":
        return osm.ce_sampled(h, Y, labels, negatives, target_mask, ignore_index=ignore_index)
    if kind == "login_ce_sampled":
        return osx.login_ce_sampled(h, Y, labels, negatives, target_mask, log_eps, clamp, ignore_index=ignore_index)
    if kind == "ce_sampled_weighted":
        return osx.ce_sampled_weighted(h, Y, labels, negatives, target_mask, weights, ignore_index=ignore_index)
    raise ValueError(kind)


def loss_and_grads(sd, specs, *args, **kwargs):
    """Loss and d(loss)/d(every parameter of ``sd``); the padding rows of the item table and the categorical tables are
    frozen (torch.nn.Embedding / EmbeddingBag padding_idx)."""
    leaves = {k: v.detach().clone().requires_grad_(v.is_floating_point()) for k, v in sd.items()}
    loss = train_loss(leaves, specs, *args, **kwargs)
    loss.backward()
    G = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in leaves.items() if v.is_floating_point()}
    G[ITEM_KEY][-1].zero_()
    for f in specs:
        if f["kind"] in ("cat", "bag"):
            G[f"{osf.PREFIX}{f['name']}.emb.weight"][f["padding_value"]].zero_()
    return loss.detach(), G


def eval_logits(sd, specs, reader, ids, feats, pad_mask, n_heads, method="sum", candidates=None):
    """TwoTower.forward_inference's logits: the last position's query state against the item tower"""
    h = query_hidden(sd, specs, ids, feats, pad_mask, n_heads, method)[:, -1]
    return h @ item_tower(sd, specs, reader, method, candidates).T
