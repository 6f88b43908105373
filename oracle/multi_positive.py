"""TEST INFRASTRUCTURE - CPU restatement of the reference's losses on multi-positive targets (labels and target mask
[B, L, P]), plain torch autograd:
  * SampledLossBase.get_sampled_logits + mask_negative_logits (replay/nn/loss/base.py:49-196): one row per (position, slot)
    pair with the mask set - the position's hidden state, the slot's positive, the position's negatives; a negative is
    masked where it equals ANY of the position's P slot values (masked-out slots included) or the ignore index;
  * CESampled (ce.py:199-249), BCESampled (bce.py:154-218), CESampledWeighted (ce.py:252-317): means over the pairs;
  * BCE (bce.py:51-95): one row per live position (any slot set), target 1 at every slot id (scatter_), sum over the
    catalog divided by the live positions.
Pinned against the real reference classes by oracle/gen_multi_positive_golden.py -> tests/golden/multi_positive_losses.npz.
"""
from __future__ import annotations

import torch


def pair_logits(hidden, table, labels, negatives, target_mask, ignore_index=-100):
    """hidden [B, L, d], labels / target_mask [B, L, P], negatives [N] | [B, N] | [B, L, N] -> (z_pos [M], masked z_neg
    [M, N]) over the M pairs."""
    B, L, P = labels.shape
    neg = negatives
    if neg.dim() == 2:
        neg = neg.unsqueeze(1).expand(B, L, -1)
    h = hidden.unsqueeze(2).expand(B, L, P, hidden.shape[-1])[target_mask]
    z_pos = (h * table[labels[target_mask]]).sum(-1)
    if neg.dim() == 1:
        z_neg = h @ table[neg].T
        negm = neg.unsqueeze(0).expand(len(h), -1)
    else:
        negm = neg.unsqueeze(2).expand(B, L, P, neg.shape[-1])[target_mask]
        z_neg = torch.einsum("md,mnd->mn", h, table[negm])
    row = labels.unsqueeze(2).expand(B, L, P, P)[target_mask]               # every pair sees its position's whole label row
    hit = (row.unsqueeze(-1) == negm.unsqueeze(-2)).any(-2)
    if ignore_index >= 0:
        hit = hit | (negm == ignore_index)
    return z_pos, z_neg.masked_fill(hit, -1e9)


def ce_sampled(hidden, table, labels, negatives, target_mask, ignore_index=-100, weights=None):
    z_pos, z_neg = pair_logits(hidden, table, labels, negatives, target_mask, ignore_index)
    logits = torch.cat((z_pos.unsqueeze(-1), z_neg), dim=-1)
    ce = torch.nn.functional.cross_entropy(logits, torch.zeros(len(logits), dtype=torch.long, device=logits.device),
                                           reduction="none")
    if weights is not None:
        ce = ce * weights[target_mask].to(ce.dtype)
    return ce.mean()


def bce_sampled(hidden, table, labels, negatives, target_mask, log_eps=1e-6, clamp=100.0, ignore_index=-100):
    z_pos, z_neg = pair_logits(hidden, table, labels, negatives, target_mask, ignore_index)
    pl = torch.clamp(torch.log(torch.sigmoid(z_pos) + log_eps), -clamp, clamp).sum()
    nl = torch.clamp(torch.log((1 - torch.sigmoid(z_neg)) + log_eps), -clamp, clamp).sum()
    return -(pl + nl) / len(z_pos)


def bce_full(hidden, table, labels, target_mask):
    """Full-catalog BCE; slot ids outside [0, n_items) are skipped (the reference's scatter_ fails on them)."""
    n_items = table.shape[0]
    live = target_mask.any(-1)
    logits = hidden[live] @ table.T
    lab = labels[live]
    tgt = torch.zeros_like(logits)
    ok = (lab >= 0) & (lab < n_items)
    rows = torch.arange(len(lab), device=lab.device).unsqueeze(-1).expand_as(lab)
    tgt[rows[ok], lab[ok]] = 1.0
    return torch.nn.functional.binary_cross_entropy_with_logits(logits, tgt, reduction="sum") / len(logits)


LOSSES = {"bce": bce_full, "ce_sampled": ce_sampled, "bce_sampled": bce_sampled, "ce_sampled_weighted": ce_sampled}


def loss_and_grads(P, ids, pad_mask, labels, target_mask, negatives, n_heads, kind, **kw):
    """Body of oracle.sasrec (new path) + one of the losses above over the catalog rows [0, n_items): (loss, gradients)."""
    from .sasrec import sasrec_body

    Pg = {}
    for k, v in P.items():
        Pg[k] = [{kk: vv.detach().clone().requires_grad_(True) for kk, vv in b.items()} for b in v] if k == "blocks" \
            else v.detach().clone().requires_grad_(True)
    h = sasrec_body(Pg, ids, pad_mask, n_heads, "new")
    n_items = Pg["item_emb"].shape[0] - 1
    table = Pg["item_emb"][:n_items]
    if kind == "bce":
        loss = bce_full(h, table, labels, target_mask)
    else:
        loss = LOSSES[kind](h, table, labels, negatives, target_mask, **kw)
    loss.backward()
    G = {}
    for k, v in Pg.items():
        if k == "blocks":
            G[k] = [{kk: (vv.grad if vv.grad is not None else torch.zeros_like(vv)) for kk, vv in b.items()} for b in v]
        else:
            G[k] = v.grad if v.grad is not None else torch.zeros_like(v)
    G["item_emb"][-1].zero_()   # the padding row is frozen (padding_idx)
    return loss.detach(), G
