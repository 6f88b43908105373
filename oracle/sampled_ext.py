"""TEST INFRASTRUCTURE - CPU restatement of the reference's LogInCESampled and CESampledWeighted (plain torch autograd), on
the logits and negative masking of oracle/sampled.py:
  * LogInCESampled.forward (replay/nn/loss/login_ce.py:240-375): -clamp(log(p + eps), -c, c) of the positive's softmax share
    p over [positive | masked negatives], mean over the valid targets;
  * CESampledWeighted.forward (replay/nn/loss/ce.py:252-330): CESampled's row losses times the sample weights of the valid
    targets, mean over the valid targets (not divided by the weights' sum).
Single positive per position.  Pinned against the real reference classes by oracle/gen_sampled_ext_golden.py ->
tests/golden/sampled_ext_losses.npz.
"""
from __future__ import annotations

import torch

from .sampled import mask_negative_logits, sampled_logits


def login_ce_sampled(hidden, table, positive_labels, negative_labels, target_mask, log_eps=1e-6, clamp=100.0,
                     ignore_index=-100):
    z_pos, z_neg, pos, neg = sampled_logits(hidden, table, positive_labels, negative_labels, target_mask)
    z_neg = mask_negative_logits(z_neg, neg, pos, ignore_index)
    p = torch.softmax(torch.cat((z_pos, z_neg), dim=-1), dim=-1)[:, 0]
    return (-torch.clamp(torch.log(p + log_eps), -clamp, clamp)).mean()


def ce_sampled_weighted(hidden, table, positive_labels, negative_labels, target_mask, weights, ignore_index=-100):
    """``weights`` [B, L, 1] or [B, L]."""
    z_pos, z_neg, pos, neg = sampled_logits(hidden, table, positive_labels, negative_labels, target_mask)
    z_neg = mask_negative_logits(z_neg, neg, pos, ignore_index)
    logits = torch.cat((z_pos, z_neg), dim=-1)
    ce = torch.nn.functional.cross_entropy(logits, torch.zeros(len(logits), dtype=torch.long), reduction="none")
    w = weights[..., 0] if weights.dim() == 3 else weights
    return (ce * w[target_mask].to(ce.dtype)).mean()


LOSSES = {"login_ce": login_ce_sampled, "ce_weighted": ce_sampled_weighted}


def loss_and_grads(P, ids, pad_mask, labels, target_mask, negatives, n_heads, kind, **kw):
    """Body of oracle.sasrec (new path) + one of the losses above: (loss, gradients of every parameter), as
    oracle.sampled.loss_and_grads returns them."""
    from .sasrec import sasrec_body

    Pg = {}
    for k, v in P.items():
        Pg[k] = [{kk: vv.detach().clone().requires_grad_(True) for kk, vv in b.items()} for b in v] if k == "blocks" \
            else v.detach().clone().requires_grad_(True)
    h = sasrec_body(Pg, ids, pad_mask, n_heads, "new")
    loss = LOSSES[kind](h, Pg["item_emb"], labels, negatives, target_mask, **kw)
    loss.backward()
    G = {}
    for k, v in Pg.items():
        if k == "blocks":
            G[k] = [{kk: (vv.grad if vv.grad is not None else torch.zeros_like(vv)) for kk, vv in b.items()} for b in v]
        else:
            G[k] = v.grad if v.grad is not None else torch.zeros_like(v)
    G["item_emb"][-1].zero_()
    return loss.detach(), G
