"""Plain-torch restatement of the legacy SASRec's scalable cross-entropy loss (replay/models/nn/loss/sce.py:43-124) with the
random draw - and optionally the row / item selections - as inputs, in any float dtype.  TEST INFRASTRUCTURE: the CPU
tests check it against the real reference (tests/golden/sce_losses.npz); the GPU tests check the CUDA head against it."""
from __future__ import annotations

import torch


def buckets_of(x, draw, mix_x: bool):
    """Bucket matrix [n_b, hd]: the draw scaled by hd^-1/4, or (mix_x) the scaled draw [T, n_b] mixing all rows of x."""
    scale = x.shape[1] ** -0.25
    b = draw.to(x.dtype) * scale
    return b.T @ x if mix_x else b


def select(x, w, padding_mask, buckets, bucket_size_x: int, bucket_size_y: int):
    """(top_x [n_b, bs_x], top_y [n_b, bs_y]): the rows / items with the largest bucket scores; pad rows score -inf."""
    sx = buckets @ x.T
    sx = sx.masked_fill(~padding_mask.view(1, -1), float("-inf"))
    return torch.topk(sx, bucket_size_x, dim=1).indices, torch.topk(buckets @ w.T, bucket_size_y, dim=1).indices


def row_losses(x, y, w, top_x, top_y):
    """CE of every (bucket, selected row): logits x_t . w[Y_b] with the label's own column at -inf, plus x_t . w[y_t]."""
    correct = (x * w[y]).sum(1)
    xb, yb = x[top_x], w[top_y]                                     # [n_b, bs_x, hd], [n_b, bs_y, hd]
    wrong = torch.einsum("bid,bjd->bij", xb, yb)
    wrong = wrong.masked_fill(y[top_x].unsqueeze(-1) == top_y.unsqueeze(1), float("-inf"))
    c = correct[top_x]
    return torch.logsumexp(torch.cat([wrong, c.unsqueeze(-1)], dim=-1), dim=-1) - c


def sce_loss(x, y, w, padding_mask, draw, bucket_size_x: int, bucket_size_y: int, mix_x: bool = False, top_x=None,
             top_y=None):
    """x [T, hd] final hidden state of every position (pad rows included), y [T] labels (all < |I|), w [|I|, hd] item table
    (no gradient flows into it), padding_mask [T] bool, draw [n_b, hd] (or [T, n_b] with mix_x) standard normals.
    Returns (loss, top_x, top_y): the mean over the rows with a non-zero per-row maximum over the buckets that selected them
    (NaN when no row is left)."""
    w = w.detach()
    with torch.no_grad():
        b = buckets_of(x.detach(), draw, mix_x)
        sel_x, sel_y = select(x.detach(), w, padding_mask, b, bucket_size_x, bucket_size_y)
    top_x = sel_x if top_x is None else top_x
    top_y = sel_y if top_y is None else top_y
    ce = row_losses(x, y, w, top_x, top_y)
    per_row = torch.zeros(x.shape[0], dtype=x.dtype, device=x.device)
    per_row = per_row.scatter_reduce(0, top_x.reshape(-1), ce.reshape(-1), reduce="amax", include_self=False)
    return per_row[(per_row != 0) & padding_mask].mean(), top_x, top_y


def loss_and_grads(P, ids, pad_mask, labels, n_heads, draw, bucket_size_x: int, bucket_size_y: int, mix_x: bool = False,
                   top_x=None, top_y=None, lnf_eps=None):
    """The legacy SASRec body (oracle/sasrec.py) + sce_loss, with autograd: (loss, grads like oracle.sasrec.loss_and_grads,
    top_x, top_y).  The table enters the loss detached (the reference scores get_all_embeddings()'s copy), so the item table
    gradient comes from the input embedding gather alone; the pad row's gradient is zeroed."""
    from . import sasrec as osr

    Pg = {k: ([{kk: vv.detach().clone().requires_grad_(True) for kk, vv in b.items()} for b in v] if k == "blocks"
              else v.detach().clone().requires_grad_(True)) for k, v in P.items()}
    h = osr.sasrec_body(Pg, ids, pad_mask, n_heads, "legacy", lnf_eps)
    n_items = P["item_emb"].shape[0] - 1
    loss, tx, ty = sce_loss(h.reshape(-1, h.shape[-1]), labels.reshape(-1), Pg["item_emb"][:n_items], pad_mask.reshape(-1),
                            draw, bucket_size_x, bucket_size_y, mix_x, top_x, top_y)
    if torch.isfinite(loss):
        loss.backward()
    G = {k: ([{kk: (vv.grad if vv.grad is not None else torch.zeros_like(vv)) for kk, vv in b.items()} for b in v]
             if k == "blocks" else (v.grad if v.grad is not None else torch.zeros_like(v))) for k, v in Pg.items()}
    G["item_emb"][-1].zero_()
    return loss.detach(), G, tx, ty
