"""float64 restatement of the sampled training heads (rp_sampled_head_* in csrc/rp_sampled_head.cu) over the compacted
rows the kernels see: hc [capacity, d] (rows < n_valid are the valid targets), labels [capacity], valid_idx [capacity]
(flat b * L + l position of each compacted row) and negatives in one of three layouts - neg_mode 0 = [N] shared, 1 =
[B * L, N] per position, 2 = [B, N] per sequence (row valid_idx[t] // L).

Per row t with positive logit z_p = h_t . E[y_t] and negative logits z_j = h_t . E[neg(t, j)]:
  kind 0 (CESampled)      z_j = -1e9 where neg == y_t or (ignore_index >= 0 and neg == ignore_index); CE over [z_p | z]
  kind 1 (BCESampled)     same masking; -(clamp(log(sigmoid(z_p) + eps)) + sum_j clamp(log(1 - sigmoid(z_j) + eps)))
  kind 2 (legacy CE)      z_j + log(V - 1) - 1e6 [neg == y_t] - log(min(N, V) - #{j: neg == y_t}); CE, no masking
  kind 3 (legacy BCE)     the BCE above without masking
and the loss is the mean over the n_valid rows (replay/nn/loss/ce.py:199-249, bce.py:154-218,
replay/models/nn/sequential/sasrec/lightning.py:310-376; oracle/sampled.py restates them over [B, L, d] hidden states).
Gradients come from autograd, in chunks of rows so that per-position negatives never gather more than
chunk x N x d table entries at once.  Pinned against oracle/sampled.py and the reference's golden values by
tests/test_sampled_reference_cpu.py.
"""
import math

import torch

CE_SAMPLED, BCE_SAMPLED, LEGACY_CE, LEGACY_BCE = 0, 1, 2, 3
CLAMP_EDGE = 1e-3    # BCE terms whose log lies this close to +-clamp may be clamped on one side of fp32 rounding only


def negative_ids(negatives, valid_idx, neg_mode, L, rows):
    """int64 [len(rows), N]: the negatives of compacted rows ``rows`` (a slice)."""
    if neg_mode == 0:
        neg = negatives.reshape(-1)
        return neg.unsqueeze(0).expand(rows.stop - rows.start, -1)
    N = negatives.shape[-1]
    r = valid_idx[rows].long()
    if neg_mode == 2:
        r = r // L
    return negatives.reshape(-1, N)[r]


def adjust_logits(z_neg, neg, y, kind, ignore_index=-100, vocab_size=None):
    """Masked / corrected negative logits and the bool [rows, N] of entries that still carry a gradient."""
    if kind in (CE_SAMPLED, BCE_SAMPLED):
        drop = neg == y[:, None]
        if ignore_index >= 0:
            drop = drop | (neg == ignore_index)
        return z_neg.masked_fill(drop, -1e9), ~drop
    if kind == LEGACY_CE:
        reject = neg == y[:, None]
        n_neg = min(neg.shape[1], vocab_size)
        z = z_neg + math.log(vocab_size - 1) - 1e6 * reject.to(z_neg.dtype)
        z = z - torch.log((n_neg - reject.sum(-1, keepdim=True)).to(z_neg.dtype))
        return z, ~reject
    return z_neg, torch.ones_like(neg, dtype=torch.bool)


def row_losses(z_pos, z_neg, kind, log_eps=1e-6, clamp=100.0):
    """Per-row loss (before the mean) from the positive logit [rows] and the adjusted negative logits [rows, N]."""
    if kind in (CE_SAMPLED, LEGACY_CE):
        return torch.logsumexp(torch.cat([z_pos[:, None], z_neg], 1), 1) - z_pos
    pos = torch.clamp(torch.log(torch.sigmoid(z_pos) + log_eps), -clamp, clamp)
    neg = torch.clamp(torch.log((1 - torch.sigmoid(z_neg)) + log_eps), -clamp, clamp).sum(-1)
    return -(pos + neg)


def clamp_edge_grads(z_pos, z_neg, log_eps, clamp):
    """|d(BCE term)/dz| of the terms whose log lies within CLAMP_EDGE of +-clamp ([rows], [rows, N]; 0 elsewhere).  Whether
    such a term is clamped (gradient 0) turns on the last bits of its fp32 logit, so its gradient is an allowed error."""
    def edge(lg):
        return ((lg.abs() - clamp).abs() < CLAMP_EDGE).to(lg.dtype)
    sp, sn = torch.sigmoid(z_pos), torch.sigmoid(z_neg)
    g_pos = edge(torch.log(sp + log_eps)) * sp * (1 - sp) / (sp + log_eps)
    g_neg = edge(torch.log((1 - sn) + log_eps)) * sn * (1 - sn) / ((1 - sn) + log_eps)
    return g_pos, g_neg


def reference(hc, table, labels, valid_idx, negatives, n_valid, kind, neg_mode, L=1, ignore_index=-100, vocab_size=None,
              log_eps=1e-6, clamp=100.0, chunk=64):
    """float64 loss, d_hc [n_valid, d] and d_table [rows of table, d] of the sampled head on the device of the inputs.

    Also returns the magnitudes the kernels' rounding scales with - mag_hc = sum_j |dz_j| |E_j| per element of d_hc,
    mag_table = sum_t |dz_tj| |h_t| per element of d_table, with dz the gradient of the loss with respect to the raw
    logits - and ``referenced``: bool [rows of table], the rows that a positive or a negative with a live gradient
    (not masked, not rejected) points at.  Every other row of d_table must be left exactly as it was.  For the BCE kinds
    edge_hc / edge_table spread the gradients of clamp_edge_grads the same way: an error the clamp's edge allows."""
    dev = hc.device
    E = table.double()
    R, d = E.shape
    M = int(n_valid)
    inv = 1.0 / max(M, 1)
    labels = labels.long()
    loss = torch.zeros((), dtype=torch.float64, device=dev)
    d_hc = torch.zeros(M, d, dtype=torch.float64, device=dev)
    mag_hc = torch.zeros_like(d_hc)
    d_table = torch.zeros(R, d, dtype=torch.float64, device=dev)
    mag_table = torch.zeros_like(d_table)
    edge_hc, edge_table = torch.zeros_like(d_hc), torch.zeros_like(d_table)
    referenced = torch.zeros(R, dtype=torch.bool, device=dev)
    shared = negatives.reshape(-1).long() if neg_mode == 0 else None
    for s in range(0, M, chunk):
        rows = slice(s, min(M, s + chunk))
        h = hc[rows].double().requires_grad_(True)
        y = labels[rows]
        neg = negative_ids(negatives, valid_idx, neg_mode, L, rows).long()
        e_pos = E[y].requires_grad_(True)
        z_pos = (h * e_pos).sum(-1)
        if neg_mode == 0:
            e_neg = E[shared].requires_grad_(True)
            z_neg = h @ e_neg.T
        else:
            e_neg = E[neg].requires_grad_(True)
            z_neg = torch.einsum("cd,cnd->cn", h, e_neg)
        z_pos.retain_grad()
        z_neg.retain_grad()
        z_adj, live = adjust_logits(z_neg, neg, y, kind, ignore_index, vocab_size)
        part = row_losses(z_pos, z_adj, kind, log_eps, clamp).sum() * inv
        part.backward()
        loss += part.detach()
        d_hc[rows] = h.grad
        referenced[y] = True
        referenced[neg[live]] = True
        d_table.index_add_(0, y, e_pos.grad)
        if neg_mode == 0:
            d_table.index_add_(0, shared, e_neg.grad)
        else:
            d_table.index_add_(0, neg.reshape(-1), e_neg.grad.reshape(-1, d))
        h_abs, ep_abs, en_abs = h.detach().abs(), e_pos.detach().abs(), e_neg.detach().abs()

        def spread(w_pos, w_neg, out_hc, out_table):
            """out_hc[rows] = w_pos |E_pos| + sum_j w_neg |E_neg|, out_table[item] += w |h| for per-logit weights w."""
            out_table.index_add_(0, y, w_pos[:, None] * h_abs)
            if neg_mode == 0:
                out_hc[rows] = w_pos[:, None] * ep_abs + w_neg @ en_abs
                out_table.index_add_(0, shared, w_neg.T @ h_abs)
            else:
                out_hc[rows] = w_pos[:, None] * ep_abs + torch.einsum("cn,cnd->cd", w_neg, en_abs)
                out_table.index_add_(0, neg.reshape(-1), (w_neg[:, :, None] * h_abs[:, None, :]).reshape(-1, d))

        spread(z_pos.grad.abs(), z_neg.grad.abs(), mag_hc, mag_table)
        if kind in (BCE_SAMPLED, LEGACY_BCE):
            with torch.no_grad():
                w_pos, w_neg = clamp_edge_grads(z_pos, z_adj, log_eps, clamp)
            spread(w_pos * inv, w_neg * inv, edge_hc, edge_table)
    return dict(loss=loss, d_hc=d_hc, d_table=d_table, mag_hc=mag_hc, mag_table=mag_table, edge_hc=edge_hc,
                edge_table=edge_table, referenced=referenced)
