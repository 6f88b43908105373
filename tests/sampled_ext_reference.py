"""float64 restatement of the sampled heads' LogInCESampled and CESampledWeighted kinds (rp_sampled_head_* kinds 4 and 5 in
csrc/rp_sampled_head.cu) over the compacted rows the kernels see; inputs and layouts as in tests/sampled_reference.py,
plus ``row_weight`` [capacity] (fp32, compacted order) for kind 5.

Both mask the negatives as CESampled does (sampled_reference.adjust_logits with kind 0) and take the softmax over
[z_p | z].  With p_t the positive's share:
  kind 4 (LogInCESampled)     loss = mean_t -clamp(log(p_t + eps), -c, c)       (replay/nn/loss/login_ce.py:240-375)
  kind 5 (CESampledWeighted)  loss = mean_t w_t (lse_t - z_p)                     (replay/nn/loss/ce.py:252-330)
Gradients come from autograd.  Pinned against oracle/sampled_ext.py by tests/test_sampled_ext_cpu.py.
"""
import torch

import sampled_reference as sr

LOGIN_CE_SAMPLED, CE_SAMPLED_WEIGHTED = 4, 5


def row_losses(z_pos, z_neg, kind, w=None, log_eps=1e-6, clamp=100.0):
    """Per-row loss (before the mean) from the positive logit [rows] and the masked negative logits [rows, N]."""
    lse = torch.logsumexp(torch.cat([z_pos[:, None], z_neg], 1), 1)
    if kind == LOGIN_CE_SAMPLED:
        return -torch.clamp(torch.log(torch.exp(z_pos - lse) + log_eps), -clamp, clamp)
    return (lse - z_pos) * w


def clamp_edge_grads(z_pos, z_neg, log_eps, clamp):
    """|d(row loss)/dz| of the LogInCE rows whose log lies within sampled_reference.CLAMP_EDGE of +-clamp ([rows], [rows,
    N]; 0 elsewhere): whether such a row is clamped turns on the last bits of its fp32 logits (the rule of the BCE kinds)."""
    lse = torch.logsumexp(torch.cat([z_pos[:, None], z_neg], 1), 1)
    p, q = torch.exp(z_pos - lse), torch.exp(z_neg - lse[:, None])
    lg = torch.log(p + log_eps)
    f = ((lg.abs() - clamp).abs() < sr.CLAMP_EDGE).to(lg.dtype) * p / (p + log_eps)
    return f * (1 - p), f[:, None] * q


def reference(hc, table, labels, valid_idx, negatives, n_valid, kind, neg_mode, L=1, ignore_index=-100, row_weight=None,
              log_eps=1e-6, clamp=100.0, chunk=64):
    """float64 loss, d_hc, d_table and the error magnitudes of sampled_reference.reference for kinds 4 and 5."""
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
        neg = sr.negative_ids(negatives, valid_idx, neg_mode, L, rows).long()
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
        z_adj, live = sr.adjust_logits(z_neg, neg, y, sr.CE_SAMPLED, ignore_index)
        w = row_weight[rows].double() if kind == CE_SAMPLED_WEIGHTED else None
        part = row_losses(z_pos, z_adj, kind, w, log_eps, clamp).sum() * inv
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
        if kind == LOGIN_CE_SAMPLED:
            with torch.no_grad():
                w_pos, w_neg = clamp_edge_grads(z_pos, z_adj, log_eps, clamp)
            spread(w_pos * inv, w_neg * inv, edge_hc, edge_table)
    return dict(loss=loss, d_hc=d_hc, d_table=d_table, mag_hc=mag_hc, mag_table=mag_table, edge_hc=edge_hc,
                edge_table=edge_table, referenced=referenced)
