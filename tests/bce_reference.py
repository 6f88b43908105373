"""float64 restatement of the full-catalog BCE head (rp_bce_head_* in csrc/rp_ce_head.cu) and the error bounds its GPU test
uses.  loss = sum_t [sum_i softplus(x_ti) - x_t,y_t] / M, dx = (sigmoid(x) - onehot) / M over the M valid rows, x = h . W^T + b
(replay/nn/loss/bce.py:10-95 ; bert4rec/lightning.py:273-305).

Error bounds.  The tensor cores take the gradient's sigmoid as a bf16 operand, so every G_ti carries a relative rounding
error of at most 2^-9; the fp32 accumulation over up to 10^5 terms and the approximate ex2 / rcp add well under that again.
A gradient element sum_i G_ti E_ik / M is therefore within 2^-8 sum_i sigma_ti |E_ik| / M of the exact value, plus the
final bf16 rounding of d_hc (2^-8 of its magnitude, half an ulp with margin).  d_bias sums fp32 sigmoids (no bf16 operand)
and takes the same bound.  The loss sums fp32 softplus terms (log1p through lg2 of a product of 32 factors): 2^-16 of
sum |softplus| / M, plus 2^-16 of |x_y| / M for the target logit's fp32 dot."""
import torch

U_G = 2.0 ** -8
U_OUT = 2.0 ** -8
U_LOSS = 2.0 ** -16


def reference(h, W, b, labels, n_valid):
    """h [cap, d], W [I, d], b [I] or None, labels [cap] (any device): fp64 loss, d_h [n_valid, d], d_W [I, d], d_b [I]
    and the bounds of each (same shapes)."""
    h = h[:n_valid].double()
    W = W.double()
    y = labels[:n_valid].long()
    x = h @ W.T
    if b is not None:
        x = x + b.double()[None, :]
    M = max(n_valid, 1)
    sig = torch.sigmoid(x)
    sp = torch.nn.functional.softplus(x)
    xy = x.gather(1, y[:, None])[:, 0] if n_valid else x.new_zeros(0)
    loss = (sp.sum() - xy.sum()) / M if n_valid else x.new_zeros(())
    g = sig.clone()
    if n_valid:
        g[torch.arange(n_valid, device=g.device), y] -= 1.0
    g /= M
    d_h, d_W, d_b = g @ W, g.T @ h, g.sum(0)
    bound_h = U_G * (sig @ W.abs() + W[y].abs()) / M + U_OUT * d_h.abs() + 1e-7
    bound_W = U_G * (sig.T @ h.abs() + torch.zeros_like(W).index_add_(0, y, h.abs())) / M + 1e-7
    bound_b = U_G * (sig.sum(0) + torch.bincount(y, minlength=W.shape[0]).double()) / M + 1e-7
    bound_loss = U_LOSS * (sp.sum() + xy.abs().sum()) / M + 1e-7
    return dict(loss=loss, d_h=d_h, d_W=d_W, d_b=d_b, bound_loss=bound_loss, bound_h=bound_h, bound_W=bound_W,
                bound_b=bound_b)


def worst(got, ref, bound):
    """largest |got - ref| / bound (1.0 = at the bound)"""
    if ref.numel() == 0:
        return 0.0
    return float(((got.double() - ref).abs() / bound).max())
