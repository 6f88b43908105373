"""float64 restatement of the scalable cross-entropy head (rp_sce_head_fwd / rp_sce_head_bwd in csrc/rp_sce_head.cu) over
the kernel's own inputs and selections: hc bf16 [capacity, d] and table bf16 [n_items, d] in the padded feature layout,
labels [capacity], pad_mask [capacity], n_rows, the bf16 bucket matrix [n_b, d] the head drew and its selections top_x /
score_x [n_b, bs_x] and top_y [n_b, bs_y].

A row t is selectable - may carry loss - iff t < n_rows, pad_mask[t] and 0 <= labels[t] < n_items (what sce_prep_kernel
masks with a -inf row bias).  A slot (b, i) carries row t = top_x[b, i] iff score_x[b, i] is finite and t is selectable.
Per carrying slot: CE = logsumexp([x_t . W[Y_b \\ {y_t}], c_t]) - c_t with c_t = x_t . W[y_t] (oracle/sce.py row_losses);
per row the maximum over its slots; loss = mean of the maxima over the counted rows; d_hc from the winning slot(s) of each
counted row, an exact tie split evenly (torch's scatter_reduce(amax) backward).

Two rules make a comparison with the fp32 kernel well defined:
- counted rows.  The kernel's CE = max(lse - c, 0) in fp32 is exactly 0 when the true CE is below about one ulp of c, and
  such a row is not counted.  Here a row is surely counted iff its max CE > COUNT_MIN * max(1, |c|) and surely not iff it
  is < AMBIG_MIN; rows in between are ``ambiguous``: the count may include any number of them, and they are left out of
  the element-wise d_hc check (their gradient is of the size of their CE: tiny).
- near-tied winners.  A row whose slot CEs within NEAR_TIE (relative) of its maximum come from slots with different
  single-slot gradients (beyond TIE_GRAD_TOL of the row's gradient) has a gradient that depends on the slot fp32 picked:
  it is left out of the element-wise check and counted in ``near_tie``.  Exact ties (duplicated buckets) are bit-equal
  in both precisions and stay in the check with the even split.

Error bounds of the kernel against this reference:
- loss: each counted CE is lse - c in fp32 (cancellation) with the fast-math exp and log, whose error is absolute: about
  k * 2^-24 * (|lse| + |c| + 1) per row for a few ulps k; ``loss_unit`` = 2^-24 * mean over the counted rows of
  (|lse| + |c| + 1), and the ambiguous rows' CE over the count comes on top.
- d_hc: the softmax reaches the dX = G . Y_b GEMM as bf16, so per element SLACK * sum_j |G_j| |Y_j| (``mag_hc``) on top of
  the final bf16 rounding; SLACK = 2^-8 as for the sampled heads' shared negatives.
Pinned against oracle/sce.py and the reference's golden values by tests/test_sce_reference_cpu.py.
"""
import math

import torch

from oracle.sce import row_losses

COUNT_MIN = 2.0 ** -20   # a max CE above COUNT_MIN * max(1, |c|) is surely non-zero in fp32
AMBIG_MIN = 2.0 ** -30   # a max CE below this is surely 0 in fp32
NEAR_TIE = 1e-5          # slot CEs within this relative distance of the row maximum may win in fp32
TIE_GRAD_TOL = 1e-3      # near-tied slots whose gradients differ by more than this (relative to the row's) are ambiguous
SLACK = 2.0 ** -8


def selectable(labels, pad_mask, n_rows, n_items):
    """bool [capacity]: rows that may carry loss (sce_prep_kernel)."""
    cap = labels.shape[0]
    t = torch.arange(cap, device=labels.device)
    lab = labels.long()
    return (t < int(n_rows)) & pad_mask.bool() & (lab >= 0) & (lab < n_items)


def selection_scores(buckets, hc, table, sel):
    """fp64 (sx [n_b, cap] with unselectable rows at -inf, sy [n_b, n_items], ax, ay): the scores the two top-Ks rank and
    the matching sums of |products| sum_j |b_j| |h_j|, the scale of their fp32 accumulation error."""
    b = buckets.double()
    h, w = hc.double(), table.double()
    sx = (b @ h.T).masked_fill(~sel.view(1, -1), float("-inf"))
    return sx, b @ w.T, b.abs() @ h.abs().T, b.abs() @ w.abs().T


def kth_best(s, k):
    """[n_b]: the k-th best score of each bucket (-inf when fewer than k are finite)."""
    return s.topk(k, dim=1).values[:, -1]


def reference(hc, table, labels, pad_mask, n_rows, top_x, score_x, top_y, chunk=8):
    """float64 loss and d_hc [capacity, d] of the head with the given selections, on the device of the inputs.

    Returns a dict: loss (over the surely counted rows, divided by ``n_counted``), n_counted, n_ambiguous, ce_sum_ambiguous,
    loss_unit, d_hc, mag_hc, checked (bool [capacity]: rows of the element-wise check), near_tie (count), ce [n_b, bs_x]
    (-1 where a slot carries nothing), row_max [capacity] (-1 = not selected), winners [capacity] (number of exact
    winners), counted / ambiguous (bool [capacity]), c [capacity] (correct logits) and lse of the winning slot."""
    dev = hc.device
    cap, d = hc.shape
    n_items = table.shape[0]
    x, W = hc.double(), table.double()
    sel = selectable(labels, pad_mask, n_rows, n_items)
    lab = labels.long().clamp(0, n_items - 1)
    tx = top_x.long()
    live = torch.isfinite(score_x) & (tx >= 0) & (tx < cap)
    live &= sel[tx.clamp(0, cap - 1)]
    txc = tx.clamp(0, cap - 1)
    ty = top_y.long()
    nb, bsx = tx.shape
    # per-slot CE (row_losses over chunks of buckets)
    ce = torch.full((nb, bsx), -1.0, dtype=torch.float64, device=dev)
    for b0 in range(0, nb, chunk):
        b1 = min(nb, b0 + chunk)
        ce[b0:b1] = row_losses(x, lab, W, txc[b0:b1], ty[b0:b1])
    ce = ce.masked_fill(~live, -1.0)
    row_max = torch.full((cap,), -1.0, dtype=torch.float64, device=dev)
    row_max = row_max.scatter_reduce(0, txc[live], ce[live], reduce="amax", include_self=True)
    c = (x * W[lab]).sum(1)
    scale = c.abs().clamp_min(1.0)
    counted = row_max > COUNT_MIN * scale
    ambiguous = (row_max >= AMBIG_MIN) & ~counted
    n_counted = int(counted.sum())
    # candidate slots: within NEAR_TIE of their row's maximum, of a counted or ambiguous row
    rm_slot = row_max[txc]
    cand = live & (counted | ambiguous)[txc] & (ce >= rm_slot * (1 - NEAR_TIE))
    exact = cand & (ce == rm_slot)
    bi = cand.nonzero()
    rows = txc[bi[:, 0], bi[:, 1]]
    # analytic single-slot gradient dCE/dx_t = sum_j p_j W[Y_bj] + (p_c - 1) W[y_t] and its magnitude sum_j |G_j| |Y_j|
    g_slot = torch.zeros(len(bi), d, dtype=torch.float64, device=dev)
    m_slot = torch.zeros_like(g_slot)
    lse_slot = torch.zeros(len(bi), dtype=torch.float64, device=dev)
    for s0 in range(0, len(bi), 64):
        s1 = min(len(bi), s0 + 64)
        b, r = bi[s0:s1, 0], rows[s0:s1]
        Y = ty[b]                                                      # [s, bs_y]
        WY = W[Y]                                                      # [s, bs_y, d]
        z = torch.einsum("sd,sjd->sj", x[r], WY).masked_fill(Y == lab[r, None], float("-inf"))
        cr = c[r]
        lse = torch.logsumexp(torch.cat([z, cr[:, None]], 1), 1)
        p, pc = torch.exp(z - lse[:, None]), torch.exp(cr - lse)
        g_slot[s0:s1] = torch.einsum("sj,sjd->sd", p, WY) + (pc - 1)[:, None] * W[lab[r]]
        m_slot[s0:s1] = torch.einsum("sj,sjd->sd", p, WY.abs()) + (1 - pc).abs()[:, None] * W[lab[r]].abs()
        lse_slot[s0:s1] = lse
    is_exact = exact[bi[:, 0], bi[:, 1]]
    winners = torch.zeros(cap, dtype=torch.float64, device=dev).index_add_(0, rows, is_exact.double())
    inv = 1.0 / max(n_counted, 1)
    wgt = torch.where(is_exact, inv / winners[rows].clamp_min(1), torch.zeros_like(lse_slot))
    d_hc = torch.zeros(cap, d, dtype=torch.float64, device=dev).index_add_(0, rows, wgt[:, None] * g_slot)
    mag_hc = torch.zeros_like(d_hc).index_add_(0, rows, wgt[:, None] * m_slot)
    # near ties: a candidate whose own gradient differs from the winners' average
    g_row = d_hc / (inv if n_counted else 1.0)
    dev_s = (g_slot - g_row[rows]).norm(dim=1) / g_row[rows].norm(dim=1).clamp_min(1e-300)
    bad = torch.zeros(cap, dtype=torch.bool, device=dev)
    bad[rows[dev_s > TIE_GRAD_TOL]] = True
    near_tie = int((bad & counted).sum())
    checked = ~(bad | ambiguous)
    d_hc[~counted] = 0.0
    mag_hc[~counted] = 0.0
    # loss and its bound
    lse_row = torch.zeros(cap, dtype=torch.float64, device=dev).index_put_((rows[is_exact],), lse_slot[is_exact])
    loss = row_max[counted].sum() / max(n_counted, 1) if n_counted else torch.tensor(math.nan, dtype=torch.float64)
    amb_sum = float(row_max[ambiguous].sum())
    unit = 2.0 ** -24 * float((lse_row.abs() + c.abs() + 1)[counted].mean()) if n_counted else 0.0
    return dict(loss=loss, n_counted=n_counted, n_ambiguous=int(ambiguous.sum()), ce_sum_ambiguous=amb_sum,
                loss_unit=unit, d_hc=d_hc, mag_hc=mag_hc, checked=checked, near_tie=near_tie, ce=ce, row_max=row_max,
                winners=winners, counted=counted, ambiguous=ambiguous, c=c, lse=lse_row, selectable=sel, live=live)
