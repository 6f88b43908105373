"""float64 restatement of the full-catalog CE head and its per-row variants (rp_ce_head_fwd_w / rp_ce_head_bwd in
csrc/rp_ce_head.cu), the per-element error bounds its GPU tests use, and the head's dispatch (tile table, split heuristic) so
that those tests can pick shapes by the tile counts they are named for.

Over the T_v valid rows, x_ti = h_t . E_i + b_i, lse_t = logsumexp_i x_ti, p_ti = exp(x_ti - lse_t), z_y = x_t,y_t:
  CE (loss_kind 0)      lt_t = lse_t - z_y                          wg_t = w_t
  LogInCE (loss_kind 1) lt_t = -clamp(log(p_y + eps), -c, c)    wg_t = w_t p_y / (p_y + eps) inside the clamp, 0 outside
  loss = sum_t w_t lt_t / T_v,   g_ti = (wg_t / T_v) (p_ti - [i == y_t]),   d_h = g E,  d_W = g^T h,  d_b = sum_t g_t
w_t is the row weight (compacted order, 1 without one).  T_v = 0 gives zeros.

Error bounds (u = 2^-24, fp32).  Every term says where it comes from.
  Logits.  The tensor cores multiply bf16 operands exactly and add d products in fp32; the bias is one more fp32 add:
      |dx_ti| <= ex_ti = d u sum_k |h_tk| |E_ik| + u |b_i|                  (z_y's gather-dot has the same bound)
  lse.  The exponentials (ex2.approx, relative 2^-22) are summed in fp32 in some order over the I items (n_items), which
      costs at most I u of the sum; the exponent argument x log2e + offset and log2 of the sum are rounded once each:
      |dlse_t| <= e_lse_t = sum_i p_ti ex_ti + I u + 2^-21 (2 + 1.5 |lse_t| + |log2(wg_t / T_v)|)
  Row weight (LogInCE).  p_y = __expf(z_y - lse) has the relative error e_p = e_lse + ex_ty + 2^-21 (1 + |z_y - lse|);
      p / (p + eps) passes eps / (p + eps) of it on, plus its own division:  e_w = eps / (p + eps) e_p + 4 u inside the clamp.
      CE: e_w = 0.  The generator of the GPU cases keeps every log(p_y + eps) at least GATE_MARGIN from +-c, far beyond
      these errors, so no row's clamp decision depends on rounding.
  G.  The gradient passes form G_ti = exp(x_ti - lse_t) wg_t / T_v and hand it to the tensor cores as a bf16 operand: a
      relative rounding of 2^-9, taken as U_G = 2^-8 (a factor two of margin), plus the error of its exponent and weight:
      rho_ti = U_G + ex_ti + e_lse_t + e_w_t.  The fp32 accumulation of the dH GEMM over the I items adds I u, the one of the
      dE GEMM and of d_bias over the T_v tokens T_v u, each of the sum of |terms|.  The one-hot part wg_t / T_v E_y (dH) /
      h_t (dE, d_bias), added in fp32, is held to U_G + e_w_t of its magnitude.
      bound_h = sum_i (wg/T_v) (rho + I u) p |E_ik| + (wg/T_v)(U_G + e_w) |E_y,k| + U_OUT |d_h|    (U_OUT: bf16 store of d_hc)
      bound_W = sum_t (wg/T_v) (rho + T_v u) p |h_tk| + sum_{t: y_t = i} (wg/T_v)(U_G + e_w) |h_tk|
      bound_b = sum_t (wg/T_v) (rho + T_v u) p + sum_{t: y_t = i} (wg/T_v)(U_G + e_w)
  Loss.  Per row, CE: e_lt = e_lse + ex_ty + u (|lse| + |z_y|) (the fp32 difference);  LogInCE inside the clamp:
      p / (p + eps) e_p, plus 2^-21 (1 + |log(p + eps)|) for __logf everywhere.  The T_v weighted row losses are summed in
      fp32 in some order (T_v u of the sum of their magnitudes) and scaled by the fp32 1 / T_v (u):
      bound_loss = (sum_t |w_t| e_lt_t + T_v u sum_t |w_t lt_t|) / T_v + u |loss|
  Every bound gets FLOOR = 1e-12 on top, so that an exact zero compares against an exact zero."""
import math

import torch

U = 2.0 ** -24
U_G = 2.0 ** -8
U_OUT = 2.0 ** -8
FLOOR = 1e-12
GATE_MARGIN = 0.01   # least distance of log(p_y + eps) from +-c in the GPU cases

# ---- dispatch of rp_ce_head.cu (test_ce_tile_table.py checks this restatement against the source)
GRID = 64                                            # column grid of the fused pass's splits (kTN)
TILE = {64: (128, 8), 128: (128, 4), 256: (64, 4)}   # ce_bwd_kernel's (column tile TN, ring depth NSTAGE) per d (dispatch_ce_bwd)
NSTAGE = {d: ns for d, (_, ns) in TILE.items()}


def cdiv(a, b):
    return (a + b - 1) // b


def pick_splits(n_row_tiles, n_col_tiles, sms, max_splits=8):
    """pick_splits of rp_ce_head.cu: the column split count of the fused pass"""
    best, best_eff = 1, 0.0
    for p in range(1, min(max_splits, n_col_tiles) + 1):
        ctas = n_row_tiles * p
        eff = ctas / (cdiv(ctas, sms) * sms)
        if eff > best_eff + 0.02:
            best, best_eff = p, eff
    return best


def fused_splits(capacity, hint, n_items, sms):
    """split count P of the fused pass (hint_row_tiles, then pick_splits over 128-item tiles)"""
    hint_tiles = cdiv(hint, 128) if 0 < hint <= capacity else cdiv(capacity, 128)
    return pick_splits(hint_tiles, cdiv(n_items, 128), sms)


def fused_tiles(capacity, hint, n_items, d, sms):
    """(split count, set of column-tile counts per CTA) of the fused pass (MODE 2)"""
    P = fused_splits(capacity, hint, n_items, sms)
    n_grid, tn = cdiv(n_items, GRID), TILE[d][0]
    spans = [min(n_items, n_grid * (s + 1) // P * GRID) - n_grid * s // P * GRID for s in range(P)]
    return P, {cdiv(c, tn) for c in spans}


def layout(n_ct, d, split, sms):
    """(capacity, n_valid, n_items, hint) whose CTAs loop over n_ct column tiles, last tiles ragged.
    split "P1": the fused pass with one split (row tiles fill the GPU), "Pn": the fused pass split over several CTAs per row
    tile, "twopass": the two-pass forward and the separate dH pass (MODE 0).  The dE pass (MODE 1) loops over
    ceil(n_valid / TN) token tiles: n_ct of them, except in "Pn" (one row tile of tokens)."""
    tn = TILE[d][0]
    if split == "Pn":
        n_valid = min(tn * n_ct - 5, 123)
        for n_items in range(GRID + 1, tn * 16 * (n_ct + 2)):
            if n_items % tn == 0:
                continue
            P, counts = fused_tiles(128, n_valid, n_items, d, sms)
            if P > 1 and n_ct in counts:
                return 128, n_valid, n_items, n_valid
        raise AssertionError(f"no catalog size splits into CTAs of {n_ct} column tiles on {sms} SMs")
    n_valid, n_items = tn * n_ct - 5, tn * n_ct - 17
    if split == "twopass":
        return cdiv(n_valid, 128) * 128, n_valid, n_items, n_valid
    capacity = sms * 128   # as many row tiles as SMs: one split is the best balance
    P, counts = fused_tiles(capacity, capacity, n_items, d, sms)
    assert P == 1 and counts == {n_ct}
    return capacity, n_valid, n_items, capacity


# ---- float64 restatement
def logits(h, W, b, n_valid):
    """fp64 logits [n_valid, I] of the valid rows"""
    x = h[:n_valid].double() @ W.double().T
    return x + b[: W.shape[0]].double()[None, :] if b is not None else x


def target_log_prob(h, W, b, labels, n_valid):
    """log p_y per valid row (fp64)"""
    x = logits(h, W, b, n_valid)
    y = labels[:n_valid].long()
    return x.gather(1, y[:, None])[:, 0] - torch.logsumexp(x, -1)


def grads(p, y, c, h, W):
    """d_h, d_W, d_b of g_ti = c_t (p_ti - [i == y_t])"""
    g = c[:, None] * p
    g[torch.arange(len(y), device=g.device), y] -= c
    return g @ W, g.T @ h, g.sum(0)


def reference(h, W, b, labels, n_valid, row_weight=None, loss_kind=0, log_eps=1e-6, clamp=100.0):
    """h [cap, d], W [I, d] (bf16 or any), b [>= I] or None, labels [cap], row_weight [cap] or None, all on one device (only
    the first n_valid entries of h, labels and row_weight are read).  Returns, in float64 on that device, the loss, d_h
    [n_valid, d], d_W [I, d], d_b [I], the bound of each (same shapes), and per row wg (gradient weight), p_y,
    lg = log(p_y + eps) and the gate (LogInCE inside the clamp)."""
    T = n_valid
    I, d = W.shape
    hh, WW = h[:T].double(), W.double()
    y = labels[:T].long().to(hh.device)
    f64 = dict(dtype=torch.float64, device=hh.device)
    bb = b[:I].double() if b is not None else torch.zeros(I, **f64)
    x = hh @ WW.T + bb[None, :]
    lse = torch.logsumexp(x, -1)
    p = torch.exp(x - lse[:, None])
    zy = x.gather(1, y[:, None])[:, 0]
    py = torch.exp(zy - lse)
    w = row_weight[:T].double() if row_weight is not None else torch.ones(T, **f64)
    inv = 1.0 / max(T, 1)
    ex = d * U * (hh.abs() @ WW.abs().T) + U * bb.abs()[None, :]
    ex_y = ex.gather(1, y[:, None])[:, 0]
    if loss_kind == 0:
        lg, gate = torch.zeros(T, **f64), torch.ones(T, dtype=torch.bool, device=hh.device)
        lt, wg = lse - zy, w
    else:
        lg = torch.log(py + log_eps)
        gate = (lg > -clamp) & (lg < clamp)
        lt = -lg.clamp(-clamp, clamp)
        wg = w * torch.where(gate, py / (py + log_eps), torch.zeros_like(py))
    c = wg * inv
    off = torch.log2(c.detach().abs().clamp_min(1e-300)).abs()
    e_lse = (p * ex).sum(1) + I * U + 2.0 ** -21 * (2 + 1.5 * lse.abs() + off)
    if loss_kind == 0:
        e_w = torch.zeros(T, **f64)
        e_lt = e_lse + ex_y + U * (lse.abs() + zy.abs())
    else:
        e_p = e_lse + ex_y + 2.0 ** -21 * (1 + (zy - lse).abs())
        e_w = torch.where(gate, log_eps / (py + log_eps) * e_p + 4 * U, torch.zeros_like(py))
        e_lt = torch.where(gate, py / (py + log_eps) * e_p, torch.zeros_like(py)) + 2.0 ** -21 * (1 + lg.abs())
    d_h, d_W, d_b = grads(p, y, c, hh, WW)
    loss = (w * lt).sum() * inv
    rho = U_G + ex + (e_lse + e_w)[:, None]
    cp = c.abs()[:, None] * p
    oh = c.abs() * (U_G + e_w)
    bound_h = (cp * (rho + I * U)) @ WW.abs() + oh[:, None] * WW[y].abs() + U_OUT * d_h.abs() + FLOOR
    A = cp * (rho + T * U)
    bound_W = A.T @ hh.abs() + torch.zeros_like(WW).index_add_(0, y, oh[:, None] * hh.abs()) + FLOOR
    bound_b = A.sum(0) + torch.zeros(I, **f64).index_add_(0, y, oh) + FLOOR
    bound_loss = ((w.abs() * e_lt).sum() + T * U * (w * lt).abs().sum()) * inv + U * loss.abs() + FLOOR
    return dict(loss=loss, d_h=d_h, d_W=d_W, d_b=d_b, bound_loss=bound_loss, bound_h=bound_h, bound_W=bound_W,
                bound_b=bound_b, wg=wg, py=py, lg=lg, gate=gate, p=p, inv=inv)


# ---- inputs of the GPU cases
# row kinds: (weighted, loss_kind, log_eps, clamp).  "login_lo" puts rows below -c (p_y + eps < e^-4), "login_hi" above +c
# (p_y > e^0.5 - 1); both keep rows inside the clamp too.
KINDS = {"plain": (False, 0, 1e-6, 100.0), "weighted": (True, 0, 1e-6, 100.0), "login": (False, 1, 1e-6, 100.0),
         "login_lo": (False, 1, 1e-3, 4.0), "login_hi": (False, 1, 1.0, 0.5), "login_w": (True, 1, 1e-3, 4.0)}
STALE = 0.25   # offset of the finite garbage in hc rows past n_valid


def make_case(cap, n_valid, n_items, d, *, bias, kind="plain", seed=0, scale_h=0.5, scale_e=0.3, bias_trap=False,
              distinct_labels=False):
    """CPU inputs of one head call.  hc rows past n_valid hold finite non-zero garbage, row weights past n_valid are NaN,
    labels are in range everywhere.  Weights: uniform in [0, 3], every 7th valid one exactly 0, the middle one 40.  LogInCE
    kinds align every other valid row with its target item (target logit uniform in [2, 25]) so that p_y spreads over
    (0, 1), and redraw any row whose log(p_y + eps) lies within GATE_MARGIN of +-c.  bias_trap: the item with the largest raw
    score of any valid row gets bias -60."""
    weighted, loss_kind, log_eps, clamp = KINDS[kind]
    g = torch.Generator().manual_seed(seed + 7919 * n_items + 131 * n_valid + d)
    h = torch.randn(cap, d, generator=g) * scale_h
    h[n_valid:] = torch.randn(cap - n_valid, d, generator=g) * 0.5 + STALE
    W = (torch.randn(n_items, d, generator=g) * scale_e).to(torch.bfloat16)
    if distinct_labels:
        assert n_items >= cap
        labels = torch.randperm(n_items, generator=g)[:cap]
    else:
        labels = torch.randint(0, n_items, (cap,), generator=g)
    b = torch.randn(n_items, generator=g) * 0.5 + 0.5 if bias else None
    if loss_kind == 1:
        for t in range(0, n_valid, 2):
            e = W[labels[t]].float()
            h[t] = e * (float(torch.rand((), generator=g)) * 23 + 2) / max(float(e.pow(2).sum()), 1e-6)
    h = h.to(torch.bfloat16)
    if bias_trap and n_valid:
        raw = h[:n_valid].double() @ W.double().T
        b[int(raw.max(0).values.argmax())] = -60.0
    if loss_kind == 1 and n_valid:
        for _ in range(50):
            lg = torch.log(torch.exp(target_log_prob(h, W, b, labels, n_valid)) + log_eps)
            near = ((lg.abs() - clamp).abs() < GATE_MARGIN).nonzero()[:, 0]
            if not len(near):
                break
            h[near] = (torch.randn(len(near), d, generator=g) * scale_h).to(torch.bfloat16)
        lg = torch.log(torch.exp(target_log_prob(h, W, b, labels, n_valid)) + log_eps)
        assert ((lg.abs() - clamp).abs() >= GATE_MARGIN).all(), "a LogInCE row sits at the clamp"
    w = None
    if weighted:
        w = torch.full((cap,), float("nan"))
        w[:n_valid] = torch.rand(n_valid, generator=g) * 3
        w[:n_valid:7] = 0.0
        if n_valid:
            w[n_valid // 2] = 40.0
    return dict(h=h, W=W, b=b, labels=labels, row_weight=w, loss_kind=loss_kind, log_eps=log_eps, clamp=clamp)


def case_reference(c, n_valid):
    return reference(c["h"], c["W"], c["b"], c["labels"], n_valid, c["row_weight"], c["loss_kind"], c["log_eps"], c["clamp"])


def worst(got, ref, bound):
    """largest |got - ref| / bound (1.0 = at the bound; NaN anywhere counts as infinitely far)"""
    if ref.numel() == 0:
        return 0.0
    r = (got.double().to(ref.device) - ref).abs() / bound
    return math.inf if torch.isnan(r).any() else float(r.max())
