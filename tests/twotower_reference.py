"""float64 restatement of TwoTower's own device code (csrc/rp_twotower.cu, engine_twotower.py, engine_swiglu.py) and the
bounds tests/test_gpu_twotower_fp64.py measures it with.

Candidate compaction (rp_tower_compact), restated on the host:
  the entries a step reads are the labels t < min(n_valid, capacity), the shared negatives (mode 0), every per-sequence row
  (mode 2) and the per-position rows valid_idx[:n_valid] (mode 1); a negative equal to ignore_index (>= 0) flags nothing,
  any other id flags itself, or item 0 when it lies outside the catalog; the flagged items take slots in ascending id,
  at most ``cap`` of them; labels become slot ids, negatives slot ids, ``cap`` when ignored and ``cap + 1`` outside the
  catalog.  ``mistake="tile_local"`` numbers the slots per scan tile of TILE items without the earlier tiles' prefix.
Row scatter (rp_tower_scatter_rows): d_table[item_of_slot[s]] += fp32(dx[s]) for s < min(n_slots, n_rows), one fp32 add per
  element, so the expected table is exact.  ``mistake="next_row"`` adds one slot's row to the next item's row.

Item tower, one SwiGLU sub-block in the engine's padded layout (x [rows, dp], [WG; W1] [2F, dp], W2 [dp, F]):
  GL = x [WG; W1]^T + [bg; b1],  U = silu(GL[:, :F]) GL[:, F:],  z = U W2^T + b2 + x,  out = RMSNorm(z) over the d true
  columns of the dp-wide row (eps = fp32 eps);
  backward from d(out):  dz = RMSNorm'(z) d(out),  dU = dz W2,  dGL = SwiGLU'(GL) dU,  dx = dGL [WG; W1] + dz,
  dW2 = dz^T U,  d[WG; W1] = dGL^T x,  db2 = sum dz,  d[bg; b1] = sum dGL,  d norm from the RMSNorm backward.
Every stage is measured on the engine's own bf16 inputs to it.  The SwiGLU and RMSNorm stages take the per-element bounds of
tests/diff_reference.py; a GEMM output gets rp_gemm's contract (tests/gemm_reference.py): ACC_SLACK of sum_k |a_k b_k| for
the fp32 accumulation and EPI_REL of every magnitude the epilogue adds, plus half a bf16 ulp of the bf16 result.

``tower`` is the whole two-layer tower in float64 autograd, with the plausible mistakes the step and chain bounds must
reject: "no_residual" (sub-block 1 without its residual), "rms_eps" (RMSNorm eps 1e-5 instead of fp32 eps), "silu_slope"
(SiLU's slope without its g (1 - sigmoid(g)) term).

The full-catalog heads are computed in row chunks (``full_head_chunked``), so that [T_v, |I|] is never held at once."""
import numpy as np
import torch

import diff_reference as dr
from gemm_reference import ACC_SLACK, EPI_REL

TILE = 4096            # items numbered by one block of the compaction's scan (kThreads x kPerThread)
PER_THREAD = 16
RMS_EPS = dr.RMS_EPS
MISTAKES = ("no_residual", "rms_eps", "silu_slope")


# ------------------------------------------------------------------------------------------------ compaction
def read_entries(n_valid, capacity, negatives, n_neg, mode, valid_idx, n_neg_rows=None):
    """(labels read: count, negative entries read: int64 flat indices into ``negatives``)"""
    nv = max(0, min(int(n_valid), capacity))
    if mode == 0:
        idx = np.arange(n_neg, dtype=np.int64)
    elif mode == 2:
        idx = np.arange(int(n_neg_rows) * n_neg, dtype=np.int64)
    else:
        rows = np.asarray(valid_idx[:nv], dtype=np.int64)
        idx = (rows[:, None] * n_neg + np.arange(n_neg)[None, :]).reshape(-1)
    return nv, idx


def compact_ref(n_items, labels, n_valid, capacity, negatives, n_neg, mode, valid_idx, ignore_index, cap, n_neg_rows=None,
                mistake=None):
    """Host restatement of rp_tower_compact.  ``negatives`` int64 array (flat), ``labels`` int array.  Returns dict:
    n_slots, item_of_slot [cap] (-1 past n_slots), labels_out [nv], neg_idx (flat indices read) and neg_out (their slots)."""
    labels = np.asarray(labels, dtype=np.int64)
    negatives = np.asarray(negatives, dtype=np.int64).reshape(-1)
    nv, idx = read_entries(n_valid, capacity, negatives, n_neg, mode, valid_idx, n_neg_rows)
    lab, neg = labels[:nv], negatives[idx]
    inside = lambda v: (v >= 0) & (v < n_items)  # noqa: E731
    ign = (neg == ignore_index) if ignore_index >= 0 else np.zeros(neg.shape, dtype=bool)
    flag = np.zeros(n_items, dtype=bool)
    flag[np.where(inside(lab), lab, 0)] = True
    live = neg[~ign]
    flag[np.where(inside(live), live, 0)] = True
    items = np.flatnonzero(flag)
    if mistake == "tile_local":
        rank = np.zeros(items.size, dtype=np.int64)
        tiles = items // TILE
        for t in np.unique(tiles):
            sel = tiles == t
            rank[sel] = np.arange(int(sel.sum()))
    else:
        rank = np.arange(items.size, dtype=np.int64)
    slot_of = np.full(n_items, -1, dtype=np.int64)
    keep = rank < cap
    slot_of[items[keep]] = rank[keep]
    n_slots = min(items.size, cap)
    item_of_slot = np.full(cap, -1, dtype=np.int64)
    item_of_slot[rank[keep]] = items[keep]
    lab_out = np.where(inside(lab), slot_of[np.clip(lab, 0, n_items - 1)], cap + 1)
    neg_out = np.where(ign, cap, np.where(inside(neg), slot_of[np.clip(neg, 0, n_items - 1)], cap + 1))
    return dict(n_slots=int(n_slots), item_of_slot=item_of_slot, labels_out=lab_out, neg_idx=idx, neg_out=neg_out, nv=nv)


# ------------------------------------------------------------------------------------------------ scatter
def scatter_ref(d_table, dx, item_of_slot, n_slots, n_rows, mistake=None):
    """fp32 [R, d] table after rp_tower_scatter_rows (item_of_slot None: the identity map); exact, on the host or device"""
    out = d_table.clone()
    ns = n_rows if item_of_slot is None else max(0, min(int(n_slots), n_rows))
    items = torch.arange(ns, device=out.device) if item_of_slot is None else item_of_slot[:ns].long().to(out.device)
    add = dx[:ns].float().to(out.device)
    if mistake == "next_row" and ns:
        items = items.clone()
        items[ns // 2] += 1
    return out.index_add_(0, items, add)


# ------------------------------------------------------------------------------------------------ one sub-block, by stage
def gemm_ref(A, W, bias=None, residual=None):
    """y = A W^T (+ bias) (+ residual) in float64 with rp_gemm's bound for a bf16 output: (y, bound)"""
    a, w = A.double(), W.double()
    acc = a @ w.T
    mag = a.abs() @ w.abs().T
    y, slack = acc, ACC_SLACK * mag
    if bias is not None:
        b = bias.double()[None, :]
        y = y + b
        slack = slack + EPI_REL * (b.abs() + y.abs())
    if residual is not None:
        r = residual.double()
        slack = slack + EPI_REL * (y.abs() + r.abs())
        y = y + r
    slack = slack + EPI_REL * y.abs()
    return y, dr.bf16_bound(y, slack)


def block_fwd_stages(x, WGW1, bgb1, W2, b2, GL, U, z, norm, F, d_true, rows):
    """references and bounds of the forward stages of one sub-block, each on the engine's input to it"""
    dp = x.shape[1]
    out = {}
    out["GL"] = gemm_ref(x[:rows], WGW1, bgb1)
    out["U"] = dr.swiglu_fwd(GL, rows, F)
    out["z"] = gemm_ref(U[:rows], W2, b2, residual=x[:rows])
    y, yb, _ = dr.rmsnorm_fwd(z, norm, RMS_EPS, 1.0, rows, dp, dp, d_true)
    out["out"] = (y, yb)
    return out


def block_bwd_stages(dout, x, WGW1, W2, GL, U, z, norm, dz, dU, dGL, F, d_true, rows):
    """references of the backward stages of one sub-block on the engine's inputs: per-element (ref, bound) of dz, dU, dGL
    and dx; float64 dW2, dWGW1, db2, dbgbl; the RMSNorm backward dict (its dw and bounds)"""
    dp = x.shape[1]
    rb = dr.rmsnorm_bwd(dout, z, norm, RMS_EPS, 1.0, rows, dp, dp, d_true)
    out = {"dz": (rb["dx"], rb["dx_b"]), "rms": rb}
    out["dU"] = gemm_ref(dz[:rows], W2.T)
    out["dGL"] = dr.swiglu_bwd(dU, GL, rows, F)
    out["dx"] = gemm_ref(dGL[:rows], WGW1.T, residual=dz[:rows])
    dzd, dgd = dz[:rows].double(), dGL[:rows].double()
    out["dW2"] = dzd.T @ U[:rows].double()
    out["dWGW1"] = dgd.T @ x[:rows].double()
    out["db2"] = dzd.sum(0)
    out["dbgb1"] = dgd.sum(0)
    return out


def tower_input(rows, d, g):
    """item rows for the tower tests: N(0, 1), every eighth row (from row 5) scaled by 1e-3, so that with a small W2 bias
    the first norm sees rows whose mean square is near eps = 1e-5 (where the eps matters)"""
    x = torch.randn(rows, d, generator=g)
    x[5::8] *= 1e-3
    return x


# ------------------------------------------------------------------------------------------------ the tower in autograd
class _SiluNoSlope(torch.autograd.Function):
    """silu with the slope sigmoid(g) only (the 'silu_slope' mistake)"""

    @staticmethod
    def forward(ctx, g):
        ctx.save_for_backward(g)
        return g * torch.sigmoid(g)

    @staticmethod
    def backward(ctx, dy):
        (g,) = ctx.saved_tensors
        return dy * torch.sigmoid(g)


def rms_norm(x, w, n_true, eps=RMS_EPS):
    """RMSNorm over the n_true true columns of a padded row (padded columns are zero in x and w)"""
    return x * torch.rsqrt(x.pow(2).sum(-1, keepdim=True) / n_true + eps) * w


def sub_block(x, P, p, F, n_true, mistake=None):
    GL = x @ P[p + "wgw1"].T + P[p + "bgb1"]
    g, l = GL[:, :F], GL[:, F:2 * F]
    s = _SiluNoSlope.apply(g) if mistake == "silu_slope" else torch.nn.functional.silu(g)
    z = (s * l) @ P[p + "w2"].T + P[p + "b2"]
    if not (mistake == "no_residual" and p == "tw0."):
        z = z + x
    return rms_norm(z, P[p + "norm"], n_true, 1e-5 if mistake == "rms_eps" else RMS_EPS)


def tower(x0, P, F, n_true, mistake=None):
    """the two-layer tower in the engine's padded layout; P: {tw0./tw1.} x {wgw1 [2F, dp], bgb1 [2F], w2 [dp, F], b2, norm}"""
    assert mistake is None or mistake in MISTAKES, mistake
    return sub_block(sub_block(x0, P, "tw0.", F, n_true, mistake), P, "tw1.", F, n_true, mistake)


# ------------------------------------------------------------------------------------------------ full-catalog heads
FULL_KINDS = ("ce", "ce_weighted", "login_ce", "bce")


def full_head_chunked(kind, h, E, labels, weights=None, log_eps=1e-6, clamp=100.0, rows=512):
    """Mean loss of float64 rows ``h`` [n, d] over the table ``E`` [I, d] in chunks of ``rows`` rows -> (loss, d_h, d_E).
    ce: lse - z_y;  ce_weighted: w (lse - z_y);  login_ce: -clamp(log(p_y + eps), -c, c);  bce: sum_i softplus(z_i) - z_y."""
    n = h.shape[0]
    d_h = torch.empty_like(h)
    d_E = torch.zeros_like(E)
    total = torch.zeros((), dtype=h.dtype, device=h.device)
    for r0 in range(0, n, rows):
        hc, y = h[r0:r0 + rows], labels[r0:r0 + rows]
        ar = torch.arange(hc.shape[0], device=h.device)
        z = hc @ E.T
        zy = z[ar, y]
        if kind == "bce":
            total += (torch.nn.functional.softplus(z).sum(1) - zy).sum()
            g = torch.sigmoid(z)
            g[ar, y] -= 1.0
        else:
            lse = torch.logsumexp(z, -1)
            g = z.sub_(lse[:, None]).exp_()
            g[ar, y] -= 1.0
            if kind == "login_ce":
                py = torch.exp(zy - lse)
                lg = torch.log(py + log_eps)
                total += (-lg.clamp(-clamp, clamp)).sum()
                c = torch.where((lg > -clamp) & (lg < clamp), py / (py + log_eps), torch.zeros_like(py))
            else:
                c = weights[r0:r0 + rows] if kind == "ce_weighted" else torch.ones_like(lse)
                total += (c * (lse - zy)).sum()
            g *= c[:, None]
        g /= n
        d_h[r0:r0 + rows] = g @ E
        d_E.addmm_(g.T, hc)
    return total / max(n, 1), d_h, d_E
