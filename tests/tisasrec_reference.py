"""float64 restatement of TiSASRec's time-interval kernels (csrc/rp_tisasrec.cu) at their own boundaries, with a
per-element error bound for every output, and the inputs the kernel tests draw.  It works one (sequence, head) at a time in
closed form: the time terms are gathered per pair from the [time_span + 1, 64] table slot, with dropout masks of one
sequence ([L, L, 64]) at most, never the [B, L, L, d] tensors of oracle/tisasrec.time_attention, so B in the hundreds is
affordable and the whole reference runs on whichever device its inputs are on.

Notation, per head h (64-wide slot, padded table columns zero), sequence b, live query row i, key j <= i (n = i + 1 keys),
r_ij = min(floor(|t_i - t_j|), span) in the timestamps' dtype; ks = 1 / (1 - p) in fp32 (1 without dropout); mk, mv, ka the
0 / 1 keep draws of the tk, tv and attention sites (tests/dropout_stream.py's stream, here as torch integer ops):
  qe_ij  = ks sum_c q_ic E_K[r_ij, c] mk_ijc                    qa_ij  = the same sum of |terms|
  x_ij   = (S_ij + qe_ij) scale,  A = softmax_j x,  Ad = A ka ks
  hpre_i = q_in_i + ks sum_j Ad'_ij E_V[r_ij] mv_ij             (Ad' the kernel's own rounded Ad, which it multiplies by)
  tvd_ij = ks sum_c dO_ic E_V[r_ij, c] mv_ijc,  dav = (dpd + tvd) keep,  dot_i = sum_j A_ij dav_ij
  ds_ij  = A_ij (dav_ij - dot_i) scale,  dq_t_i = ks sum_j ds_ij E_K[r_ij] mk_ij
  d_time_k[r] += sum_{pairs with r_ij = r} ds_ij q_i ks mk_ij,  d_time_v[r] += sum A_ij keep_ij dO_i ks mv_ij
keep is ka ks with dropout and 1 without; A in the backward is the forward's bf16 save, an input.

Error bounds (u = 2^-24).  bf16 outputs get half a bf16 ulp of |ref| + slack (HULP(|ref| + e)) plus the fp32 slack e.  The
kernels build with fast math: ks and 1 / sum are MUFU.RCP reciprocals, within 2 u of the quotient, so every term that
carries ks or the row's 1 / sum gets 2 u more than one rounding:
  Logit.  The fp32 dot over the slot's 64 columns (bf16 x bf16 products are exact in fp32) costs 63 u qa; the ks product
      (and ks itself), the S add and the scale product:  e_x = scale (66 u qa + u |S + qe|) + u |x|.
  Softmax.  x - m rounds once (u |z|, z = x - m; the max's own error cancels in the ratio), __expf is within 2 + 1.173 |z|
      fp32 ulps (CUDA programming guide), i.e. 2 u (2 + 1.173 |z|) relative; so each exponential carries
      delta = e_x + u (4 + 3.35 |z|).  The sum of n positive terms costs n u of itself, 1 / sum 2 u and the product u:
      A_ij has the relative error rho_ij = delta_ij + sum_k A_ik delta_ik + (n + 3) u.
  A (bf16):  HULP + rho A.   Ad (bf16, a ks product before the store):  HULP + (rho + 3 u) Ad.
  hpre (bf16).  The n bf16 x bf16 products of Ad' E_V are exact and summed in fp32 (n u), times ks and plus q_in (one u of
      the result each):  e = ks (n + 3) u sum_j |Ad'_ij E_V mv| + u |hpre|.
  dS (bf16).  tvd as qe: e_tvd = 67 u tva;  dav:  e_dav = keep (e_tvd + u |dpd + tvd|) + u |dav|;  the row dot, each of n
      products rounded and summed:  e_dot = sum_j A_ij e_dav_ij + (n + 1) u sum_j |A_ij dav_ij|;  the subtraction, the A
      product and the scale one u each:  e_ds = scale A (e_dav + e_dot + u |dav - dot|) + 2 u |ds|.  Stored: HULP + e_ds.
  Ad (backward, bf16 of the fp32 product bf16(A) * keep):  HULP + 3 u |Ad|.
  dq_t (bf16).  The kernel multiplies the fp32 ds (not the stored bf16) by E_K:  e = ks sum_j (e_ds + (n + 3) u |ds|)
      |E_K mk| + u |dq_t|.
  d_time_k, d_time_v (fp32, added to the start value).  Each term is a product of the fp32 ds (or bf16(A) keep) by q ks
      (dO ks): two (three) roundings, and ks's own 2 u.  The terms of bucket r are summed with shared-memory atomics in an unknown order
      inside each of the G CTAs of the head, then the G partials in order, then added to the start value: at most
      (N_r + G) u of the sum of |terms| (N_r the pairs in bucket r), and u |out|.  d_time_k also carries ds's error:
          bound_k = sum_terms e_ds |q| ks mk + (N_r + G + 5) u sum |terms| + u |out|
          bound_v = (N_r + G + 6) u sum |terms| + u |out|
  d_pos (fp32).  dropout'(dkv) over the B sequences in order, a ks product each: (B + 4) u sum |terms| + u |out|.
Every bound gets FLOOR = 1e-30 on top, so that an exact zero compares against an exact zero."""
import math

import numpy as np
import torch

from dropout_stream import _fmix32

U = 2.0 ** -24
FLOOR = 1e-30
SLOT = 64
BWD_CTAS = 256      # kBwdCtas: the backward runs min(BWD_CTAS // H, B) CTAs per head, CTA g taking b = g, g + G, ...
SITE_ATT, SITE_TK, SITE_TV = 1 << 40, 4002 << 40, 4003 << 40
DTYPE_CODE = {torch.int64: 0, torch.float32: 1, torch.float64: 2}
_M32 = 0xFFFFFFFF


def bwd_ctas(B, H):
    return max(1, min(BWD_CTAS // H, B))


def f32(x):
    return float(np.float32(x))


def ks_of(p):
    """1 / (1 - p) as the kernels compute it (fp32)"""
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(p))) if p > 0 else 1.0


def hulp(x):
    """half a bf16 ulp of |x| (x float64)"""
    a = x.abs().clamp_min(1e-300)
    return torch.exp2(torch.floor(torch.log2(a)) - 8)


def bf16_bound(ref, slack):
    return hulp(ref.abs() + slack) + slack + FLOOR


# ------------------------------------------------------------------------------------------------ intervals, dropout
def intervals(t, span):
    """r[i, j] = min(floor(|t_i - t_j|), span) of one sequence's timestamps t [L], in t's dtype (int64 skips the floor)"""
    d = (t[:, None] - t[None, :]).abs()
    if d.dtype != torch.int64:
        d = torch.floor(d)
        return torch.where(d > span, torch.full_like(d, span), d).long()
    return d.clamp_max(span)


def _mul32(h, c):
    """(h * c) mod 2^32 for int64 tensors h in [0, 2^32) and a constant c, without int64 overflow"""
    lo, hi = c & 0xFFFF, c >> 16
    return (h * lo + (((h * hi) & 0xFFFF) << 16)) & _M32


def _fmix(h):
    h = h ^ (h >> 16)
    h = _mul32(h, 0x85EBCA6B)
    h = h ^ (h >> 13)
    h = _mul32(h, 0xC2B2AE35)
    return h ^ (h >> 16)


def row_key(seed_eff, off, rows):
    """drop_row_key for an int64 tensor of row indices (< 2^62)"""
    seed, off = int(seed_eff) & 0xFFFFFFFFFFFFFFFF, int(off)
    s = int(_fmix32((seed & _M32) ^ (((seed >> 32) * 0x85EBCA77) & _M32) ^ ((((off >> 32) & _M32) * 0xC2B2AE3D) & _M32)
                    ^ (((off & _M32) * 0x27D4EB2F) & _M32)))
    return _fmix((s + _mul32(rows & _M32, 0x9E3779B1) + _mul32(rows >> 32, 0x165667B1)) & _M32)


def col_key(cols):
    return _fmix((_mul32(cols, 0x9E3779B1) + 0x27D4EB2F) & _M32)


def mix(rk, ck):
    x = _mul32(rk ^ ck, 0x9E3779B1)
    x = x ^ (x >> 15)
    return _mul32(x, 0x85EBCA77)


def threshold(p):
    return int(float(np.float32(p)) * 4294967296.0)


def keep(seed_eff, off, p, rows, cols):
    """bool [*rows.shape, *cols.shape]: element (row, col) of a dropout site is kept"""
    rk = row_key(seed_eff, off, rows)
    ck = col_key(cols)
    return mix(rk.reshape(*rows.shape, *([1] * cols.dim())), ck) >= threshold(p)


# ------------------------------------------------------------------------------------------------ problem description
class Problem:
    """The kernels' inputs (torch tensors on one device) and scalars.  q, q_in, d_o: bf16 [B*L, ldq]; times [B, L] in their
    dtype; pad bool [B, L]; tk, tv: bf16 [span + 1, ld_t] (padded slot columns zero); S fp32 [B*H, Lp, Lp]; dpd bf16
    [B*H, Lp, Lp].  seed_eff = seed + *seed_ptr (or seed when seed_ptr is null)."""

    def __init__(self, **kw):
        self.__dict__.update(kw)
        self.Lp = (self.L + 63) // 64 * 64
        self.scale = f32(1.0 / math.sqrt(self.head_dim))
        self.ks = ks_of(self.p)

    def slot(self, x, b, h):
        """[L, 64] float64 of head h's slot of sequence b's rows of a [B*L, ld] array"""
        return x[b * self.L:(b + 1) * self.L, h * SLOT:(h + 1) * SLOT].double()

    def table(self, x, h):
        return x[:, h * SLOT:(h + 1) * SLOT].double()

    def masks(self, b, h):
        """(mk, mv) float64 [L, L, 64] keep factors 0 / ks of the tk / tv sites, ka [L, Lp] 0 / ks of the attention site"""
        dev, L = self.q.device, self.L
        if self.p <= 0:
            return None, None, None
        rows = (b * L + torch.arange(L, device=dev))[:, None] * L + torch.arange(L, device=dev)[None, :]
        cols = h * SLOT + torch.arange(SLOT, device=dev)
        tks = getattr(self, "time_ks", self.ks)     # a test may restate a kernel that forgets ks on the time terms
        mk = keep(self.seed_eff, self.tk_off, self.p, rows, cols).double() * tks
        mv = keep(self.seed_eff, self.tv_off, self.p, rows, cols).double() * tks
        arows = (b * self.H + h) * self.Lp + torch.arange(L, device=dev)
        ka = keep(self.seed_eff, self.att_off, self.p, arows, torch.arange(L, device=dev)).double() * self.ks
        return mk, mv, ka


def _pair_dot(x, E, r, m):
    """(sum_c x_ic E[r_ij, c] m_ijc, the sum of |terms|) for x [L, 64], E [n_r, 64], r [L, L], m [L, L, 64] or None"""
    if m is None:
        return (x @ E.T).gather(1, r), (x.abs() @ E.abs().T).gather(1, r)
    t = x[:, None, :] * E[r] * m
    return t.sum(-1), t.abs().sum(-1)


def _pair_sum(w, E, r, m):
    """sum_j w_ij E[r_ij] m_ij -> [L, 64], and the sum of |terms|"""
    if m is None:
        n_r = E.shape[0]
        W = torch.zeros(w.shape[0], n_r, dtype=w.dtype, device=w.device).scatter_add_(1, r, w)
        Wa = torch.zeros_like(W).scatter_add_(1, r, w.abs())
        return W @ E, Wa @ E.abs()
    t = w[:, :, None] * E[r] * m
    return t.sum(1), t.abs().sum(1)


def _table_grad(w, x, r, m, n_r):
    """sum over pairs of bucket r of w_ij x_ic m_ijc -> [n_r, 64], |terms| sum [n_r, 64], pair count per bucket [n_r]"""
    L = r.shape[0]
    idx = r.reshape(-1)
    cnt = torch.zeros(n_r, dtype=torch.float64, device=r.device).index_add_(0, idx, (w != 0).double().reshape(-1))
    if m is None:
        t = w[:, :, None] * x[:, None, :]
    else:
        t = w[:, :, None] * x[:, None, :] * m
    t = t.reshape(L * L, -1)
    z = torch.zeros(n_r, t.shape[1], dtype=torch.float64, device=r.device)
    return z.clone().index_add_(0, idx, t), z.index_add_(0, idx, t.abs()), cnt


def forward(P, S=None, ad_kernel=None, r=None):
    """Reference and bounds of rp_ti_attn_fwd.  S: the fp32 scores the kernel is given (P.S by default; float64 for the
    stage reference).  ad_kernel: the kernel's Ad output [B*H, Lp, Lp] (its own rounding, which hpre multiplies by); None
    uses the reference Ad.  r: intervals [B, L, L] to use instead of the timestamps'.  Returns dict of float64 tensors: A, Ad [B*H, L, L], hpre [B*L, H*64] and their bounds
    (A_b, Ad_b, hpre_b), and, for the backward, the per-sequence intervals r [B, L, L]."""
    S = P.S if S is None else S
    B, H, L, dev = P.B, P.H, P.L, P.q.device
    out = {k: torch.zeros(B * H, L, L, dtype=torch.float64, device=dev) for k in ("A", "Ad", "A_b", "Ad_b")}
    out["hpre"] = torch.zeros(B * L, H * SLOT, dtype=torch.float64, device=dev)
    out["hpre_b"] = torch.zeros_like(out["hpre"])
    out["r"] = torch.zeros(B, L, L, dtype=torch.long, device=dev)
    causal = torch.ones(L, L, dtype=torch.bool, device=dev).tril()
    n = torch.arange(1, L + 1, device=dev, dtype=torch.float64)[:, None]
    for b in range(B):
        rb = intervals(P.times[b].to(dev), P.span) if r is None else r[b]
        out["r"][b] = rb
        live = P.pad[b].to(dev)
        rowm = causal & live[:, None]
        for h in range(H):
            bz = b * H + h
            mk, mv, ka = P.masks(b, h)
            q = P.slot(P.q, b, h)
            qe, qa = _pair_dot(q, P.table(P.tk, h), rb, mk)     # mk carries ks (1 without dropout)
            Sb = S[bz, :L, :L].double()
            x = (Sb + qe) * P.scale
            ex = P.scale * (66 * U * qa + U * (Sb + qe).abs()) + U * x.abs()
            xm = torch.where(rowm, x, torch.full_like(x, -math.inf))
            m = xm.max(1, keepdim=True).values.clamp_min(-1e300)
            z = torch.where(rowm, x - m, torch.zeros_like(x))
            A = torch.where(rowm, torch.exp(z), torch.zeros_like(x))
            A = A / A.sum(1, keepdim=True).clamp_min(1e-300)
            delta = torch.where(rowm, ex + U * (4 + 3.35 * z.abs()), torch.zeros_like(x))
            rho = delta + (A * delta).sum(1, keepdim=True) + (n + 3) * U
            Ad = A if ka is None else A * ka[:, :L]
            out["A"][bz], out["Ad"][bz] = A, Ad
            out["A_b"][bz] = bf16_bound(A, rho * A)
            out["Ad_b"][bz] = bf16_bound(Ad, (rho + 3 * U) * Ad)
            adk = Ad if ad_kernel is None else ad_kernel[bz, :L, :L].double() * rowm
            o, oa = _pair_sum(adk, P.table(P.tv, h), rb, mv)
            qin = P.slot(P.q_in, b, h)
            hp = torch.where(live[:, None], qin + o, qin)
            e = (n + 3) * U * oa + U * hp.abs()
            rows = slice(b * L, (b + 1) * L)
            out["hpre"][rows, h * SLOT:(h + 1) * SLOT] = hp
            out["hpre_b"][rows, h * SLOT:(h + 1) * SLOT] = torch.where(live[:, None], bf16_bound(hp, e),
                                                                       torch.full_like(hp, FLOOR))
    return out


def backward(P, A=None, dpd=None, r=None):
    """Reference and bounds of rp_ti_attn_bwd.  A: the forward's probabilities [B*H, >=L, >=L] (the kernel's bf16 a_save);
    dpd: dO . v'^T [B*H, >=L, >=L] (P.dpd by default).  Returns dS, Ad [B*H, L, L], dq_t [B*L, H*64], d_time_k / d_time_v
    [span + 1, H*64] (the sums alone: the test adds its start values) and their bounds."""
    dpd = P.dpd if dpd is None else dpd
    B, H, L, dev, n_r = P.B, P.H, P.L, P.q.device, P.span + 1
    G = bwd_ctas(B, H)
    out = {k: torch.zeros(B * H, L, L, dtype=torch.float64, device=dev) for k in ("dS", "Ad", "dS_b", "Ad_b")}
    for k in ("dq_t", "dq_t_b"):
        out[k] = torch.zeros(B * L, H * SLOT, dtype=torch.float64, device=dev)
    acc = {k: torch.zeros(n_r, H * SLOT, dtype=torch.float64, device=dev)
           for k in ("dtk", "dtv", "dtk_abs", "dtv_abs", "dtk_eds")}
    cnt = {k: torch.zeros(n_r, H, dtype=torch.float64, device=dev) for k in ("k", "v")}
    used = torch.zeros(n_r, H, dtype=torch.float64, device=dev)
    causal = torch.ones(L, L, dtype=torch.bool, device=dev).tril()
    n = torch.arange(1, L + 1, device=dev, dtype=torch.float64)[:, None]
    for b in range(B):
        rb = intervals(P.times[b].to(dev), P.span) if r is None else r[b]
        live = P.pad[b].to(dev)
        rowm = (causal & live[:, None]).double()
        for h in range(H):
            bz = b * H + h
            cs = slice(h * SLOT, (h + 1) * SLOT)
            mk, mv, ka = P.masks(b, h)
            dO, q = P.slot(P.d_o, b, h), P.slot(P.q, b, h)
            a = A[bz, :L, :L].double() * rowm
            tvd, tva = _pair_dot(dO, P.table(P.tv, h), rb, mv)
            kp = rowm if ka is None else ka[:, :L] * rowm
            dp = dpd[bz, :L, :L].double()
            dav = (dp + tvd) * kp
            e_dav = kp * (67 * U * tva + U * (dp + tvd).abs()) + U * dav.abs()
            dot = (a * dav).sum(1, keepdim=True)
            e_dot = (a * e_dav).sum(1, keepdim=True) + (n + 1) * U * (a * dav).abs().sum(1, keepdim=True)
            ds = a * (dav - dot) * P.scale * rowm
            e_ds = (P.scale * a * (e_dav + e_dot + U * (dav - dot).abs()) + 2 * U * ds.abs()) * rowm
            ad = a * kp
            out["dS"][bz], out["dS_b"][bz] = ds, bf16_bound(ds, e_ds)
            out["Ad"][bz], out["Ad_b"][bz] = ad, bf16_bound(ad, 3 * U * ad.abs())
            g, _ = _pair_sum(ds, P.table(P.tk, h), rb, mk)
            _, ga = _pair_sum(e_ds + (n + 3) * U * ds.abs(), P.table(P.tk, h), rb, mk)
            rows = slice(b * L, (b + 1) * L)
            out["dq_t"][rows, cs] = g
            out["dq_t_b"][rows, cs] = bf16_bound(g, ga + U * g.abs())
            tk, tka, ck = _table_grad(ds, q, rb, mk, n_r)
            tke, _, _ = _table_grad(e_ds, q.abs(), rb, mk, n_r)
            tv, tva2, cv = _table_grad(ad, dO, rb, mv, n_r)
            acc["dtk"][:, cs] += tk
            acc["dtk_abs"][:, cs] += tka
            acc["dtk_eds"][:, cs] += tke
            acc["dtv"][:, cs] += tv
            acc["dtv_abs"][:, cs] += tva2
            cnt["k"][:, h] += ck
            cnt["v"][:, h] += cv
            used[:, h] += torch.bincount(rb[rowm.bool()], minlength=n_r).double()
    Nk = cnt["k"].repeat_interleave(SLOT, 1)
    Nv = cnt["v"].repeat_interleave(SLOT, 1)
    out["d_time_k"], out["d_time_v"] = acc["dtk"], acc["dtv"]
    out["used"] = used.repeat_interleave(SLOT, 1) > 0      # [span + 1, H*64]: a live pair of the head falls in the bucket
    out["d_time_k_b"] = acc["dtk_eds"] + (Nk + G + 5) * U * acc["dtk_abs"]
    out["d_time_v_b"] = (Nv + G + 6) * U * acc["dtv_abs"]
    return out


def table_bound(b_sum, start, ref_sum):
    """the bound of a time-table / positional gradient added to ``start``: the sum's bound and u of the result"""
    return b_sum + U * (start.double() + ref_sum).abs() + FLOOR


# ------------------------------------------------------------------------------------------------ positional terms
def pos_add(kv, pos_k, pos_v, L, d, p, seed_eff, off_k, off_v):
    """rp_ti_pos_add emulated on the host, bit for bit: kv[t, c] = bf16(fp32(kv) + dropout(pos[t % L, c]))"""
    T = kv.shape[0]
    out = kv.clone()
    dev = kv.device
    ks = torch.tensor(ks_of(p), dtype=torch.float32)
    tok = torch.arange(T, device=dev)
    for half, (pos, off) in enumerate(((pos_k, off_k), (pos_v, off_v))):
        v = pos[tok % L, :d].float()
        if p > 0:
            kp = keep(seed_eff, off, p, tok, torch.arange(d, device=dev))
            v = torch.where(kp, v * ks.to(dev), torch.zeros_like(v))
        cs = slice(half * d, (half + 1) * d)
        out[:, cs] = (kv[:, cs].float() + v).to(torch.bfloat16)
    return out


def pos_bwd(dkv, B, L, d, head_dim, p, seed_eff, off_k, off_v):
    """rp_ti_pos_bwd's sums (d_pos_k, d_pos_v [L, d]), their bounds before the start add, and the true-column mask [d]"""
    dev = dkv.device
    ks = ks_of(p)
    tok = torch.arange(B * L, device=dev)
    res = []
    for half, off in enumerate((off_k, off_v)):
        g = dkv[:, half * d:(half + 1) * d].double()
        if p > 0:
            g = g * keep(seed_eff, off, p, tok, torch.arange(d, device=dev)).double() * ks
        g = g.view(B, L, d)
        res += [g.sum(0), (B + 4) * U * g.abs().sum(0)]
    true_cols = (torch.arange(d, device=dev) % SLOT) < head_dim
    return res[0], res[1], res[2], res[3], true_cols


# ------------------------------------------------------------------------------------------------ the whole attention stage
def attention_stage(q, kv, q_in, d_o, times, pad, tk, tv, H, head_dim, span, p, seed_eff, att_off, tk_off=SITE_TK,
                    tv_off=SITE_TV):
    """One block's attention forward and backward in float64 from the engine's Q, KV = [K' | V'], q_in and dO = dh (all
    [B*L, *] in the padded layout, dpad = H * 64 columns per half): h = q_in + Ad (V' + TVm), dQ, dK', dV' and the time
    tables' gradients (sums only).  Returns a dict of float64 tensors."""
    B, L = pad.shape
    d = H * SLOT
    P = Problem(q=q, q_in=q_in, d_o=d_o, times=times, pad=pad, tk=tk, tv=tv, B=B, H=H, L=L, head_dim=head_dim,
                span=span, p=p, seed_eff=seed_eff, att_off=att_off, tk_off=tk_off, tv_off=tv_off)
    dev = q.device
    S = torch.zeros(B * H, L, L, dtype=torch.float64, device=dev)
    dpd = torch.zeros_like(S)
    for b in range(B):
        rows = slice(b * L, (b + 1) * L)
        for h in range(H):
            cs = slice(h * SLOT, (h + 1) * SLOT)
            k, v = kv[rows, cs].double(), kv[rows, d + h * SLOT:d + (h + 1) * SLOT].double()
            S[b * H + h] = q[rows, cs].double() @ k.T
            dpd[b * H + h] = d_o[rows, cs].double() @ v.T
    f = forward(P, S=S)
    bw = backward(P, A=f["A"], dpd=dpd, r=f["r"])
    h = f["hpre"].clone()
    dQ = bw["dq_t"].clone()
    dKV = torch.zeros(B * L, 2 * d, dtype=torch.float64, device=dev)
    for b in range(B):
        rows = slice(b * L, (b + 1) * L)
        for hh in range(H):
            bz, cs = b * H + hh, slice(hh * SLOT, (hh + 1) * SLOT)
            k, v = kv[rows, cs].double(), kv[rows, d + hh * SLOT:d + (hh + 1) * SLOT].double()
            live = pad[b].to(dev)[:, None]
            h[rows, cs] += torch.where(live, f["Ad"][bz] @ v, torch.zeros_like(v))
            dQ[rows, cs] += bw["dS"][bz] @ k
            dKV[rows, cs] = bw["dS"][bz].T @ q[rows, cs].double()
            dKV[rows, d + hh * SLOT:d + (hh + 1) * SLOT] = bw["Ad"][bz].T @ d_o[rows, cs].double()
    return {"h": h, "dQ": dQ, "dK": dKV[:, :d], "dV": dKV[:, d:], "d_time_k": bw["d_time_k"], "d_time_v": bw["d_time_v"]}


# ------------------------------------------------------------------------------------------------ inputs
def make_times(kind, B, L, span, g, dtype=torch.int64):
    """[B, L] timestamps of one kind (see the GPU tests), CPU"""
    if kind == "mixed":
        t = torch.randint(0, 2 * span + 2, (B, L), generator=g).sort(1).values
    elif kind == "edges":      # every gap span - 1, span or span + 1, some zero
        steps = torch.randint(0, 4, (B, L), generator=g)
        steps = torch.tensor([0, span - 1, span, span + 1])[steps]
        t = steps.cumsum(1)
    elif kind == "decreasing":  # decreasing and negative
        t = -torch.randint(0, max(2, span // 3 + 2), (B, L), generator=g).cumsum(1)
    elif kind == "unsorted":
        t = torch.randint(-span, span, (B, L), generator=g)
    elif kind == "big_int":     # near 2^62, gaps >= 2^32 beside small ones
        small = torch.randint(0, span + 2, (B, L), generator=g)
        big = torch.randint(0, 2, (B, L), generator=g) << 32
        t = (1 << 62) + (small + big).cumsum(1)
    elif kind == "epoch_f32":   # epoch seconds ~1.7e9, where float32's ulp is 128: 64 s steps round
        return (1.7e9 + (torch.randint(0, 4, (B, L), generator=g).double() * 64).cumsum(1)).to(torch.float32)
    elif kind == "frac":        # fractional gaps at floor edges
        steps = torch.tensor([0.0, 2.999, 3.0, 3.5, 0.25, float(span) - 0.001, float(span), float(span) + 0.5])
        t = 1000.0 + steps[torch.randint(0, len(steps), (B, L), generator=g)].double().cumsum(1)
        return t.to(dtype)
    elif kind == "epoch_f64":   # epoch seconds with sub-second steps
        t = 1.7e9 + (torch.randint(0, 8, (B, L), generator=g).double() * 0.37).cumsum(1)
        return t.to(dtype)
    else:
        raise ValueError(kind)
    return t if dtype == torch.int64 else t.to(dtype)


def make_pad(B, L, pattern):
    """bool [B, L]: pattern 'mixed' = full, left padding, one live row, all dead, a dead row between live ones (cyclic
    over the sequences); 'full' = all live"""
    pad = torch.ones(B, L, dtype=torch.bool)
    if pattern == "full":
        return pad
    for b in range(B):
        k = b % 5
        if k == 1:
            pad[b, : L // 3] = False
        elif k == 2:
            pad[b, : L - 1] = False
        elif k == 3:
            pad[b] = False
        elif k == 4 and L > 2:
            pad[b, L // 2] = False
    return pad


def make_problem(B, L, head_dim, H, span, p=0.0, times="mixed", dtype=torch.int64, pad="mixed", seed=0, seed_eff=0x5EED,
                 ld_extra=0, device="cpu"):
    """The kernels' inputs, drawn so that a pair put in a wrong bucket moves its logit by O(1): adjacent table rows are
    independent, scaled 0.5; padded slot columns of the tables are zero, padded slot columns of q / dO are finite.  q, q_in,
    dO and the tables have ``ld_extra`` columns beyond H * 64 (the GPU tests fill them with NaN)."""
    g = torch.Generator().manual_seed(seed)
    T, d = B * L, H * SLOT
    Lp = (L + 63) // 64 * 64
    ld = d + ld_extra

    def rnd(*shape, s=1.0):
        return (torch.randn(*shape, generator=g) * s).to(torch.bfloat16)

    colmask = ((torch.arange(d) % SLOT) < head_dim)
    q, q_in, d_o = (torch.zeros(T, ld, dtype=torch.bfloat16) for _ in range(3))
    q[:, :d], q_in[:, :d], d_o[:, :d] = rnd(T, d), rnd(T, d), rnd(T, d)
    tk, tv = (torch.zeros(span + 1, ld, dtype=torch.bfloat16) for _ in range(2))
    tk[:, :d] = rnd(span + 1, d, s=0.5) * colmask.to(torch.bfloat16)
    tv[:, :d] = rnd(span + 1, d, s=0.5) * colmask.to(torch.bfloat16)
    S = torch.randn(B * H, Lp, Lp, generator=g) * 2.0
    dpd = rnd(B * H, Lp, Lp)
    tm = make_times(times, B, L, span, g, dtype)
    pm = make_pad(B, L, pad)
    P = Problem(q=q, q_in=q_in, d_o=d_o, times=tm, pad=pm, tk=tk, tv=tv, S=S, dpd=dpd, B=B, H=H, L=L, head_dim=head_dim,
                span=span, p=p, seed_eff=seed_eff, att_off=SITE_ATT, tk_off=SITE_TK, tv_off=SITE_TV, ldq=ld)
    return P


def to(P, device):
    """a copy of P with every tensor on ``device``"""
    kw = {k: (v.to(device) if torch.is_tensor(v) else v) for k, v in P.__dict__.items() if k not in ("Lp", "scale", "ks")}
    return Problem(**kw)


def ratio(got, ref, bound, mask=None):
    """max |got - ref| / bound (over ``mask``)"""
    e = (got.double() - ref).abs() / bound
    if mask is not None:
        e = e[mask]
    return float(e.max()) if e.numel() else 0.0
