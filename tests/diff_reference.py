"""float64 restatement of the DiffTransformer kernels (csrc/rp_diff.cu) at their own boundaries, with a per-element error
bound for every output, and the inputs the kernel tests draw.  The attention is computed one sequence at a time, its heads
batched, in closed form ([H, L, L] tensors at most), so B * H in the hundreds is affordable and the reference runs on
whichever device its inputs are on.  Every backward takes the kernel's own saves (bf16 e1 / e2, fp32 inv, O32, O2) as its
inputs, so each kernel is measured alone.

Notation, per head h of sequence b, query row i, key j <= i (n = i + 1 keys; visible: j == i or pad[j]):
  s_m = scale q_m . k_m (m = 1, 2; scale = fp32(1 / sqrt(hd)); q, k bf16 of the 64-wide slot, columns >= hd zero)
  M_m = max_{j visible} s_m,  e_m = exp(s_m - M_m) (0 where not visible),  Z_m = sum_j e_m,  inv_m = 1 / Z_m,
  A_m = e_m inv_m
  lambda = exp(lq1 . lk1) - exp(lq2 . lk2) + li    (li = fp32(lambda_init), E1 / E2 the two exponentials)
  A = A1 - lambda A2,  O = A V,  O2 = A2 V    (V bf16 [L, 2 hd] of the v_slot-wide slot)
  out = O r rs alpha,  r = 1 / sqrt(mean_c O^2 + eps) over the 2 hd true columns,  alpha = 1 - li
  backward, from the saves and dA: A_m = e_m' inv_m' (the kernel's rounded saves), r1 = sum_{j<=i} A1 dA,
  gw = dOn rs alpha,  r2 = r (gw . O2) - r^3 (gw . O)(O . O2) / (2 hd)  (= dO_pre . O2 with O, O2 the fp32 saves),
  dS1 = A1 (dA - r1) scale,  dS2 = -lambda A2 (dA - r2) scale,  A = A1 - lambda A2,  dlam_part = -r2
  dlambda_h = sum_{b, i} dlam_part;  g_q1 += dlambda E1 k1,  g_k1 += dlambda E1 q1,  g_q2 -= dlambda E2 k2,  g_k2 -= ... q2
RMSNorm over groups of G columns with n_true true ones: y = x r w alpha, r = 1 / sqrt(sum_G x^2 / n_true + eps);
  dx = r g - x r^3 (g . x) / n_true with g = dy w alpha;  dw += sum over items of dy x r alpha.
SwiGLU: u = silu(g) l;  dg = du l sig (1 + g (1 - sig)),  dl = du g sig,  sig = 1 / (1 + exp(-g)).

Error bounds (u = 2^-24; first order: every relative error below is under 1e-3, so second-order terms are below 1e-3 of
the bound and are dropped).  The library builds with --use_fast_math:
  - expf and __expf are ex2.approx of a rounded product: within 2 + 1.173 |z| fp32 ulps of exp(z) (CUDA programming
    guide), i.e. X(z) = 2 u (2 + 1.173 |z|) relative, and results below 2^-126 flush to zero (FLUSH absolute);
  - x / y and 1.f / y are approximate: within 2 ulps, DIV = 4 u relative;
  - rsqrtf is MUFU.RSQ: within 2 ulps, RSQ = 4 u relative.
A sequential fp32 sum of N terms (or an FMA chain of N steps) is within N u of the sum of |terms|; a warp's butterfly adds
5 levels.  bf16 outputs get half a bf16 ulp of |ref| + slack (HULP(|ref| + e)) plus the fp32 slack e.
  lambda (every kernel computes it the same way, one thread, index order):  the dot of hd fp32 products, product and add
      rounded apart:  e_s = 2 hd u sum |lq lk|;  E = exp(s):  e_E = E (e_s + X(s));  the difference and the li add:
          e_lambda = e_E1 + e_E2 + u |E1 - E2| + u |lambda|     (in terms of E1 + E2: lambda itself may cancel)
  Forward (rp_diff_attn_fwd).
    Logit.  hd bf16 x bf16 products (exact) in an FMA chain (hd + 1 steps at most, the odd width's extra column is
        0 x 0), times scale:  e_s = scale (hd + 1) u sum |q k| + u |s|.
    Row max.  The max of the rounded logits is within e_M = max_{j visible} e_s of the exact max.
    e (bf16, unnormalised).  s - M rounds once (u |z|, z = s - M), __expf adds X(z):  delta_j = e_s + u |z| + X(z) is the
        error of e_j besides the max's; stored:  HULP + e_j (delta_j + e_M) + FLUSH.
    inv (fp32).  The sum of n positives, ceil(n / 32) per lane and 5 butterfly levels (D = ceil(n / 32) + 5), the
        reciprocal DIV:  inv (sum_j A_j delta_j + e_M + D u + DIV).
    A_m (fp32, e inv rounded; the max's error cancels):  alpha_m = delta + sum_j A_j delta_j + (D + 1) u + DIV relative,
        plus FLUSH inv.
    A (fp32):  e_A = alpha_1 A1 + |lambda| (alpha_2 + 2 u) A2 + e_lambda A2 + u |A|   (in terms of A1 + |lambda| A2: A
        may cancel, e.g. lambda -> 1 with q2 = q1 and k2 = k1).
    O, O2 (fp32; the FMA chain over the n keys of row i):  e_O = sum_j e_A |V| + n u sum_j |A V|,
        e_O2 = sum_j alpha_2 A2 |V| + n u sum_j A2 |V|.  o_pre (bf16):  HULP + e_O.
    out (bf16).  rstd's own error: the sum of squares over v_slot columns (v_slot / 32 per lane + 5 levels + the square),
        the division by 2 hd, the eps add, then RSQ:  eps_r = (v_slot / 32 + 6 + 1) u / 2 + DIV / 2 + RSQ.  O's error
        passes through the norm's Jacobian (r' = r at mean(O^2) lowered by O's error):
          e_out = |rs| alpha (r' e_O,c + r'^3 |O_c| sum_k |O_k| e_O,k / (2 hd)) + |out| (eps_r + 4 u)
        (the products by rstd, rs and 1 - li, and 1 - li's own rounding).
  Softmax backward (rp_diff_attn_softmax_bwd).
    r1:  each term e1 inv1 dA rounded twice, D levels of sums:  e_r1 = (D + 2) u sum_j |A1 dA|.
    r2:  gw = dOn rs alpha (3 roundings with alpha's), sums over v_slot columns in D_v = v_slot / 32 + 5 levels:
        e_g2 = (D_v + 4) u sum |gw O2|,  e_gx = (D_v + 4) u sum |gw O|,  e_x2 = (D_v + 1) u sum |O O2|;  rstd as above
        (eps_r);  t1 = r g2 (one product), t2 = r^3 gx / (2 hd) x2 (four products and a division):
          e_r2 = r e_g2 + |t1| (eps_r + u) + r^3 / (2 hd) (e_gx |x2| + |gx| e_x2) + |t2| (3 eps_r + 4 u + DIV) + u |r2|
        Computing r2 from the bf16-rounded dO_pre instead would cost half a bf16 ulp of every dO_pre element, 2^15 u.
    dS1 (bf16):  HULP + scale A1 (e_r1 + u |dA - r1|) + 3 u |dS1|   (A1's product, the difference, the two products).
    dS2 (bf16):  HULP + scale |lambda| A2 (e_r2 + u |dA - r2|) + scale e_lambda A2 |dA - r2| + 4 u |dS2|.
    A (bf16):  HULP + u A1 + 2 u |lambda| A2 + e_lambda A2 + u |A|.   dlam_part (fp32):  e_r2.
  Lambda backward (rp_diff_lambda_bwd).  The partials of a head: ceil(B L / 256) per thread, then 8 tree levels:
      e_dl = (ceil(B L / 256) + 8) u sum |part|;  g_q1 = dl E1 k1 in two products:
      e_g = |E k| e_dl + |dl k| e_E + 2 u |dl E k|,  and u |result| for the add onto the start value.
  RMSNorm forward (rp_rmsnorm_fwd).  eps_r = (G / 32 + 6 + 1) u / 2 + DIV / 2 + RSQ;  y (bf16): HULP + |y| (eps_r + 3 u)
      (the products by rstd, w and alpha).
  RMSNorm backward (rp_rmsnorm_bwd).  g = dy w alpha (2 roundings);  dot = g . x:  e_dot = (G / 32 + 5 + 3) u sum |g x|;
      k = r^3 dot / n_true (three products, DIV):  e_k = r^3 e_dot / n_true + |k| (3 eps_r + 3 u + DIV);
      dx (bf16):  HULP + |r g| (eps_r + 3 u) + |x| e_k + u |x k| + u |dx|.
      dw: each term dy x (exact) r alpha:  (eps_r + 2 u) |term|;  warp w sums its C_w <= C items in order, then the 1024
      partials are summed as 8 strided chains of 128 and the 8 chain sums are added onto the start value in order:
          e_dw = (eps_r + (C + 130) u) sum |terms| + 8 u (|start| + sum |terms|) + u |result|.
  SwiGLU (rp_swiglu_fwd / _bwd).  E = exp(-g):  e_E = E X(g) + FLUSH;  1 + E: e_1E = e_E + u (1 + E);
      sig and silu (a DIV-approximate quotient):  eps_sig = e_1E / (1 + E) + DIV;
      u (bf16):  HULP + |u| (eps_sig + u) + FLUSH (1 + |l|);
      dl (bf16):  HULP + |du g| sig eps_sig + u |dl| + FLUSH;
      dg (bf16):  1 - sig:  e_om = sig eps_sig + u |1 - sig|;  T = 1 + g (1 - sig):
          e_T = |g| e_om + u |g (1 - sig)| + u |T|;
          HULP + |du l| (sig e_T + |T| sig eps_sig) + 2 u |dg| + FLUSH (1 + |T|).
      Below g = -88 (ln FLT_MAX = 88.72, less __expf's error) exp(-g) may overflow: the kernel's sig and silu become 0,
      so the bound there also admits |ref| (the references are below 1e-36 there).
Every bound gets FLOOR = 1e-30 on top, so that an exact zero compares against an exact zero."""
import math

import numpy as np
import torch

from tisasrec_reference import FLOOR, U, bf16_bound, f32, ratio  # noqa: F401  (ratio is part of this module's interface)
from tisasrec_reference import table_bound as accum_bound  # noqa: F401  (an increment's bound after the add onto a start)

FLUSH = 2.0 ** -126
DIV = 4 * U
RSQ = 4 * U
SLOT = 64               # kQkSlot: q1 / q2 / k1 / k2 slot width
MAX_L = 256
BWD_WARPS_PER_SM = 128  # rp_diff_attn_softmax_bwd: at most SMs * 16 blocks of 8 warps, one row per warp at a time
RMS_PARTS = 1024        # kRmsParts: per-warp weight-gradient partials of rp_rmsnorm_bwd
GRID_PER_SM = 16 * 256  # rp_swiglu_*: at most SMs * 16 blocks of 256 threads, one element per thread at a time
OVERFLOW_G = -88.0
RMS_EPS = float(np.finfo(np.float32).eps)


def exp_err(z):
    """relative error of __expf at argument z"""
    return 2 * U * (2 + 1.173 * z.abs())


def lp_of(L):
    return (L + 63) // 64 * 64


def v_slot_of(hd):
    return 64 if hd <= 32 else 128


# ------------------------------------------------------------------------------------------------ lambda
def lambda_ref(lq1, lk1, lq2, lk2, li):
    """head_lambda for every head: dict of float64 [H] tensors lam, E1, E2 and their bounds e_lam, e_E1, e_E2"""
    hd = lq1.shape[-1]
    out = {}
    for m, (a, b) in ((1, (lq1, lk1)), (2, (lq2, lk2))):
        p = a.double() * b.double()
        s = p.sum(-1)
        E = torch.exp(s)
        out[f"E{m}"] = E
        out[f"e_E{m}"] = E * (2 * hd * U * p.abs().sum(-1) + exp_err(s))
    out["lam"] = out["E1"] - out["E2"] + f32(li)
    out["e_lam"] = out["e_E1"] + out["e_E2"] + U * (out["E1"] - out["E2"]).abs() + U * out["lam"].abs()
    return out


# ------------------------------------------------------------------------------------------------ problem description
class Attn:
    """The attention kernels' inputs (torch tensors on one device) and scalars.  qkv bf16 [B*L, ld] in the engine's
    layout: q at q_c0 + h * 128 (q1 | q2, 64 columns each), k at k_c0 + h * 128, v at v_c0 + h * VS; pad bool [B, L];
    lq1 / lk1 / lq2 / lk2 fp32 [H, hd]; rs fp32 [VS] (zero past 2 hd); li the block's lambda_init."""

    def __init__(self, **kw):
        self.__dict__.update(kw)
        self.Lp = lp_of(self.L)
        self.VS = v_slot_of(self.hd)
        self.scale = f32(1.0 / math.sqrt(self.hd))

    def heads(self, b):
        """(q [H, 2, L, hd], k [H, 2, L, hd], v [H, L, 2 hd]) float64 of sequence b"""
        H, L, hd, VS = self.H, self.L, self.hd, self.VS
        X = self.qkv[b * L:(b + 1) * L].double()
        q = X[:, self.q_c0:self.q_c0 + H * 2 * SLOT].reshape(L, H, 2, SLOT)[..., :hd].permute(1, 2, 0, 3)
        k = X[:, self.k_c0:self.k_c0 + H * 2 * SLOT].reshape(L, H, 2, SLOT)[..., :hd].permute(1, 2, 0, 3)
        v = X[:, self.v_c0:self.v_c0 + H * VS].reshape(L, H, VS)[..., :2 * hd].permute(1, 0, 2)
        return q, k, v

    def visible(self, b):
        L, dev = self.L, self.qkv.device
        causal = torch.ones(L, L, dtype=torch.bool, device=dev).tril()
        eye = torch.eye(L, dtype=torch.bool, device=dev)
        return causal & (self.pad[b].to(dev)[None, :] | eye)

    def lam(self):
        return lambda_ref(self.lq1, self.lk1, self.lq2, self.lk2, self.li)


def _rows_n(L, dev):
    n = torch.arange(1, L + 1, device=dev, dtype=torch.float64)[:, None]
    return n, torch.ceil(n / 32) + 5


def _heads_to_rows(x, VS):
    """[H, L, w] -> [L, H * VS] (columns past w zero)"""
    H, L, w = x.shape
    out = torch.zeros(L, H, VS, dtype=x.dtype, device=x.device)
    out[..., :w] = x.permute(1, 0, 2)
    return out.reshape(L, H * VS)


def _rows_to_heads(x, L, H, VS):
    """[L, >= H * VS] -> [H, L, VS]"""
    return x[:, :H * VS].double().reshape(L, H, VS).permute(1, 0, 2)


def forward(P, visible=None, lam=None, alpha=None):
    """Reference and bounds of rp_diff_attn_fwd.  Returns float64 tensors: e1, e2, A1, A2, A [B*H, L, L], inv1, inv2
    [B*H, L], out, o_pre, O32, O2 [B*L, H*VS] (padded columns zero) and a ``<name>_b`` bound for each kernel output.
    ``visible`` (callable b -> [L, L] bool), ``lam`` (dict as lambda_ref) and ``alpha`` restate a kernel with another
    mask, lambda or output scale (the mutation tests)."""
    B, H, L, hd, VS = P.B, P.H, P.L, P.hd, P.VS
    dev = P.qkv.device
    lam = P.lam() if lam is None else lam
    lv, el = lam["lam"][:, None, None], lam["e_lam"][:, None, None]
    alpha = 1.0 - f32(P.li) if alpha is None else alpha
    eps = f32(P.eps)
    rs = P.rs[:2 * hd].double()
    n, D = _rows_n(L, dev)
    nc = 2 * hd
    eps_r = 0.5 * ((VS / 32 + 7) * U + DIV) + RSQ
    z3 = lambda: torch.zeros(B * H, L, L, dtype=torch.float64, device=dev)  # noqa: E731
    z2 = lambda: torch.zeros(B * H, L, dtype=torch.float64, device=dev)  # noqa: E731
    zr = lambda: torch.zeros(B * L, H * VS, dtype=torch.float64, device=dev)  # noqa: E731
    out = {k: z3() for k in ("e1", "e2", "e1_b", "e2_b", "A1", "A2", "A")}
    out.update({k: z2() for k in ("inv1", "inv2", "inv1_b", "inv2_b")})
    out.update({k: zr() for k in ("out", "out_b", "o_pre", "o_pre_b", "O32", "O32_b", "O2", "O2_b")})
    for b in range(B):
        q, k, v = P.heads(b)
        vis = (P.visible(b) if visible is None else visible(b))[None]
        bz = slice(b * H, (b + 1) * H)
        rows = slice(b * L, (b + 1) * L)
        Am, al = [], []
        for m in (0, 1):
            s = q[:, m] @ k[:, m].transpose(-1, -2) * P.scale
            sa = q[:, m].abs() @ k[:, m].abs().transpose(-1, -2) * P.scale
            es = (hd + 1) * U * sa + U * s.abs()
            M = s.masked_fill(~vis, -math.inf).amax(-1, keepdim=True)
            eM = es.masked_fill(~vis, 0).amax(-1, keepdim=True)
            z = (s - M).masked_fill(~vis, 0)
            e = torch.exp(z) * vis
            delta = (es + U * z.abs() + exp_err(z)) * vis
            Z = e.sum(-1, keepdim=True)
            A = e / Z
            sd = (A * delta).sum(-1, keepdim=True)
            out[f"e{m + 1}"][bz], out[f"e{m + 1}_b"][bz] = e, bf16_bound(e, e * (delta + eM) + FLUSH * vis)
            out[f"inv{m + 1}"][bz] = 1 / Z[..., 0]
            out[f"inv{m + 1}_b"][bz] = (1 / Z * (sd + eM + D * U + DIV))[..., 0] + FLOOR
            out[f"A{m + 1}"][bz] = A
            Am.append(A)
            al.append((delta + sd + (D + 1) * U + DIV) * A + FLUSH / Z * vis)
        A1, A2 = Am
        A = A1 - lv * A2
        out["A"][bz] = A
        eA = al[0] + lv.abs() * (al[1] + 2 * U * A2) + el * A2 + U * A.abs()
        O, O2 = A @ v, A2 @ v
        eO = eA @ v.abs() + n * U * (A.abs() @ v.abs())
        eO2 = al[1] @ v.abs() + n * U * (A2 @ v.abs())
        ms = O.pow(2).mean(-1, keepdim=True)
        r = 1 / torch.sqrt(ms + eps)
        oe = (O.abs() * eO).sum(-1, keepdim=True)
        dms = (2 * oe + eO.pow(2).sum(-1, keepdim=True)) / nc
        rh = 1 / torch.sqrt((ms - dms).clamp_min(0) + eps)
        y = O * r * rs * alpha
        ey = rs.abs() * alpha * (rh * eO + rh ** 3 * O.abs() * oe / nc) + y.abs() * (eps_r + 4 * U)
        for name, val, bound in (("out", y, bf16_bound(y, ey)), ("o_pre", O, bf16_bound(O, eO)), ("O32", O, eO + FLOOR),
                                 ("O2", O2, eO2 + FLOOR)):
            out[name][rows] = _heads_to_rows(val, VS)
            out[name + "_b"][rows] = _heads_to_rows(bound, VS) + FLOOR
    return out


def softmax_bwd(P, e1, e2, inv1, inv2, dA, d_on, o32, o2, lam=None):
    """Reference and bounds of rp_diff_attn_softmax_bwd on the kernel's inputs (e1 / e2 / dA [B*H, Lp, Lp], inv [B*H, Lp],
    d_on / o32 / o2 [B*L, >= H*VS]).  Returns float64 dS1, dS2, A, A1, A2 [B*H, L, L] and dlam [B*H, L] with bounds
    (``<name>_b``)."""
    B, H, L, hd, VS = P.B, P.H, P.L, P.hd, P.VS
    dev = e1.device
    lam = P.lam() if lam is None else lam
    lv, el = lam["lam"][:, None, None], lam["e_lam"][:, None, None]
    alpha = 1.0 - f32(P.li)
    eps = f32(P.eps)
    rs = P.rs[:VS].double()
    n, D = _rows_n(L, dev)
    nc = 2 * hd
    Dv = VS / 32 + 5
    eps_r = 0.5 * ((VS / 32 + 7) * U + DIV) + RSQ
    causal = torch.ones(L, L, dtype=torch.bool, device=dev).tril()
    out = {k: torch.zeros(B * H, L, L, dtype=torch.float64, device=dev)
           for k in ("dS1", "dS2", "A", "A1", "A2", "dS1_b", "dS2_b", "A_b")}
    out["dlam"] = torch.zeros(B * H, L, dtype=torch.float64, device=dev)
    out["dlam_b"] = torch.zeros_like(out["dlam"])
    for b in range(B):
        bz = slice(b * H, (b + 1) * H)
        rows = slice(b * L, (b + 1) * L)
        A1 = e1[bz, :L, :L].double() * inv1[bz, :L, None].double()
        A2 = e2[bz, :L, :L].double() * inv2[bz, :L, None].double()
        g = dA[bz, :L, :L].double()
        t1 = A1 * g * causal
        r1 = t1.sum(-1, keepdim=True)
        e_r1 = (D + 2) * U * t1.abs().sum(-1, keepdim=True)
        x, x2v, don = (_rows_to_heads(t[rows], L, H, VS) for t in (o32, o2, d_on))
        gw = don * rs * alpha
        ss = x.pow(2).sum(-1, keepdim=True)
        gx, g2, x2 = ((p * q).sum(-1, keepdim=True) for p, q in ((gw, x), (gw, x2v), (x, x2v)))
        e_g2 = (Dv + 4) * U * (gw * x2v).abs().sum(-1, keepdim=True)
        e_gx = (Dv + 4) * U * (gw * x).abs().sum(-1, keepdim=True)
        e_x2 = (Dv + 1) * U * (x * x2v).abs().sum(-1, keepdim=True)
        r = 1 / torch.sqrt(ss / nc + eps)
        tt1, tt2 = r * g2, r ** 3 * gx * x2 / nc
        r2 = tt1 - tt2
        e_r2 = (r * e_g2 + tt1.abs() * (eps_r + U) + r ** 3 / nc * (e_gx * x2.abs() + gx.abs() * e_x2)
                + tt2.abs() * (3 * eps_r + 4 * U + DIV) + U * r2.abs())
        dS1 = A1 * (g - r1) * P.scale
        dS2 = -lv * A2 * (g - r2) * P.scale
        A = A1 - lv * A2
        out["A1"][bz], out["A2"][bz] = A1, A2
        out["dS1"][bz] = dS1
        out["dS1_b"][bz] = bf16_bound(dS1, P.scale * A1 * (e_r1 + U * (g - r1).abs()) + 3 * U * dS1.abs())
        out["dS2"][bz] = dS2
        out["dS2_b"][bz] = bf16_bound(dS2, P.scale * lv.abs() * A2 * (e_r2 + U * (g - r2).abs())
                                      + P.scale * el * A2 * (g - r2).abs() + 4 * U * dS2.abs())
        out["A"][bz] = A
        out["A_b"][bz] = bf16_bound(A, U * A1 + 2 * U * lv.abs() * A2 + el * A2 + U * A.abs())
        out["dlam"][bz] = -r2[..., 0]
        out["dlam_b"][bz] = e_r2[..., 0] + FLOOR
    return out


def lambda_bwd(dlam_part, B, H, L, lq1, lk1, lq2, lk2, li):
    """Reference of rp_diff_lambda_bwd's increments on the kernel's partials (fp32 [B*H, Lp]): dict of dl [H] and the
    four increments g_q1, g_k1, g_q2, g_k2 [H, hd] with their bounds (before the add onto a start value)"""
    lam = lambda_ref(lq1, lk1, lq2, lk2, li)
    part = dlam_part.double().reshape(B, H, -1)[:, :, :L]
    dl = part.sum((0, 2))
    e_dl = (math.ceil(B * L / 256) + 8) * U * part.abs().sum((0, 2))
    out = {"dl": dl}
    for name, E, eE, other, sign in (("q1", "E1", "e_E1", lk1, 1), ("k1", "E1", "e_E1", lq1, 1),
                                     ("q2", "E2", "e_E2", lk2, -1), ("k2", "E2", "e_E2", lq2, -1)):
        Ev, eEv, o = lam[E][:, None], lam[eE][:, None], other.double()
        g = sign * dl[:, None] * Ev * o
        out["g_" + name] = g
        out["g_" + name + "_b"] = (Ev * o).abs() * e_dl[:, None] + (dl[:, None] * o).abs() * eEv + 2 * U * g.abs()
    return out


# ------------------------------------------------------------------------------------------------ the attention stage
def attention_stage(QKV, dOn, pad, lq1, lk1, lq2, lk2, rs, li, H, hd, eps=1e-5):
    """One block's attention forward and backward in float64 from the engine's QKV (q | k | v in the padded layout) and
    dOn (the gradient of the normalised output, [B*L, H*VS]): On, O_pre [B*L, H*VS], dQKV [B*L, n_qkv] and the
    gradients of rs [2 hd] and lambda_q1 / k1 / q2 / k2 [H, hd]."""
    B, L = pad.shape
    VS = v_slot_of(hd)
    dev = QKV.device
    P = Attn(qkv=QKV, q_c0=0, k_c0=H * 2 * SLOT, v_c0=H * 4 * SLOT, pad=pad, lq1=lq1, lk1=lk1, lq2=lq2, lk2=lk2, li=li,
             rs=rs, eps=eps, B=B, H=H, L=L, hd=hd)
    lam = P.lam()
    lv = (lam["lam"] - f32(li) + li)[:, None, None]
    alpha = 1.0 - li
    rsd = rs[:2 * hd].double()
    nc = 2 * hd
    res = {k: torch.zeros(B * L, H * VS, dtype=torch.float64, device=dev) for k in ("On", "Opre")}
    dQKV = torch.zeros(B * L, QKV.shape[1], dtype=torch.float64, device=dev)
    d_rs = torch.zeros(2 * hd, dtype=torch.float64, device=dev)
    dl = torch.zeros(H, dtype=torch.float64, device=dev)
    for b in range(B):
        q, k, v = P.heads(b)
        vis = P.visible(b)[None]
        rows = slice(b * L, (b + 1) * L)
        A12 = []
        for m in (0, 1):
            s = (q[:, m] @ k[:, m].transpose(-1, -2) / math.sqrt(hd)).masked_fill(~vis, -math.inf)
            A12.append(torch.softmax(s, -1))
        A1, A2 = A12
        A = A1 - lv * A2
        O = A @ v
        r = 1 / torch.sqrt(O.pow(2).mean(-1, keepdim=True) + eps)
        res["Opre"][rows] = _heads_to_rows(O, VS)
        res["On"][rows] = _heads_to_rows(O * r * rsd * alpha, VS)
        don = _rows_to_heads(dOn[rows], L, H, VS)[..., :nc]
        d_rs += (don * O * r * alpha).sum((0, 1))
        g = don * rsd * alpha
        dO = r * g - O * r ** 3 * (g * O).sum(-1, keepdim=True) / nc
        dAm = dO @ v.transpose(-1, -2)
        dv = A.transpose(-1, -2) @ dO
        dl -= (A2 * dAm).sum((1, 2))
        dS1 = A1 * (dAm - (A1 * dAm).sum(-1, keepdim=True)) / math.sqrt(hd)
        dS2 = -lv * A2 * (dAm - (A2 * dAm).sum(-1, keepdim=True)) / math.sqrt(hd)
        blk = dQKV[rows]
        for h in range(H):
            for m, dS in ((0, dS1), (1, dS2)):
                c = h * 2 * SLOT + m * SLOT
                blk[:, c:c + hd] = dS[h] @ k[h, m]
                blk[:, H * 2 * SLOT + c:H * 2 * SLOT + c + hd] = dS[h].T @ q[h, m]
            blk[:, H * 4 * SLOT + h * VS:H * 4 * SLOT + h * VS + nc] = dv[h]
    res["dQKV"] = dQKV
    res["d_rs"] = d_rs
    res["dl"] = dl
    res["d_q1"] = dl[:, None] * lam["E1"][:, None] * lk1.double()
    res["d_k1"] = dl[:, None] * lam["E1"][:, None] * lq1.double()
    res["d_q2"] = -dl[:, None] * lam["E2"][:, None] * lk2.double()
    res["d_k2"] = -dl[:, None] * lam["E2"][:, None] * lq2.double()
    return res


# ------------------------------------------------------------------------------------------------ RMSNorm
def rms_rows(n_rows, n_rows_dev, gather, dev):
    """the (output row, input row) pairs the kernels process"""
    rows = n_rows if n_rows_dev is None else max(0, min(n_rows, n_rows_dev))
    out = torch.arange(rows, device=dev)
    return out, (out if gather is None else gather[:rows].to(dev).long())


def rmsnorm_fwd(x, w, eps, alpha, n_rows, d, G, n_true, n_rows_dev=None, gather=None):
    """-> (y [rows, d] float64 for the processed output rows, its bound, the output row indices)"""
    dev = x.device
    orow, src = rms_rows(n_rows, n_rows_dev, gather, dev)
    X = x[src].double().reshape(-1, d // G, G)
    W = w[:G].double()
    r = 1 / torch.sqrt(X.pow(2).sum(-1, keepdim=True) / n_true + f32(eps))
    y = X * r * W * f32(alpha)
    eps_r = 0.5 * ((G / 32 + 7) * U + DIV) + RSQ
    return y.reshape(-1, d), bf16_bound(y, y.abs() * (eps_r + 3 * U)).reshape(-1, d), orow


def rmsnorm_bwd(dy, x, w, eps, alpha, n_rows, d, G, n_true, n_rows_dev=None, gather=None):
    """-> dict: dx [rows, d] float64 and its bound at input rows ``src``; the weight-gradient increment dw [G], the sum of
    |terms| dw_abs [G], the per-warp partials dw_parts [1024, G], and the largest item count of a warp"""
    dev = x.device
    orow, src = rms_rows(n_rows, n_rows_dev, gather, dev)
    rows = orow.numel()
    X = x[src].double().reshape(rows, d // G, G)
    Dy = dy[orow].double().reshape(rows, d // G, G)
    W = w[:G].double()
    a = f32(alpha)
    r = 1 / torch.sqrt(X.pow(2).sum(-1, keepdim=True) / n_true + f32(eps))
    eps_r = 0.5 * ((G / 32 + 7) * U + DIV) + RSQ
    g = Dy * W * a
    dot = (g * X).sum(-1, keepdim=True)
    e_dot = (G / 32 + 8) * U * (g * X).abs().sum(-1, keepdim=True)
    kk = r ** 3 * dot / n_true
    e_k = r ** 3 * e_dot / n_true + kk.abs() * (3 * eps_r + 3 * U + DIV)
    dx = r * g - X * kk
    e_dx = (r * g).abs() * (eps_r + 3 * U) + X.abs() * e_k + U * (X * kk).abs() + U * dx.abs()
    terms = (Dy * X * r * a).reshape(-1, G)   # item it = row * groups + group
    items = terms.shape[0]
    warp = torch.arange(items, device=dev) % RMS_PARTS
    parts = torch.zeros(RMS_PARTS, G, dtype=torch.float64, device=dev).index_add_(0, warp, terms)
    cmax = -(-items // RMS_PARTS) if items else 0
    tabs = terms.abs().sum(0)
    return {"dx": dx.reshape(rows, d), "dx_b": bf16_bound(dx, e_dx).reshape(rows, d), "src": src, "dw": terms.sum(0),
            "dw_abs": tabs, "dw_parts": parts, "dw_inc_b": (eps_r + (cmax + 130) * U) * tabs}


def dw_bound(ref, start):
    """the bound of rp_rmsnorm_bwd's dw after the add onto ``start``"""
    s = start.double()
    return ref["dw_inc_b"] + 8 * U * (s.abs() + ref["dw_abs"]) + U * (s + ref["dw"]).abs() + FLOOR


# ------------------------------------------------------------------------------------------------ SwiGLU
def _sig(g):
    E = torch.exp(-g)
    e1E = E * exp_err(g) + FLUSH + U * (1 + E)
    sig = 1 / (1 + E)
    return sig, e1E / (1 + E) + DIV


def swiglu_fwd(gl, n, F):
    """-> (u [n, F] float64, bound)"""
    g, l = gl[:n, :F].double(), gl[:n, F:2 * F].double()
    sig, eps = _sig(g)
    u = g * sig * l
    e = u.abs() * (eps + U) + FLUSH * (1 + l.abs()) + torch.where(g < OVERFLOW_G, u.abs(), torch.zeros_like(u))
    return u, bf16_bound(u, e)


def swiglu_bwd(du, gl, n, F, with_silu_slope=True):
    """-> (dgl [n, 2F] float64, bound).  ``with_silu_slope`` False restates a kernel that drops g (1 - sig)."""
    g, l = gl[:n, :F].double(), gl[:n, F:2 * F].double()
    d = du[:n, :F].double()
    sig, eps = _sig(g)
    esig = sig * eps
    om = 1 - sig
    T = 1 + g * om if with_silu_slope else torch.ones_like(g)
    e_T = g.abs() * (esig + U * om.abs()) + U * (g * om).abs() + U * T.abs()
    dg = d * l * sig * T
    dl = d * g * sig
    ovf = g < OVERFLOW_G
    e_dg = (d * l).abs() * (sig * e_T + T.abs() * esig) + 2 * U * dg.abs() + FLUSH * (1 + T.abs())
    e_dl = (d * g).abs() * esig + U * dl.abs() + FLUSH
    e_dg = e_dg + torch.where(ovf, dg.abs(), torch.zeros_like(dg))
    e_dl = e_dl + torch.where(ovf, dl.abs(), torch.zeros_like(dl))
    return torch.cat([dg, dl], 1), torch.cat([bf16_bound(dg, e_dg), bf16_bound(dl, e_dl)], 1)


# ------------------------------------------------------------------------------------------------ inputs
PAD_KINDS = ("all", "last", "none", "left", "holes")


def make_pad(B, L, kind, g):
    """bool [B, L]: all live, only the last token live, none live, left-padded with random lengths, random holes"""
    if kind == "all":
        return torch.ones(B, L, dtype=torch.bool)
    if kind == "last":
        pm = torch.zeros(B, L, dtype=torch.bool)
        pm[:, -1] = True
        return pm
    if kind == "none":
        return torch.zeros(B, L, dtype=torch.bool)
    if kind == "left":
        lens = torch.randint(0, L + 1, (B,), generator=g)
        return torch.arange(L)[None, :] >= (L - lens)[:, None]
    if kind == "holes":
        return torch.rand(B, L, generator=g) < 0.7
    raise ValueError(kind)


def lambda_params(H, hd, lam_target, li, g):
    """fp32 [H, hd] lambda_q1, _k1, _q2, _k2 with lambda of head h near lam_target + 0.05 h: lq1 . lk1 = 0.5 and
    lq2 . lk2 = log(e^0.5 - (lambda - li))"""
    lams = torch.tensor(lam_target, dtype=torch.float64) + 0.05 * torch.arange(H, dtype=torch.float64)
    lq1 = torch.randn(H, hd, generator=g, dtype=torch.float64) * 0.3
    lk1 = 0.5 * lq1 / (lq1 * lq1).sum(-1, keepdim=True)
    bt = torch.log(math.exp(0.5) - (lams - li))
    lq2 = torch.randn(H, hd, generator=g, dtype=torch.float64) * 0.3
    lk2 = lq2 * (bt / (lq2 * lq2).sum(-1))[:, None]
    return tuple(t.float() for t in (lq1, lk1, lq2, lk2))


def make_attn(B, L, hd, H, pad="holes", lam_target=0.3, li=0.2, qk_std=1.0, identical=False, seed=0, ld_extra=8,
              rs_std=0.25, device="cpu"):
    """Attention inputs in the engine's layout: qkv bf16 [B*L, H * (256 + VS) + ld_extra] (slot padding zero, the extra
    columns zero here: the GPU tests fill them with NaN), pad, lambda parameters aimed at lam_target, rs around 1.
    qk_std scales q and k (|logit| ~ qk_std^2); identical: q2 = q1 and k2 = k1."""
    g = torch.Generator().manual_seed(seed)
    VS = v_slot_of(hd)
    T, n_qkv = B * L, H * (4 * SLOT + VS)
    qkv = torch.zeros(T, n_qkv + ld_extra)
    for c0 in (0, H * 2 * SLOT):
        x = torch.randn(T, H, 2, hd, generator=g) * qk_std
        if identical:
            x[:, :, 1] = x[:, :, 0]
        blk = torch.zeros(T, H, 2, SLOT)
        blk[..., :hd] = x
        qkv[:, c0:c0 + H * 2 * SLOT] = blk.reshape(T, -1)
    vb = torch.zeros(T, H, VS)
    vb[..., :2 * hd] = torch.randn(T, H, 2 * hd, generator=g)
    qkv[:, H * 4 * SLOT:n_qkv] = vb.reshape(T, -1)
    rs = torch.zeros(VS)
    rs[:2 * hd] = 1 + rs_std * torch.randn(2 * hd, generator=g)
    lq1, lk1, lq2, lk2 = lambda_params(H, hd, lam_target, li, g)
    P = Attn(qkv=qkv.to(torch.bfloat16), q_c0=0, k_c0=H * 2 * SLOT, v_c0=H * 4 * SLOT, pad=make_pad(B, L, pad, g),
             lq1=lq1, lk1=lk1, lq2=lq2, lk2=lk2, li=li, rs=rs, eps=1e-5, B=B, H=H, L=L, hd=hd, n_qkv=n_qkv,
             ld=n_qkv + ld_extra)
    return to(P, device)


def to(P, device):
    kw = {k: (v.to(device) if torch.is_tensor(v) else v) for k, v in P.__dict__.items() if k not in ("Lp", "VS", "scale")}
    return Attn(**kw)


def bwd_inputs(P, fwd, seed=1):
    """softmax-backward inputs from forward saves (dict of e1, e2, inv1, inv2 [B*H, Lp(, Lp)], o32, o2 [B*L, >= H*VS],
    any dtype): random dA (bf16 [B*H, Lp, Lp]) and d_on (bf16 [B*L, ld] with ld = H*VS + 8, padded columns zero)"""
    g = torch.Generator().manual_seed(seed)
    B, H, L, Lp, VS, hd = P.B, P.H, P.L, P.Lp, P.VS, P.hd
    dA = torch.randn(B * H, Lp, Lp, generator=g).to(torch.bfloat16)
    don = torch.zeros(B * L, H, VS)
    don[..., :2 * hd] = torch.randn(B * L, H, 2 * hd, generator=g)
    d_on = torch.zeros(B * L, H * VS + 8)
    d_on[:, :H * VS] = don.reshape(B * L, -1)
    return dA.to(P.qkv.device), d_on.to(torch.bfloat16).to(P.qkv.device)


def saves_from_reference(P, ref):
    """the forward's saves in the kernel's layout and dtypes, rounded from the reference (CPU tests)"""
    B, H, L, Lp, VS = P.B, P.H, P.L, P.Lp, P.VS
    dev = ref["e1"].device
    s = {}
    for k in ("e1", "e2"):
        t = torch.zeros(B * H, Lp, Lp, dtype=torch.float64, device=dev)
        t[:, :L, :L] = ref[k]
        s[k] = t.to(torch.bfloat16)
    for k in ("inv1", "inv2"):
        t = torch.zeros(B * H, Lp, dtype=torch.float64, device=dev)
        t[:, :L] = ref[k]
        s[k] = t.float()
    for k in ("O32", "O2"):
        t = torch.zeros(B * L, H * VS + 8, dtype=torch.float64, device=dev)
        t[:, :H * VS] = ref[k]
        s[k.lower()] = t.float()
    return s


def make_rms(rows, d, G, n_true_kind, seed=0, zero_row=None):
    """RMSNorm inputs: x bf16 [rows, d] and w fp32 [G] (zero in the padded columns), dy bf16 [rows, d] (random in every
    column) and n_true.  n_true_kind: "one" (column 0 of each group), "full", or "slots" (the first 50 of every 64
    columns, or 100 of every 128 for a group of 128 or more)."""
    g = torch.Generator().manual_seed(seed)
    if isinstance(n_true_kind, int):
        mask = torch.arange(G) < n_true_kind
    elif n_true_kind == "one":
        mask = torch.arange(G) < 1
    elif n_true_kind == "full":
        mask = torch.ones(G, dtype=torch.bool)
    else:
        slot, valid = (64, 50) if G == 64 else (128, 100)
        mask = (torch.arange(G) % slot) < valid
    x = torch.randn(rows, d // G, G, generator=g) * (0.5 + 2 * torch.rand(rows, d // G, 1, generator=g))
    x = (x * mask).reshape(rows, d)
    if zero_row is not None and rows > zero_row:
        x[zero_row] = 0
    w = (0.5 + torch.rand(G, generator=g)) * mask
    dy = torch.randn(rows, d, generator=g)
    return x.to(torch.bfloat16), w, dy.to(torch.bfloat16), int(mask.sum())


EDGE_GATES = (-100.0, -89.5, -89.0, -88.5, -88.0, -87.5, -87.0, -80.0, -20.0, -1.28125, 0.0, 1.28125, 20.0, 80.0, 87.5,
              88.0, 88.5, 89.0, 100.0)


def make_swiglu(n, F, seed=0, rows_extra=3):
    """gl bf16 [n + rows_extra, 2F]: gates N(0, 9), a quarter of them uniform in (-100, 100), plus every EDGE_GATES value;
    linear halves N(0, 1) with some scaled down to 1e-3; du bf16 [n + rows_extra, F]"""
    g = torch.Generator().manual_seed(seed)
    R = n + rows_extra
    gate = torch.randn(R, F, generator=g) * 3
    wide = torch.rand(R, F, generator=g) < 0.25
    gate = torch.where(wide, torch.rand(R, F, generator=g) * 200 - 100, gate)
    flat = gate.view(-1)
    k = min(len(EDGE_GATES), n * F)
    pos = torch.randperm(n * F, generator=g)[:k]
    flat[pos] = torch.tensor(EDGE_GATES[:k])
    lin = torch.randn(R, F, generator=g)
    lin = torch.where(torch.rand(R, F, generator=g) < 0.1, lin * 1e-3, lin)
    du = torch.randn(R, F, generator=g)
    return torch.cat([gate, lin], 1).to(torch.bfloat16), du.to(torch.bfloat16)
