"""Kernel-level tests of the four attention entry points of csrc/rp_attention.cu (rp_attn_fwd, the fused rp_attn_bwd,
rp_attn_softmax_bwd behind the un-fused backward, rp_attn_last) against a float64 restatement of masked multi-head
attention, at the tile, block and mask edges where the kernels change behaviour.

Layout as the engine calls them (engine.py SasRecEngine._attention_forward / _attention_backward, the rp_attn_last call of
_body_forward): Q is [T, d], K and V share one packed [T, 2d] array (k_c0 = 0, v_c0 = d), dK and dV go into one packed
array, H = 2 heads so head column offsets matter, and B >= 3 sequences so the 128-row tiles of sequence b run into the
rows of sequence b + 1 and the last sequence's tiles run past the end of the arrays.

Errors are measured per (sequence, head, 64-row block) - a norm relative to the reference block's norm - so that one
wrong 64-key chunk or 64-row block cannot hide in a global norm.  Run with -s to print the worst error of each family.
"""
import ctypes
import math
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from dropout_stream import drop_keep, keep_draws
from replay_b200._lib import AttnBwdDesc, AttnDesc, check, lib

LOG2E = 1.4426950408889634
SENT = -3.25            # sentinel for memory a kernel must not write (exact in bf16)
BIG = 300.0             # masked key rows hold +-BIG: a masked key that leaks into a max, a sum or P.V is a large error
SHARP = 5.6             # "sharp" scale = SHARP / sqrt(head_dim): logits * scale span about +-20
SEED, OFF, CTR = 0x5EED1234ABC, 3 << 40, 987654321   # dropout stream of the kernel-level tests (seed_ptr holds CTR)
P_DROP = 0.2

# Tolerances.  P, dS and Pd pass through bf16, so ~2^-9 relative error per element is expected.  Each bound is about 3x
# the worst error observed over every case of this file on one H100 80GB HBM3 (400 W power limit), and never looser than
# 1e-2 (norms) / 2e-2 (max-abs).  The inputs are seeded and the kernels deterministic, so the observed errors reproduce.
TOL_O = 1e-2            # O: per (b, h, 64-query block) ||O - O_ref|| / ||O_ref||; worst seen 3.1e-3
TOL_O_MAX = 1.1e-2      # O: max |O - O_ref| / max |V| over the visible keys; worst seen 3.7e-3
TOL_GRAD = 1e-2         # dQ / dK / dV: per (b, h, 64-row block) norm-relative error; worst seen 9.8e-3 (fused dK),
                        #   7.7e-3 (un-fused dK): dS is rounded to bf16 before the sums over queries / keys
TOL_GRAD_MAX = 2e-2     # dQ / dK / dV: max |g - g_ref| / max |g_ref|; worst seen 7.8e-3
TOL_LAST = 6.5e-3       # rp_attn_last: per (b, h) norm-relative error of the one output row; worst seen 2.1e-3
TOL_M_ABS, TOL_M_REL = 4e-5, 1e-5   # m_save (exp2 units); worst seen 1.1e-5 absolute
TOL_INV_REL = 1e-5      # inv_sum; worst seen 2.8e-6
BLOCK_FLOOR = 1e-4      # blocks whose reference is ~0 are compared absolutely at this RMS level
BF16_ROUND = 2.0 ** -8 * 1.005   # bf16 unit roundoff (round to nearest) + 0.5 % for ex2.approx and fp32 sums


def _ru(x, m):
    return (x + m - 1) // m * m


# ----------------------------------------------------------------------------------------------------------------------
# float64 reference
# ----------------------------------------------------------------------------------------------------------------------
def visibility(pad, L, causal, mask_pad_keys):
    """bool [B, 1, L, L]: key j is visible to query i iff j < L, pad[b, j] (if mask_pad_keys) and j <= i (if causal)."""
    vis = torch.ones(pad.shape[0], 1, L, L, dtype=torch.bool)
    if mask_pad_keys:
        vis = vis & pad.view(-1, 1, 1, L)
    if causal:
        vis = vis & torch.ones(L, L, dtype=torch.bool).tril()
    return vis


def _attn(q, k, v, vis, scale, keep=None):
    s = (q @ k.transpose(-1, -2)) * scale
    s = s.masked_fill(~vis, float("-inf"))
    has = vis.any(-1, keepdim=True)
    m = torch.where(has, s.detach().amax(-1, keepdim=True), torch.zeros((), dtype=s.dtype))
    e = torch.exp(s - m)
    den = e.sum(-1, keepdim=True)
    ok = den > 0
    inv = torch.where(ok, 1.0 / torch.where(ok, den, torch.ones_like(den)), torch.zeros_like(den))
    p = e * inv
    o = (p if keep is None else p * keep) @ v
    return o, (m * LOG2E).squeeze(-1), inv.squeeze(-1), e


def attn_ref(q, k, v, pad_mask, causal, mask_pad_keys, scale, keep=None):
    """Masked attention of [B, H, L, hd] float64 inputs.  Returns O [B, H, L, hd], the row max in exp2 units
    (max_j s_ij * scale * log2 e, 0 for a row with no visible key), 1 / row sum (0 for such a row) and the un-normalised
    exp(s - max) [B, H, L, L].  ``keep`` (0 or 1/(1-p)) multiplies the normalised P that multiplies V."""
    return _attn(q, k, v, visibility(pad_mask, q.shape[2], causal, mask_pad_keys), scale, keep)


def _attn_grads(q, k, v, vis, scale, keep, d_o):
    """O and fp64 autograd dQ, dK, dV for the output gradient ``d_o``."""
    q, k, v = (t.detach().clone().requires_grad_(True) for t in (q, k, v))
    o = _attn(q, k, v, vis, scale, keep)[0]
    o.backward(d_o)
    return o.detach(), q.grad, k.grad, v.grad


def attn_grads_given_o(q, k, v, vis, scale, keep, d_o, o):
    """dQ, dK, dV by the softmax-backward formula dS = P (dP * keep - delta) * scale, delta_i = sum_c dO_ic O_ic, with O
    an INPUT: the fused backward reads the forward's stored bf16 O, and where dP * keep and delta cancel (a row with one
    visible key has dS = 0 exactly) the rounding of O is the whole answer.  With the exact O this is autograd
    (test_grad_formula_matches_autograd)."""
    _, _, inv, e = _attn(q, k, v, vis, scale)
    p = e * inv[..., None]
    dp = d_o @ v.transpose(-1, -2)
    pd = p if keep is None else p * keep
    dp = dp if keep is None else dp * keep
    ds = p * (dp - (d_o * o).sum(-1, keepdim=True)) * scale
    return ds @ k, ds.transpose(-1, -2) @ q, pd.transpose(-1, -2) @ d_o


def block_err(got, ref, blk=64):
    """Largest norm-relative error over the (b, h, blk-row block)s of [B, H, L, D] arrays.  A block whose reference is
    ~0 is measured against an RMS floor of BLOCK_FLOOR instead."""
    B, H, L, D = ref.shape
    nb = -(-L // blk)
    pad = (0, 0, 0, nb * blk - L)
    diff = F.pad(got - ref, pad).reshape(B, H, nb, blk * D).norm(dim=-1)
    den = F.pad(ref, pad).reshape(B, H, nb, blk * D).norm(dim=-1)
    n = torch.tensor([min(blk, L - i * blk) * D for i in range(nb)], dtype=torch.float64)
    return float((diff / torch.maximum(den, BLOCK_FLOOR * n.sqrt())).max())


MODES = {"sasrec": (1, 1), "legacy": (1, 0), "bert": (0, 1), "none": (0, 0)}   # (causal, mask_pad_keys)


def _pad_pattern(L, bert=False, B=4, seed=0):
    """bool [B, L], True = real token.  0: full; 1: left padded, the first 128-row tile all padding when L > 128;
    2: one token; 3: all padding; BERT4Rec: interior holes in 0; more sequences: random holes."""
    pad = torch.ones(B, L, dtype=torch.bool)
    n_pad = min(L - 1, 128 + (L - 128) // 3) if L > 128 else L - max(1, L // 3)
    pad[1, :n_pad] = False
    pad[2, : L - 1] = False
    pad[3] = False
    if bert:
        pad[0, 5::7] = False
    g = torch.Generator().manual_seed(seed)
    for b in range(4, B):
        pad[b] = torch.rand(L, generator=g) > 0.3
    return pad


def _heads(x, B, L, H, hd):
    """[T, >= H*hd] -> float64 [B, H, L, hd]"""
    return x[:, : H * hd].double().reshape(B, L, H, hd).permute(0, 2, 1, 3)


def _case(pad, H, hd, mpk, seed, hd_true=None, dev=None):
    """Inputs on the engine's layout: q bf16 [T, d], kv bf16 [T, 2d]; with ``hd_true`` < hd the head columns
    [hd_true, hd) are zero (a padded head slot)."""
    B, L = pad.shape
    T, d = B * L, H * hd
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(T, d, generator=g)
    kv = torch.randn(T, 2 * d, generator=g)
    if mpk:
        sign = torch.randint(0, 2, (T, 1), generator=g).float() * 2 - 1
        kv = torch.where((~pad).reshape(T, 1), BIG * sign, kv)
    if hd_true is not None:
        cols = ((torch.arange(d) % hd) < hd_true).float()
        q, kv = q * cols, kv * torch.cat([cols, cols])
    q, kv = q.to(torch.bfloat16), kv.to(torch.bfloat16)
    c = SimpleNamespace(B=B, L=L, H=H, hd=hd, d=d, T=T, Lp=_ru(L, 64), pad=pad, q=q, kv=kv, hd_true=hd_true or hd)
    ht = c.hd_true
    c.q64 = _heads(q, B, L, H, hd)[..., :ht]
    c.k64 = _heads(kv[:, :d], B, L, H, hd)[..., :ht]
    c.v64 = _heads(kv[:, d:], B, L, H, hd)[..., :ht]
    if dev is not None:
        c.qd, c.kvd, c.padd = q.to(dev), kv.to(dev), pad.to(dev).contiguous()
    return c


def _d_out(c, seed):
    g = torch.Generator().manual_seed(seed)
    d_o = torch.randn(c.T, c.d, generator=g)
    d_o = d_o * ((torch.arange(c.d) % c.hd) < c.hd_true).float()
    return d_o.to(torch.bfloat16)


_WORST = {}


def _note(family, value):
    """Record the worst error of a family (and the case it came from) for the report printed at the end."""
    if float(value) >= _WORST.get(family, (0.0, ""))[0]:
        _WORST[family] = (float(value), os.environ.get("PYTEST_CURRENT_TEST", "").split("::")[-1].split(" ")[0])
    return value


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if _WORST:
        print("\nworst observed error per family:")
        for k, (v, case) in sorted(_WORST.items()):
            print(f"  {k:24s} {v:.3g}  {case}")


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda")


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ----------------------------------------------------------------------------------------------------------------------
# kernel calls
# ----------------------------------------------------------------------------------------------------------------------
def _attn_fwd(c, causal, mpk, scale, train=True, drop=0.0, ctr=None):
    """rp_attn_fwd -> (out [T, d + 64] with sentinel columns, p_save, inv_sum, m_save) (the last three None at
    inference).  p_save is zero-initialised; inv_sum / m_save start at -1 so that every row < L must be written."""
    B, L, H, hd, d, T, Lp, dev = c.B, c.L, c.H, c.hd, c.d, c.T, c.Lp, c.qd.device
    out = torch.full((T, d + 64), SENT, dtype=torch.bfloat16, device=dev)
    ad = AttnDesc()
    ad.q, ad.q_rows, ad.q_cols, ad.ldq, ad.q_c0 = c.qd.data_ptr(), T, d, d, 0
    ad.k, ad.k_rows, ad.k_cols, ad.ldk, ad.k_c0 = c.kvd.data_ptr(), T, 2 * d, 2 * d, 0
    ad.v, ad.v_rows, ad.v_cols, ad.ldv, ad.v_c0 = c.kvd.data_ptr(), T, 2 * d, 2 * d, d
    ad.B, ad.H, ad.L, ad.head_dim = B, H, L, hd
    ad.causal, ad.mask_pad_keys = causal, mpk
    ad.scale = scale
    ad.pad_mask = c.padd.data_ptr()
    ad.out, ad.ldo = out.data_ptr(), d + 64
    p_save = inv = m = None
    if train:
        p_save = torch.zeros(B * H, Lp, Lp, dtype=torch.bfloat16, device=dev)
        inv = torch.full((B * H, Lp), -1.0, device=dev)
        m = torch.full((B * H, Lp), -1.0, device=dev)
        ad.p_save, ad.inv_sum, ad.m_save = p_save.data_ptr(), inv.data_ptr(), m.data_ptr()
    ad.drop_p, ad.seed, ad.drop_off = drop, SEED, OFF
    ad.seed_ptr = None if ctr is None else ctr.data_ptr()
    check(lib().rp_attn_fwd(ctypes.byref(ad), _stream()), "rp_attn_fwd")
    torch.cuda.synchronize()
    return out, p_save, inv, m


def _attn_bwd(c, causal, mpk, scale, fwd, d_o, drop=0.0, ctr=None):
    """rp_attn_bwd on the forward's own O / m_save / inv_sum -> (dq [T + 64, d + 64], dkv [T + 64, 2d + 64]), both
    sentinel-filled outside what the kernel may write (64 rows past the last sequence, columns past the heads)."""
    B, L, H, hd, d, T, dev = c.B, c.L, c.H, c.hd, c.d, c.T, c.qd.device
    out, _, inv, m = fwd
    dq = torch.full((T + 64, d + 64), SENT, dtype=torch.bfloat16, device=dev)
    dkv = torch.full((T + 64, 2 * d + 64), SENT, dtype=torch.bfloat16, device=dev)
    bd = AttnBwdDesc()
    bd.q, bd.q_rows, bd.q_cols, bd.ldq, bd.q_c0 = c.qd.data_ptr(), T, d, d, 0
    bd.k, bd.k_rows, bd.k_cols, bd.ldk, bd.k_c0 = c.kvd.data_ptr(), T, 2 * d, 2 * d, 0
    bd.v, bd.v_rows, bd.v_cols, bd.ldv, bd.v_c0 = c.kvd.data_ptr(), T, 2 * d, 2 * d, d
    bd.d_out, bd.do_rows, bd.do_cols, bd.ld_do = d_o.data_ptr(), T, d, d
    bd.out, bd.ldo = out.data_ptr(), out.shape[1]
    bd.B, bd.H, bd.L, bd.head_dim = B, H, L, hd
    bd.causal, bd.mask_pad_keys = causal, mpk
    bd.scale = scale
    bd.pad_mask = c.padd.data_ptr()
    bd.m_save, bd.inv_sum = m.data_ptr(), inv.data_ptr()
    bd.dq, bd.ld_dq, bd.dq_c0 = dq.data_ptr(), d + 64, 0
    bd.dk, bd.ld_dk, bd.dk_c0 = dkv.data_ptr(), 2 * d + 64, 0
    bd.dv, bd.ld_dv, bd.dv_c0 = dkv.data_ptr(), 2 * d + 64, d
    bd.drop_p, bd.seed, bd.drop_off = drop, SEED, OFF
    bd.seed_ptr = None if ctr is None else ctr.data_ptr()
    check(lib().rp_attn_bwd(ctypes.byref(bd), _stream()), "rp_attn_bwd")
    torch.cuda.synchronize()
    return dq, dkv


def _attn_last(c, mpk, scale):
    """rp_attn_last on the last query row of every sequence -> out [B + 1, d] (row B is a sentinel row)."""
    B, L, H, hd, d = c.B, c.L, c.H, c.hd, c.d
    q_last = c.qd.view(B, L, d)[:, -1].contiguous()
    out = torch.full((B + 1, d), SENT, dtype=torch.bfloat16, device=c.qd.device)
    check(lib().rp_attn_last(q_last.data_ptr(), c.kvd.data_ptr(), c.kvd.data_ptr(), 2 * d, 2 * d, 0, d, c.padd.data_ptr(),
                             B, H, L, hd, mpk, out.data_ptr(), scale, _stream()), "rp_attn_last")
    torch.cuda.synchronize()
    return out


def _ref_scale(c, scale):
    return scale if scale > 0 else 1.0 / math.sqrt(c.hd)


# ----------------------------------------------------------------------------------------------------------------------
# checks shared by the tests
# ----------------------------------------------------------------------------------------------------------------------
def _check_fwd(c, causal, mpk, scale, res, keep=None):
    B, L, H, hd, d, Lp, ht = c.B, c.L, c.H, c.hd, c.d, c.Lp, c.hd_true
    out, p_save, inv, m = res
    o_ref, m_ref, inv_ref, e_ref = attn_ref(c.q64, c.k64, c.v64, c.pad, causal, mpk, _ref_scale(c, scale), keep)
    o_all = _heads(out.cpu(), B, L, H, hd)
    o = o_all[..., :ht]
    assert (o_all[..., ht:] == 0).all(), "padded head columns of O must stay zero"
    assert _note("fwd O block", block_err(o, o_ref)) < TOL_O
    key_ok = c.pad if mpk else torch.ones_like(c.pad)
    vmax = c.v64.abs().amax(dim=(1, 3))[key_ok].max()
    assert _note("fwd O max/|V|", (o - o_ref).abs().max() / vmax) < TOL_O_MAX
    vis = visibility(c.pad, L, causal, mpk)
    dead = (~vis.any(-1)).expand(B, H, L)
    assert (o[dead] == 0).all(), "fully masked query rows must give exactly zero"
    assert (out[:, d:] == SENT).all(), "columns past the heads were written"
    if p_save is None:
        return
    inv_k = inv.cpu().double().view(B, H, Lp)[:, :, :L]
    m_k = m.cpu().double().view(B, H, Lp)[:, :, :L]
    _note("fwd m_save abs", (m_k - m_ref).abs().max())
    torch.testing.assert_close(m_k, m_ref, rtol=TOL_M_REL, atol=TOL_M_ABS)
    _note("fwd inv_sum rel", ((inv_k - inv_ref).abs() / inv_ref.clamp_min(1e-300)).max())
    torch.testing.assert_close(inv_k, inv_ref, rtol=TOL_INV_REL, atol=0)   # atol 0: fully masked rows exactly 0
    P = p_save.cpu().double().view(B, H, Lp, Lp)
    vis_full = torch.zeros(B, 1, Lp, Lp, dtype=torch.bool)
    vis_full[:, :, :L, :L] = vis
    vis_full = vis_full.expand(B, H, Lp, Lp)
    assert (P[~vis_full] == 0).all(), "p_save must be zero above the diagonal, at masked keys, at columns >= L, rows >= L"
    e = e_ref[vis.expand(B, H, L, L)]
    pe = P[:, :, :L, :L][vis.expand(B, H, L, L)]
    rel = ((pe - e).abs() / (e + 1e-30)).max() if e.numel() else torch.tensor(0.0)
    assert _note("fwd p_save rel", rel) < BF16_ROUND   # the un-dropped exp(s - max), rounded to bf16


def _check_grads(c, causal, mpk, got, ref, family):
    """got / ref: (dQ, dK, dV) as [B, H, L, hd_true] float64."""
    for name, g, r in zip(("dQ", "dK", "dV"), got, ref):
        assert _note(f"{family} {name} block", block_err(g, r)) < TOL_GRAD, name
        assert _note(f"{family} {name} max", (g - r).abs().max() / r.abs().max().clamp_min(BLOCK_FLOOR)) < TOL_GRAD_MAX, name
    B, H, L = c.B, c.H, c.L
    vis = visibility(c.pad, L, causal, mpk)
    dead_q = (~vis.any(-1)).expand(B, H, L)
    assert (got[0][dead_q] == 0).all(), "dQ of fully masked query rows must be exactly zero"
    if mpk:
        pad_k = (~c.pad).view(B, 1, L).expand(B, H, L)
        assert (got[1][pad_k] == 0).all() and (got[2][pad_k] == 0).all(), "dK / dV of masked pad keys must be exactly zero"


# ----------------------------------------------------------------------------------------------------------------------
# CPU: the reference and the tolerances
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", list(MODES))
def test_attn_ref_matches_sdpa_and_zeroes_masked_rows(mode):
    causal, mpk = MODES[mode]
    B, H, L, hd = 4, 2, 70, 16
    g = torch.Generator().manual_seed(3)
    q, k, v = (torch.randn(B, H, L, hd, generator=g, dtype=torch.float64) for _ in range(3))
    pad = _pad_pattern(L, bert=mode == "bert")
    scale = 0.37
    o, m2, inv, e = attn_ref(q, k, v, pad, causal, mpk, scale)
    vis = visibility(pad, L, causal, mpk)
    sd = F.scaled_dot_product_attention(q, k, v, attn_mask=vis, scale=scale)
    live = vis.any(-1).expand(B, H, L)
    torch.testing.assert_close(o[live], sd[live], rtol=1e-12, atol=1e-12)
    assert (o[~live] == 0).all() and (inv[~live] == 0).all() and (m2[~live] == 0).all()
    s = (q @ k.transpose(-1, -2)) * scale
    ref_m = s.masked_fill(~vis, float("-inf")).amax(-1) * LOG2E
    torch.testing.assert_close(m2[live], ref_m[live], rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(inv[live], 1.0 / e.sum(-1)[live], rtol=1e-12, atol=0)
    assert (e[~vis.expand(B, H, L, L)] == 0).all()


@pytest.mark.parametrize("mode", list(MODES))
def test_attn_ref_matches_oracle_mha_core(mode):
    """attn_ref is the attention core of oracle/sasrec.py::mha (identity projections)."""
    from oracle.sasrec import mha

    causal, mpk = MODES[mode]
    B, H, L, hd = 4, 2, 70, 16
    d = H * hd
    g = torch.Generator().manual_seed(4)
    q_in, kv_in = (torch.randn(B, L, d, generator=g, dtype=torch.float64) for _ in range(2))
    eye = torch.eye(d, dtype=torch.float64)
    blk = {"in_w": torch.cat([eye, eye, eye]), "in_b": torch.zeros(3 * d, dtype=torch.float64), "out_w": eye,
           "out_b": torch.zeros(d, dtype=torch.float64)}
    pad = _pad_pattern(L, bert=mode == "bert", B=B)
    got = mha(q_in, kv_in, blk, H, visibility(pad, L, causal, mpk)[:, 0])
    split = lambda x: x.view(B, L, H, hd).transpose(1, 2)  # noqa: E731
    ref = attn_ref(split(q_in), split(kv_in), split(kv_in), pad, causal, mpk, 1.0 / math.sqrt(hd))[0]
    torch.testing.assert_close(got, ref.transpose(1, 2).reshape(B, L, d), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("dropout", [False, True])
def test_grad_formula_matches_autograd(mode, dropout):
    """attn_grads_given_o with the exact O is fp64 autograd of attn_ref (incl. fully masked rows and dropout)."""
    causal, mpk = MODES[mode]
    L = 70
    c = _case(_pad_pattern(L, bert=mode == "bert"), 2, 16, mpk, seed=6)
    keep = drop_keep(SEED + CTR, OFF, P_DROP, c.B, c.H, L, c.Lp) if dropout else None
    vis = visibility(c.pad, L, causal, mpk)
    d_o = _heads(_d_out(c, 7), c.B, L, c.H, c.hd)
    o, *auto = _attn_grads(c.q64, c.k64, c.v64, vis, 0.3, keep, d_o)
    for a, f in zip(auto, attn_grads_given_o(c.q64, c.k64, c.v64, vis, 0.3, keep, d_o, o)):
        torch.testing.assert_close(f, a, rtol=1e-10, atol=1e-10)


def test_dropout_port_keep_rate():
    keep = keep_draws(SEED + CTR, OFF, P_DROP, np.arange(2048), 256)
    assert abs(float(keep.double().mean()) - (1 - P_DROP)) < 5e-3
    assert not torch.equal(keep, keep_draws(SEED + CTR + 1, OFF, P_DROP, np.arange(2048), 256))


_PERTURBATIONS = ["causal_strict", "drop_last_chunk", "slot_scale", "row_key_pitch", "keep_twice"]


@pytest.mark.parametrize("L", [65, 200, 300])
@pytest.mark.parametrize("perturbation", _PERTURBATIONS)
def test_tolerances_discriminate_perturbed_references(perturbation, L):
    """At the GPU tests' shapes and tolerances, each plausible kernel mistake - causal j < i instead of j <= i, the last
    visible 64-key chunk dropped, 1/sqrt(64) instead of 1/sqrt(48) in a padded slot, the dropout row key at bz*L + i
    instead of bz*Lp + i, the keep-scale applied twice - moves O and the gradients by at least 10x the tolerance."""
    hd_true = 48 if perturbation == "slot_scale" else None
    pad = _pad_pattern(L)
    c = _case(pad, 2, 64, 1, seed=L, hd_true=hd_true)
    B, H, Lp = c.B, c.H, c.Lp
    scale = 1.0 / math.sqrt(c.hd_true)
    vis = visibility(pad, L, 1, 1)
    dropout = perturbation in ("row_key_pitch", "keep_twice")
    keep = drop_keep(SEED + CTR, OFF, P_DROP, B, H, L, Lp) if dropout else None
    pvis, pscale, pkeep = vis, scale, keep
    if perturbation == "causal_strict":
        pvis = vis & torch.ones(L, L, dtype=torch.bool).tril(-1)
    elif perturbation == "drop_last_chunk":
        j = torch.arange(L)
        last_chunk = torch.where(vis, j, -1).amax(-1, keepdim=True) // 64
        pvis = vis & (j // 64 != last_chunk)
    elif perturbation == "slot_scale":
        pscale = 1.0 / math.sqrt(64)
    elif perturbation == "row_key_pitch":
        pkeep = drop_keep(SEED + CTR, OFF, P_DROP, B, H, L, L)
    else:
        pkeep = keep / (1.0 - P_DROP)
    d_o = _heads(_d_out(c, 5), B, L, H, 64)[..., : c.hd_true]
    ref = _attn_grads(c.q64, c.k64, c.v64, vis, scale, keep, d_o)
    bad = _attn_grads(c.q64, c.k64, c.v64, pvis, pscale, pkeep, d_o)
    assert block_err(bad[0], ref[0]) >= 10 * TOL_O
    assert max(block_err(b, r) for b, r in zip(bad[1:], ref[1:])) >= 10 * TOL_GRAD


# ----------------------------------------------------------------------------------------------------------------------
# GPU: rp_attn_fwd
# ----------------------------------------------------------------------------------------------------------------------
_FWD_L_KB1 = [1, 7, 63, 64, 65, 127, 128, 129, 200, 255, 256]   # one resident 256-key block
_FWD_L_KB2 = [257, 300, 383, 384, 449, 512]                      # two (head_dim 64 only)
_FWD_L_HD128 = [1, 65, 128, 129, 200, 256]
_FWD_SPREAD = [1, 65, 129, 255, 300, 449]                       # 1, 2, 3 and 4 query tiles, both key-block counts
_FWD_CASES = ([("sasrec", 64, L) for L in _FWD_L_KB1 + _FWD_L_KB2]
              + [(m, 64, L) for m in ("legacy", "bert", "none") for L in _FWD_SPREAD]
              + [("sasrec", 128, L) for L in _FWD_L_HD128]
              + [(m, 128, L) for m in ("legacy", "bert", "none") for L in (65, 129, 256)])


@pytest.mark.gpu
@pytest.mark.parametrize("mode,hd,L", _FWD_CASES)
def test_attn_fwd_matches_reference(cuda, mode, hd, L):
    """out, m_save, inv_sum and p_save against attn_ref at the default and a sharp scale; exact zeros where nothing is
    visible; inference (no saved statistics) bitwise equal to training on every query tile with a real row and zero on
    all-padding tiles; bitwise equal reruns."""
    causal, mpk = MODES[mode]
    c = _case(_pad_pattern(L, bert=mode == "bert"), 2, hd, mpk, seed=7 * L + hd, dev=cuda)
    B, d = c.B, c.d
    for scale in (0.0, SHARP / math.sqrt(hd)):
        res = _attn_fwd(c, causal, mpk, scale)
        _check_fwd(c, causal, mpk, scale, res)
        again = _attn_fwd(c, causal, mpk, scale)
        assert all(torch.equal(a, b) for a, b in zip(res, again)), "reruns differ"
        inf_out = _attn_fwd(c, causal, mpk, scale, train=False)[0].view(B, L, -1)
        tr_out = res[0].view(B, L, -1)
        assert (inf_out[..., d:] == SENT).all()
        for b in range(B):
            for t0 in range(0, L, 128):
                rows = slice(t0, min(L, t0 + 128))
                if c.pad[b, rows].any():
                    assert torch.equal(inf_out[b, rows], tr_out[b, rows]), (b, t0)
                else:
                    assert (inf_out[b, rows, :d] == 0).all(), (b, t0)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,hd,L", [("sasrec", 64, 65), ("sasrec", 64, 200), ("sasrec", 64, 300), ("sasrec", 64, 512),
                                       ("bert", 64, 129), ("bert", 64, 449), ("sasrec", 128, 129), ("bert", 128, 256)])
def test_attn_fwd_dropout_matches_reference(cuda, mode, hd, L):
    """Attention dropout p = 0.2 with the step counter behind seed_ptr: O equals attn_ref under the ported mask, and
    p_save / inv_sum hold the un-dropped probabilities."""
    causal, mpk = MODES[mode]
    c = _case(_pad_pattern(L, bert=mode == "bert"), 2, hd, mpk, seed=11 * L + hd, dev=cuda)
    ctr = torch.tensor([CTR], dtype=torch.int64, device=cuda)
    keep = drop_keep(SEED + CTR, OFF, P_DROP, c.B, c.H, L, c.Lp)
    res = _attn_fwd(c, causal, mpk, 0.0, drop=P_DROP, ctr=ctr)
    _check_fwd(c, causal, mpk, 0.0, res, keep=keep)


@pytest.mark.gpu
@pytest.mark.parametrize("hd,hd_true,L", [(64, 48, 65), (64, 48, 200), (64, 48, 300), (128, 96, 129), (128, 96, 256)])
def test_attn_fwd_scale_override_for_padded_head_slots(cuda, hd, hd_true, L):
    """A 48-wide head in a 64-wide slot (96 in 128) with zero columns past the true width: with scale = 1/sqrt(true
    width) the kernel computes the true-width attention, and the padded output columns stay exactly zero."""
    c = _case(_pad_pattern(L), 2, hd, 1, seed=L + hd_true, hd_true=hd_true, dev=cuda)
    scale = 1.0 / math.sqrt(hd_true)
    _check_fwd(c, 1, 1, scale, _attn_fwd(c, 1, 1, scale))


@pytest.mark.gpu
def test_dropout_port_matches_device_stream(cuda):
    """The Python port of the dropout stream equals rp_dropout_bwd's mask on an all-ones [B*H*Lp, Lp] array (same seed,
    site offset and step counter), bit for bit."""
    B, H, L = 3, 2, 200
    Lp = _ru(L, 64)
    rows = B * H * Lp
    ctr = torch.tensor([CTR], dtype=torch.int64, device=cuda)
    ones = torch.ones(rows, Lp, dtype=torch.bfloat16, device=cuda)
    out = torch.empty_like(ones)
    check(lib().rp_dropout_bwd(ones.data_ptr(), out.data_ptr(), rows, Lp, None, P_DROP, SEED, OFF, ctr.data_ptr(), _stream()),
          "rp_dropout_bwd")
    got = (out.cpu() > 0)
    assert torch.equal(got, keep_draws(SEED + CTR, OFF, P_DROP, np.arange(rows), Lp))
    port = drop_keep(SEED + CTR, OFF, P_DROP, B, H, L, Lp) > 0
    assert torch.equal(got.view(B, H, Lp, Lp)[:, :, :L, :L], port)


# ----------------------------------------------------------------------------------------------------------------------
# GPU: the fused backward (head_dim 64, L <= 256)
# ----------------------------------------------------------------------------------------------------------------------
def _fused_bwd_case(cuda, c, causal, mpk, scale, drop):
    ctr = torch.tensor([CTR], dtype=torch.int64, device=cuda)
    keep = drop_keep(SEED + CTR, OFF, drop, c.B, c.H, c.L, c.Lp) if drop > 0 else None
    fwd = _attn_fwd(c, causal, mpk, scale, drop=drop, ctr=ctr)
    d_o = _d_out(c, seed=c.L + 1)
    d_od = d_o.to(cuda)
    dq, dkv = _attn_bwd(c, causal, mpk, scale, fwd, d_od, drop=drop, ctr=ctr)
    dq2, dkv2 = _attn_bwd(c, causal, mpk, scale, fwd, d_od, drop=drop, ctr=ctr)
    assert torch.equal(dq, dq2) and torch.equal(dkv, dkv2), "reruns differ"
    T, d, ht = c.T, c.d, c.hd_true
    assert (dq[T:] == SENT).all() and (dq[:, d:] == SENT).all(), "dQ written outside [T, d)"
    assert (dkv[T:] == SENT).all() and (dkv[:, 2 * d:] == SENT).all(), "dK / dV written outside [T, 2d)"
    dq, dkv = dq[:T].cpu(), dkv[:T].cpu()
    got = [_heads(x, c.B, c.L, c.H, c.hd) for x in (dq, dkv[:, :d], dkv[:, d: 2 * d])]
    assert all((g[..., ht:] == 0).all() for g in got), "padded head columns of the gradients must stay zero"
    vis = visibility(c.pad, c.L, causal, mpk)
    d_o64 = _heads(d_o, c.B, c.L, c.H, c.hd)[..., :ht]
    o64 = _heads(fwd[0].cpu(), c.B, c.L, c.H, c.hd)[..., :ht]
    ref = attn_grads_given_o(c.q64, c.k64, c.v64, vis, _ref_scale(c, scale), keep, d_o64, o64)
    _check_grads(c, causal, mpk, [g[..., :ht] for g in got], ref, "fused bwd")


@pytest.mark.gpu
@pytest.mark.parametrize("drop", [0.0, P_DROP])
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("L", [1, 33, 64, 65, 128, 129, 192, 200, 255, 256])
def test_attn_bwd_fused_matches_autograd(cuda, L, mode, drop):
    """dQ, dK, dV of rp_attn_bwd (fed the kernel forward's O, m_save, inv_sum) against the fp64 backward formula on the
    same O (attn_grads_given_o), per 64-row block:
    both warpgroups' key blocks, the second 128-row tile, causal block skipping, masked keys exactly zero, nothing
    written outside the heads / rows, bitwise equal reruns."""
    causal, mpk = MODES[mode]
    c = _case(_pad_pattern(L, bert=mode == "bert"), 2, 64, mpk, seed=13 * L + causal + 2 * mpk, dev=cuda)
    _fused_bwd_case(cuda, c, causal, mpk, 0.0, drop)


@pytest.mark.gpu
@pytest.mark.parametrize("drop", [0.0, P_DROP])
@pytest.mark.parametrize("L", [65, 200, 256])
def test_attn_bwd_fused_scale_override_for_padded_head_slot(cuda, L, drop):
    c = _case(_pad_pattern(L), 2, 64, 1, seed=L + 48, hd_true=48, dev=cuda)
    _fused_bwd_case(cuda, c, 1, 1, 1.0 / math.sqrt(48), drop)


# ----------------------------------------------------------------------------------------------------------------------
# GPU: the un-fused backward (head_dim 128, and head_dim 64 at L > 256)
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("drop", [0.0, P_DROP])
@pytest.mark.parametrize("hd,L", [(64, 65), (64, 200), (64, 256), (128, 129), (64, 257), (64, 300), (64, 449), (64, 512)])
def test_attn_softmax_bwd_matches_formula(cuda, hd, L, drop):
    """rp_attn_softmax_bwd on forward-produced p_save / inv_sum and a random dpd, against its formula
    (P = p_save * inv_sum, dP = dpd * mask / keep, dS = P (dP - sum_j P_j dP_j) scale, Pd = P mask / keep) in fp64:
    128-column blocks NK = 2 (L <= 256) and NK = 4, ragged L; nothing written past the row's last 4-column group."""
    c = _case(_pad_pattern(L), 2, hd, 1, seed=17 * L, dev=cuda)
    B, H, Lp = c.B, c.H, c.Lp
    BH = B * H
    scale = 1.0 / math.sqrt(hd)
    ctr = torch.tensor([CTR], dtype=torch.int64, device=cuda)
    _, p_save, inv, _ = _attn_fwd(c, 1, 1, 0.0, drop=drop, ctr=ctr)
    g = torch.Generator().manual_seed(L)
    dpd = torch.randn(BH, Lp, Lp, generator=g).to(torch.bfloat16).to(cuda)
    p0, d0 = p_save.cpu(), dpd.cpu()
    check(lib().rp_attn_softmax_bwd(p_save.data_ptr(), dpd.data_ptr(), inv.data_ptr(), BH, L, scale, drop, SEED, OFF,
                                    ctr.data_ptr(), _stream()), "rp_attn_softmax_bwd")
    torch.cuda.synchronize()
    pd_k, ds_k = p_save.cpu(), dpd.cpu()
    keep = (drop_keep(SEED + CTR, OFF, drop, B, H, L, Lp).view(BH, L, L) if drop > 0
            else torch.ones(BH, L, L, dtype=torch.float64))
    P = p0[:, :L, :L].double() * inv.cpu().double()[:, :L, None]
    dP = d0[:, :L, :L].double() * keep
    dot = (P * dP).sum(-1, keepdim=True)
    ds = P * (dP - dot) * scale
    pd = P * keep
    for name, got, ref, rowscale in (("dS", ds_k, ds, (P * (dP.abs() + dot.abs())).amax(-1, keepdim=True) * scale),
                                     ("Pd", pd_k, pd, pd.amax(-1, keepdim=True))):
        err = ((got[:, :L, :L].double() - ref).abs() / (ref.abs() + 1e-3 * rowscale).clamp_min(1e-300)).max()
        assert _note(f"softmax bwd {name} rel", err) < BF16_ROUND, name
    c4 = _ru(L, 4)
    for got, before in ((pd_k, p0), (ds_k, d0)):
        assert torch.equal(got[:, L:], before[:, L:]), "rows >= L were written"
        assert torch.equal(got[:, :L, c4:], before[:, :L, c4:]), "columns past the last 4-column group were written"
        assert (got[:, :L, L:c4] == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("d,H,L,variant,drop", [(128, 1, 65, "new", 0.0), (256, 2, 200, "new", P_DROP),
                                                (256, 2, 256, "legacy", 0.0), (256, 2, 65, "legacy", P_DROP),
                                                (128, 2, 300, "new", P_DROP), (128, 2, 512, "new", 0.0),
                                                (128, 2, 512, "legacy", P_DROP)])
def test_attention_drivers_unfused_backward_matches_autograd(cuda, d, H, L, variant, drop):
    """The engine's un-fused attention backward (dPd = dO.V^T, rp_attn_softmax_bwd over the saved probabilities, three
    batched GEMMs) run through the shared attention drivers SasRecEngine._attention_forward / _attention_backward, with
    SASRec's Q and packed [K | V] as sources and dQ / packed [dK | dV] as destinations, on planted Q, K, V and dO: O, dQ, dK,
    dV against fp64 autograd per 64-row block, at head_dim 128 and at head_dim 64 with L > 256."""
    from replay_b200.engine import EncoderConfig, SasRecEngine

    cfg = EncoderConfig(n_items=500, d=d, n_heads=H, n_blocks=1, max_len=L, dropout=drop, variant=variant)
    eng = SasRecEngine(cfg, 4, L, cuda, seed=SEED)
    assert not eng.fused_attn_bwd
    mpk = int(variant == "new")
    c = _case(_pad_pattern(L), H, d // H, mpk, seed=19 * L + d, dev=cuda)
    a = eng.act[0]
    eng.in_pad.copy_(c.padd.view(-1))
    a["Q"].copy_(c.qd)
    a["KV"].copy_(c.kvd)
    eng.rng_counter.fill_(CTR)
    qkv = (a["Q"], 0), (a["KV"], 0), (a["KV"], d)
    eng._attention_forward(0, True, *qkv, causal=True, mask_pad_keys=bool(mpk))
    d_o = _d_out(c, seed=L)
    eng.s["d_o"].copy_(d_o.to(cuda))
    eng._attention_backward(0, *qkv, (eng.s["dQ"], 0), (eng.s["dKV"], 0), (eng.s["dKV"], d), causal=True, mask_pad_keys=bool(mpk))
    torch.cuda.synchronize()
    B, hd, T = c.B, c.hd, c.T
    keep = drop_keep(eng.seed + CTR, eng._site(0, 0) << 40, drop, B, H, L, c.Lp) if drop > 0 else None
    vis = visibility(c.pad, L, 1, mpk)
    o_ref, *ref = _attn_grads(c.q64, c.k64, c.v64, vis, 1.0 / math.sqrt(hd), keep, _heads(d_o, B, L, H, hd))
    o = _heads(a["O"].cpu(), B, L, H, hd)
    assert _note("unfused O block", block_err(o, o_ref)) < TOL_O
    dkv = eng.s["dKV"][:T].cpu()
    got = [_heads(x, B, L, H, hd) for x in (eng.s["dQ"][:T].cpu(), dkv[:, :d], dkv[:, d:])]
    _check_grads(c, 1, mpk, got, ref, "unfused bwd")


# ----------------------------------------------------------------------------------------------------------------------
# GPU: rp_attn_last
# ----------------------------------------------------------------------------------------------------------------------
def _row_err(got, ref):
    """per (b, h) norm-relative error of [B, H, D] rows (a ~0 reference row: against the RMS floor)"""
    den = torch.maximum(ref.norm(dim=-1), torch.tensor(BLOCK_FLOOR * math.sqrt(ref.shape[-1]), dtype=torch.float64))
    return float(((got - ref).norm(dim=-1) / den).max())


@pytest.mark.gpu
@pytest.mark.parametrize("mpk", [0, 1])
@pytest.mark.parametrize("hd,L", [(64, L) for L in (1, 31, 32, 33, 200, 511, 512)] + [(128, L) for L in (1, 31, 32, 33, 200, 256)])
def test_attn_last_matches_reference(cuda, hd, L, mpk):
    """One query (the last position) per (sequence, head) against the last row of attn_ref, for B*H = 10 (not a
    multiple of the 8 warps per CTA) with K and V in the packed [T, 2d] array; an all-padding sequence with masked pad
    keys gives exactly 0; and the result agrees with the last row of rp_attn_fwd on the same inputs."""
    B, H = 5, 2   # five sequences: the second CTA has two live warps
    c = _case(_pad_pattern(L, B=B), H, hd, mpk, seed=23 * L + hd + mpk, dev=cuda)
    for scale in (0.0, SHARP / math.sqrt(hd)):
        out = _attn_last(c, mpk, scale)
        assert (out[B] == SENT).all()
        got = out[:B].cpu().double().view(B, H, hd)
        ref = attn_ref(c.q64, c.k64, c.v64, c.pad, 1, mpk, _ref_scale(c, scale))[0][:, :, -1]
        assert _note("last row", _row_err(got, ref)) < TOL_LAST
        if mpk:
            assert (got[~c.pad.any(-1)] == 0).all(), "an all-padding sequence must give exactly zero"
        if hd == 64 or L <= 256:
            fwd = _attn_fwd(c, 1, mpk, scale)[0].cpu().double()
            last = fwd.view(B, L, -1)[:, -1, : c.d].reshape(B, H, hd)
            assert _note("last vs fwd", _row_err(got, last)) < 2 * TOL_LAST   # worst seen 3.7e-3 (both rounded to bf16)


@pytest.mark.gpu
@pytest.mark.parametrize("hd,hd_true,L", [(64, 48, 200), (128, 96, 200)])
def test_attn_last_scale_override_for_padded_head_slots(cuda, hd, hd_true, L):
    B, H = 5, 2
    c = _case(_pad_pattern(L, B=B), H, hd, 1, seed=L + hd_true, hd_true=hd_true, dev=cuda)
    scale = 1.0 / math.sqrt(hd_true)
    got = _attn_last(c, 1, scale)[:B].cpu().double().view(B, H, hd)
    assert (got[..., hd_true:] == 0).all()
    ref = attn_ref(c.q64, c.k64, c.v64, c.pad, 1, 1, scale)[0][:, :, -1]
    assert _note("last row", _row_err(got[..., :hd_true], ref)) < TOL_LAST


# ----------------------------------------------------------------------------------------------------------------------
# GPU: engine-level paths the model tests do not reach
# ----------------------------------------------------------------------------------------------------------------------
def _cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


@pytest.mark.gpu
@pytest.mark.parametrize("d,H", [(128, 1), (256, 2)])
def test_head_slot_128_train_step_matches_oracle(cuda, d, H):
    """SASRec with 128-wide heads (attn_fwd_kernel<128, 1>, the un-fused backward at head_dim 128, attn_last_kernel<128>)
    at L = 200 against the oracle: hidden states, loss, every parameter gradient, and the predict-path last hidden state;
    thresholds of test_config5_shape_train_step_matches_oracle."""
    from oracle import sasrec as osr
    from replay_b200.engine import EncoderConfig, SasRecEngine
    from replay_b200.synthetic import make_sequences

    B, L, I = 3, 200, 1500
    P = osr.random_params(I, d, L, 2, seed=29)
    ids, pm, lab, tm = make_sequences(B, I, L, seed=6)
    ids[0, :150], pm[0, :150] = I, False          # the first 128-row query tile of sequence 0 is all padding
    lab[0, :149], tm[0, :149] = I, False
    cfg = EncoderConfig(n_items=I, d=d, n_heads=H, n_blocks=2, max_len=L, dropout=0.0, variant="new")
    eng = SasRecEngine(cfg, B, L, cuda)
    assert cfg.head_slot == 128 and not eng.fused_attn_bwd
    eng.load_canonical(P)
    eng.set_batch(ids.cuda(), pm.cuda(), lab.cuda(), tm.cuda())
    hid = eng.forward_hidden_all().float().cpu().view(B, L, d)
    ref_h = osr.sasrec_body(P, ids, pm, H, "new")
    assert (hid - ref_h).abs().max() < 8e-2, (hid - ref_h).abs().max()
    loss = eng.forward_train()
    ref_loss, Gref = osr.loss_and_grads(P, ids, pm, lab, tm, H, "new")
    assert abs(loss[0].item() - float(ref_loss)) < 5e-3 * float(ref_loss), (loss[0].item(), float(ref_loss))
    eng.g32.zero_()
    eng.backward()
    torch.cuda.synchronize()
    G = eng.export_canonical(eng.grads)
    bad = []
    for k, (a, b) in enumerate(zip(osr.flat_param_list(G), osr.flat_param_list(Gref))):
        c, r = _cos(a, b), float(a.double().norm() / (b.double().norm() + 1e-30))
        if c < 0.99 or abs(r - 1) > 0.04:
            bad.append((k, round(c, 5), round(r, 4)))
    assert not bad, bad
    eng.set_batch(ids.cuda(), pm.cuda())
    hq = eng.forward_last_hidden().float().cpu()
    ref_e = osr.sasrec_body(P, ids, pm, H, "new", mode="eval")[:, -1]
    assert (hq - ref_e).abs().max() < 8e-2


@pytest.mark.gpu
def test_fused_attention_backward_matches_unfused_at_L200(cuda):
    """The fused attention backward and the un-fused path share the forward and its dropout masks: at L = 200 (four
    64-row blocks, both warpgroups, two 128-row tiles) with attention dropout 0.2 their gradients agree to bf16 round-off."""
    from oracle import sasrec as osr
    from replay_b200.engine import EncoderConfig, SasRecEngine
    from replay_b200.synthetic import make_sequences

    B, L, d, H, I = 4, 200, 128, 2, 1500
    P = osr.random_params(I, d, L, 2, seed=31)
    batch = [t.cuda() for t in make_sequences(B, I, L, seed=8)]
    grads = []
    for fused in (True, False):
        cfg = EncoderConfig(n_items=I, d=d, n_heads=H, n_blocks=2, max_len=L, dropout=P_DROP, variant="new")
        eng = SasRecEngine.__new__(SasRecEngine)
        SasRecEngine.__init__(eng, cfg, B, L, cuda, seed=77)
        assert eng.fused_attn_bwd
        if not fused:  # rebuild the workspace for the un-fused path
            eng.fused_attn_bwd = False
            eng._alloc_workspace()
        eng.load_canonical(P)
        eng.set_batch(*batch)
        eng.forward_train()
        eng.g32.zero_()
        eng.backward()
        torch.cuda.synchronize()
        grads.append(eng.g32.clone())
    a, b = grads
    assert torch.isfinite(a).all() and torch.isfinite(b).all()
    cos = float((a.double() @ b.double()) / (a.double().norm() * b.double().norm()))
    assert cos > 0.9995, cos
    assert abs(float(a.norm() / b.norm()) - 1) < 5e-3
