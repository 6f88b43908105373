"""float64 restatement of SasRecEngine's training step, shared by the SASRec step tests (test_gpu_sasrec_body.py at the
config-2 shape, test_gpu_config5_fp64.py at the config-5 shape).

- ``engine_keeps``: the keep masks of every dropout site, ported from csrc/rp_philox.cuh (tests/dropout_stream.py);
- ``sasrec_body_ref`` / ``sasrec_ref``: oracle.sasrec's body and full-catalog CE with a keep mask at every site;
- ``ref_loss_and_grads``: loss, x[-1], hidden states and autograd gradients, the CE head unchunked ([T_v, I] logits);
- ``ce_head_chunked`` / ``ref_loss_and_grads_chunked``: the same with the head computed in row chunks, so that a catalog of
  a million items never materialises [T_v, I];
- ``step_batch``, ``_Case``, ``engine_view``: the batches, configurations and parameter view of the step tests.
"""
import math

import numpy as np
import torch

from dropout_stream import drop_keep, keep_draws

SEED, CTR = 0x5EED1234ABC, 987654321   # dropout stream of the kernel-level tests (seed_ptr holds CTR)
P_DROP = 0.2                           # configs 2 and 5
EPS = 1e-8                             # LayerNorm 1 / 2 of a SASRec block


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _bf(x):
    return x.to(torch.bfloat16)


def _ks(p):
    return 1.0 / (1.0 - float(np.float32(p)))


def _ru(x, m):
    return (x + m - 1) // m * m


def _site(blk, k):
    """SasRecEngine._site: dropout site k of block blk (offset = site << 40; the embedding is offset 0)."""
    return 1 + 8 * blk + k


# ----------------------------------------------------------------------------------------------------------------------
# float64 reference of the SASRec training loss with every dropout site
# ----------------------------------------------------------------------------------------------------------------------
def engine_keeps(seed_eff, p, B, L, cfg, site_shift=0, dev=None):
    """Keep masks (0 or 1/(1-p), float64) of every dropout site of SasRecEngine's training body, in the model's true
    feature space: the embedding at offset 0; per block attention probabilities at _site(i, 0) << 40 (row key
    bz * Lp + i), the FFN hidden activation after the ReLU at _site(i, 1) << 40 and the FFN output before the residual at
    _site(i, 2) << 40.  Token sites are drawn over the padded width dp (the kernels' column keys) and gathered at
    cfg.feat_index().  ``site_shift`` moves every block site number (a plausible mistake)."""
    T, Lp, ks = B * L, _ru(L, 64), _ks(p)
    rows = np.arange(T)
    feat = cfg.feat_index()

    def tok(off):
        return (keep_draws(seed_eff, off, p, rows, cfg.dp)[:, feat].double() * ks).view(B, L, cfg.d).to(dev)

    out = {"emb": tok(0), "blocks": []}
    for i in range(cfg.n_blocks):
        s = lambda k: (_site(i, k) + site_shift) << 40  # noqa: E731
        out["blocks"].append({"attn": drop_keep(seed_eff, s(0), p, B, cfg.n_heads, L, Lp).to(dev), "ffn1": tok(s(1)),
                              "ffn2": tok(s(2))})
    return out


def unit_keeps(B, L, d, H, n_blocks):
    ones = lambda *s: torch.ones(*s, dtype=torch.float64)  # noqa: E731
    return {"emb": ones(B, L, d), "blocks": [{"attn": ones(B, H, L, L), "ffn1": ones(B, L, d), "ffn2": ones(B, L, d)}
                                             for _ in range(n_blocks)]}


def _ln64(x, w, b, eps, width=None):
    """LayerNorm; ``width`` > d takes the statistics over ``width`` features of which the extra ones are zero (the
    padded-width mistake)."""
    n = x.shape[-1] if width is None else width
    mu = x.sum(-1, keepdim=True) / n
    var = (((x - mu) ** 2).sum(-1, keepdim=True) + (n - x.shape[-1]) * mu ** 2) / n
    return (x - mu) / torch.sqrt(var + eps) * w + b


def sasrec_body_ref(P, ids, pad, H, variant, lnf_eps, keeps=None, mistake=None, dp=None):
    """oracle.sasrec.sasrec_body restated with a keep mask at every dropout site -> (x[-1] [B, L, d] before the final
    LayerNorm, hidden [B, L, d] after it).  ``mistake`` (a plausible kernel / engine error, for the tolerance checks):
    'ffn_drop_after_residual', 'ln_padded_width' (LayerNorm statistics over ``dp`` features), 'no_row_mask' (legacy),
    'kv_from_normed', 'pos_first_rows' (the new path's positional window from the front), 'attn_keep_transposed' (the
    attention keep mask drawn with query and key swapped)."""
    B, L = ids.shape
    item_emb, pos = P["item_emb"], P["pos_emb"]
    d = item_emb.shape[1]
    hd = d // H
    I = item_emb.shape[0] - 1
    width = dp if mistake == "ln_padded_width" else None
    legacy = variant == "legacy"
    real = pad[..., None].to(item_emb.dtype)
    x = item_emb[ids.masked_fill(~pad, I)] * math.sqrt(d)
    x = x + (pos[:L] if legacy or mistake == "pos_first_rows" else pos[pos.shape[0] - L:])
    if keeps is not None:
        x = x * keeps["emb"]
    if legacy:
        x = x * real
    causal = torch.tril(torch.ones(L, L, dtype=torch.bool, device=ids.device))
    vis = (causal[None] if legacy else causal[None] & pad[:, None, :])[:, None]
    for i, blk in enumerate(P["blocks"]):
        kb = keeps["blocks"][i] if keeps is not None else None
        q_in = _ln64(x, blk["ln1_w"], blk["ln1_b"], EPS, width)
        kv_in = q_in if mistake == "kv_from_normed" else x
        w, b = blk["in_w"], blk["in_b"]
        q = (q_in @ w[:d].T + b[:d]).view(B, L, H, hd).transpose(1, 2)
        k = (kv_in @ w[d:2 * d].T + b[d:2 * d]).view(B, L, H, hd).transpose(1, 2)
        v = (kv_in @ w[2 * d:].T + b[2 * d:]).view(B, L, H, hd).transpose(1, 2)
        s = ((q @ k.transpose(-1, -2)) / math.sqrt(hd)).masked_fill(~vis, float("-inf"))
        m = s.detach().amax(-1, keepdim=True)
        m = torch.where(torch.isinf(m), torch.zeros_like(m), m)
        e = torch.exp(s - m)
        den = e.sum(-1, keepdim=True)
        pr = torch.where(den > 0, e / den.clamp_min(1e-300), torch.zeros_like(e))
        if kb is not None:
            pr = pr * (kb["attn"].transpose(-1, -2) if mistake == "attn_keep_transposed" else kb["attn"])
        o = (pr @ v).transpose(1, 2).reshape(B, L, d)
        h = q_in + o @ blk["out_w"].T + blk["out_b"]
        y = _ln64(h, blk["ln2_w"], blk["ln2_b"], EPS, width)
        u = torch.relu(y @ blk["w1"].T + blk["b1"])
        if kb is not None:
            u = u * kb["ffn1"]
        t = u @ blk["w2"].T + blk["b2"]
        if kb is not None and mistake == "ffn_drop_after_residual":
            x = (y + t) * kb["ffn2"]
        else:
            x = y + (t * kb["ffn2"] if kb is not None else t)
        if legacy and mistake != "no_row_mask":
            x = x * real
    return x, _ln64(x, P["lnf_w"], P["lnf_b"], lnf_eps, width)


def _targets(labels, tmask, I):
    return tmask & (labels >= 0) & (labels < I)


def sasrec_ref(P, ids, pad, labels, tmask, H, variant, lnf_eps, keeps=None, mistake=None, dp=None):
    """sasrec_body_ref + the full-catalog CE -> (loss, x[-1], hidden)."""
    x, hid = sasrec_body_ref(P, ids, pad, H, variant, lnf_eps, keeps, mistake, dp)
    item_emb = P["item_emb"]
    I = item_emb.shape[0] - 1
    sel = _targets(labels, tmask, I)
    logits = hid[sel] @ item_emb[:I].T
    loss = (torch.logsumexp(logits, -1) - logits.gather(1, labels[sel][:, None])[:, 0]).mean()
    return loss, x, hid


_BLOCK_KEYS = ("ln1_w", "ln1_b", "in_w", "in_b", "out_w", "out_b", "ln2_w", "ln2_b", "w1", "b1", "w2", "b2")


def _leaves(P):
    """[(name, tensor)] of a canonical parameter dict in SasRecEngine's naming."""
    out = [("item_emb", P["item_emb"]), ("pos_emb", P["pos_emb"])]
    for i, blk in enumerate(P["blocks"]):
        out += [(f"b{i}.{k}", blk[k]) for k in _BLOCK_KEYS]
    return out + [("lnf_w", P["lnf_w"]), ("lnf_b", P["lnf_b"])]


def _map(P, f):
    Q = {k: f(k, v) for k, v in P.items() if k != "blocks"}
    Q["blocks"] = [{k: f(f"b{i}.{k}", v) for k, v in blk.items()} for i, blk in enumerate(P["blocks"])]
    return Q


def _grads(leaves, grads):
    G = {k: (g if g is not None else torch.zeros_like(t)) for (k, t), g in zip(leaves, grads)}
    G["item_emb"][-1] = 0
    return G


def ref_loss_and_grads(P, ids, pad, labels, tmask, H, variant, lnf_eps, keeps=None, mistake=None, dp=None):
    """float64 loss, x[-1], hidden states and autograd gradients {name: tensor} (the pad row of item_emb frozen)."""
    Q = _map(P, lambda k, v: v.detach().double().clone().requires_grad_(True))
    loss, x, hid = sasrec_ref(Q, ids, pad, labels, tmask, H, variant, lnf_eps, keeps, mistake, dp)
    leaves = _leaves(Q)
    grads = torch.autograd.grad(loss, [t for _, t in leaves], allow_unused=True)
    return loss.detach(), x.detach(), hid.detach(), _grads(leaves, grads)


def ce_head_chunked(h, E, labels, rows=512, skip=None):
    """Mean full-catalog CE of float64 rows ``h`` [n, d] over the table ``E`` [I, d], in chunks of at most ``rows`` rows ->
    (loss, lse [n], d_h [n, d], d_E [I, d]); peak memory one [rows, I] chunk.  ``skip`` = (r0, r1): rows whose d_E
    contribution is left out (a plausible mistake of a chunked kernel)."""
    n = h.shape[0]
    lse = torch.empty(n, dtype=h.dtype, device=h.device)
    d_h = torch.empty_like(h)
    d_E = torch.zeros_like(E)
    total = torch.zeros((), dtype=h.dtype, device=h.device)
    for r0 in range(0, n, rows):
        hc, y = h[r0:r0 + rows], labels[r0:r0 + rows]
        z = hc @ E.T
        lse[r0:r0 + rows] = l = torch.logsumexp(z, -1)
        total += (l - z.gather(1, y[:, None])[:, 0]).sum()
        g = z.sub_(l[:, None]).exp_()                  # softmax, in place
        g[torch.arange(g.shape[0], device=g.device), y] -= 1.0
        g /= n
        d_h[r0:r0 + rows] = g @ E
        if skip is None or not skip[0] <= r0 < skip[1]:
            d_E.addmm_(g.T, hc)
    return total / max(n, 1), lse, d_h, d_E


def ref_loss_and_grads_chunked(P, ids, pad, labels, tmask, H, variant, lnf_eps, keeps=None, mistake=None, dp=None,
                               rows=512):
    """ref_loss_and_grads with the CE head from ce_head_chunked: the body's gradients by autograd from d(hidden), the
    tied table receiving both its head and its input-gather contributions."""
    Q = _map(P, lambda k, v: v.detach().double().clone().requires_grad_(True))
    x, hid = sasrec_body_ref(Q, ids, pad, H, variant, lnf_eps, keeps, mistake, dp)
    E = Q["item_emb"].detach()
    I = E.shape[0] - 1
    sel = _targets(labels, tmask, I)
    loss, _, d_h, d_E = ce_head_chunked(hid.detach()[sel], E[:I], labels[sel], rows)
    d_hid = torch.zeros_like(hid)
    d_hid[sel] = d_h
    del d_h
    leaves = _leaves(Q)
    torch.autograd.backward(hid, d_hid)
    G = _grads(leaves, [t.grad for _, t in leaves])
    G["item_emb"][:I] += d_E
    return loss, x.detach(), hid.detach(), G


# the bf16-consumed parameters of SasRecEngine (the kernels read their bf16 shadow): the reference uses them rounded
_BF16_PARAMS = ("item_emb", "in_w", "out_w", "w1", "w2")


def engine_view(P):
    """The parameters as SasRecEngine computes with them: bf16-consumed ones rounded to bf16, the rest fp32."""
    return _map(P, lambda k, v: (_bf(v).float() if k.split(".")[-1] in _BF16_PARAMS else v.float()))


_LENGTHS = [200, 200, 150, 57, 13, 1, 120]


def step_batch(B, L, I, seed, lengths=_LENGTHS):
    """Left-padded histories of the given ``lengths`` (repeated; capped at L), next-item labels on ~90 % of the real
    positions."""
    g = _gen(seed)
    pad = torch.zeros(B, L, dtype=torch.bool)
    for b in range(B):
        pad[b, L - min(lengths[b % len(lengths)], L):] = True
    items = torch.randint(0, I, (B, L + 1), generator=g)
    ids = torch.where(pad, items[:, :-1], torch.zeros_like(pad, dtype=torch.int64))
    labels = items[:, 1:]
    tmask = pad & (torch.rand(B, L, generator=g) > 0.1)
    return ids, pad, labels, tmask


class _Case:
    """One configuration of the step test: the engine's EncoderConfig, the reference's view of it, the fused-body flag.
    ``max_len`` defaults to L for the legacy model and L + 10 (an offset positional window) for the new path."""

    def __init__(self, variant, d, H, fused=True, L=200, I=2000, max_len=None):
        from replay_b200.engine import EncoderConfig

        self.variant, self.d, self.H, self.fused, self.L, self.I = variant, d, H, fused, L, I
        self.max_len = max_len or (L if variant == "legacy" else L + 10)
        self.cfg = EncoderConfig(n_items=I, d=d, n_heads=H, n_blocks=2, max_len=self.max_len, variant=variant)
        self.lnf_eps = self.cfg.lnf_eps

    def params(self, seed):
        from oracle import sasrec as osr

        return engine_view(osr.random_params(self.I, self.d, self.max_len, 2, seed=seed, bias_scale=0.1))
