"""Plain-torch restatement of RePlay's SasRec with the DiffTransformer encoder (TEST INFRASTRUCTURE - see oracle/__init__.py).

Parameters are the reference's own ``state_dict`` (keys of ``SasRec(body=SasRecBody(..., encoder=DiffTransformerLayer(...)))``);
everything is computed in their dtype (fp64 to adjudicate).

Reference files restated (under replay/ of the reference project):
  nn/sequential/sasrec/diff_transformer.py (blocks, lambda_init) ; nn/attention.py:67-157 (differential attention) ;
  nn/ffn.py:60-99 (SwiGLU) ; nn/mask.py:29-80 (DefaultAttentionMask) ; nn/sequential/sasrec/agg.py (positions) ;
  nn/sequential/sasrec/model.py (SasRecBody.forward, output normalization)
"""
from __future__ import annotations

import math

import numpy as np
import torch

from .sasrec import ce_loss

RMS_EPS = float(torch.finfo(torch.float32).eps)   # torch.nn.RMSNorm(eps=None) on the reference's fp32 activations
ENC = "body.encoder.layers."


def lambda_init(block: int) -> float:
    return 0.8 - 0.6 * math.exp(-0.3 * block)


def n_blocks_of(sd) -> int:
    n = 0
    while f"{ENC}{n}.attn.W_q.weight" in sd:
        n += 1
    return n


def rms_norm(x, w, eps=RMS_EPS):
    return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps) * w


def visible_mask(pad_mask):
    """[B, L, L]: key j visible to query i iff j <= i and (pad_mask[j] or j == i) (mask.py:29-51)"""
    L, dev = pad_mask.shape[1], pad_mask.device
    causal = torch.tril(torch.ones(L, L, dtype=torch.bool, device=dev))
    eye = torch.eye(L, dtype=torch.bool, device=dev)
    return causal.unsqueeze(0) & (pad_mask.unsqueeze(1) | eye.unsqueeze(0))


def diff_attention(x, sd, i, n_heads, visible, return_parts=False):
    """MultiHeadDifferentialAttention.forward (attention.py:86-157) of block ``i`` on x [B, L, d]."""
    p = f"{ENC}{i}.attn."
    B, L, d = x.shape
    hd = d // n_heads
    q = (x @ sd[p + "W_q.weight"].T).view(B, L, n_heads, 2 * hd).transpose(1, 2)
    k = (x @ sd[p + "W_k.weight"].T).view(B, L, n_heads, 2 * hd).transpose(1, 2)
    v = (x @ sd[p + "W_v.weight"].T).view(B, L, n_heads, 2 * hd).transpose(1, 2)
    q1, q2 = q.chunk(2, dim=-1)
    k1, k2 = k.chunk(2, dim=-1)
    li = lambda_init(i)
    lam = (torch.exp((sd[p + "lambda_q1"] * sd[p + "lambda_k1"]).sum(-1))
           - torch.exp((sd[p + "lambda_q2"] * sd[p + "lambda_k2"]).sum(-1)) + li)
    scale = 1.0 / math.sqrt(hd)
    m = torch.where(visible, 0.0, -torch.inf).to(x.dtype).unsqueeze(1)
    a1 = torch.softmax(q1 @ k1.transpose(-2, -1) * scale + m, dim=-1)
    a2 = torch.softmax(q2 @ k2.transpose(-2, -1) * scale + m, dim=-1)
    A = a1 - lam.view(1, n_heads, 1, 1) * a2
    o_pre = A @ v
    o = o_pre / torch.sqrt(o_pre.pow(2).mean(-1, keepdim=True) + 1e-5) * sd[p + "rms_scale"] * (1 - li)
    out = o.transpose(1, 2).reshape(B, L, 2 * d) @ sd[p + "W_o.weight"].T
    if return_parts:
        return out, dict(lam=lam, a1=a1, a2=a2, o_pre=o_pre, o=o)
    return out


def diff_block(x, sd, i, n_heads, visible):
    """DiffTransformerBlock.forward (diff_transformer.py): post-norm attention and SwiGLU."""
    p = f"{ENC}{i}."
    y = rms_norm(diff_attention(x, sd, i, n_heads, visible) + x, sd[p + "attn_norm.weight"])
    g = y @ sd[p + "ff.WG.weight"].T + sd[p + "ff.WG.bias"]
    lin = y @ sd[p + "ff.W1.weight"].T + sd[p + "ff.W1.bias"]
    ff = (torch.nn.functional.silu(g) * lin) @ sd[p + "ff.W2.weight"].T + sd[p + "ff.W2.bias"]
    return rms_norm(ff + y, sd[p + "ff_norm.weight"])


def diff_body(sd, ids, pad_mask, n_heads, lnf_eps=None, item_feature="item_id"):
    """Hidden states [B, L, d] of every position (dropout off).  The output normalization is LayerNorm when the state
    dict has ``body.output_normalization.bias``, RMSNorm otherwise; ``lnf_eps`` None = torch's default of either."""
    E = sd[f"body.embedder.feature_embedders.{item_feature}.emb.weight"]
    pe = sd["body.embedding_aggregator.pe.weight"]
    B, L = ids.shape
    d = E.shape[1]
    ids = ids.masked_fill(~pad_mask, E.shape[0] - 1)
    x = E[ids] * math.sqrt(d) + pe[pe.shape[0] - L:].unsqueeze(0)
    vis = visible_mask(pad_mask)
    for i in range(n_blocks_of(sd)):
        x = diff_block(x, sd, i, n_heads, vis)
    w = sd["body.output_normalization.weight"]
    if "body.output_normalization.bias" in sd:
        return torch.nn.functional.layer_norm(x, (d,), w, sd["body.output_normalization.bias"], 1e-5 if lnf_eps is None else lnf_eps)
    return rms_norm(x, w, RMS_EPS if lnf_eps is None else lnf_eps)


def params_of(sd):
    """the trainable entries of a reference state_dict (the ``scaling`` buffers excluded)"""
    return {k: v for k, v in sd.items() if not k.endswith(".attn.scaling")}


def loss_and_grads(sd, ids, pad_mask, labels, target_mask, n_heads, item_feature="item_id", loss_fn=None):
    """Full-catalog CE (or ``loss_fn(hidden, table)``) and its gradient with respect to every parameter; the pad row's
    gradient is zeroed (torch.nn.Embedding(padding_idx=...))."""
    P = {k: v.detach().clone().requires_grad_(True) for k, v in params_of(sd).items()}
    full = dict(sd, **P)
    h = diff_body(full, ids, pad_mask, n_heads, item_feature=item_feature)
    table = P[f"body.embedder.feature_embedders.{item_feature}.emb.weight"]
    n_items = table.shape[0] - 1
    loss = ce_loss(h, table[:n_items], labels, target_mask) if loss_fn is None else loss_fn(h, table[:n_items])
    loss.backward()
    G = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in P.items()}
    G[f"body.embedder.feature_embedders.{item_feature}.emb.weight"][-1].zero_()
    return loss.detach(), G


# ----------------------------------------------------------------------------------------------------------------------
# golden vectors (oracle/gen_diff_golden.py): the weights are not stored but drawn from a seed; the file keeps the reference's
# key list and a checksum of every tensor, and the gradients as bf16
# ----------------------------------------------------------------------------------------------------------------------


def seeded_state_dict(n_items, d, n_heads, max_len, n_blocks, norm, seed, item_feature="item_id"):
    """Weights under the reference's state_dict keys, drawn from a CPU torch.Generator: xavier-normal matrices (lambda_*
    included, as DiffTransformerLayer.reset_parameters), 1-D parameters at their init value (norm weights and rms_scale 1,
    biases 0) plus N(0, 0.05) noise, the item table's pad row zero, attn.scaling = 1/sqrt(head_dim)."""
    g = torch.Generator().manual_seed(seed)
    hd = d // n_heads

    def xav(r, c):
        return torch.randn(r, c, generator=g) * math.sqrt(2.0 / (r + c))

    def vec(n, base):
        return torch.full((n,), float(base)) + torch.randn(n, generator=g) * 0.05

    E = xav(n_items + 1, d)
    E[n_items] = 0
    sd = {f"body.embedder.feature_embedders.{item_feature}.emb.weight": E, "body.embedding_aggregator.pe.weight": xav(max_len, d)}
    for i in range(n_blocks):
        p = f"{ENC}{i}."
        sd.update({p + "attn.W_q.weight": xav(2 * d, d), p + "attn.W_k.weight": xav(2 * d, d), p + "attn.W_v.weight": xav(2 * d, d),
                   p + "attn.W_o.weight": xav(d, 2 * d)})
        for k in ("q1", "k1", "q2", "k2"):
            sd[p + "attn.lambda_" + k] = xav(n_heads, hd)
        sd[p + "attn.scaling"] = torch.tensor(1.0 / math.sqrt(hd), dtype=torch.float32)
        sd.update({p + "attn.rms_scale": vec(2 * hd, 1), p + "attn_norm.weight": vec(d, 1), p + "ff_norm.weight": vec(d, 1),
                   p + "ff.WG.weight": xav(2 * d, d), p + "ff.WG.bias": vec(2 * d, 0), p + "ff.W1.weight": xav(2 * d, d),
                   p + "ff.W1.bias": vec(2 * d, 0), p + "ff.W2.weight": xav(d, 2 * d), p + "ff.W2.bias": vec(d, 0)})
    sd["body.output_normalization.weight"] = vec(d, 1)
    if norm == "layernorm":
        sd["body.output_normalization.bias"] = vec(d, 0)
    return sd


def checksum(t) -> float:
    return float(t.double().sum())


def to_bf16_bits(t) -> np.ndarray:
    return t.detach().to(torch.bfloat16).view(torch.int16).numpy().copy()


def from_bf16_bits(a) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a)).view(torch.bfloat16).float()


def load_golden(path):
    """(npz, reference state_dict, reference gradients fp32 from bf16) of a golden file; raises if the seeded weights
    are not the ones the reference ran with"""
    z = np.load(path)
    sd = seeded_state_dict(int(z["n_items"]), int(z["d"]), int(z["H"]), int(z["L"]), int(z["n_blocks"]), str(z["norm"]),
                           int(z["seed"]))
    keys = [str(k) for k in z["sd_keys"]]
    if sorted(keys) != sorted(sd):
        raise ValueError(f"{path}: the seeded state_dict has other keys than the reference's")
    for k, c in zip(keys, z["sd_sums"]):
        if abs(checksum(sd[k]) - float(c)) > 1e-9 * max(1.0, abs(float(c))):
            raise ValueError(f"{path}: the seeded {k} differs from the weights the reference ran with")
    grads = {k[6:]: from_bf16_bits(z[k]) for k in z.files if k.startswith("grad::")}
    return z, sd, grads
