"""Plain-torch restatement of RePlay's TiSASRec (the legacy SasRecModel(ti_modification=True)) - TEST INFRASTRUCTURE.

Reference restated: replay/models/nn/sequential/sasrec/model.py TiSasRecEmbeddings (532-646), TiSasRecLayers (649-707),
TiSasRecAttention (710-800), SasRecPointWiseFeedForward, SasRecNormalizer; loss as oracle.sasrec.ce_loss.

Canonical parameter dict ``P`` (the layout of replay_b200.engine_tisasrec, true shapes)::

    item_emb [I+1, d]  pos_k [Lmax, d]  pos_v [Lmax, d]  time_k [span+1, d]  time_v [span+1, d]
    blocks: ln1_w ln1_b qw[d,d] kw vw qb[d] kb vb ln2_w ln2_b w1[d,d] b1 w2[d,d] b2
    lnf_w lnf_b
Computed in the dtype of the parameters handed in.  Dropout is given as explicit keep factors (0 or 1/(1-p)) so that a test
can replay the masks the kernels drew; None means no dropout.
"""
import torch

from .sasrec import ce_loss, layer_norm

_BLOCK = ("ln1_w", "ln1_b", "qw", "kw", "vw", "qb", "kb", "vb", "ln2_w", "ln2_b", "w1", "b1", "w2", "b2")


def time_matrix(times, span):
    """r[b, i, j] = min(floor(|t_bi - t_bj|), span) in the timestamps' own dtype; int64 skips the floor."""
    r = torch.abs(times.unsqueeze(-1) - times.unsqueeze(1))
    if r.dtype != torch.int64:
        r = torch.floor(r).long()
    return r.masked_fill(r > span, span)


def random_params(n_items, d, max_len, n_blocks, span, seed=0, dtype=torch.float32, bias_scale=0.05):
    g = torch.Generator().manual_seed(seed)

    def xavier(*shape):
        return torch.randn(*shape, generator=g) * (2.0 / (shape[0] + shape[1])) ** 0.5

    def vec(base=0.0):
        return base + torch.randn(d, generator=g) * bias_scale

    P = {"item_emb": xavier(n_items + 1, d), "pos_k": xavier(max_len, d), "pos_v": xavier(max_len, d),
         "time_k": xavier(span + 1, d), "time_v": xavier(span + 1, d), "blocks": []}
    for _ in range(n_blocks):
        P["blocks"].append({"ln1_w": vec(1.0), "ln1_b": vec(), "qw": xavier(d, d), "kw": xavier(d, d), "vw": xavier(d, d),
                            "qb": vec(), "kb": vec(), "vb": vec(), "ln2_w": vec(1.0), "ln2_b": vec(), "w1": xavier(d, d),
                            "b1": vec(), "w2": xavier(d, d), "b2": vec()})
    P["lnf_w"], P["lnf_b"] = vec(1.0), vec()
    return params_to(P, dtype)


def params_to(P, dtype):
    return {k: ([{kk: vv.to(dtype) for kk, vv in b.items()} for b in v] if k == "blocks" else v.to(dtype)) for k, v in P.items()}


def params_from_state_dict(sd):
    """reference SasRecModel(ti_modification=True).state_dict() -> canonical dict"""
    e = "item_embedder."
    P = {"item_emb": sd[e + "item_emb.weight"], "pos_k": sd[e + "abs_pos_k_emb.pe.weight"],
         "pos_v": sd[e + "abs_pos_v_emb.pe.weight"], "time_k": sd[e + "time_matrix_k_emb.weight"],
         "time_v": sd[e + "time_matrix_v_emb.weight"], "lnf_w": sd["output_normalization.last_layernorm.weight"],
         "lnf_b": sd["output_normalization.last_layernorm.bias"], "blocks": []}
    i = 0
    while f"sasrec_layers.attention_layernorms.{i}.weight" in sd:
        s = "sasrec_layers."
        blk = {"ln1_w": sd[f"{s}attention_layernorms.{i}.weight"], "ln1_b": sd[f"{s}attention_layernorms.{i}.bias"],
               "ln2_w": sd[f"{s}forward_layernorms.{i}.weight"], "ln2_b": sd[f"{s}forward_layernorms.{i}.bias"]}
        for k, m in (("q", "query_w"), ("k", "key_w"), ("v", "value_w")):
            blk[k + "w"], blk[k + "b"] = sd[f"{s}attention_layers.{i}.{m}.weight"], sd[f"{s}attention_layers.{i}.{m}.bias"]
        for k in ("1", "2"):
            blk["w" + k] = sd[f"{s}forward_layers.{i}.conv{k}.weight"][:, :, 0]
            blk["b" + k] = sd[f"{s}forward_layers.{i}.conv{k}.bias"]
        P["blocks"].append(blk)
        i += 1
    return P


def time_attention(q, k, v, r, time_k, time_v, pad_mask, n_heads, keep_att=None, keep_tk=None, keep_tv=None):
    """TiSasRecAttention's core after the projections.  q, k, v [B, L, d] with k, v already holding the dropped positional
    terms; r [B, L, L] intervals; time_k / time_v [span+1, d]; pad_mask bool [B, L].  keep_att [B, H, L, L], keep_tk /
    keep_tv [B, L, L, d]: dropout keep factors.  Padded query rows get the reference's uniform row (their output is
    zeroed by the block).  Returns o [B, L, d]."""
    B, L, d = q.shape
    hs = d // n_heads
    TK, TV = time_k[r], time_v[r]                        # [B, L, L, d]: affordable at test sizes only
    if keep_tk is not None:
        TK, TV = TK * keep_tk, TV * keep_tv
    qh = q.view(B, L, n_heads, hs).transpose(1, 2)       # [B, H, L, hs]
    kh = k.view(B, L, n_heads, hs).transpose(1, 2)
    vh = v.view(B, L, n_heads, hs).transpose(1, 2)
    TKh = TK.view(B, L, L, n_heads, hs).permute(0, 3, 1, 2, 4)   # [B, H, L, L, hs]
    TVh = TV.view(B, L, L, n_heads, hs).permute(0, 3, 1, 2, 4)
    s = qh @ kh.transpose(-1, -2) + (TKh @ qh.unsqueeze(-1)).squeeze(-1)
    s = s / hs ** 0.5
    causal = torch.ones(L, L, dtype=torch.bool, device=q.device).triu(1)
    masked = causal[None, None] | ~pad_mask[:, None, :, None]
    s = torch.where(masked, torch.full_like(s, -(2.0 ** 32) + 1), s)
    a = torch.softmax(s, dim=-1)
    if keep_att is not None:
        a = a * keep_att
    o = a @ vh + (a.unsqueeze(-2) @ TVh).squeeze(-2)
    return o.transpose(1, 2).reshape(B, L, d)


def body(P, ids, pad_mask, times, n_heads, span, keep=None):
    """Hidden states after the final LayerNorm, [B, L, d].  keep: dict of keep factors (see time_attention and the
    embedder's: item [B, L, d], pos_k / pos_v [B, L, d]; per block: att [B, H, L, L], ffn1 / ffn2 [B, L, d]) or None."""
    keep = keep or {}
    n_items = P["item_emb"].shape[0] - 1
    d = P["item_emb"].shape[1]
    B, L = ids.shape
    ids = ids.masked_fill(~pad_mask, n_items)
    pm = pad_mask.unsqueeze(-1).to(P["item_emb"].dtype)
    x = P["item_emb"][ids] * d ** 0.5
    if "item" in keep:
        x = x * keep["item"]
    x = x * pm
    pk = P["pos_k"][:L].expand(B, L, d)
    pv = P["pos_v"][:L].expand(B, L, d)
    if "pos_k" in keep:
        pk, pv = pk * keep["pos_k"], pv * keep["pos_v"]
    r = time_matrix(times, span)
    for i, blk in enumerate(P["blocks"]):
        kb = keep.get("blocks", [{}] * len(P["blocks"]))[i]
        q_in = layer_norm(x, blk["ln1_w"], blk["ln1_b"], 1e-8)
        q = q_in @ blk["qw"].T + blk["qb"]
        k = x @ blk["kw"].T + blk["kb"] + pk
        v = x @ blk["vw"].T + blk["vb"] + pv
        o = time_attention(q, k, v, r, P["time_k"], P["time_v"], pad_mask, n_heads, kb.get("att"), keep.get("time_k"),
                           keep.get("time_v"))
        y = layer_norm(q_in + o, blk["ln2_w"], blk["ln2_b"], 1e-8)
        u = torch.relu(y @ blk["w1"].T + blk["b1"])
        if "ffn1" in kb:
            u = u * kb["ffn1"]
        z = u @ blk["w2"].T + blk["b2"]
        if "ffn2" in kb:
            z = z * kb["ffn2"]
        x = (z + y) * pm
    return layer_norm(x, P["lnf_w"], P["lnf_b"], 1e-8)


def train_loss(P, ids, pad_mask, times, labels, target_mask, n_heads, span, keep=None):
    n_items = P["item_emb"].shape[0] - 1
    return ce_loss(body(P, ids, pad_mask, times, n_heads, span, keep), P["item_emb"][:n_items], labels, target_mask)


def loss_and_grads(P, ids, pad_mask, times, labels, target_mask, n_heads, span, keep=None):
    """Loss and d(loss)/d(param) by autograd; the item table's padding row is frozen (Embedding(padding_idx=...))."""
    Pg = {k: ([{kk: vv.detach().clone().requires_grad_(True) for kk, vv in b.items()} for b in v] if k == "blocks"
              else v.detach().clone().requires_grad_(True)) for k, v in P.items()}
    loss = train_loss(Pg, ids, pad_mask, times, labels, target_mask, n_heads, span, keep)
    loss.backward()
    G = {k: ([{kk: vv.grad if vv.grad is not None else torch.zeros_like(vv) for kk, vv in b.items()} for b in v]
             if k == "blocks" else (v.grad if v.grad is not None else torch.zeros_like(v))) for k, v in Pg.items()}
    G["item_emb"][-1].zero_()
    return loss.detach(), G
