"""Attention with 128-wide head slots at 256 < L <= 512: rp_attn_fwd's attn_fwd_kernel<128, 2> (Q and K resident, V streamed
through a ring of 64-key stages), the un-fused backward that consumes its saved statistics, rp_attn_last at the same
lengths, and the SASRec / BERT4Rec engines and the legacy SasRec module at these shapes.

Kernel-level checks reuse the float64 reference, the inputs and the tolerances of test_gpu_attention.py; engine-level
checks compare against the oracle with the thresholds of test_head_slot_128_train_step_matches_oracle.
"""
import math

import numpy as np
import pytest
import torch

from dropout_stream import drop_keep
from test_gpu_attention import (CTR, MODES, OFF, P_DROP, SEED, SENT, SHARP, TOL_LAST, TOL_O, _attn_fwd, _attn_grads,
                                _attn_last, _case, _check_fwd, _check_grads, _cos, _d_out, _heads, _note, _pad_pattern,
                                _ref_scale, _row_err, attn_ref, block_err, visibility)

pytestmark = pytest.mark.gpu

HD = 128
_FWD_L = [257, 300, 383, 384, 449, 511, 512]   # 3 and 4 query tiles; 5 to 8 64-key chunks, ragged and whole


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda")


# ----------------------------------------------------------------------------------------------------------------------
# rp_attn_fwd
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("L", _FWD_L)
@pytest.mark.parametrize("mode", list(MODES))
def test_attn_fwd_hd128_long_matches_reference(cuda, mode, L):
    """out, m_save, inv_sum and p_save against attn_ref at the default and a sharp scale (including zeros above the
    diagonal and at masked keys, and nothing written past the heads); inference bitwise equal to training on every query
    tile with a real row and zero on all-padding tiles; bitwise equal reruns."""
    causal, mpk = MODES[mode]
    c = _case(_pad_pattern(L, bert=mode == "bert"), 2, HD, mpk, seed=7 * L + HD + 1, dev=cuda)
    B, d = c.B, c.d
    for scale in (0.0, SHARP / math.sqrt(HD)):
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


@pytest.mark.parametrize("L", [300, 512])
@pytest.mark.parametrize("mode", ["sasrec", "bert"])
def test_attn_fwd_hd128_long_dropout_matches_reference(cuda, mode, L):
    """Attention dropout p = 0.2 with the step counter behind seed_ptr: O equals attn_ref under the ported mask (the
    row keys bz * Lp + row, the column keys of every streamed chunk), and p_save / inv_sum hold the un-dropped values."""
    causal, mpk = MODES[mode]
    c = _case(_pad_pattern(L, bert=mode == "bert"), 2, HD, mpk, seed=11 * L + HD + 1, dev=cuda)
    ctr = torch.tensor([CTR], dtype=torch.int64, device=cuda)
    keep = drop_keep(SEED + CTR, OFF, P_DROP, c.B, c.H, L, c.Lp)
    res = _attn_fwd(c, causal, mpk, 0.0, drop=P_DROP, ctr=ctr)
    _check_fwd(c, causal, mpk, 0.0, res, keep=keep)


@pytest.mark.parametrize("L", [300, 512])
@pytest.mark.parametrize("hd_true", [96, 75])
def test_attn_fwd_hd128_long_scale_override_for_padded_head_slot(cuda, hd_true, L):
    """A 96- or 75-wide head in a 128-wide slot with scale = 1/sqrt(true width): the true-width attention, and the
    padded output columns stay exactly zero."""
    c = _case(_pad_pattern(L), 2, HD, 1, seed=L + hd_true + 1, hd_true=hd_true, dev=cuda)
    scale = 1.0 / math.sqrt(hd_true)
    _check_fwd(c, 1, 1, scale, _attn_fwd(c, 1, 1, scale))


# ----------------------------------------------------------------------------------------------------------------------
# the un-fused backward on the streamed forward's saves
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("drop", [0.0, P_DROP])
@pytest.mark.parametrize("variant", ["new", "legacy"])
@pytest.mark.parametrize("L", [300, 512])
@pytest.mark.parametrize("d,H", [(128, 1), (256, 2)])
def test_attention_drivers_hd128_long_backward_matches_autograd(cuda, d, H, L, variant, drop):
    """SasRecEngine._attention_forward / _attention_backward at head slot 128 and L > 256 (the streamed forward, then
    dPd = dO.V^T, rp_attn_softmax_bwd with four 128-column blocks and three batched GEMMs) on planted Q, K, V and dO:
    O, dQ, dK, dV against fp64 autograd per 64-row block."""
    from replay_b200.engine import EncoderConfig, SasRecEngine

    cfg = EncoderConfig(n_items=500, d=d, n_heads=H, n_blocks=1, max_len=L, dropout=drop, variant=variant)
    eng = SasRecEngine(cfg, 4, L, cuda, seed=SEED)
    assert cfg.head_slot == HD and not eng.fused_attn_bwd
    mpk = int(variant == "new")
    c = _case(_pad_pattern(L), H, d // H, mpk, seed=19 * L + d + 1, dev=cuda)
    a = eng.act[0]
    eng.in_pad.copy_(c.padd.view(-1))
    a["Q"].copy_(c.qd)
    a["KV"].copy_(c.kvd)
    eng.rng_counter.fill_(CTR)
    qkv = (a["Q"], 0), (a["KV"], 0), (a["KV"], d)
    eng._attention_forward(0, True, *qkv, causal=True, mask_pad_keys=bool(mpk))
    d_o = _d_out(c, seed=L + 1)
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
# rp_attn_last
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mpk", [0, 1])
@pytest.mark.parametrize("L", [257, 300, 511, 512])
def test_attn_last_hd128_long_matches_reference_and_fwd(cuda, L, mpk):
    """The last query row per (sequence, head) at head_dim 128 against attn_ref and against the last row of the streamed
    rp_attn_fwd on the same inputs; an all-padding sequence with masked pad keys gives exactly 0."""
    B, H = 5, 2
    c = _case(_pad_pattern(L, B=B), H, HD, mpk, seed=23 * L + HD + mpk + 1, dev=cuda)
    for scale in (0.0, SHARP / math.sqrt(HD)):
        out = _attn_last(c, mpk, scale)
        assert (out[B] == SENT).all()
        got = out[:B].cpu().double().view(B, H, HD)
        ref = attn_ref(c.q64, c.k64, c.v64, c.pad, 1, mpk, _ref_scale(c, scale))[0][:, :, -1]
        assert _note("last row", _row_err(got, ref)) < TOL_LAST
        if mpk:
            assert (got[~c.pad.any(-1)] == 0).all(), "an all-padding sequence must give exactly zero"
        fwd = _attn_fwd(c, 1, mpk, scale)[0].cpu().double()
        last = fwd.view(B, L, -1)[:, -1, : c.d].reshape(B, H, HD)
        assert _note("last vs fwd", _row_err(got, last)) < 2 * TOL_LAST


# ----------------------------------------------------------------------------------------------------------------------
# engines against the oracle
# ----------------------------------------------------------------------------------------------------------------------
def _named(P, name):
    """entry ``name`` of the engine's layout in an oracle parameter / gradient dict"""
    blk, _, leaf = name.partition(".")
    return P["blocks"][int(blk[1:])][leaf] if leaf else P[name]


def _check_grads_against(eng, G):
    """every parameter gradient at its true shape: cosine >= 0.99 and norm ratio within 4 % of the oracle's"""
    bad = []
    for name in eng.layout:
        a, b = eng.export_named(name, eng.grads).cpu(), _named(G, name)
        assert tuple(a.shape) == tuple(b.shape), name
        if b.norm() < 1e-12:
            assert a.norm() < 1e-6, name
            continue
        c, r = _cos(a, b), float(a.double().norm() / b.double().norm())
        if c < 0.99 or abs(r - 1) > 0.04:
            bad.append((name, round(c, 5), round(r, 4)))
    assert not bad, bad


def _oracle_grads(loss_fn, P):
    Pg = {k: ([{kk: vv.detach().clone().requires_grad_(True) for kk, vv in b.items()} for b in v] if k == "blocks"
              else v.detach().clone().requires_grad_(True)) for k, v in P.items()}
    loss = loss_fn(Pg)
    loss.backward()
    grad = lambda t: t.grad if t.grad is not None else torch.zeros_like(t)  # noqa: E731
    G = {k: ([{kk: grad(vv) for kk, vv in b.items()} for b in v] if k == "blocks" else grad(v)) for k, v in Pg.items()}
    return float(loss.detach()), G


@pytest.mark.parametrize("variant,d,H,L", [("new", 128, 1, 512), ("legacy", 100, 1, 384)])
def test_sasrec_hd128_long_train_step_and_predict_match_oracle(cuda, variant, d, H, L):
    """SASRec at head slot 128 and L > 256 (new path d = 128 at L = 512; legacy hidden 100 in a 128 slot at L = 384):
    hidden states, loss, every parameter gradient, the predict-path last hidden state, and top-10 with the seen filter
    against the oracle.  The first 128-row query tile of sequence 0 is all padding."""
    from oracle import sasrec as osr
    from replay_b200 import ops
    from replay_b200.engine import EncoderConfig, SasRecEngine
    from replay_b200.synthetic import make_sequences

    B, I = 3, 1500
    P = osr.random_params(I, d, L, 2, seed=29)
    ids, pm, lab, tm = make_sequences(B, I, L, seed=6)
    ids[0, :150], pm[0, :150] = I, False
    lab[0, :149], tm[0, :149] = I, False
    cfg = EncoderConfig(n_items=I, d=d, n_heads=H, n_blocks=2, max_len=L, dropout=0.0, variant=variant)
    eng = SasRecEngine(cfg, B, L, cuda)
    assert cfg.head_slot == HD and cfg.hd_valid == (0 if d == HD else d) and not eng.fused_attn_bwd
    eng.load_canonical(P)
    eng.set_batch(ids.cuda(), pm.cuda(), lab.cuda(), tm.cuda())
    hid = eng.unpad_features(eng.forward_hidden_all()).float().cpu().view(B, L, d)
    ref_h = osr.sasrec_body(P, ids, pm, H, variant)
    assert (hid - ref_h).abs().max() < 8e-2, (hid - ref_h).abs().max()
    loss = eng.forward_train()
    ref_loss, G = osr.loss_and_grads(P, ids, pm, lab, tm, H, variant)
    assert abs(loss[0].item() - float(ref_loss)) < 5e-3 * float(ref_loss), (loss[0].item(), float(ref_loss))
    eng.g32.zero_()
    eng.backward()
    torch.cuda.synchronize()
    _check_grads_against(eng, G)
    eng.set_batch(ids.cuda(), pm.cuda())
    hq = eng.forward_last_hidden()
    ref_e = osr.sasrec_body(P, ids, pm, H, variant, mode="eval")[:, -1]
    assert (eng.unpad_features(hq).float().cpu() - ref_e).abs().max() < 8e-2
    table = eng.params16["item_emb"][:I]
    ids_k, _ = ops.score_topk(hq, table, 10, ops.seen_prepare(ids.cuda(), I))
    ids_o, _ = osr.score_topk(hq.float().cpu(), table.float().cpu(), ids, 10)
    assert torch.equal(ids_k.cpu(), ids_o)


def _bert_params(I, d, L, n_blocks, seed):
    """random BERT4Rec parameters in the oracle's canonical layout (untied head with bias)"""
    g = torch.Generator().manual_seed(seed)

    def xn(*shape):
        return torch.randn(*shape, generator=g) * math.sqrt(2.0 / (shape[0] + shape[1]))

    def small(n):
        return torch.randn(n, generator=g) * 0.02

    P = {"item_emb": xn(I, d), "mask_emb": xn(1, d), "pos_emb": xn(L, d), "blocks": [], "head_w": xn(I, d), "head_b": small(I)}
    for _ in range(n_blocks):
        P["blocks"].append({"ln1_w": 1 + small(d), "ln1_b": small(d), "in_w": xn(3 * d, d), "in_b": small(3 * d),
                            "out_w": xn(d, d), "out_b": small(d), "ln2_w": 1 + small(d), "ln2_b": small(d),
                            "w1": xn(4 * d, d), "b1": small(4 * d), "w2": xn(d, 4 * d), "b2": small(d)})
    return P


def test_bert4rec_300h4_long_train_step_and_predict_match_oracle(cuda):
    """BERT4Rec at the tutorial's hidden 300 / 4 heads (head_dim 75 in 128-wide slots) with a 512-item window: hidden
    states on real rows, loss, every parameter gradient, the predict-path hidden state of the shifted window, and top-10
    with the seen filter against a float64 ranking of the same bf16 query rows and head."""
    from oracle import bert4rec as ob
    from oracle import sasrec as osr
    from replay_b200 import ops
    from replay_b200.engine_bert import Bert4RecEngine, BertConfig

    B, L, d, H, I = 3, 512, 300, 4, 700
    P = _bert_params(I, d, L, 2, seed=37)
    g = torch.Generator().manual_seed(38)
    ids = torch.randint(0, I, (B, L), generator=g)
    pm = torch.ones(B, L, dtype=torch.bool)
    pm[0, :150] = False                       # the first 128-row query tile of sequence 0 is all padding
    pm[2] = torch.rand(L, generator=g) > 0.3  # interior holes
    ids = ids.masked_fill(~pm, 0)
    tok = pm & (torch.rand(B, L, generator=g) > 0.2)
    cfg = BertConfig(n_items=I, d=d, n_heads=H, n_blocks=2, max_len=L, dropout=0.0)
    eng = Bert4RecEngine(cfg, B, L, cuda)
    assert cfg.head_slot == HD and cfg.hd_valid == 75 and not eng.fused_attn_bwd
    eng.load_canonical(P)
    eng.set_batch(ids.cuda(), pm.cuda(), tok.cuda(), ids.cuda())
    hid = eng.unpad_features(eng.forward_hidden_all()).float().cpu().view(B, L, d)
    ref_h = ob.bert4rec_body(P, ids, pm, tok, H)
    assert (hid[pm] - ref_h[pm]).abs().max() < 8e-2, (hid[pm] - ref_h[pm]).abs().max()
    loss = eng.forward_train()
    ref_loss, G = _oracle_grads(lambda Q: ob.train_loss(Q, ids, pm, tok, ids, H), P)
    assert abs(loss[0].item() - ref_loss) < 5e-3 * ref_loss, (loss[0].item(), ref_loss)
    eng.g32.zero_()
    eng.backward()
    torch.cuda.synchronize()
    _check_grads_against(eng, G)
    sids, spm, stm = ob.shift_for_predict(ids, pm, pm)
    eng.set_batch(sids.cuda(), spm.cuda(), stm.cuda())
    hq = eng.forward_last_hidden()
    ref_e = ob.bert4rec_body(P, sids, spm, stm, H)[:, -1]
    assert (eng.unpad_features(hq).float().cpu() - ref_e).abs().max() < 8e-2
    W, bias = eng.head_for_scoring()
    ids_k, _ = ops.score_topk(hq, W, 10, ops.seen_prepare(ids.cuda(), I), bias=bias)
    logits = hq.double().cpu() @ W.double().cpu().T + bias[:I].double().cpu()
    ref = torch.argsort(-osr.seen_filter(logits, ids, I), dim=1, stable=True)[:, :10]
    assert torch.equal(ids_k.cpu(), ref)


# ----------------------------------------------------------------------------------------------------------------------
# the public module
# ----------------------------------------------------------------------------------------------------------------------
def test_legacy_sasrec_module_trains_and_predicts_at_L512(cuda):
    """The legacy SasRec with the reference's head_count=1 and hidden 100 (one 128-wide slot, 28 padded columns) at
    max_seq_len=512 and dropout 0.2: CUDA-graph training steps lower the loss; padded columns of every parameter,
    gradient and Adam moment stay exactly zero; predict_topk returns valid, distinct ids."""
    from replay_b200.models.nn.sequential import SasRec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema
    from replay_b200.synthetic import make_sequences

    n_items, d, L, B = 2000, 100, 512, 16
    torch.manual_seed(0)
    m = SasRec(TensorSchema(TensorFeatureInfo("item_id", n_items, 0, d)), block_count=2, head_count=1, hidden_size=d,
               max_seq_len=L, dropout_rate=0.2)
    ids, pm, lab, tm = make_sequences(B, n_items, L, seed=12)
    batch = {"feature_tensor": {"item_id": ids.cuda()}, "padding_mask": pm.cuda(),
             "positive_labels": lab.clamp(max=n_items - 1).cuda(), "target_padding_mask": tm.cuda()}
    losses = [float(m.training_step(batch, i)) for i in range(30)]
    assert all(np.isfinite(losses)) and np.mean(losses[-5:]) < np.mean(losses[:5]) - 0.3, (losses[:5], losses[-5:])
    eng = m._model.core.engine
    assert eng.cfg.head_slot == HD and eng.cfg.hd_valid == d and eng.L == L
    for name in eng.layout:
        real = torch.zeros(eng.layout[name][1], dtype=torch.bool, device=cuda)
        rk, ck = eng._pad_kind(name)
        rows = eng._axis_index(rk) if rk else torch.arange(real.shape[0], device=cuda)
        if real.dim() == 1:
            real[rows] = True
        else:
            cols = eng._axis_index(ck) if ck else torch.arange(real.shape[1], device=cuda)
            real[rows[:, None], cols[None, :]] = True
        o, shp = eng.layout[name]
        n = torch.Size(shp).numel()
        for flat, what in ((eng.p32, "param"), (eng.g32, "grad"), (eng.adam_m, "adam_m"), (eng.adam_v, "adam_v")):
            assert not flat[o:o + n].view(shp)[~real].any(), (what, name)
    m.eval()
    top, _ = m.predict_topk({"feature_tensor": {"item_id": ids.cuda()}, "padding_mask": pm.cuda()}, 10, seen_ids=ids.cuda())
    top = top.cpu()
    assert top.shape == (B, 10) and ((top >= 0) & (top < n_items)).all()
    assert all(len(set(r.tolist())) == 10 for r in top)
