"""BERT4Rec at any hidden size and head count, without a GPU: the feature-slot geometry of BertConfig, the float64 BERT4Rec of
oracle/bert4rec.py against the real reference at padded shapes (tests/golden/bert4rec_d*.npz, tools/gen_bert_shapes_golden.py),
the module surface, and the C ABI's argument errors of the biased d = 512 heads."""
import os

import numpy as np
import pytest
import torch

from bert_shapes_golden import SHAPES, load, unpack_grads


# (d, H) -> (head_dim, slot, dp, hd_valid, FFN inner columns): EncoderConfig's slots, the inner axis rounded up to 128
GEOMETRY = [((64, 1), (64, 64, 64, 0, 256)), ((128, 2), (64, 64, 128, 0, 512)), ((256, 4), (64, 64, 256, 0, 1024)),
            ((256, 2), (128, 128, 256, 0, 1024)), ((512, 8), (64, 64, 512, 0, 2048)), ((512, 4), (128, 128, 512, 0, 2048)),
            ((300, 4), (75, 128, 512, 75, 1280)), ((96, 2), (48, 64, 128, 48, 384)), ((64, 4), (16, 64, 256, 16, 256)),
            ((192, 4), (48, 64, 256, 48, 768)), ((50, 1), (50, 64, 64, 50, 256)), ((100, 2), (50, 64, 128, 50, 512)),
            ((320, 4), (80, 128, 512, 80, 1280))]


@pytest.mark.parametrize("dh,geo", GEOMETRY, ids=[f"d{d}h{h}" for (d, h), _ in GEOMETRY])
def test_bert_config_geometry(dh, geo):
    from replay_b200.engine import EncoderConfig
    from replay_b200.engine_bert import BertConfig

    d, H = dh
    c = BertConfig(n_items=10, d=d, n_heads=H, n_blocks=1, max_len=8)
    assert (c.head_dim, c.head_slot, c.dp, c.hd_valid, c.ffn_p) == geo
    assert c.ffn == 4 * d and c.ffn_p % 128 == 0 and c.ffn_p <= 4 * c.dp   # fits the weight-gradient workspace
    e = EncoderConfig(n_items=10, d=d, n_heads=H, n_blocks=1, max_len=8)
    assert (e.head_dim, e.head_slot, e.dp, e.hd_valid) == geo[:4]
    assert torch.equal(c.feat_index(), e.feat_index())


@pytest.mark.parametrize("d,H", [(300, 2), (640, 8), (300, 7), (100, 3), (1024, 8)])
def test_bert_config_rejects(d, H):
    """300 / 2: head_dim 150 > 128; 640 / 8: 8 slots of 128 = 1024 columns; d % H != 0; 1024 / 8: 1024 columns."""
    from replay_b200.engine import EncoderConfig
    from replay_b200.engine_bert import BertConfig

    with pytest.raises(ValueError) as eb:
        BertConfig(n_items=10, d=d, n_heads=H, n_blocks=1, max_len=8)
    with pytest.raises(ValueError) as ee:
        EncoderConfig(n_items=10, d=d, n_heads=H, n_blocks=1, max_len=8)
    assert str(eb.value) == str(ee.value)   # one layout rule, one wording


def test_bert4rec_module_constructs_at_the_tutorial_shape():
    """The reference tutorial's Bert4Rec(hidden_size=300, head_count=4), with the BCE head too (biased, 512 padded columns)."""
    from replay_b200.models.nn.sequential import Bert4Rec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    schema = TensorSchema(TensorFeatureInfo("item_id", 1000, 0, 300))
    for lt in ("CE", "BCE"):
        m = Bert4Rec(schema, block_count=2, head_count=4, max_seq_len=100, hidden_size=300, dropout_rate=0.5, loss_type=lt,
                     device="cpu")
        assert m._model.core.cfg.dp == 512 and m._model.core.loss_kind == lt.lower()
    with pytest.raises(ValueError):
        Bert4Rec(schema, block_count=2, head_count=2, hidden_size=300, device="cpu")


def _leaf(P):
    return {k: ([{kk: vv.double().requires_grad_() for kk, vv in b.items()} for b in v] if k == "blocks"
                else v.double().requires_grad_()) for k, v in P.items()}


def _close(got, ref, rtol):
    got, ref = got.detach().double(), ref.double()
    assert got.shape == ref.shape, (got.shape, ref.shape)
    err = float((got - ref).abs().max())
    assert err <= rtol * float(ref.abs().max()) + 1e-9, (err, float(ref.abs().max()))


def _oracle(golden_dir, tag):
    from oracle import bert4rec as ob

    z, sd, grads = load(os.path.join(golden_dir, f"bert4rec_{tag}.npz"))
    P = _leaf(ob.params_from_state_dict(sd))
    ids, pm, tok = (torch.from_numpy(z[k]) for k in ("ids", "pad_mask", "token_mask"))
    h = ob.bert4rec_body(P, ids, pm, tok, int(z["H"]))
    W, b = ob.head_weights(P)
    sel = pm & ~tok
    return z, P, h, h[sel] @ W.T + b, torch.from_numpy(z["labels"])[sel], grads


@pytest.mark.parametrize("tag", list(SHAPES))
def test_oracle_matches_reference_at_padded_shapes(golden_dir, tag):
    """Loss, hidden states and EVERY gradient of the float64 BERT4Rec against the reference (fp32 run, fp16-packed gradients:
    2^-11 of the largest entry; large matrices on their stored rows)."""
    z, P, h, logits, y, grads = _oracle(golden_dir, tag)
    d, H = SHAPES[tag][:2]
    assert (int(z["d"]), int(z["H"])) == (d, H)
    _close(h, torch.from_numpy(z["train_hidden"]), 1e-5)
    loss = torch.nn.functional.cross_entropy(logits, y)
    loss.backward()
    assert abs(float(loss.detach()) - float(z["train_loss"])) <= 1e-6 * float(z["train_loss"])
    got = _grads_by_key(P, int(z["tying"]))
    assert set(got) == set(grads)
    for k, (rows, ref) in grads.items():
        _close(got[k] if rows is None else got[k][rows], ref, 2e-3)


def _grads_by_key(P, tying):
    """the oracle's gradients under the reference's state_dict keys (params_from_state_dict inverted)"""
    out = {"item_embedder.cat_embeddings.item_id.weight": P["item_emb"].grad, "item_embedder.mask_embedding.weight": P["mask_emb"].grad,
           "item_embedder.position.pe.weight": P["pos_emb"].grad}
    leaf = {"ln1_w": "attention_norm.weight", "ln1_b": "attention_norm.bias", "in_w": "attention.in_proj_weight",
            "in_b": "attention.in_proj_bias", "out_w": "attention.out_proj.weight", "out_b": "attention.out_proj.bias",
            "ln2_w": "pff_norm.weight", "ln2_b": "pff_norm.bias", "w1": "pff.w_1.weight", "b1": "pff.w_1.bias",
            "w2": "pff.w_2.weight", "b2": "pff.w_2.bias"}
    for i, b in enumerate(P["blocks"]):
        out.update({f"transformer_blocks.{i}.{leaf[k]}": v.grad for k, v in b.items()})
    if tying:
        out["_head.out_bias"] = P["head_b"].grad
    else:
        out["_head.linear.weight"], out["_head.linear.bias"] = P["head_w"].grad, P["head_b"].grad
    return out


def test_oracle_bce_matches_reference_at_the_tutorial_shape(golden_dir):
    """Bert4Rec(loss_type="BCE") at 300 / 4: loss and the item table, in_proj, head weight and bias gradients."""
    z, P, h, logits, y, _ = _oracle(golden_dir, "d300h4")
    zb = np.load(os.path.join(golden_dir, "bert4rec_bce_d300h4.npz"))
    loss = (torch.nn.functional.softplus(logits).sum() - logits.gather(1, y[:, None]).sum()) / logits.shape[0]
    loss.backward()
    assert abs(float(loss.detach()) - float(zb["train_loss"])) <= 1e-6 * float(zb["train_loss"])
    g = _grads_by_key(P, 0)
    packed = unpack_grads(zb)
    assert len(packed) == 4
    for k, (rows, ref) in packed.items():
        _close(g[k] if rows is None else g[k][rows], ref, 2e-3)


def test_c_abi_biased_wide_head_argument_errors():
    """d = 512 with a bias: NULL arguments and a bias without d_bias (or the reverse) are EINVAL, decided before any CUDA
    call (the BCE backward checks its buffers and workspace size first, then the pair)."""
    import ctypes

    from replay_b200._lib import lib

    L = lib()
    EINVAL = -1
    buf = ctypes.create_string_buffer(64)
    p = ctypes.cast(buf, ctypes.c_void_p)
    big = 1 << 50
    assert L.rp_ce_head_bwd(None, None, p, None, None, 128, 100, 512, None, None, None, None, p, 0, 0, p, big, None) == EINVAL
    assert L.rp_ce_head_bwd(p, p, p, p, p, 128, 100, 512, p, p, p, p, None, 0, 0, p, big, None) == EINVAL   # bias, no d_bias
    assert L.rp_ce_head_bwd(p, p, None, p, p, 128, 100, 512, p, p, p, p, p, 0, 0, p, big, None) == EINVAL   # d_bias, no bias
    assert L.rp_bce_head_bwd(None, None, p, None, None, 128, 100, 512, None, None, None, p, 0, 0, p, big, None) == EINVAL
    assert L.rp_bce_head_bwd(p, p, p, p, p, 128, 100, 512, p, p, p, None, 0, 0, p, big, None) == EINVAL
    assert L.rp_bce_head_bwd(p, p, None, p, p, 128, 100, 512, p, p, p, p, 0, 0, p, big, None) == EINVAL
    assert L.rp_bce_head_fwd(None, p, p, p, p, 128, 100, 512, p, None, 0, p, big, None) == EINVAL
