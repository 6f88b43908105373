"""GPU parity of BERT4Rec at hidden sizes that the kernels see padded (300 / 4, 96 / 2 tied, 64 / 4) and at 512 / 8 with its
biased d = 512 head, against the real reference (tests/golden/bert4rec_d*.npz, tools/gen_bert_shapes_golden.py).  Tolerances
as in test_gpu_bert4rec.py.  Padded feature columns and the FFN's padded inner columns must stay exactly zero in every
parameter, gradient and Adam moment through training."""
import os

import pytest
import torch

from bert_shapes_golden import SHAPES, load

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda")


def _cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def _engine(golden_dir, tag, cuda, dropout=0.0, with_grad=True):
    from oracle import bert4rec as ob
    from replay_b200.engine_bert import Bert4RecEngine, BertConfig

    z, sd, grads = load(os.path.join(golden_dir, f"bert4rec_{tag}.npz"))
    P = ob.params_from_state_dict(sd)
    B, L = z["ids"].shape
    cfg = BertConfig(n_items=int(z["n_items"]), d=int(z["d"]), n_heads=int(z["H"]), n_blocks=int(z["n_blocks"]), max_len=L,
                     dropout=dropout, tying=bool(int(z["tying"])))
    eng = Bert4RecEngine(cfg, B, L, cuda, with_grad=with_grad)
    eng.load_canonical(P)
    return z, sd, grads, P, eng


def _batch(z, cuda):
    return tuple(torch.from_numpy(z[k]).to(cuda) for k in ("ids", "pad_mask", "token_mask", "labels"))


def _pad_mask_of(eng, name):
    """True on the padded entries of parameter ``name`` (feature slots, FFN inner tail, head bias tail)"""
    real = torch.zeros(eng.layout[name][1], dtype=torch.bool, device=eng.dev)
    rk, ck = eng._pad_kind(name)
    rows = eng._axis_index(rk) if rk else torch.arange(real.shape[0], device=eng.dev)
    if real.dim() == 1:
        real[rows] = True
    else:
        cols = eng._axis_index(ck) if ck else torch.arange(real.shape[1], device=eng.dev)
        real[rows[:, None], cols[None, :]] = True
    return ~real


@pytest.mark.parametrize("tag", list(SHAPES))
def test_engine_step_matches_reference(golden_dir, cuda, tag):
    """Hidden states on real rows, n_valid, the loss and EVERY gradient (at the true shapes) against the reference."""
    from replay_b200.models.nn.sequential.bert4rec import bert_key_map

    z, sd, grads, P, eng = _engine(golden_dir, tag, cuda)
    ids, pm, tok, labels = _batch(z, cuda)
    B, L = ids.shape
    eng.set_batch(ids, pm, tok, labels)
    hid = eng.unpad_features(eng.forward_hidden_all()).float().cpu().view(B, L, -1)
    ref_h = torch.from_numpy(z["train_hidden"])
    real = torch.from_numpy(z["pad_mask"])
    assert hid.shape[-1] == int(z["d"])
    assert (hid[real] - ref_h[real]).abs().max() < 6e-2
    loss = eng.forward_train()
    torch.cuda.synchronize()
    ref_loss = float(z["train_loss"])
    assert abs(loss[0].item() - ref_loss) < 5e-3 * ref_loss, (loss[0].item(), ref_loss)
    assert int(eng.n_valid.item()) == int((real & ~torch.from_numpy(z["token_mask"])).sum())
    eng.g32.zero_()
    eng.backward()
    torch.cuda.synchronize()
    keymap = bert_key_map(eng.cfg.n_blocks, eng.cfg.tying)
    assert set(keymap.values()) == set(grads)   # every gradient of the model
    bad = []
    for nm, rk in keymap.items():
        a = eng.export_named(nm, eng.grads).cpu()
        assert tuple(a.shape) == eng.true_shape(nm) == tuple(sd[rk].shape), nm
        rows, b = grads[rk]
        if rows is not None:   # large matrices: the stored rows (all columns)
            a = a[rows]
        assert a.shape == b.shape, (nm, a.shape, b.shape)
        if b.norm() < 1e-12:
            assert a.norm() < 1e-6, nm
            continue
        c, r = _cos(a, b), float(a.double().norm() / b.double().norm())
        if c < 0.995 or abs(r - 1) > 0.03:
            bad.append((nm, round(c, 5), round(r, 4)))
    assert not bad, bad
    # padded entries of every gradient are exactly zero
    for name in eng.layout:
        assert not eng.grads[name][_pad_mask_of(eng, name)].any(), name


@pytest.mark.parametrize("tag", ["d300h4", "d96h2_tied", "d512h8"])
def test_padded_columns_stay_zero_through_fused_steps(golden_dir, cuda, tag):
    """Two fused steps (forward + backward + Adam) with dropout 0.1: padded columns of every parameter, gradient and both
    Adam moments are exactly 0, and the true entries moved."""
    z, sd, grads, P, eng = _engine(golden_dir, tag, cuda, dropout=0.1)
    ids, pm, tok, labels = _batch(z, cuda)
    before = eng.p32.clone()
    for _ in range(2):
        eng.set_batch(ids, pm, tok, labels)
        loss = eng.train_step()
    torch.cuda.synchronize()
    assert torch.isfinite(loss).all()
    moved = False
    for name in eng.layout:
        pad = _pad_mask_of(eng, name)
        for buf, what in ((eng.params, "param"), (eng.grads, "grad")):
            assert not buf[name][pad].any(), (what, name)
        o, shp = eng.layout[name]
        n = torch.Size(shp).numel()
        for flat, what in ((eng.adam_m, "adam_m"), (eng.adam_v, "adam_v"), (eng.p16.float(), "bf16 shadow")):
            assert not flat[o:o + n].view(shp)[pad].any(), (what, name)
        moved |= bool((eng.params[name] != before[o:o + n].view(shp)).any())
    assert moved
    if eng.cfg.hd_valid:
        # activations: padded feature columns of the last block's output and of the head's input rows
        nv = int(eng.n_valid.item())
        padcol = torch.ones(eng.cfg.dp, dtype=torch.bool, device=cuda)
        padcol[eng._feat] = False
        assert not eng.x[-1][:, padcol].any() and not eng.hc[:nv, padcol].any()


@pytest.mark.parametrize("tag", list(SHAPES))
def test_biased_topk_matches_fp64_argsort(golden_dir, cuda, tag):
    """Top-10 with seen items and with candidates (fused score_topk through the module) equal a float64 argsort of the same
    bf16 query rows and head; the module's logits equal the reference's eval logits within bf16 tolerance."""
    from replay_b200.models.nn.sequential import Bert4Rec
    from replay_b200.models.nn.sequential.bert4rec import shift_features
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    z, sd, _ = load(os.path.join(golden_dir, f"bert4rec_{tag}.npz"))
    n_items, d, H, L, nb, tied = (int(z[k]) for k in ("n_items", "d", "H", "L", "n_blocks", "tying"))
    m = Bert4Rec(TensorSchema(TensorFeatureInfo("item_id", n_items, 0, d)), block_count=nb, head_count=H, hidden_size=d,
                 max_seq_len=L, dropout_rate=0.0, enable_embedding_tying=bool(tied))
    m.load_state_dict({"_model." + k: v for k, v in sd.items()})
    ids, pm, tok, _ = _batch(z, cuda)
    sids, spm, stm = shift_features(ids, pm, pm, 0)
    batch = {"inputs": {"item_id": sids}, "pad_mask": spm, "token_mask": stm}
    core = m._model.core
    hq = core._query_padded(sids, spm, stm).float()
    q = m._model.get_query_embeddings({"item_id": sids}, spm, stm)
    assert q.shape == (ids.shape[0], d)
    assert torch.equal(q, core.engine.unpad_features(hq))
    W, b = core.engine.head_for_scoring()
    logits = (hq.double() @ W.double().T + b[:n_items].double()).cpu()
    sc = m.predict(batch)
    assert sc.shape == (ids.shape[0], n_items)
    assert (sc.cpu().double() - logits).abs().max() < 1e-3 * (logits.abs().max() + 1)
    seen = torch.zeros(ids.shape[0], n_items, dtype=torch.bool)
    seen.scatter_(1, ids.cpu(), True)
    top, _ = m.predict_topk(batch, 10, seen_ids=ids)
    ref = torch.argsort(-logits.masked_fill(seen, float("-inf")), dim=1, stable=True)[:, :10]
    assert torch.equal(top.cpu(), ref)
    cands = torch.arange(3, n_items, 7, device=cuda)
    top_c, _ = m.predict_topk(batch, 10, seen_ids=ids, candidates_to_score=cands)
    lc = logits[:, cands.cpu()].masked_fill(seen[:, cands.cpu()], float("-inf"))
    assert torch.equal(top_c.cpu(), cands.cpu()[torch.argsort(-lc, dim=1, stable=True)[:, :10]])
    # eval logits of the reference on the un-shifted batch
    ref_eval = torch.from_numpy(z["eval_logits"])
    got_eval = m._model.predict({"item_id": ids}, pm, tok).cpu()
    assert (got_eval - ref_eval).abs().max() < 0.1


@pytest.mark.parametrize("tag", ["d300h4", "d96h2_tied"])
def test_module_training_step_and_state_dict_round_trip(golden_dir, cuda, tag):
    """Bert4Rec training_step gives the reference loss; state_dict has the reference's keys and TRUE shapes (tied: the head's
    alias keys too) and a round trip through a fresh module reproduces the weights and the scores."""
    from replay_b200.models.nn.sequential import Bert4Rec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    z, sd, _ = load(os.path.join(golden_dir, f"bert4rec_{tag}.npz"))
    n_items, d, H, L, nb, tied = (int(z[k]) for k in ("n_items", "d", "H", "L", "n_blocks", "tying"))

    def make():
        return Bert4Rec(TensorSchema(TensorFeatureInfo("item_id", n_items, 0, d)), block_count=nb, head_count=H, hidden_size=d,
                        max_seq_len=L, dropout_rate=0.0, enable_embedding_tying=bool(tied))

    m = make()
    m.load_state_dict({"_model." + k: v for k, v in sd.items()})
    sd1 = m.state_dict()
    for k, v in sd.items():
        assert tuple(sd1["_model." + k].shape) == tuple(v.shape), k
        assert torch.equal(sd1["_model." + k].cpu(), v), k
    if tied:
        assert any(k.startswith("_model._head._item_embedder.") for k in sd1)
    ids, pm, tok, labels = _batch(z, cuda)
    batch = {"query_id": torch.arange(ids.shape[0]).view(-1, 1), "inputs": {"item_id": ids}, "pad_mask": pm,
             "token_mask": tok, "positive_labels": labels}
    loss = m.training_step(batch, 0)
    assert abs(float(loss) - float(z["train_loss"])) < 5e-3 * float(z["train_loss"])
    sd2 = m.state_dict()
    assert set(sd2) == set(sd1) and all(sd2[k].shape == sd1[k].shape for k in sd1)
    m2 = make()
    m2.load_state_dict(sd2)
    sd3 = m2.state_dict()
    for k in sd2:
        assert torch.equal(sd3[k].cpu(), sd2[k].cpu()), k
    pbatch = {"inputs": {"item_id": ids}, "pad_mask": pm, "token_mask": tok}
    torch.testing.assert_close(m2.validation_step(pbatch, 0), m.validation_step(pbatch, 0))
