"""GPU: the full-catalog BCE through the public surfaces against the REAL reference classes (tests/golden/full_bce_losses.npz,
tools/gen_bce_golden.py) - new-path ``SasRec.loss = BCE()`` fused and un-fused, ``Bert4Rec(loss_type="BCE")`` untied and
tied - and the engines at the config-2 shape (SASRec d = 128, |I| = 50 K) and the config-3 shape (BERT4Rec d = 256,
|I| = 100 K, biased head), dropout 0, against the float64 head on the rows the engine selected.

Reference bounds as for the other losses: loss within 5e-3 relative; gradients with cosine > 0.995 and a norm ratio within 3%."""
import os

import numpy as np
import pytest
import torch

from bce_reference import reference, worst

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda")


def _agree(name, a, b):
    a, b = a.detach().double().cpu().reshape(-1), torch.as_tensor(b).double().reshape(-1)
    c = float(a @ b / (a.norm() * b.norm() + 1e-30))
    r = float(a.norm() / b.norm())
    assert c > 0.995 and abs(r - 1) < 0.03, (name, c, r)


@pytest.mark.parametrize("fused", [True, False], ids=["fused", "unfused"])
def test_new_path_sasrec_bce_matches_reference(golden_dir, cuda, fused):
    from replay_b200.nn.loss import BCE
    from replay_b200.nn.sequential import SasRec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    z = np.load(os.path.join(golden_dir, "sasrec_new_tiny.npz"))
    zb = np.load(os.path.join(golden_dir, "full_bce_losses.npz"))
    sd = {k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd::")}
    n_items, d, Lmax = int(z["n_items"]), int(z["d"]), z["ids"].shape[1]
    model = SasRec.from_params(TensorSchema(TensorFeatureInfo("item_id", n_items, n_items, d)), embedding_dim=d,
                               num_heads=int(z["H"]), num_blocks=int(z["n_blocks"]), max_sequence_length=Lmax, dropout=0.0,
                               device=cuda)
    model.load_state_dict(sd)
    model.loss = BCE()
    model.train()
    ids, pm = torch.from_numpy(z["ids"]).cuda(), torch.from_numpy(z["pad_mask"]).cuda()
    lab, tm = torch.from_numpy(z["labels"]).cuda(), torch.from_numpy(z["target_mask"]).cuda()
    eng = model.core.ensure_engine(ids.shape[0], Lmax, with_grad=True)
    eng.fused_ce = fused
    out = model(feature_tensors={"item_id": ids}, padding_mask=pm, positive_labels=lab.unsqueeze(-1),
                target_padding_mask=tm.unsqueeze(-1))
    out["loss"].backward()
    torch.cuda.synchronize()
    ref = float(zb["new_loss"])
    assert abs(float(out["loss"]) - ref) < 5e-3 * abs(ref), (float(out["loss"]), ref)
    G = eng.export_canonical(eng.grads)
    _agree("item_emb", G["item_emb"], zb["new_gE"])
    _agree("in_w", G["blocks"][0]["in_w"], zb["new_gW"])


@pytest.mark.parametrize("tag,name", [("tiny", "untied"), ("tiny_tied", "tied")])
def test_bert4rec_bce_matches_reference(golden_dir, cuda, tag, name):
    from replay_b200.models.nn.sequential import Bert4Rec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    z = np.load(os.path.join(golden_dir, f"bert4rec_{tag}.npz"))
    zb = np.load(os.path.join(golden_dir, "full_bce_losses.npz"))
    sd = {"_model." + k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd::")}
    n_items, d, H, L = int(z["n_items"]), int(z["d"]), int(z["H"]), int(z["L"])
    m = Bert4Rec(TensorSchema(TensorFeatureInfo("item_id", n_items, 0, d)), block_count=int(z["n_blocks"]), head_count=H,
                 hidden_size=d, max_seq_len=L, dropout_rate=0.0, enable_embedding_tying=bool(int(z["tying"])), loss_type="BCE",
                 fused_optimizer=False)
    m.load_state_dict(sd)
    ids, pm, tok = (torch.from_numpy(z[k]).cuda() for k in ("ids", "pad_mask", "token_mask"))
    loss = m._model.core.loss(ids, pm, tok, torch.from_numpy(z["labels"]).cuda())
    loss.backward()
    torch.cuda.synchronize()
    ref = float(zb[f"bert_{name}_loss"])
    assert abs(float(loss) - ref) < 5e-3 * abs(ref), (float(loss), ref)
    G = m._model.core.engine.grads
    _agree("item_emb", G["item_emb"], zb[f"bert_{name}_gE"])
    _agree("in_w", G["b0.in_w"], zb[f"bert_{name}_gW"])
    _agree("head_b", G["head_b"][:n_items], zb[f"bert_{name}_gBias"])
    if name == "untied":
        _agree("head_w", G["head_w"], zb[f"bert_{name}_gHead"])


def _head_at_engine_rows(eng, W, bias, n_items):
    """the engine's compacted rows through the head again, against float64 (loss, d_hc, d_table, d_bias)"""
    from replay_b200 import ops

    nv = int(eng.n_valid.item())
    st = ops.CEHeadState(eng.hc.shape[0], n_items, W.shape[1], eng.hc.device)
    d_hc = torch.zeros_like(eng.hc)
    d_W = torch.zeros(n_items, W.shape[1], device=W.device)
    d_b = torch.zeros(n_items, device=W.device) if bias is not None else None
    loss = ops.bce_head_fwd(st, eng.hc, W, eng.labels_c, eng.n_valid, bias=bias, d_hc=d_hc, n_valid_hint=nv).clone()
    ops.bce_head_bwd(st, eng.hc, W, eng.labels_c, eng.n_valid, d_hc, d_W, bias=bias, d_bias=d_b, n_valid_hint=nv)
    torch.cuda.synchronize()
    r = reference(eng.hc, W, None if bias is None else bias[:n_items], eng.labels_c, nv)
    assert abs(float(loss[0]) - float(r["loss"])) <= float(r["bound_loss"])
    assert worst(d_hc[:nv], r["d_h"], r["bound_h"]) <= 1.0
    assert worst(d_W, r["d_W"], r["bound_W"]) <= 1.0
    if bias is not None:
        assert worst(d_b, r["d_b"], r["bound_b"]) <= 1.0
    return float(r["loss"])


def test_engine_config2_shape(cuda):
    """SASRec d = 128, |I| = 50 K, L = 200, dropout 0: the step's loss and the head at the engine's own rows."""
    from replay_b200.nn.loss import BCE
    from replay_b200.nn.sequential import SasRec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema
    from replay_b200.synthetic import make_sequences

    n_items, d, L, B = 50_000, 128, 200, 32
    model = SasRec.from_params(TensorSchema(TensorFeatureInfo("item_id", n_items, n_items, d)), embedding_dim=d, num_heads=2,
                               num_blocks=2, max_sequence_length=L, dropout=0.0, seed=4)
    model.loss = BCE()
    model.train()
    ids, pm, lab, tm = (t.cuda() for t in make_sequences(B, n_items, L, seed=9))
    loss = float(model.core.loss(ids, pm, lab, tm))
    eng = model.core.engine
    ref = _head_at_engine_rows(eng, eng.params16["item_emb"][:n_items], None, n_items)
    assert abs(loss - ref) < 1e-4 * abs(ref), (loss, ref)
    assert int(eng.n_valid.item()) == int(tm.sum())


def test_engine_config3_shape(cuda):
    """BERT4Rec d = 256, |I| = 100 K, untied biased head, L = 200, dropout 0."""
    from replay_b200.models.nn.sequential import Bert4Rec
    from replay_b200.models.nn.sequential.bert4rec import uniform_masker
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    n_items, d, L, B = 100_000, 256, 200, 24
    m = Bert4Rec(TensorSchema(TensorFeatureInfo("item_id", n_items, 0, d)), block_count=2, head_count=4, hidden_size=d,
                 max_seq_len=L, dropout_rate=0.0, loss_type="BCE", fused_optimizer=False)
    g = torch.Generator().manual_seed(5)
    ids = torch.randint(1, n_items, (B, L), generator=g)
    pm = torch.ones(B, L, dtype=torch.bool)
    pm[: B // 2, : L // 2] = False
    tok = uniform_masker(pm, 0.2, generator=g)
    core = m._model.core
    core.ensure_engine(B, L, with_grad=True).params["head_b"][:n_items].copy_(torch.randn(n_items, generator=g).cuda() * 0.3)
    core.mark_params_updated()
    loss = float(core.loss(ids.cuda(), pm.cuda(), tok.cuda(), ids.cuda()))
    eng = core.engine
    ref = _head_at_engine_rows(eng, eng.params16["head_w"], eng.params["head_b"], n_items)
    assert abs(loss - ref) < 1e-4 * abs(ref), (loss, ref)
    assert int(eng.n_valid.item()) == int((pm & ~tok).sum())
