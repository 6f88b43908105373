"""Side features of the legacy BERT4Rec on the CPU: the plain-torch restatement (oracle/bert4rec_side_features.py) against
the goldens of the real reference, the mirror's checkpoint keys, the item-only configuration, every configuration that
raises, ``get_all_embeddings`` and the exported kernels' argument checks."""
import os

import numpy as np
import pytest
import torch

from oracle import bert4rec_passes as op
from oracle import bert4rec_side_features as obs
from replay_b200.engine import SideFeature
from replay_b200.engine_bert import BertConfig
from replay_b200.models.nn.sequential import Bert4Rec
from replay_b200.models.nn.sequential.bert4rec import Bert4RecModel, bert_key_map
from replay_b200.schema import TensorFeatureInfo, TensorSchema, bert_side_features_of

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = ["d64h2", "d300h4", "d96h2_tied_bce"]


def _load(tag):
    z = np.load(os.path.join(GOLDEN, f"bert4rec_side_{tag}.npz"))
    specs = [(str(n), "cat" if str(k) == "cat" else "ident") for n, k in zip(z["f_name"], z["f_kind"])]
    specs = [s for s in specs if s[1] == "cat"] + [s for s in specs if s[1] == "ident"]   # the reference's sum order
    return z, specs, op.golden_state_dict(z)


def _schema_of(z, d=None):
    """the stand-in schema of a golden (the item id, then its side features in the golden's order)"""
    d = int(z["d"]) if d is None else d
    fs = []
    for n, k, c, p in zip(z["f_name"], z["f_kind"], z["f_card"], z["f_pad"]):
        if str(k) == "cat":
            fs.append(TensorFeatureInfo(str(n), int(c), int(p), d))
        else:
            fs.append(TensorFeatureInfo(str(n), None, 0, d, is_cat=False, is_list=str(k) == "num_list", tensor_dim=d))
    return TensorSchema(TensorFeatureInfo("item_id", int(z["n_items"]), 0, d), features=fs)


def _model(z, cls=Bert4RecModel, **kw):
    args = dict(max_len=int(z["L"]), hidden_size=int(z["d"]), num_blocks=int(z["n_blocks"]), num_heads=int(z["H"]),
                num_passes_over_block=int(z["passes"]), dropout=0.0, enable_positional_embedding=bool(int(z["positional"])),
                enable_embedding_tying=bool(int(z["tying"])), device="cpu")
    args.update(kw)
    return cls(_schema_of(z), **args)


def _leaves(P):
    """engine-style name -> leaf tensor of the canonical dict (block parameters as b{i}.{k}, side tables as feat.{name})"""
    out = {k: v for k, v in P.items() if k not in ("blocks", "feat")}
    out.update({f"b{i}.{k}": v for i, blk in enumerate(P["blocks"]) for k, v in blk.items()})
    out.update({f"feat.{n}": v for n, v in P["feat"].items()})
    for v in out.values():
        v.requires_grad_(True)
    return out


@pytest.mark.parametrize("tag", CASES)
def test_restatement_matches_reference_golden(tag):
    """Train loss, every gradient and the shifted window's eval logits of the restatement against the reference's."""
    z, specs, sd = _load(tag)
    t = lambda k: torch.from_numpy(z[k])  # noqa: E731
    P = obs.params_from_state_dict(sd, specs)
    leaves = _leaves(P)
    feats = {n: t("feat::" + n) for n, _ in specs}
    loss = obs.train_loss(P, t("ids"), t("pad_mask"), t("token_mask"), t("labels"), feats, specs, int(z["H"]),
                          int(z["passes"]), str(z["loss"]).lower())
    assert abs(loss.item() - float(z["train_loss"])) < 1e-5 * max(1.0, abs(float(z["train_loss"])))
    grads = torch.autograd.grad(loss, list(leaves.values()))
    keys = bert_key_map(int(z["n_blocks"]), bool(int(z["tying"])), "item_id", bool(int(z["positional"])),
                        [SideFeature(n, k) for n, k in specs])
    assert sorted(keys[k] for k in leaves) == sorted(k[6:] for k in z.files if k.startswith("grad::"))
    for name, g in zip(leaves, grads):
        ref = t("grad::" + keys[name])
        assert torch.allclose(g, ref, atol=1e-5, rtol=1e-4), name
    with torch.no_grad():
        pf = {n: t("pfeat::" + n) for n, _ in specs}
        h = obs.body(P, t("pfeat::item_id"), t("p_pad_mask"), t("p_token_mask"), pf, specs, int(z["H"]), int(z["passes"]))
        lg = obs.logits(P, h[:, -1])
    torch.testing.assert_close(lg, t("eval_logits"), atol=1e-4, rtol=1e-4)


@pytest.mark.parametrize("tag", CASES)
def test_state_dict_keys_follow_the_reference(tag):
    """Keys in the reference's order, the tied head's aliases included; a strict load of the golden weights succeeds."""
    z, _, sd = _load(tag)
    m = _model(z)
    m.load_state_dict(sd, strict=True)
    assert list(m.state_dict()) == [str(k) for k in z["sd_keys"]]
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k]), k
    lm = Bert4Rec(_schema_of(z), **_lightning_args(z))
    lm.load_state_dict({"_model." + k: v for k, v in sd.items()})
    assert list(lm.state_dict()) == ["_model." + str(k) for k in z["sd_keys"]]


def _lightning_args(z):
    return dict(block_count=int(z["n_blocks"]), head_count=int(z["H"]), hidden_size=int(z["d"]), max_seq_len=int(z["L"]),
                dropout_rate=0.0, pass_per_transformer_block_count=int(z["passes"]),
                enable_positional_embedding=bool(int(z["positional"])), enable_embedding_tying=bool(int(z["tying"])),
                loss_type=str(z["loss"]), device="cpu")


def test_state_dict_misses_side_tables_strictly():
    z, _, sd = _load("d64h2")
    m = _model(z)
    with pytest.raises(RuntimeError, match="missing keys"):
        m.load_state_dict({k: v for k, v in sd.items() if "genre" not in k}, strict=True)


def test_item_only_schema_builds_todays_model():
    s = TensorSchema(TensorFeatureInfo("item_id", 500, 0, 64))
    m = Bert4RecModel(s, max_len=32, hidden_size=64, num_blocks=2, num_heads=2, device="cpu")
    today = BertConfig(n_items=500, d=64, n_heads=2, n_blocks=2, max_len=32, dropout=0.1, tying=False, pad_id=0)
    assert m.core.cfg == today and m.core.cfg.features == ()
    assert m.core.cfg.param_layout() == today.param_layout()
    assert not any(k.startswith("feat.") for k, _, _ in today.param_layout())


def test_side_layout_follows_the_item_only_layout():
    """The side tables come after head_b, with cardinality rows (no padding row), so the item-only offsets are unchanged."""
    base = dict(n_items=100, d=300, n_heads=4, n_blocks=1, max_len=16)
    fs = (SideFeature("genre", "cat", 11, 0, 1), SideFeature("vec", "ident", 0, 0, 300))
    a, b = BertConfig(**base).param_layout(), BertConfig(**base, features=fs).param_layout()
    assert b[:len(a)] == a and b[len(a):] == [("feat.genre", (11, 512), (None, "f"))]
    assert BertConfig(**base, features=fs).true_shapes()["feat.genre"] == (11, 300)


def test_schema_conversion_order_and_kinds():
    z, _, _ = _load("d64h2")
    assert bert_side_features_of(_schema_of(z)) == [SideFeature("genre", "cat", 7, 3, 1), SideFeature("flag", "cat", 1, 0, 1),
                                                    SideFeature("vec", "ident", 0, 0, 64), SideFeature("vl", "ident", 0, 0, 64)]
    # numericals after categoricals whatever the schema order: the order of the reference's sum
    s = TensorSchema(TensorFeatureInfo("item_id", 10, 0, 64), features=[
        TensorFeatureInfo("v", None, 0, 64, is_cat=False, tensor_dim=64), TensorFeatureInfo("g", 3, 0, 64)])
    assert [f.name for f in bert_side_features_of(s)] == ["g", "v"]


def _base(*extra, d=64):
    return TensorSchema(TensorFeatureInfo("item_id", 100, 0, d), features=list(extra))


def test_raising_configurations():
    mk = lambda s, d=64: Bert4RecModel(s, max_len=16, hidden_size=d, num_blocks=1, num_heads=2, device="cpu")  # noqa: E731
    with pytest.raises(NotImplementedError, match="Non-sequential features is not yet supported"):
        mk(_base(TensorFeatureInfo("u", 5, 0, 64, is_seq=False)))
    with pytest.raises(ValueError, match="Dimension of all features must be the same for sum aggregation"):
        mk(_base(TensorFeatureInfo("g", 5, 0, 32)))
    with pytest.raises(ValueError, match="Dimension of all features must be the same for sum aggregation"):
        mk(_base(TensorFeatureInfo("timestamp", None, 0, 64, is_cat=False, tensor_dim=1)))
    with pytest.raises(NotImplementedError, match="categorical list"):
        mk(_base(TensorFeatureInfo("tags", 5, 0, 64, is_list=True)))
    # the reference's own constructor error wins over the list: a later feature of another dim
    with pytest.raises(ValueError, match="Dimension"):
        mk(_base(TensorFeatureInfo("tags", 5, 0, 64, is_list=True), TensorFeatureInfo("g", 5, 0, 32)))
    # an identity feature as wide as the first feature but not as the model
    with pytest.raises(ValueError, match="tensor_dim == 96"):
        mk(_base(TensorFeatureInfo("v", None, 0, 64, is_cat=False, tensor_dim=64)), d=96)
    base = dict(n_items=10, d=64, n_heads=1, n_blocks=1, max_len=8)
    for f in (SideFeature("b", "bag_sum", 5, 0, 1), SideFeature("n", "num", width=3)):
        with pytest.raises(ValueError, match="unknown kind"):
            BertConfig(**base, features=(f,))
    with pytest.raises(ValueError, match="distinct names"):
        BertConfig(**base, features=(SideFeature("g", "cat", 5), SideFeature("g", "cat", 5)))
    with pytest.raises(ValueError, match="at most 16"):
        BertConfig(**base, features=tuple(SideFeature(f"g{i}", "cat", 5) for i in range(17)))
    with pytest.raises(ValueError, match="cardinality"):
        BertConfig(**base, features=(SideFeature("g", "cat", 0),))


def test_short_prediction_batch_with_a_numerical_feature_raises():
    z, _, _ = _load("d64h2")
    m = Bert4Rec(_schema_of(z), **_lightning_args(z))
    B, L = 3, int(z["L"]) - 4
    batch = {"query_id": torch.arange(B), "pad_mask": torch.ones(B, L, dtype=torch.bool),
             "token_mask": torch.ones(B, L, dtype=torch.bool),
             "inputs": {"item_id": torch.zeros(B, L, dtype=torch.int64), "genre": torch.zeros(B, L, dtype=torch.int64),
                        "flag": torch.zeros(B, L, dtype=torch.int64), "vec": torch.zeros(B, L, 64),
                        "vl": torch.zeros(B, L, 64)}}
    with pytest.raises(ValueError, match="numerical features"):
        m.predict_step(batch, 0)


def test_short_categorical_batch_is_padded_and_shifted_per_feature():
    s = _base(TensorFeatureInfo("genre", 7, 3, 64))
    m = Bert4Rec(s, block_count=1, head_count=2, hidden_size=64, max_seq_len=6, dropout_rate=0.0, device="cpu")
    batch = {"pad_mask": torch.tensor([[False, True, True, True]]), "token_mask": torch.tensor([[False, True, True, True]]),
             "inputs": {"item_id": torch.tensor([[0, 5, 6, 7]]), "genre": torch.tensor([[3, 1, 2, 0]])}}
    ids, pm, tm, feats = m._prepared(batch)
    assert ids.tolist() == [[0, 0, 5, 6, 7, 0]] and feats["item_id"] is ids
    assert feats["genre"].tolist() == [[3, 3, 1, 2, 0, 3]]
    assert pm.tolist() == [[False, False, True, True, True, True]]
    assert tm.tolist() == [[False, False, True, True, True, False]]


def test_get_all_embeddings_keys():
    z, _, sd = _load("d64h2")
    s = _base(TensorFeatureInfo("genre", 7, 3, 64), TensorFeatureInfo("flag", 1, 0, 64))
    m = Bert4RecModel(s, max_len=16, hidden_size=64, num_blocks=2, num_heads=2, device="cpu")
    m.load_state_dict({k: v for k, v in sd.items() if not k.startswith("_head._item_embedder.")})
    e = m.get_all_embeddings()
    assert list(e) == ["item_embedding", "genre", "flag", "positional_embedding"]
    assert torch.equal(e["genre"], sd["item_embedder.cat_embeddings.genre.weight"]) and e["flag"].shape == (1, 64)
    m2 = _model(z)
    m2.load_state_dict(sd)
    with pytest.raises(KeyError):
        m2.get_all_embeddings()   # the reference indexes cat_embeddings[name] for the numerical "vec" too


def test_bert_feature_kernels_are_exported():
    from replay_b200 import _lib

    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    L = _lib.lib()
    for name in ("rp_bert_feature_embed_fwd", "rp_bert_feature_embed_bwd"):
        getattr(L, name)
    arr = (_lib.RpFeature * 1)()
    arr[0].values, arr[0].table, arr[0].d_table, arr[0].n_rows, arr[0].width = 1, 1, 1, 5, 1
    # argument checks run before any launch, so they answer without a device
    assert L.rp_bert_feature_embed_fwd(None, 1, None, 1, 1, arr, 1, 16, 8, 64, 0, 0.0, 0, 0, None, 1, None) == -1
    assert L.rp_bert_feature_embed_bwd(None, 1, 1, arr, 1, 16, 64, 0, 0.0, 0, 0, None, None) == -1
    for kind in (_lib.FEAT_BAG_SUM, _lib.FEAT_BAG_MEAN, _lib.FEAT_NUM):
        arr[0].kind = kind
        assert L.rp_bert_feature_embed_fwd(1, 1, None, 1, 1, arr, 1, 16, 8, 64, 0, 0.0, 0, 0, None, 1, None) == -1
        assert L.rp_bert_feature_embed_bwd(1, 1, 1, arr, 1, 16, 64, 0, 0.0, 0, 0, None, None) == -1
