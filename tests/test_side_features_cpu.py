"""Side features of the new-path SASRec on the CPU: the plain-torch restatement (oracle/side_features.py) against the
goldens of the real reference, the schema surface, the configurations that still raise, the reference key map and
``from_params`` on an item-only schema."""
import os

import numpy as np
import pytest
import torch

from oracle import sasrec as osr
from oracle import side_features as osf
from replay_b200.engine import EncoderConfig, SideFeature
from replay_b200.nn.agg import SumAggregator
from replay_b200.nn.embedding import SequenceEmbedding
from replay_b200.nn.mask import DefaultAttentionMask
from replay_b200.nn.sequential.sasrec import (DiffTransformerLayer, PositionAwareAggregator, SasRec, SasRecBody,
                                              SasRecTransformerLayer)
from replay_b200.schema import TensorFeatureInfo, TensorSchema

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CPU = torch.device("cpu")


@pytest.mark.parametrize("tag", ["d64h2_sum", "d50h1_mean"])
def test_restatement_matches_reference_golden(tag):
    z = np.load(os.path.join(GOLDEN, f"sasrec_side_{tag}.npz"))
    sd, specs = osf.golden_state_dict(z), osf.golden_specs(z)
    P = osr.params_from_new_state_dict(sd)
    P["side"] = osf.side_from_state_dict(sd, specs)
    feats = {f["name"]: torch.from_numpy(z["feat::" + f["name"]]) for f in specs}
    t = lambda k: torch.from_numpy(z[k])  # noqa: E731
    loss, G = osf.loss_and_grads(P, specs, t("ids"), feats, t("pad_mask"), t("labels"), t("target_mask"), int(z["H"]),
                                 str(z["method"]))
    assert abs(float(loss) - float(z["train_loss"])) < 1e-5
    pre = "body.embedder.feature_embedders."
    for f in specs:
        if f["kind"] in ("cat", "bag"):
            pairs = [(G["side"][f["name"]], pre + f["name"] + ".emb.weight")]
        elif f["kind"] == "num":
            pairs = [(G["side"][f["name"] + ".w"], pre + f["name"] + ".linear.weight"),
                     (G["side"][f["name"] + ".b"], pre + f["name"] + ".linear.bias")]
        else:
            pairs = []
        for g, k in pairs:
            assert torch.allclose(g, torch.from_numpy(z["grad::" + k]), atol=1e-6), k
    assert torch.allclose(G["item_emb"], torch.from_numpy(z[f"grad::{pre}item_id.emb.weight"]), atol=1e-6)


def _info(name, kind, d=64, **kw):
    base = dict(cat=dict(cardinality=10, padding_value=10), bag=dict(cardinality=10, padding_value=10, is_list=True),
                num=dict(cardinality=None, padding_value=0, is_cat=False, tensor_dim=3),
                ident=dict(cardinality=None, padding_value=0, is_cat=False, tensor_dim=d))[kind]
    base.update(kw)
    return TensorFeatureInfo(name=name, embedding_dim=d, **base)


def _schema(*extra, d=64):
    return TensorSchema(TensorFeatureInfo("item_id", 100, 100, d), features=list(extra))


def test_schema_stand_in_keeps_item_only_behaviour():
    s = TensorSchema(TensorFeatureInfo("item_id", 100, 100, 64))
    assert s.items() == [("item_id", s["item_id"])] and list(s.categorical_features) == ["item_id"]
    assert s.numerical_features == {}
    f = TensorFeatureInfo("item_id", 100, 100, 64, True, True)
    assert (f.is_list, f.tensor_dim) == (False, None)
    s2 = _schema(_info("g", "cat"), _info("p", "num"))
    assert [k for k, _ in s2.items()] == ["item_id", "g", "p"]
    assert list(s2.numerical_features) == ["p"] and s2["g"].cardinality == 10


def test_from_params_item_only_is_todays_config():
    m = SasRec.from_params(_schema(), embedding_dim=64, num_heads=2, num_blocks=2, max_sequence_length=32, dropout=0.1,
                           device=CPU)
    assert m.core.cfg == EncoderConfig(n_items=100, d=64, n_heads=2, n_blocks=2, max_len=32, dropout=0.1, variant="new")


def test_from_params_embeds_side_features_and_maps_reference_keys():
    s = _schema(_info("g", "cat"), _info("t", "bag"), _info("p", "num"), _info("v", "ident"), _info("q", "cat"))
    m = SasRec.from_params(s, embedding_dim=64, num_heads=2, max_sequence_length=16, excluded_features=["q"],
                           categorical_list_feature_aggregation_method="mean", device=CPU)
    assert m.core.cfg.features == (SideFeature("g", "cat", 10, 10, 1), SideFeature("t", "bag_mean", 10, 10, 1),
                                   SideFeature("p", "num", 0, 0, 3), SideFeature("v", "ident", 0, 0, 64))
    km, pre = m.core._keymap, "body.embedder.feature_embedders."
    assert km["feat.g"] == pre + "g.emb.weight" and km["feat.t"] == pre + "t.emb.weight"
    assert km["feat.p.w"] == pre + "p.linear.weight" and km["feat.p.b"] == pre + "p.linear.bias"
    assert m.core.cfg.true_shapes()["feat.p.w"] == (64, 3) and m.core.cfg.true_shapes()["feat.g"] == (11, 64)
    assert not any("feat.v" in k or "feat.q" in k for k in km)


def _body(schema, enc=None, method="sum", d=64):
    return SasRecBody(SequenceEmbedding(schema, categorical_list_feature_aggregation_method=method),
                      PositionAwareAggregator(SumAggregator(d), 16, 0.1), DefaultAttentionMask("item_id", 2),
                      enc or SasRecTransformerLayer(d, 2, 2, 0.1, "relu"), torch.nn.LayerNorm(d))


def test_still_raising_configurations():
    with pytest.raises(ValueError, match="max"):
        _body(_schema(_info("t", "bag")), method="max").build_core(CPU)
    with pytest.raises(NotImplementedError, match="Non-sequential"):
        _body(_schema(_info("g", "cat", is_seq=False))).build_core(CPU)
    with pytest.raises(ValueError, match="embedding_dim"):
        _body(_schema(_info("g", "cat", d=32))).build_core(CPU)
    with pytest.raises(ValueError, match="SasRecTransformerLayer"):
        _body(_schema(_info("g", "cat")), enc=DiffTransformerLayer(64, 2, 2)).build_core(CPU)
    with pytest.raises(ValueError, match="new-path"):
        EncoderConfig(n_items=10, d=64, n_heads=1, n_blocks=1, max_len=8, variant="legacy",
                      features=(SideFeature("g", "cat", 3, 3),))
    with pytest.raises(ValueError, match="at most 64"):
        EncoderConfig(n_items=10, d=64, n_heads=1, n_blocks=1, max_len=8, features=(SideFeature("p", "num", width=65),))
    assert _body(_schema(_info("g", "cat"))).build_core(CPU).cfg.features == (SideFeature("g", "cat", 10, 10, 1),)


def test_feature_kernels_are_exported():
    from replay_b200 import _lib

    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    L = _lib.lib()
    for name in ("rp_feature_embed_fwd", "rp_feature_embed_fwd_rows", "rp_feature_embed_bwd", "rp_feature_embed_bwd_rows"):
        getattr(L, name)
    arr = (_lib.RpFeature * 1)()
    # argument checks run before any launch, so they answer without a device
    assert L.rp_feature_embed_fwd(None, None, None, arr, 1, 8, 8, 64, 0, 0, 8.0, 0.0, 0, 0, None, None, None) == -1
    assert L.rp_feature_embed_bwd(None, arr, 1, 8, 64, 0, 8.0, 0.0, 0, 0, None, None, None, 64, None) == -1
    assert L.rp_feature_embed_fwd_rows(1, 1, 1, arr, 1, None, None, 8, 8, 64, 0, 0, 8.0, 0.0, 0, 0, None, 1, None) == -1
