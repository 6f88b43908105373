"""ConcatAggregator on the new-path SASRec, on the CPU: the plain-torch restatement (oracle/concat_features.py) against the
goldens of the real reference, the concat body's configuration and reference key map, every configuration that raises,
the item-only concat model, and the exported kernels' argument errors."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import concat_features as ocf
from oracle import side_features as osf
from replay_b200.engine import EncoderConfig, SideFeature
from replay_b200.nn.agg import ConcatAggregator, SumAggregator
from replay_b200.nn.embedding import SequenceEmbedding
from replay_b200.nn.mask import DefaultAttentionMask
from replay_b200.nn.sequential.sasrec import (DiffTransformerLayer, PositionAwareAggregator, SasRec, SasRecBody,
                                              SasRecTransformerLayer)
from replay_b200.schema import TensorFeatureInfo, TensorSchema

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CPU = torch.device("cpu")
PRE = "body.embedder.feature_embedders."


@pytest.mark.parametrize("tag", ["d64h2", "d50h1_mean", "item_only"])
def test_restatement_matches_reference_golden(tag):
    z = np.load(os.path.join(GOLDEN, f"sasrec_concat_{tag}.npz"))
    sd, specs = osf.golden_state_dict(z), ocf.golden_specs(z)
    P = ocf.params_from_state_dict(sd, specs)
    ids, pm, lab, tm, feats = ocf.batch_of(z, specs)
    loss, G = ocf.loss_and_grads(P, specs, ids, feats, pm, lab, tm, int(z["H"]), str(z["item_name"]), str(z["method"]))
    assert abs(float(loss) - float(z["train_loss"])) < 1e-5
    pairs = [(G["item_emb"], f"{PRE}item_id.emb.weight"), (G["pos_emb"], "body.embedding_aggregator.pe.weight")]
    if specs:
        pairs += [(G["proj_w"], ocf.PROJ + "weight"), (G["proj_b"], ocf.PROJ + "bias")]
    for f in specs:
        if f["kind"] in ("cat", "bag"):
            pairs.append((G["side"][f["name"]], PRE + f["name"] + ".emb.weight"))
        elif f["kind"] == "num":
            pairs += [(G["side"][f["name"] + ".w"], PRE + f["name"] + ".linear.weight"),
                      (G["side"][f["name"] + ".b"], PRE + f["name"] + ".linear.bias")]
    for g, k in pairs:
        assert torch.allclose(g, torch.from_numpy(z["grad::" + k]), atol=1e-5), k


def _info(name, kind, dim, **kw):
    base = dict(cat=dict(cardinality=10, padding_value=10), bag=dict(cardinality=10, padding_value=10, is_list=True),
                num=dict(cardinality=None, padding_value=0, is_cat=False, tensor_dim=3),
                ident=dict(cardinality=None, padding_value=0, is_cat=False, tensor_dim=dim))[kind]
    base.update(kw)
    return TensorFeatureInfo(name=name, embedding_dim=dim, **base)


def _fixture_schema(d=10):
    """the reference's own ConcatAggregator fixture (tests/nn/conftest.py): widths 10 .. 14 around the item"""
    return TensorSchema(TensorFeatureInfo("item_id", 15, 15, d), features=[
        _info("cat_list_feature", "bag", 11, cardinality=4, padding_value=4), _info("num_feature", "num", 12, tensor_dim=1),
        _info("num_list_feature", "num", 13, tensor_dim=6), _info("emb_list_feature", "ident", 14)])


def _body(schema, dims=None, d=10, heads=1, enc=None):
    dims = [f.embedding_dim for _, f in schema.items()] if dims is None else dims
    return SasRecBody(SequenceEmbedding(schema), PositionAwareAggregator(ConcatAggregator(dims, d), 7, 0.2),
                      DefaultAttentionMask("item_id", heads), enc or SasRecTransformerLayer(d, heads, 1, 0.2, "relu"),
                      torch.nn.LayerNorm(d))


def test_concat_body_config_and_key_map():
    cfg = _body(_fixture_schema()).build_core(CPU).cfg
    # sorted names: cat_list_feature 11 | emb_list_feature 14 | item_id 10 | num_feature 12 | num_list_feature 13
    assert cfg.aggregator == "concat" and cfg.concat_item_at == 2
    assert [f.name for f in cfg.features] == ["cat_list_feature", "emb_list_feature", "num_feature", "num_list_feature"]
    assert cfg.features[1] == SideFeature("emb_list_feature", "ident", 0, 0, 14, 14)
    assert cfg.concat_width == 60 and cfg.concat_kp == 64 and cfg.concat_columns() == (25, [0, 11, 35, 47])
    shapes = cfg.true_shapes()
    assert shapes["feat_proj.w"] == (10, 60) and shapes["feat_proj.b"] == (10,)
    assert shapes["feat.cat_list_feature"] == (5, 11) and shapes["feat.num_list_feature.w"] == (13, 6)
    # the projection comes after every other parameter
    assert [n for n, _, _ in cfg.param_layout()][-2:] == ["feat_proj.w", "feat_proj.b"]
    km = SasRec(_body(_fixture_schema()), device=CPU).core._keymap
    assert km["feat_proj.w"] == ocf.PROJ + "weight" and km["feat_proj.b"] == ocf.PROJ + "bias"
    assert km["feat.num_feature.w"] == PRE + "num_feature.linear.weight"
    assert not any("emb_list_feature" in v for v in km.values())
    # the golden's keys are exactly the concat model's (the identity buffer aside)
    z = np.load(os.path.join(GOLDEN, "sasrec_concat_d64h2.npz"))
    specs = ocf.golden_specs(z)
    feats = [_info(f["name"], f["kind"], f["dim"], **({"cardinality": f["cardinality"], "padding_value": f["padding_value"]}
                                                      if f["kind"] in ("cat", "bag") else {"tensor_dim": f["width"]}))
             for f in specs]
    sch = TensorSchema(TensorFeatureInfo("item_id", 200, 200, 64), features=feats)
    core = _body(sch, d=64, heads=2, enc=SasRecTransformerLayer(64, 2, 2, 0.2, "relu")).build_core(CPU)
    want = {str(k) for k in z["sd_keys"] if not str(k).endswith("._weight")}
    assert set(core._keymap.values()) == want
    assert core.cfg.concat_item_at == 1 and core.cfg.concat_kp == 128


def test_item_only_concat_is_the_item_only_model():
    sch = TensorSchema(TensorFeatureInfo("item_id", 100, 100, 64))
    cat = _body(sch, d=64, heads=2).build_core(CPU).cfg
    body = SasRecBody(SequenceEmbedding(sch), PositionAwareAggregator(SumAggregator(64), 7, 0.2),
                      DefaultAttentionMask("item_id", 2), SasRecTransformerLayer(64, 2, 1, 0.2, "relu"), torch.nn.LayerNorm(64))
    assert cat == body.build_core(CPU).cfg
    assert cat.aggregator == "sum" and cat.features == ()


def test_concat_value_errors():
    with pytest.raises(ValueError, match=r"Input embedding dim is not equal to embedding_dim \(32 != 64\)"):
        ConcatAggregator([32], 64)
    with pytest.raises(ValueError, match="do not match the embedder"):
        _body(_fixture_schema(), dims=[10, 11, 12, 13]).build_core(CPU)
    with pytest.raises(ValueError, match="do not match the embedder"):
        _body(_fixture_schema(), dims=[10, 11, 12, 13, 15]).build_core(CPU)
    with pytest.raises(ValueError, match="the item feature"):
        _body(_fixture_schema(d=16), d=10).build_core(CPU)
    wide = TensorSchema(TensorFeatureInfo("item_id", 15, 15, 64), features=[_info(f"f{i}", "cat", 200) for i in range(5)])
    with pytest.raises(ValueError, match="at most 1024"):
        _body(wide, d=64).build_core(CPU)
    assert _body(TensorSchema(TensorFeatureInfo("item_id", 15, 15, 64), features=[_info(f"f{i}", "cat", 192) for i in range(5)]),
                 d=64).build_core(CPU).cfg.concat_kp == 1024
    with pytest.raises(ValueError, match="needs its embedding_dim"):
        EncoderConfig(n_items=10, d=64, n_heads=1, n_blocks=1, max_len=8, aggregator="concat",
                      features=(SideFeature("g", "cat", 3, 3),))
    with pytest.raises(ValueError, match="needs side features"):
        EncoderConfig(n_items=10, d=64, n_heads=1, n_blocks=1, max_len=8, aggregator="concat")
    with pytest.raises(ValueError, match="unknown aggregator"):
        EncoderConfig(n_items=10, d=64, n_heads=1, n_blocks=1, max_len=8, aggregator="max")


class _Reader:
    def __init__(self, cols):
        self.cols = cols

    def __getitem__(self, k):
        return self.cols[k]

    @property
    def feature_names(self):
        return list(self.cols)


def test_still_raising_with_concat():
    # side features with the DiffTransformer encoder, "max" bags and ConcatAggregator in TwoTower keep their errors
    with pytest.raises(ValueError, match="SasRecTransformerLayer"):
        _body(_fixture_schema(), enc=DiffTransformerLayer(10, 1, 1)).build_core(CPU)
    sch = _fixture_schema()
    with pytest.raises(ValueError, match="max"):
        SasRecBody(SequenceEmbedding(sch, categorical_list_feature_aggregation_method="max"),
                   PositionAwareAggregator(ConcatAggregator([10, 11, 12, 13, 14], 10), 7, 0.2), DefaultAttentionMask("item_id", 1),
                   SasRecTransformerLayer(10, 1, 1, 0.2, "relu"), torch.nn.LayerNorm(10)).build_core(CPU)
    from replay_b200.nn.ffn import SwiGLUEncoder
    from replay_b200.nn.sequential.twotower import TwoTowerBody

    sch = TensorSchema(TensorFeatureInfo("item_id", 30, 30, 64))
    agg = ConcatAggregator([64], 64)
    tt = TwoTowerBody(schema=sch, embedder=SequenceEmbedding(sch), attn_mask_builder=DefaultAttentionMask("item_id", 2),
                      query_tower_feature_names=["item_id"], query_embedding_aggregator=PositionAwareAggregator(agg, 16, 0.1),
                      item_embedding_aggregator=agg, query_encoder=SasRecTransformerLayer(64, 2, 1, 0.1, activation="relu"),
                      query_tower_output_normalization=torch.nn.LayerNorm(64), item_encoder=SwiGLUEncoder(64, 128),
                      item_features_reader=_Reader({"item_id": torch.arange(30)}))
    with pytest.raises(ValueError, match="SumAggregator"):
        tt.build_core(device="cpu")


def test_concat_kernels_are_exported():
    from replay_b200 import _lib

    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    L = _lib.lib()
    arr = (_lib.RpFeature * 1)()
    col, dim = (ctypes.c_int * 1)(64), (ctypes.c_int * 1)(16)
    # argument checks run before any launch, so they answer without a device
    assert L.rp_concat_gather(None, None, arr, col, dim, 1, 0, 8, 64, 0, 128, None, None) == -1
    assert L.rp_concat_gather_rows(1, 1, arr, col, dim, 1, 0, None, None, 8, 64, 0, 128, 1, None) == -1
    assert L.rp_concat_embed_fwd(None, None, None, None, 8, 8, 64, 0, 8.0, 0.0, 0, 0, None, None, None) == -1
    assert L.rp_concat_embed_fwd(1, 1, 1, None, 8, 8, 64, 0, 8.0, 0.0, 0, 0, None, 1, None) == -1   # row_tok without count
    assert L.rp_concat_embed_fwd(1, 1, None, None, 8, 8, 96, 0, 8.0, 0.0, 0, 0, None, 1, None) == -2
    assert L.rp_concat_scatter(None, 1, 1, 0, arr, col, dim, 1, 0, None, None, 8, 64, 0, 128, None, 0, None) == -1
    assert L.rp_embed_pos_bwd(None, None, None, 1, 8, 64, 0, 0.0, 0, 0, None, 1, None) == -1
    assert L.rp_embed_pos_bwd(1, None, None, 1, 8, 96, 0, 0.0, 0, 0, None, 1, None) == -2
    # segment layout: the item at 0..63 and a 16-wide categorical at 64 tile [0, 80), so kp 128 is accepted by the checks
    # and anything that leaves a gap, overlaps or overflows is RP_ESHAPE
    vals = (ctypes.c_int32 * 8)()
    arr[0].kind, arr[0].width, arr[0].n_rows, arr[0].padding_value = _lib.FEAT_CAT, 1, 4, 3
    arr[0].values, arr[0].table = ctypes.addressof(vals), ctypes.addressof(vals)

    def gather(c=64, w=16, kp=128, d=64, item_col=0):
        return L.rp_concat_gather(1, 1, arr, (ctypes.c_int * 1)(c), (ctypes.c_int * 1)(w), 1, item_col, 8, d, 0, kp, 1, None)

    assert gather(c=65) == -2 and gather(c=60) == -2 and gather(kp=64) == -2 and gather(kp=96) == -2
    assert gather(kp=2048) == -2 and gather(d=96) == -2 and gather(c=0, item_col=0) == -2
    arr[0].kind = 9
    assert gather() == -1
