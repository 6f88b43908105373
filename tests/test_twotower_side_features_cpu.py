"""TwoTower with side features without a GPU: the reference's key list, shapes and dtypes from the goldens
(oracle/gen_twotower_side_features_golden.py), the engine layout, the catalog gradient plan, and the construction errors."""
import os

import numpy as np
import pytest
import torch

from replay_b200.engine import SideFeature
from replay_b200.engine_twotower import TwoTowerConfig, TwoTowerEngine
from replay_b200.schema import TensorFeatureInfo, TensorSchema

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


class _Reader:
    def __init__(self, cols):
        self.cols = cols

    def __getitem__(self, k):
        return self.cols[k]

    @property
    def feature_names(self):
        return list(self.cols)


def _golden(tag):
    z = dict(np.load(os.path.join(GOLD, f"twotower_side_{tag}.npz")))
    n, d = int(z["n_items"]), int(z["d"])
    fs = []
    for name, kind, pad, width, card in zip(z["f_name"], z["f_kind"], z["f_padding_value"], z["f_width"], z["f_cardinality"]):
        if str(kind) in ("cat", "bag"):
            fs.append(TensorFeatureInfo(str(name), int(card), int(pad), d, is_list=str(kind) == "bag"))
        else:
            fs.append(TensorFeatureInfo(str(name), None, 0, d, is_cat=False, tensor_dim=int(width)))
    sch = TensorSchema(TensorFeatureInfo("item_id", n, n, d), features=fs)
    reader = _Reader({str(k): torch.from_numpy(z["item::" + str(k)]) for k in z["reader"]})
    return z, sch, reader


def _model(sch, reader, z, **kw):
    from replay_b200.nn.sequential.twotower import TwoTower

    args = dict(embedding_dim=int(z["d"]), num_heads=int(z["H"]), num_blocks=int(z["n_blocks"]),
                max_sequence_length=int(z["L"]), dropout=0.0, categorical_list_feature_aggregation_method=str(z["method"]),
                device="cpu")
    args.update(kw)
    return TwoTower.from_params(sch, reader, **args)


@pytest.mark.parametrize("tag", ["d64h2", "d50h1"])
def test_state_dict_keys_shapes_dtypes_match_reference(tag):
    from oracle import side_features as osf

    z, sch, reader = _golden(tag)
    m = _model(sch, reader, z)
    m.load_state_dict(osf.golden_state_dict(z), strict=False)
    sd = m.state_dict()
    assert list(sd) == [str(k) for k in z["keys"]]
    for k, shp, dt in zip(z["keys"], z["key_shapes"], z["key_dtypes"]):
        assert "x".join(map(str, sd[str(k)].shape)) == str(shp), k
        assert str(sd[str(k)].dtype) == str(dt), k
    for k in z["reader"]:
        assert torch.equal(sd[f"body.item_tower.item_reference_{k}"], reader[str(k)])
    cfg = m.core.cfg
    assert cfg.item_features == ("genre", "brand", "tags", "stats", "vec")
    assert [f.name for f in cfg.features] == ["genre", "brand", "tags", "stats", "vec", "ctx"]


def test_item_only_layout_is_unchanged():
    """side tables come after every item-only parameter: the item-only prefix of the layout is the item-only model's"""
    base = TwoTowerConfig(n_items=50, d=64, n_heads=2, n_blocks=2, max_len=16, dropout=0.0)
    side = TwoTowerConfig(n_items=50, d=64, n_heads=2, n_blocks=2, max_len=16, dropout=0.0,
                          features=(SideFeature("g", "cat", 5, 5), SideFeature("x", "num", width=3)), item_features=("g",))
    a, b = base.param_layout(), side.param_layout()
    assert b[:len(a)] == a
    assert [n for n, _, _ in b[len(a):]] == ["feat.g", "feat.x.w", "feat.x.b"]


def test_item_features_must_be_embedder_features():
    with pytest.raises(ValueError, match="Feature names found that embedder does not support"):
        TwoTowerConfig(n_items=50, d=64, n_heads=2, n_blocks=1, max_len=16, features=(SideFeature("g", "cat", 5, 5),),
                       item_features=("h",))


def test_catalog_plan_groups_rows_in_fixed_order():
    """_build_item_plan: live entries only (padding, out-of-table ids and all-padding bags dropped), grouped by (feature,
    row), ascending items, chunks inside one group, mean weights 1 / count"""
    class _E:
        ITEM_PLAN_CHUNK = 2
        dev = torch.device("cpu")
        cfg = type("C", (), {"dp": 64})()

    e = _E()
    e.item_feats = (SideFeature("g", "cat", 3, 3), SideFeature("t", "bag_mean", 4, 4, 1), SideFeature("x", "num", width=2))
    e.item_in = {"g": torch.tensor([[0], [3], [0], [2], [0], [-1], [7]], dtype=torch.int32),
                 "t": torch.tensor([[4, 4], [1, 1], [0, 2], [4, 4], [1, 4], [4, 9], [2, 2]], dtype=torch.int32),
                 "x": torch.zeros(7, 2)}
    p = TwoTowerEngine._build_item_plan(e, e.item_in)
    assert p["ent_item"].tolist() == [0, 2, 4, 3, 2, 1, 1, 4, 2, 6, 6]
    assert p["grp_feat"].tolist() == [0, 0, 1, 1, 1]
    assert p["grp_row"].tolist() == [0, 2, 0, 1, 2]
    assert p["grp_chunk"].tolist() == [0, 2, 3, 4, 6, 8]
    assert p["chunk_off"].tolist() == [0, 2, 3, 4, 5, 7, 8, 10, 11]
    assert p["ent_w"].tolist() == [1, 1, 1, 1, 0.5, 0.5, 0.5, 1, 0.5, 0.5, 0.5]
    assert p["desc"].n_chunks == 8 and p["desc"].n_groups == 5


def test_construction_errors():
    from replay_b200.nn.agg import ConcatAggregator, SumAggregator
    from replay_b200.nn.embedding import SequenceEmbedding
    from replay_b200.nn.ffn import SwiGLUEncoder
    from replay_b200.nn.mask import DefaultAttentionMask
    from replay_b200.nn.sequential import DiffTransformerLayer, PositionAwareAggregator, SasRecTransformerLayer
    from replay_b200.nn.sequential.twotower import TwoTower, TwoTowerBody

    z, sch, reader = _golden("d64h2")
    with pytest.raises(ValueError, match="max"):
        _model(sch, reader, z, categorical_list_feature_aggregation_method="max")
    bad = _Reader({**reader.cols, "nope": torch.zeros(60)})
    with pytest.raises(ValueError, match="Feature names found that embedder does not support"):
        _model(sch, bad, z)
    with pytest.raises(ValueError, match="context_merger"):
        TwoTower(_model(sch, reader, z).core, context_merger=object(), device="cpu")
    names = [n for n, _ in sch.items()]

    def body(**over):
        agg = SumAggregator(64)
        kw = dict(schema=sch, embedder=SequenceEmbedding(sch), attn_mask_builder=DefaultAttentionMask("item_id", 2),
                  query_tower_feature_names=names, query_embedding_aggregator=PositionAwareAggregator(agg, 12, 0.0),
                  item_embedding_aggregator=agg, query_encoder=SasRecTransformerLayer(64, 2, 1, 0.0, activation="relu"),
                  query_tower_output_normalization=torch.nn.LayerNorm(64), item_encoder=SwiGLUEncoder(64, 128),
                  item_features_reader=reader)
        kw.update(over)
        return TwoTowerBody(**kw).build_core(device="cpu")

    assert body().cfg.item_features == ("genre", "brand", "tags", "stats", "vec")
    cat = ConcatAggregator([64] * len(names), 64)
    with pytest.raises(ValueError, match="SumAggregator"):
        body(item_embedding_aggregator=cat)
    with pytest.raises(ValueError, match="SumAggregator"):
        body(query_embedding_aggregator=PositionAwareAggregator(cat, 12, 0.0))
    with pytest.raises(ValueError, match="SasRecTransformerLayer"):
        body(query_encoder=DiffTransformerLayer(64, 2, 1))
    with pytest.raises(ValueError, match="side features"):
        body(query_tower_feature_names=["item_id", "genre"])
    with pytest.raises(ValueError, match="arange"):
        body(item_features_reader=_Reader({**reader.cols, "item_id": torch.arange(60).flip(0)}))


# ------------------------------------------------------------------------------------------ the oracle against the goldens
CASES = {"ce": ("ce", None), "bce": ("bce", None), "ce_sampled_shared": ("ce_sampled", "shared"),
         "ce_sampled_perseq": ("ce_sampled", "perseq"), "ce_sampled_perpos": ("ce_sampled", "perpos"),
         "login_ce_sampled_perseq": ("login_ce_sampled", "perseq"), "ce_sampled_weighted_shared": ("ce_sampled_weighted", "shared")}


def _oracle_inputs(z):
    from oracle import side_features as osf
    from oracle import twotower_side_features as ots

    specs = ots.golden_specs(z)
    sd = {k: v.double() for k, v in osf.golden_state_dict(z).items()}
    reader = {str(k): torch.from_numpy(z["item::" + str(k)]) for k in z["reader"] if str(k) != "item_id"}
    reader = {k: (v.double() if v.is_floating_point() else v) for k, v in reader.items()}
    feats = {k[len("feat::"):]: torch.from_numpy(z[k]) for k in z if k.startswith("feat::")}
    feats = {k: (v.double() if v.is_floating_point() else v) for k, v in feats.items()}
    t = lambda k: torch.from_numpy(z[k])  # noqa: E731
    return ots, specs, sd, reader, feats, t("ids"), t("pad_mask"), t("labels"), t("target_mask")


def _oracle_case(z, name):
    ots, specs, sd, reader, feats, ids, pm, lab, tm = _oracle_inputs(z)
    kind, layout = CASES[name]
    kw = {}
    if layout:
        kw = dict(negatives=torch.from_numpy(z[f"neg_{layout}"]), ignore_index=int(z["ignore_index"]))
    if kind == "ce_sampled_weighted":
        kw["weights"] = torch.from_numpy(z["weights"]).double()
    return ots.loss_and_grads(sd, specs, reader, ids, feats, pm, lab, tm, int(z["H"]), str(z["method"]), kind, **kw)


@pytest.mark.parametrize("tag", ["d64h2", "d50h1"])
@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_reference_golden(tag, name):
    """oracle/twotower_side_features.py (float64) reproduces the reference's loss, its full gradients (CE: every one;
    the others: the embedder's tables) and the sum and norm of every gradient"""
    z, _, _ = _golden(tag)
    loss, G = _oracle_case(z, name)
    ref = float(z[f"{name}::loss"])
    assert abs(float(loss) - ref) < 1e-5 * max(1.0, abs(ref)), (float(loss), ref)
    full = [k for k in z if k.startswith(f"{name}::grad::")]
    assert full
    for k in full:
        key = k.split("::")[2]
        want = torch.from_numpy(z[k]).double()
        assert torch.allclose(G[key].reshape(want.shape), want, rtol=1e-3, atol=1e-4 * float(want.abs().max()) + 1e-9), key
    for k in z:
        if k.startswith(f"{name}::gsum::"):
            key = k.split("::")[2]
            s, nrm = z[k]
            assert abs(float(G[key].norm()) - nrm) <= 1e-4 * nrm + 1e-9, key
            assert abs(float(G[key].sum()) - s) <= 1e-4 * nrm * G[key].numel() ** 0.5 + 1e-9, key


@pytest.mark.parametrize("tag", ["d64h2", "d50h1"])
def test_oracle_adam_step_matches_reference_golden(tag):
    """one Adam step of the CE loss (betas 0.9, 0.98, lr 1e-3) from the oracle's gradients: the reference's checksums.
    in_proj_bias is left out: its key third's exact gradient is zero (softmax is invariant to q . b_k), so Adam's first
    step moves it by +-lr on the sign of rounding noise on either side."""
    from oracle import sasrec as osr

    z, _, _ = _golden(tag)
    _, _, sd, *_ = _oracle_inputs(z)
    _, G = _oracle_case(z, "ce")
    for (k, p), (s, sq) in zip(sd.items(), z["adam_checksum"]):
        if k.endswith("in_proj_bias"):
            continue
        g = G[k]
        q, _, _ = osr.adam_step(p, g, torch.zeros_like(g), torch.zeros_like(g), 1)
        moved = float((q - p).abs().sum())
        assert abs(float(q.sum()) - s) <= 1e-6 * max(1.0, abs(s)) + 1e-3 * moved, k
        assert abs(float((q * q).sum()) - sq) <= 1e-6 * sq + 1e-9, k


@pytest.mark.parametrize("tag", ["d64h2", "d50h1"])
def test_oracle_inference_matches_reference_golden(tag):
    z, _, _ = _golden(tag)
    ots, specs, sd, reader, feats, ids, pm, _, _ = _oracle_inputs(z)
    H, method = int(z["H"]), str(z["method"])
    live = pm.any(1)   # a window without any item: the reference's eval attention over no key is not restated
    with torch.no_grad():
        lo = ots.eval_logits(sd, specs, reader, ids, feats, pm, H, method)
        cand = torch.from_numpy(z["candidates"])
        lc = ots.eval_logits(sd, specs, reader, ids, feats, pm, H, method, cand)
    assert torch.allclose(lo[live], torch.from_numpy(z["eval_logits"]).double()[live], atol=1e-4)
    for key in ("cand_logits", "cand_logits_nocache"):
        assert torch.allclose(lc[live], torch.from_numpy(z[key]).double()[live], atol=1e-4), key
    for b in range(ids.shape[0]):
        lo[b, ids[b][pm[b]]] = -torch.inf
    assert torch.equal(torch.topk(lo, 10, dim=-1).indices[live], torch.from_numpy(z["top10"])[live])
