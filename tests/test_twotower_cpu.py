"""TwoTower without a GPU: oracle/twotower.py against the golden vectors of the real reference (tests/golden/twotower_*.npz,
written by oracle/gen_twotower_golden.py), the reference's state_dict keys, and every configuration the CUDA path
rejects at construction."""
import os

import numpy as np
import pytest
import torch

from oracle import twotower as ott
from oracle.diff import from_bf16_bits
from replay_b200.schema import TensorFeatureInfo, TensorSchema

GOLD = os.path.join(os.path.dirname(__file__), "golden")
TAGS = ("d64h2", "d50h1", "d128h2")


def load(tag):
    return dict(np.load(os.path.join(GOLD, f"twotower_{tag}.npz")))


def case_inputs(z):
    t = lambda k: torch.from_numpy(z[k])  # noqa: E731
    return t("ids"), t("pad_mask"), t("labels"), t("target_mask")


def golden_sd(z, dtype=torch.float64):
    n, d, H, L, nb = (int(z[k]) for k in ("n_items", "d", "H", "L", "n_blocks"))
    sd = ott.seeded_state_dict(n, d, H, L, nb, int(z["seed"]))
    keys = list(z["sd_keys"])
    assert list(sd) == keys
    for k, s in zip(keys, z["sd_sums"]):
        assert abs(float(sd[k].double().sum()) - s) <= 1e-6 * max(1.0, abs(s)), k
    return ott.to_dtype(sd, dtype)


CASES = {"bce": dict(kind="bce"), "ce_sampled_shared": dict(kind="ce_sampled", neg="shared"),
         "ce_sampled_perseq": dict(kind="ce_sampled", neg="perseq"), "ce_sampled_perpos": dict(kind="ce_sampled", neg="perpos"),
         "login_ce_sampled_perseq": dict(kind="login_ce_sampled", neg="perseq"),
         "ce_sampled_weighted_shared": dict(kind="ce_sampled_weighted", neg="shared")}


def oracle_case(z, sd, name):
    ids, pm, lab, tm = case_inputs(z)
    H = int(z["H"])
    if name == "ce":
        return ott.loss_and_grads(sd, ids, pm, lab, tm, H, "ce")
    c = CASES[name]
    kw = {}
    if "neg" in c:
        kw = dict(negatives=torch.from_numpy(z[f"neg_{c['neg']}"]), ignore_index=int(z["ignore_index"]))
    if c["kind"] == "ce_sampled_weighted":
        kw["weights"] = torch.from_numpy(z["weights"]).double()
    return ott.loss_and_grads(sd, ids, pm, lab, tm, H, c["kind"], **kw)


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_ce_matches_reference(tag):
    z = load(tag)
    sd = golden_sd(z)
    loss, G = oracle_case(z, sd, "ce")
    assert abs(float(loss) - float(z["ce::loss"])) < 1e-5 * abs(float(z["ce::loss"]))
    keys = [k[len("ce::grad::"):] for k in z if k.startswith("ce::grad::")]
    assert sorted(keys) == sorted(G)
    for k in keys:
        ref = from_bf16_bits(z[f"ce::grad::{k}"]).double()
        assert torch.allclose(G[k].reshape(ref.shape), ref, rtol=2e-2, atol=1e-2 * float(ref.abs().max()) + 1e-9), k


@pytest.mark.parametrize("tag", TAGS)
@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_losses_match_reference(tag, name):
    z = load(tag)
    loss, G = oracle_case(z, golden_sd(z), name)
    ref = float(z[f"{name}::loss"])
    assert abs(float(loss) - ref) < 1e-5 * max(1.0, abs(ref)), (float(loss), ref)
    for k, g in G.items():
        s, nrm = z[f"{name}::gsum::{k}"]
        assert abs(float(g.norm()) - nrm) <= 1e-4 * nrm + 1e-9, k
        assert abs(float(g.sum()) - s) <= 1e-4 * nrm * g.numel() ** 0.5 + 1e-9, k


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_inference_matches_reference(tag):
    z = load(tag)
    sd = golden_sd(z)
    ids, pm, _, _ = case_inputs(z)
    H = int(z["H"])
    with torch.no_grad():
        lo = ott.eval_logits(sd, ids, pm, H)
        cand = torch.from_numpy(z["candidates"])
        lc = ott.eval_logits(sd, ids, pm, H, cand)
    live = pm.any(1)   # a window without any item: the reference's eval attention over no key is not restated
    assert torch.allclose(lo[live], torch.from_numpy(z["eval_logits"]).double()[live], atol=1e-4)
    assert torch.allclose(lc[live], torch.from_numpy(z["cand_logits"]).double()[live], atol=1e-4)
    for b in range(ids.shape[0]):
        lo[b, ids[b][pm[b]]] = -torch.inf
    assert torch.equal(torch.topk(lo, 10, dim=-1).indices[live], torch.from_numpy(z["top10"])[live])


@pytest.mark.parametrize("tag", TAGS)
def test_key_list_matches_reference(tag):
    from replay_b200.nn.sequential.twotower import twotower_keys

    z = load(tag)
    keys = twotower_keys(int(z["n_blocks"]))
    assert keys == list(z["sd_keys"])
    with_cache = list(z["cache_keys"])
    i = with_cache.index("body.item_tower.cache")
    assert with_cache[:i] + with_cache[i + 1:] == keys and with_cache[i - 1] == "body.item_tower.item_reference_item_id"


def test_key_map_covers_every_engine_parameter():
    from replay_b200.engine_twotower import TwoTowerConfig
    from replay_b200.nn.sequential.twotower import twotower_key_map, twotower_keys

    cfg = TwoTowerConfig(n_items=40, d=64, n_heads=2, n_blocks=2, max_len=12)
    m = twotower_key_map(2)
    names = [n for n, _, _ in cfg.param_layout()]
    assert sorted(m) == sorted(names)
    assert set(m.values()) <= set(twotower_keys(2))
    shapes = cfg.true_shapes()
    assert shapes["tw0.wg"] == (128, 64) and shapes["tw1.w2"] == (64, 128) and shapes["tw0.norm"] == (64,)


# ---------------------------------------------------------------------------------------------------------------- construction
class _Reader:
    def __init__(self, cols):
        self.cols = cols

    def __getitem__(self, k):
        return self.cols[k]

    @property
    def feature_names(self):
        return list(self.cols)


class _SideFeatureSchema(TensorSchema):
    """the item feature and one categorical side feature"""

    def items(self):
        return super().items() + [("genre", TensorFeatureInfo("genre", 5, 5, 64))]


def _schema(n=30, d=64, extra=False):
    return (_SideFeatureSchema if extra else TensorSchema)(TensorFeatureInfo("item_id", n, n, d))


def _body(**over):
    from replay_b200.nn.agg import SumAggregator
    from replay_b200.nn.embedding import SequenceEmbedding
    from replay_b200.nn.ffn import SwiGLUEncoder
    from replay_b200.nn.mask import DefaultAttentionMask
    from replay_b200.nn.sequential import PositionAwareAggregator, SasRecTransformerLayer
    from replay_b200.nn.sequential.twotower import TwoTowerBody

    sch = over.pop("schema", _schema())
    d = 64
    agg = SumAggregator(d)
    kw = dict(schema=sch, embedder=SequenceEmbedding(sch), attn_mask_builder=DefaultAttentionMask("item_id", 2),
              query_tower_feature_names=["item_id"], query_embedding_aggregator=PositionAwareAggregator(agg, 16, 0.1),
              item_embedding_aggregator=agg, query_encoder=SasRecTransformerLayer(d, 2, 1, 0.1, activation="relu"),
              query_tower_output_normalization=torch.nn.LayerNorm(d), item_encoder=SwiGLUEncoder(d, 2 * d),
              item_features_reader=_Reader({"item_id": torch.arange(30)}))
    kw.update(over)
    return TwoTowerBody(**kw)


def _core(**over):
    return _body(**over).build_core(device="cpu")


def test_default_body_builds():
    core = _core()
    assert core.cfg.n_items == 30 and core.cfg.d == 64 and core.cfg.ffn_p == 128


@pytest.mark.parametrize("over, match", [
    (lambda: dict(query_encoder=__import__("replay_b200.nn.sequential", fromlist=["x"]).SasRecTransformerLayer(64, 2, 1, 0.1)),
     "activation"),
    (lambda: dict(query_encoder=__import__("replay_b200.nn.sequential", fromlist=["x"]).DiffTransformerLayer(64, 2, 1)),
     "SasRecTransformerLayer"),
    (lambda: dict(query_tower_output_normalization=torch.nn.RMSNorm(64)), "LayerNorm"),
    (lambda: dict(item_encoder=__import__("replay_b200.nn.ffn", fromlist=["x"]).SwiGLUEncoder(64, 100)), "hidden_dim"),
    (lambda: dict(item_encoder=object()), "SwiGLUEncoder"),
    (lambda: dict(item_features_reader=_Reader({"item_id": torch.arange(30).flip(0)})), "arange"),
    (lambda: dict(item_features_reader=_Reader({"item_id": torch.arange(29)})), "arange"),
    (lambda: dict(item_embedding_aggregator=object()), "SumAggregator"),
])
def test_unsupported_parts_raise(over, match):
    with pytest.raises(ValueError, match=match):
        _core(**over())


def test_side_features_raise():
    from replay_b200.nn.embedding import SequenceEmbedding

    sch = _schema(extra=True)
    with pytest.raises(ValueError, match="side features"):
        _core(schema=sch, embedder=SequenceEmbedding(sch))
    with pytest.raises(ValueError, match="genre"):
        _core(schema=sch, embedder=SequenceEmbedding(sch, excluded_features=["genre"]),
              item_features_reader=_Reader({"item_id": torch.arange(30), "genre": torch.zeros(30, dtype=torch.long)}))


def test_context_merger_raises():
    from replay_b200.nn.sequential.twotower import TwoTower

    with pytest.raises(ValueError, match="context_merger"):
        TwoTower(_body(), context_merger=object(), device="cpu")


def test_from_params_builds_the_reference_shape():
    from replay_b200.nn.sequential.twotower import TwoTower

    m = TwoTower.from_params(_schema(), _Reader({"item_id": torch.arange(30)}), embedding_dim=64, num_heads=2, num_blocks=2,
                             max_sequence_length=16, dropout=0.0, device="cpu")
    cfg = m.core.cfg
    assert (cfg.n_items, cfg.d, cfg.n_heads, cfg.n_blocks, cfg.max_len, cfg.lnf_eps) == (30, 64, 2, 2, 16, 1e-5)
    assert type(m.loss).__name__ == "CE" and m.loss.ignore_index == 30
    assert m.loss.logits_callback == m.get_logits
    assert list(m.state_dict()) == ["body.item_tower.item_reference_item_id"]   # no engine without a GPU


def test_features_reader_reads_parquet(tmp_path):
    import pandas as pd

    from replay_b200.nn.sequential.twotower import FeaturesReader

    sch = _schema()
    path = tmp_path / "items.parquet"
    pd.DataFrame({"item_id": np.random.default_rng(0).permutation(30)}).to_parquet(path)
    r = FeaturesReader(sch, {"item_id": {}}, str(path))
    assert list(r.feature_names) == ["item_id"] and torch.equal(r["item_id"], torch.arange(30))
