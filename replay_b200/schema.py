"""Minimal stand-ins for ``replay.data.nn.TensorSchema`` / ``TensorFeatureInfo`` exposing only the duck-typed surface
the sequential models touch (SURVEY.md §8b "Duck-type surface"): when RePlay itself is importable, pass its own schema
objects instead - the models accept either."""
from __future__ import annotations

from dataclasses import dataclass


@dataclass
class TensorFeatureInfo:
    """``is_list``: a categorical / numerical list; ``tensor_dim``: the last dimension of a numerical feature's values."""
    name: str
    cardinality: int | None
    padding_value: int
    embedding_dim: int
    is_seq: bool = True
    is_cat: bool = True
    is_list: bool = False
    tensor_dim: int | None = None

    def _set_cardinality(self, n: int) -> None:
        self.cardinality = n


class _Single:
    def __init__(self, f):
        self._f = f

    def item(self):
        return self._f


class TensorSchema:
    """The categorical sequential item-id feature (what SASRec / BERT4Rec need on the hot path), optionally followed by
    ``features``: the side features the new-path SASRec embeds next to it."""

    def __init__(self, item_feature: TensorFeatureInfo, query_id_feature_name: str = "query_id",
                 timestamp_feature_name: str | None = None, features=()):
        self._item = item_feature
        self._extra = list(features)
        self.query_id_feature_name = query_id_feature_name
        self.timestamp_feature_name = timestamp_feature_name

    @property
    def item_id_features(self):
        return _Single(self._item)

    @property
    def item_id_feature_name(self) -> str:
        return self._item.name

    def items(self):
        return [(f.name, f) for f in [self._item, *self._extra]]

    def __getitem__(self, name):
        for k, f in self.items():
            if k == name:
                return f
        raise KeyError(name)

    @property
    def categorical_features(self):
        return {k: f for k, f in self.items() if f.is_cat}

    @property
    def numerical_features(self):
        return {k: f for k, f in self.items() if not f.is_cat}


def item_feature_of(schema):
    """(name, cardinality, padding_value, embedding_dim) from a RePlay TensorSchema or the stand-in above."""
    f = schema.item_id_features.item()
    return schema.item_id_feature_name, int(f.cardinality), int(f.padding_value), getattr(f, "embedding_dim", None)


def side_features_of(schema, excluded=(), list_aggregation: str = "sum") -> list:
    """The side features ``SequenceEmbedding`` embeds next to the item id (replay/nn/embedding.py:52-70), as
    ``engine.SideFeature``s: every feature of the schema that is neither excluded nor the item id.  Raises as the reference
    does for a non-sequential feature (NotImplementedError), and ValueError for a list aggregation the CUDA path does not
    implement ("max": a bf16 argmax may pick another element than the fp32 reference)."""
    from .engine import SideFeature

    item = schema.item_id_feature_name
    out = []
    for name, f in schema.items():
        if name in excluded or name == item:
            continue
        if not f.is_seq:
            raise NotImplementedError(f"Non-sequential features is not yet supported. Got {name}")
        if f.is_cat:
            if getattr(f, "is_list", False):
                if list_aggregation not in ("sum", "mean"):
                    raise ValueError(f"categorical_list_feature_aggregation_method={list_aggregation!r} is not supported "
                                     "on the CUDA path (sum, mean)")
                kind = "bag_" + list_aggregation
            else:
                kind = "cat"
            out.append(SideFeature(name, kind, int(f.cardinality), int(f.padding_value), 1))
        else:
            td = int(f.tensor_dim)
            out.append(SideFeature(name, "ident" if td == f.embedding_dim else "num", 0, 0, td))
    return out


def bert_side_features_of(schema) -> list:
    """The side features the legacy BERT4Rec sums into its item embedding (BertEmbedding, bert4rec/model.py:173-296), as
    ``engine.SideFeature``s: every categorical feature but the item id (kind "cat", an Embedding of ``cardinality`` rows
    without a padding row), then every numerical one (kind "ident": its values are added as they are), each in schema order,
    the order of the reference's sum.  Raises as the reference's constructor does: NotImplementedError for a non-sequential
    feature, ValueError when a feature's dim (``embedding_dim`` of a categorical, ``tensor_dim`` of a numerical) differs from
    the first feature's.  A categorical list raises NotImplementedError here; the reference fails later, at forward."""
    from .engine import SideFeature

    item = schema.item_id_feature_name
    common, cats, nums = None, [], []
    for name, f in schema.items():
        if not f.is_seq:
            raise NotImplementedError("Non-sequential features is not yet supported")
        dim = f.embedding_dim if f.is_cat else f.tensor_dim
        if common is None:
            common = dim
        if dim != common:
            raise ValueError("Dimension of all features must be the same for sum aggregation")
        if name == item:
            continue
        if f.is_cat:
            cats.append(SideFeature(name, "bag_sum" if getattr(f, "is_list", False) else "cat", int(f.cardinality),
                                    int(f.padding_value), 1))
        else:
            nums.append(SideFeature(name, "ident", 0, 0, int(f.tensor_dim)))
    for f in cats:   # after the loop: the reference's own construction errors come first
        if f.kind != "cat":
            raise NotImplementedError(f"BERT4Rec cannot sum the categorical list feature {f.name!r} into its input")
    return cats + nums
