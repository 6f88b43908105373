"""Mirror of ``replay.nn.sequential.twotower`` (replay/nn/sequential/twotower/{model,reader}.py) backed by the H100 engine
(replay_b200/engine_twotower.py).

Same construction (``TwoTower(body, loss)`` and ``from_params(schema, item_features_reader, ...)``), the same ``forward`` /
``forward_train`` / ``forward_inference`` / ``get_logits`` contracts and the same ``state_dict`` keys as the reference: the
query tower is the new-path SASRec body, the item tower SwiGLUEncoder(d, 2d) over the sum of the reader's item features,
embedded by the tables both towers share.  The query tower reads the schema's side features from ``feature_tensors`` as
``SasRec`` does; the item tower reads the reader's columns, held on the device."""
from __future__ import annotations

import torch

from ...core import _LEAF, SasRecCore
from ...engine import _BLOCK_PARAMS
from ...engine_twotower import TOWER_LAYERS, TwoTowerConfig, TwoTowerEngine
from ...schema import item_feature_of, side_features_of
from ..agg import SumAggregator
from ..embedding import SequenceEmbedding
from ..ffn import SwiGLUEncoder
from ..loss import CE
from ..mask import DefaultAttentionMask
from .sasrec import PositionAwareAggregator, SasRec, SasRecTransformerLayer, _check_side

_TOWER_LEAF = {"wg": "WG.weight", "bg": "WG.bias", "w1": "W1.weight", "b1": "W1.bias", "w2": "W2.weight", "b2": "W2.bias"}


class FeaturesReader:
    """replay/nn/sequential/twotower/reader.py: the item features of a parquet file (encoded columns), sorted by item id,
    as tensors by feature name.  Any object with ``__getitem__`` and ``feature_names`` can stand in for it."""

    def __init__(self, schema, metadata: dict, path: str, **kwargs):
        import numpy as np
        import pandas as pd

        item = schema.item_id_feature_name
        if item is None:
            raise ValueError("Items identifier doesn't specified.Please pass a `TensorFeatureInfo` to `TensorSchema` with "
                             "parameter feature_hint setted to FeatureHint.ITEM_ID.")
        extra = set(metadata) - {item} - {n for n, f in schema.items() if _source_is_item_features(f)}
        if extra:
            raise ValueError(f"The metadata contains information about the following columns,which are not described in "
                             f"schema: {extra}.")
        features = pd.read_parquet(path=path, columns=list({*metadata, item}), **kwargs)
        for k, v in metadata.items():
            if v:
                features[k] = features[k].apply(lambda r, v=v: np.concatenate(([v["padding"]] * (v["shape"] - len(r)), r)))
        features = features.sort_values(by=item).reset_index(drop=True)
        self._features = {}
        for k in metadata:
            num = bool(getattr(schema[k], "is_num", False))
            col = features[k]
            arr = np.asarray(col.to_list() if getattr(schema[k], "is_list", False) else col.to_numpy(),
                             dtype=np.float32 if num else np.int64)
            self._features[k] = torch.from_numpy(arr.copy())

    def __getitem__(self, key: str) -> torch.Tensor:
        return self._features[key]

    @property
    def feature_names(self):
        return self._features.keys()


def _source_is_item_features(info) -> bool:
    src = getattr(info, "feature_source", None)
    return src is not None and str(getattr(src, "source", "")).upper().endswith("ITEM_FEATURES")


def _embedder_keys(pre: str, item_feature: str, features=()) -> list:
    """the keys of SequenceEmbedding's feature_embedders under ``pre``: the item table, then each side feature's
    (nn/embedding.py: CategoricalEmbedding.emb, NumericalEmbedding.linear, IdentityEmbedding's _weight buffer)"""
    keys = [f"{pre}embedder.feature_embedders.{item_feature}.emb.weight"]
    for f in features:
        e = f"{pre}embedder.feature_embedders.{f.name}."
        keys += ([e + "emb.weight"] if f.categorical else [e + "linear.weight", e + "linear.bias"] if f.kind == "num"
                 else [e + "_weight"])
    return keys


def twotower_keys(n_blocks: int, item_feature: str = "item_id", features=(), item_features=()) -> list:
    """Every parameter / buffer key of the reference's TwoTower in its ``state_dict`` order, without the item tower's
    ``cache`` (which follows the last ``body.item_tower.item_reference_<f>`` while the reference holds one).  ``features``:
    the embedder's side features (engine.SideFeature, schema order); ``item_features``: the names of those the item
    features reader holds besides the item id."""
    enc = "body.query_tower.encoder."
    keys = _embedder_keys("body.", item_feature, features) + _embedder_keys("body.query_tower.", item_feature, features)
    keys.append("body.query_tower.embedding_aggregator.pe.weight")
    for group in (("in_w", "in_b", "out_w", "out_b"), ("ln1_w", "ln1_b"), ("w1", "b1", "w2", "b2"), ("ln2_w", "ln2_b")):
        keys += [enc + _LEAF[k].format(i=i) for i in range(n_blocks) for k in group]
    keys += ["body.query_tower.output_normalization.weight", "body.query_tower.output_normalization.bias"]
    keys += [f"body.item_tower.item_reference_{n}" for n in (item_feature, *item_features)]
    keys += _embedder_keys("body.item_tower.", item_feature, features)
    for layer in (1, 2):
        keys += [f"body.item_tower.encoder.sw{layer}.{_TOWER_LEAF[k]}" for k in ("wg", "bg", "w1", "b1", "w2", "b2")]
        keys.append(f"body.item_tower.encoder.norm{layer}.weight")
    return keys


def twotower_key_map(n_blocks: int, item_feature: str = "item_id", features=()) -> dict:
    """engine parameter name -> reference key (the shared tables under ``body.embedder``)"""
    m = {"item_emb": f"body.embedder.feature_embedders.{item_feature}.emb.weight",
         "pos_emb": "body.query_tower.embedding_aggregator.pe.weight",
         "lnf_w": "body.query_tower.output_normalization.weight", "lnf_b": "body.query_tower.output_normalization.bias"}
    for i in range(n_blocks):
        m.update({f"b{i}.{k}": "body.query_tower.encoder." + _LEAF[k].format(i=i) for k in _BLOCK_PARAMS})
    for layer, p in enumerate(TOWER_LAYERS, start=1):
        m.update({p + k: f"body.item_tower.encoder.sw{layer}.{v}" for k, v in _TOWER_LEAF.items()})
        m[p + "norm"] = f"body.item_tower.encoder.norm{layer}.weight"
    for f in features:
        pre = f"body.embedder.feature_embedders.{f.name}."
        if f.categorical:
            m[f"feat.{f.name}"] = pre + "emb.weight"
        elif f.kind == "num":
            m.update({f"feat.{f.name}.w": pre + "linear.weight", f"feat.{f.name}.b": pre + "linear.bias"})
    return m


class TwoTowerCore(SasRecCore):
    """SasRecCore on the TwoTower engine: the item table of every head is the item tower's output over the catalog, kept
    until the parameters change.  ``cache_live`` follows the reference's ``item_tower.cache`` (set by an eval forward over
    the whole catalog, cleared by a training forward): the ``state_dict`` carries the cache while it is live."""

    def __init__(self, cfg: TwoTowerConfig, item_feature: str = "item_id", device=None, seed: int = 0, item_values=None):
        self.cache_live = False
        # the item features reader's side columns (cfg.item_features) as it gave them: the state_dict's item_reference_<f>
        self.item_values = {n: torch.as_tensor(item_values[n]).detach().cpu().clone() for n in cfg.item_features}
        super().__init__(cfg, item_feature=item_feature, device=device, seed=seed)

    def _init_args(self) -> dict:
        return {**super()._init_args(), "item_values": self.item_values}

    def _key_map(self):
        return twotower_key_map(self.cfg.n_blocks, self.item_feature, self.cfg.features)

    def _make_engine(self, batch, seq_len, with_grad):
        return TwoTowerEngine(self.cfg, batch, seq_len, self._device, seed=self._seed, with_grad=with_grad,
                              item_values=self.item_values)

    def _keys(self):
        return twotower_keys(self.cfg.n_blocks, self.item_feature, self.cfg.features, self.cfg.item_features)

    def _shared_keys(self):
        """reference key under body.embedder -> its two aliases (the query and item towers share the embedder)"""
        main = _embedder_keys("body.", self.item_feature, self.cfg.features)
        q = _embedder_keys("body.query_tower.", self.item_feature, self.cfg.features)
        it = _embedder_keys("body.item_tower.", self.item_feature, self.cfg.features)
        return {m: (a, b) for m, a, b in zip(main, q, it)}

    def _ref_keys(self):
        return {f"body.item_tower.item_reference_{n}": n for n in (self.item_feature, *self.cfg.item_features)}

    def _cache_key(self):
        return "body.item_tower.cache"

    def _reference_buffer(self, name):
        return torch.arange(self.cfg.n_items, dtype=torch.int64) if name == self.item_feature else self.item_values[name]

    def state_dict(self, *args, destination=None, prefix="", keep_vars=False):  # noqa: D102
        src = self._export() if self.engine is not None else dict(self._pending_state or {})
        for f in self.cfg.features:   # IdentityEmbedding's buffer (nn/embedding.py): eye(d), no parameter
            if f.kind == "ident":
                src[f"body.embedder.feature_embedders.{f.name}._weight"] = torch.eye(self.cfg.d)
        for main, aliases in self._shared_keys().items():
            if main in src:
                for a in aliases:
                    src[a] = src[main]
        refs = self._ref_keys()
        for k, n in refs.items():
            src[k] = self._reference_buffer(n)
        last_ref = list(refs)[-1]
        out = destination if destination is not None else {}
        for k in self._keys():
            if k in src:
                out[prefix + k] = src[k]
            if k == last_ref and self.cache_live and self.engine is not None:
                out[prefix + self._cache_key()] = self.engine.unpad_features(self.item_table()).float().cpu()
        return out

    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):  # noqa: D102
        """The reference's keys; a shared table is read from whichever of its three keys comes last in the reference's
        order.  The item_reference_<f> buffers must hold the reader the model was built with (the item id's: arange).
        ``body.item_tower.cache`` is optional and, when present, is the tower output the next eval forward uses (the
        reference's shape checks apply)."""
        keys = self._keys()
        missing = [k for k in keys if k not in state_dict]
        if strict and missing:
            raise RuntimeError(f"missing keys in state_dict: {missing[:5]} ...")
        for k, n in self._ref_keys().items():
            ref = state_dict.get(k)
            if ref is None:
                continue
            mine = self._reference_buffer(n)
            ref = torch.as_tensor(ref).cpu()
            if ref.shape != mine.shape or not torch.equal(ref.to(mine.dtype), mine):
                if n == self.item_feature:
                    raise ValueError(f"{k} must equal arange({self.cfg.n_items}) (logit column i is item i)")
                raise ValueError(f"{k} differs from the item features reader this model was built with")
        cache = state_dict.get(self._cache_key())
        if cache is not None and (cache.dim() != 2 or cache.shape[0] != self.cfg.n_items or cache.shape[1] != self.cfg.d):
            raise AssertionError(f"cache of shape {tuple(cache.shape)} does not fit [{self.cfg.n_items}, {self.cfg.d}]")
        inv = {v: k for k, v in self._keymap.items()}
        for main, aliases in self._shared_keys().items():
            for a in aliases:
                if main in inv:
                    inv[a] = inv[main]
        ordered = {}
        for k in keys:   # the reference's order: the last of a shared table's three keys wins
            if k in state_dict and k in inv:
                ordered[self._keymap[inv[k]]] = state_dict[k]
        if self.engine is None:
            self._pending_state = {k: torch.as_tensor(v).detach().clone() for k, v in ordered.items()}
        else:
            self._import(ordered)
            if cache is not None:
                eng = self._eval_engine_ready()
                eng._alloc_tower()["cache"].copy_(eng.pad_features(cache.to(eng.dev, torch.float32)).to(torch.bfloat16))
                eng.tower_valid = True
        self.cache_live = cache is not None
        return torch.nn.modules.module._IncompatibleKeys(missing, [])

    def _eval_engine_ready(self):
        eng = self.engine
        if self._shadow_dirty:
            eng.refresh_shadow()
            self._shadow_dirty = False
        return eng

    def _to_ref(self, k, v):
        return v if k.startswith(TOWER_LAYERS) else super()._to_ref(k, v)   # Linear weights (no Conv1d axis)

    def _from_ref(self, k, v):
        return v if k.startswith(TOWER_LAYERS) else super()._from_ref(k, v)

    def _import(self, state: dict):
        super()._import(state)
        if self.engine is not None:
            self.engine.tower_valid = False

    def mark_params_updated(self):
        super().mark_params_updated()
        if self.engine is not None:
            self.engine.tower_valid = False

    def loss(self, *args, **kwargs):
        self.cache_live = False
        out = super().loss(*args, **kwargs)
        self.engine.tower_valid = False
        return out

    def fused_step(self, *args, **kwargs):
        """A replayed step graph runs no Python of the engine: the tower over the catalog is marked stale here, after the
        step changed the parameters (and, with a full-catalog loss, wrote the cache with the pre-step tower)."""
        self.cache_live = False
        out = super().fused_step(*args, **kwargs)
        self.engine.tower_valid = False
        return out

    @torch.no_grad()
    def item_table(self, candidates=None) -> torch.Tensor:
        """The item tower's output (bf16, padded width) over the catalog or the given candidates."""
        t = self._eval_engine_ready().tower_table()
        return t if candidates is None else t[candidates].contiguous()

    @torch.no_grad()
    def predict_topk(self, ids, pad_mask, k: int, seen_ids=None, candidates=None, feats=None):
        # the tower runs outside any captured predict graph, which then reads its (stable) output buffer
        self._eval_engine(ids)
        self.item_table()
        return super().predict_topk(ids, pad_mask, k, seen_ids, candidates, feats=feats)


class TwoTowerBody:
    """replay/nn/sequential/twotower/model.py ``TwoTowerBody`` (config only): the parts are read when ``TwoTower(body, loss)``
    builds the engine."""

    def __init__(self, schema, embedder, attn_mask_builder, query_tower_feature_names, query_embedding_aggregator,
                 item_embedding_aggregator, query_encoder, query_tower_output_normalization, item_encoder,
                 item_features_reader) -> None:
        missing = (set(query_tower_feature_names) | set(item_features_reader.feature_names)) - set(_embedder_features(embedder))
        if missing:
            raise ValueError(f"Feature names found that embedder does not support {list(missing)}")
        self.schema = schema
        self.embedder = embedder
        self.attn_mask_builder = attn_mask_builder
        self.query_tower_feature_names = query_tower_feature_names
        self.query_embedding_aggregator = query_embedding_aggregator
        self.item_embedding_aggregator = item_embedding_aggregator
        self.query_encoder = query_encoder
        self.query_tower_output_normalization = query_tower_output_normalization
        self.item_encoder = item_encoder
        self.item_features_reader = item_features_reader

    def build_core(self, device=None, seed: int = 0) -> TwoTowerCore:
        """The engine configuration this body describes; ValueError for anything the CUDA path does not implement."""
        emb, qagg, iagg, mask = self.embedder, self.query_embedding_aggregator, self.item_embedding_aggregator, self.attn_mask_builder
        enc, norm, ienc, reader = self.query_encoder, self.query_tower_output_normalization, self.item_encoder, self.item_features_reader
        if not isinstance(emb, SequenceEmbedding):
            raise ValueError(f"embedder must be SequenceEmbedding, got {type(emb).__name__}")
        name, card, pad, feat_dim = item_feature_of(self.schema)
        if pad != card:
            raise ValueError("the item feature's padding_value must equal its cardinality (replay/data/nn/schema.py:89-90)")
        skip = set(emb.excluded_features) | {self.schema.query_id_feature_name, self.schema.timestamp_feature_name}
        side = side_features_of(emb.schema, skip, emb.categorical_list_feature_aggregation_method)
        unused = sorted({name, *(f.name for f in side)} - set(self.query_tower_feature_names))
        if unused:   # the query tower's input sums every embedder table (the CUDA path has no per-tower feature subset)
            raise ValueError(f"side features {unused} are in the embedder but not in query_tower_feature_names; the query tower "
                             "must embed every feature of the embedder (exclude the others from the SequenceEmbedding)")
        if name not in reader.feature_names:
            raise ValueError(f"the item features reader must hold the item feature {name!r}")
        item_side = [f.name for f in side if f.name in set(reader.feature_names)]
        ref = torch.as_tensor(reader[name]).cpu()
        if ref.dim() != 1 or not torch.equal(ref.long(), torch.arange(card)):
            raise ValueError(f"the item features reader's {name!r} column must equal arange({card}): the rows of a complete, "
                             "encoded item table")
        if not isinstance(qagg, PositionAwareAggregator) or not isinstance(qagg.embedding_aggregator, SumAggregator):
            raise ValueError("query_embedding_aggregator must be PositionAwareAggregator(SumAggregator(...), ...)")
        if not isinstance(iagg, SumAggregator):
            raise ValueError(f"item_embedding_aggregator must be SumAggregator, got {type(iagg).__name__}")
        if not isinstance(mask, DefaultAttentionMask) or mask.reference_feature_name != name:
            raise ValueError(f"attn_mask_builder must be DefaultAttentionMask on the item feature {name!r}")
        if not isinstance(enc, SasRecTransformerLayer):
            raise ValueError(f"query_encoder must be SasRecTransformerLayer, got {type(enc).__name__}")
        if enc.activation != "relu":
            raise ValueError(f"SasRecTransformerLayer supports activation='relu' only, got {enc.activation!r}")
        d = enc.embedding_dim
        _check_side(emb.schema, side, d)
        if qagg.embedding_aggregator.embedding_dim != d or iagg.embedding_dim != d or (feat_dim is not None and feat_dim != d):
            raise ValueError("the embedder, the aggregators and the encoders must share one embedding_dim")
        if mask.num_heads != enc.num_heads:
            raise ValueError("attn_mask_builder.num_heads must equal the query encoder's num_heads")
        if enc.dropout != qagg.dropout:
            raise ValueError("the aggregator and SasRecTransformerLayer must share one dropout")
        if not (isinstance(norm, torch.nn.LayerNorm) and norm.elementwise_affine and norm.bias is not None):
            raise ValueError("query_tower_output_normalization must be torch.nn.LayerNorm with affine weights and bias "
                             f"(got {type(norm).__name__})")
        if tuple(norm.normalized_shape) != (d,):
            raise ValueError(f"query_tower_output_normalization must normalise {d} features")
        if not isinstance(ienc, SwiGLUEncoder):
            raise ValueError(f"item_encoder must be SwiGLUEncoder, got {type(ienc).__name__}")
        if ienc.embedding_dim != d or ienc.hidden_dim != 2 * d:
            raise ValueError(f"item_encoder must be SwiGLUEncoder(embedding_dim={d}, hidden_dim={2 * d}), got "
                             f"({ienc.embedding_dim}, {ienc.hidden_dim})")
        cfg = TwoTowerConfig(n_items=card, d=d, n_heads=enc.num_heads, n_blocks=enc.num_blocks, max_len=qagg.max_sequence_length,
                             dropout=qagg.dropout, variant="new", lnf_eps=norm.eps, features=tuple(side),
                             item_features=tuple(item_side))
        return TwoTowerCore(cfg, item_feature=name, device=device, seed=seed,
                            item_values={n: reader[n] for n in item_side})


def _embedder_features(emb) -> list:
    """the features a SequenceEmbedding embeds (the schema's, less its exclusions, the query id and the timestamp)"""
    if not isinstance(emb, SequenceEmbedding):
        return list(getattr(emb, "feature_names", []))
    sch = emb.schema
    skip = set(emb.excluded_features) | {sch.query_id_feature_name, sch.timestamp_feature_name}
    return [f for f, _ in sch.items() if f not in skip]


class TwoTower(SasRec):
    """replay/nn/sequential/twotower/model.py ``TwoTower``: query tower (SASRec body) and item tower (SwiGLUEncoder) fused
    by a dot product.  The losses of ``replay_b200.nn.loss`` select the fused heads (full-catalog and sampled); the sampled
    losses run the item tower on the step's distinct candidates only."""

    multi_positive = False   # the sampled losses' candidate compaction takes one label per position

    def __init__(self, body, loss=None, context_merger=None, device=None, seed: int = 0):
        if context_merger is not None:
            raise ValueError("context_merger is not supported (only None)")
        core = body.build_core(device=device, seed=seed) if isinstance(body, TwoTowerBody) else body
        super().__init__(core, loss=loss, device=device, seed=seed)
        self.context_merger = None

    @SasRec.loss.setter
    def loss(self, spec):
        SasRec.loss.fset(self, spec)
        if hasattr(spec, "logits_callback"):
            spec.logits_callback = self.get_logits

    @classmethod
    def from_params(cls, schema, item_features_reader, embedding_dim: int = 192, num_heads: int = 4, num_blocks: int = 2,
                    max_sequence_length: int = 50, dropout: float = 0.3, excluded_features=None,
                    categorical_list_feature_aggregation_method: str = "sum", device=None, seed: int = 0) -> "TwoTower":
        """replay/nn/sequential/twotower/model.py:535-626: SASRec query tower with a LayerNorm output, SwiGLUEncoder(d, 2d)
        item tower, one SumAggregator for both towers, CE loss."""
        excluded = list({schema.query_id_feature_name, schema.timestamp_feature_name, *(excluded_features or [])} - {None})
        names = {n for n, _ in schema.items()} - set(excluded)
        common = SumAggregator(embedding_dim)
        body = TwoTowerBody(
            schema=schema,
            embedder=SequenceEmbedding(schema, excluded_features=excluded,
                                       categorical_list_feature_aggregation_method=categorical_list_feature_aggregation_method),
            attn_mask_builder=DefaultAttentionMask(schema.item_id_feature_name, num_heads),
            query_tower_feature_names=names,
            query_embedding_aggregator=PositionAwareAggregator(common, max_sequence_length, dropout),
            item_embedding_aggregator=common,
            query_encoder=SasRecTransformerLayer(embedding_dim, num_heads, num_blocks, dropout, activation="relu"),
            query_tower_output_normalization=torch.nn.LayerNorm(embedding_dim),
            item_encoder=SwiGLUEncoder(embedding_dim, 2 * embedding_dim),
            item_features_reader=item_features_reader)
        _, card, pad, _ = item_feature_of(schema)
        return cls(body, loss=CE(ignore_index=pad), device=device, seed=seed)

    def forward_train(self, *args, **kwargs):
        self.core.cache_live = False
        return super().forward_train(*args, **kwargs)

    def forward_inference(self, feature_tensors, padding_mask, candidates_to_score=None):
        """As the reference: the first eval forward over the whole catalog fills the item tower's cache."""
        out = super().forward_inference(feature_tensors, padding_mask, candidates_to_score)
        if candidates_to_score is None:
            self.core.cache_live = True
        return out
