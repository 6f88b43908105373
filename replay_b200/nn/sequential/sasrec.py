"""Mirror of ``replay.nn.sequential.SasRec`` (replay/nn/sequential/sasrec/model.py:116-378) backed by the H100 engine.

Same construction (``from_params``), same ``forward`` signature and train / inference output contracts, same
``state_dict`` key names (SURVEY.md Appendix B); the computation is the fused CUDA path (``replay_b200.core``)."""
from __future__ import annotations

import dataclasses
import math
import warnings

import torch

from ...core import SasRecCore
from ..loss import CE, check_multi_positive
from ...engine import EncoderConfig
from ...engine_diff import DiffConfig, DiffEngine
from ...schema import item_feature_of, side_features_of
from ..agg import ConcatAggregator, SumAggregator
from ..embedding import SequenceEmbedding
from ..mask import DefaultAttentionMask

_DIFF_LEAF = {"wq": "attn.W_q.weight", "wk": "attn.W_k.weight", "wv": "attn.W_v.weight", "wo": "attn.W_o.weight",
              "lambda_q1": "attn.lambda_q1", "lambda_k1": "attn.lambda_k1", "lambda_q2": "attn.lambda_q2",
              "lambda_k2": "attn.lambda_k2", "rms_scale": "attn.rms_scale", "attn_norm": "attn_norm.weight",
              "ff_norm": "ff_norm.weight", "ff_wg": "ff.WG.weight", "ff_w1": "ff.W1.weight", "ff_bg": "ff.WG.bias",
              "ff_b1": "ff.W1.bias", "ff_w2": "ff.W2.weight", "ff_b2": "ff.W2.bias"}


def diff_key_map(cfg: DiffConfig, item_feature: str = "item_id") -> dict:
    """engine parameter name -> key of the reference's ``SasRec(body=SasRecBody(..., encoder=DiffTransformerLayer(...)))``"""
    m = {"item_emb": f"body.embedder.feature_embedders.{item_feature}.emb.weight",
         "pos_emb": "body.embedding_aggregator.pe.weight", "lnf_w": "body.output_normalization.weight"}
    if cfg.out_norm == "layernorm":
        m["lnf_b"] = "body.output_normalization.bias"
    for i in range(cfg.n_blocks):
        m.update({f"b{i}.{k}": f"body.encoder.layers.{i}.{v}" for k, v in _DIFF_LEAF.items()})
    return m


class _DiffCore(SasRecCore):
    """SasRecCore on the DiffTransformer engine.  ``state_dict`` also carries each block's ``attn.scaling`` buffer
    (1/sqrt(head_dim)), which ``load_state_dict`` checks."""

    def _key_map(self):
        return diff_key_map(self.cfg, self.item_feature)

    def _make_engine(self, batch, seq_len, with_grad):
        return DiffEngine(self.cfg, batch, seq_len, self._device, seed=self._seed, with_grad=with_grad)

    def _scaling(self) -> dict:
        v = torch.tensor(1.0 / math.sqrt(self.cfg.head_dim), dtype=torch.float32)
        return {f"body.encoder.layers.{i}.attn.scaling": v.clone() for i in range(self.cfg.n_blocks)}

    def state_dict(self, *args, destination=None, prefix="", keep_vars=False):  # noqa: D102
        out = super().state_dict(*args, destination=destination, prefix=prefix, keep_vars=keep_vars)
        for k, v in self._scaling().items():
            out[prefix + k] = v
        return out

    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):  # noqa: D102
        for k, v in self._scaling().items():
            if k in state_dict and not torch.allclose(torch.as_tensor(state_dict[k]).float().cpu(), v):
                raise ValueError(f"{k} = {float(state_dict[k])} does not match this model's 1/sqrt(head_dim) = {float(v)}")
            if strict and k not in state_dict:
                raise RuntimeError(f"missing keys in state_dict: [{k!r}] ...")
        return super().load_state_dict(state_dict, strict=strict, assign=assign)


class PositionAwareAggregator:
    """replay/nn/sequential/sasrec/agg.py: item embedding * sqrt(d) + the last-L positional embedding, then dropout."""

    def __init__(self, embedding_aggregator, max_sequence_length: int, dropout: float) -> None:
        self.embedding_aggregator = embedding_aggregator
        self.max_sequence_length = max_sequence_length
        self.dropout = dropout


class SasRecTransformerLayer:
    """replay/nn/sequential/sasrec/transformer.py (config only): pre-LN blocks with a ReLU FFN."""

    def __init__(self, embedding_dim: int, num_heads: int, num_blocks: int, dropout: float, activation: str = "gelu") -> None:
        self.embedding_dim, self.num_heads, self.num_blocks = embedding_dim, num_heads, num_blocks
        self.dropout, self.activation = dropout, activation


class DiffTransformerLayer:
    """replay/nn/sequential/sasrec/diff_transformer.py (config only): post-norm blocks of multi-head differential
    attention and a SwiGLU FFN of width 2 * embedding_dim.  Head width <= 64, at most 256 padded columns (heads x 64)."""

    def __init__(self, embedding_dim: int, num_heads: int, num_blocks: int) -> None:
        self.embedding_dim, self.num_heads, self.num_blocks = embedding_dim, num_heads, num_blocks


class SasRecBody:
    """replay/nn/sequential/sasrec/model.py ``SasRecBody`` (config only): the parts are read when ``SasRec(body, loss)``
    builds the engine.  ``output_normalization`` is a ``torch.nn.LayerNorm`` or ``torch.nn.RMSNorm`` of the model width."""

    def __init__(self, embedder, embedding_aggregator, attn_mask_builder, encoder, output_normalization) -> None:
        self.embedder = embedder
        self.embedding_aggregator = embedding_aggregator
        self.attn_mask_builder = attn_mask_builder
        self.encoder = encoder
        self.output_normalization = output_normalization

    def build_core(self, device=None, seed: int = 0) -> SasRecCore:
        """The engine configuration this body describes; ValueError for anything the CUDA path does not implement."""
        emb, agg, mask, enc, norm = (self.embedder, self.embedding_aggregator, self.attn_mask_builder, self.encoder,
                                     self.output_normalization)
        if not isinstance(emb, SequenceEmbedding):
            raise ValueError(f"embedder must be SequenceEmbedding, got {type(emb).__name__}")
        schema = emb.schema
        name, card, pad, feat_dim = item_feature_of(schema)
        if pad != card:
            raise ValueError("the item feature's padding_value must equal its cardinality (replay/data/nn/schema.py:89-90)")
        skip = set(emb.excluded_features) | {schema.query_id_feature_name, schema.timestamp_feature_name}
        side = side_features_of(schema, skip, emb.categorical_list_feature_aggregation_method)
        if (not isinstance(agg, PositionAwareAggregator)
                or not isinstance(agg.embedding_aggregator, (SumAggregator, ConcatAggregator))):
            raise ValueError("embedding_aggregator must be PositionAwareAggregator(SumAggregator(...) or ConcatAggregator(...), ...)")
        concat = isinstance(agg.embedding_aggregator, ConcatAggregator)
        if not isinstance(mask, DefaultAttentionMask) or mask.reference_feature_name != name:
            raise ValueError(f"attn_mask_builder must be DefaultAttentionMask on the item feature {name!r}")
        if not isinstance(enc, (SasRecTransformerLayer, DiffTransformerLayer)):
            raise ValueError(f"encoder must be SasRecTransformerLayer or DiffTransformerLayer, got {type(enc).__name__}")
        d = enc.embedding_dim
        if concat and feat_dim is not None and feat_dim != d:
            raise ValueError(f"the item feature {name!r} has embedding_dim {feat_dim}; ConcatAggregator's model scores against "
                             f"its table, so it must be the model's {d}")
        if agg.embedding_aggregator.embedding_dim != d or (feat_dim is not None and feat_dim != d):
            raise ValueError("the embedder, the aggregator and the encoder must share one embedding_dim")
        agg_kw = {}
        if concat:
            side, agg_kw = _concat_side(schema, name, side, agg.embedding_aggregator.input_embedding_dims, d)
        else:
            _check_side(schema, side, d)
        if side and not isinstance(enc, SasRecTransformerLayer):
            raise ValueError(f"side features {[f.name for f in side]} need the SasRecTransformerLayer encoder")
        if mask.num_heads != enc.num_heads:
            raise ValueError("attn_mask_builder.num_heads must equal the encoder's num_heads")
        if isinstance(norm, torch.nn.LayerNorm) and norm.elementwise_affine and norm.bias is not None:
            out_norm = "layernorm"
        elif isinstance(norm, torch.nn.RMSNorm) and norm.elementwise_affine:
            out_norm = "rmsnorm"
        else:
            raise ValueError("output_normalization must be torch.nn.LayerNorm or torch.nn.RMSNorm with affine weights")
        if tuple(norm.normalized_shape) != (d,):
            raise ValueError(f"output_normalization must normalise {d} features")
        eps = norm.eps
        if isinstance(enc, SasRecTransformerLayer):
            if enc.activation != "relu":
                raise ValueError(f"SasRecTransformerLayer supports activation='relu' only, got {enc.activation!r}")
            if out_norm != "layernorm":
                raise ValueError("SasRecTransformerLayer supports a LayerNorm output normalization only")
            if enc.dropout != agg.dropout:
                raise ValueError("the aggregator and SasRecTransformerLayer must share one dropout")
            cfg = EncoderConfig(n_items=card, d=d, n_heads=enc.num_heads, n_blocks=enc.num_blocks,
                                max_len=agg.max_sequence_length, dropout=agg.dropout, variant="new", lnf_eps=eps,
                                features=tuple(side), **agg_kw)
            return SasRecCore(cfg, item_feature=name, device=device, seed=seed)
        cfg = DiffConfig(n_items=card, d=d, n_heads=enc.num_heads, n_blocks=enc.num_blocks, max_len=agg.max_sequence_length,
                         dropout=agg.dropout, out_norm=out_norm, lnf_eps=eps)
        return _DiffCore(cfg, item_feature=name, device=device, seed=seed)


def _concat_side(schema, item: str, side, input_dims, d: int):
    """ConcatAggregator's side features at their own embedding_dim, in its concatenation order (ascending feature name),
    and the EncoderConfig arguments that place the item's segment among them.  ValueError when ``input_dims`` are not the
    embedder's features' widths.  Without side features (the item alone, no projection) it is the item-only model."""
    widths = {item: d, **{f.name: int(schema[f.name].embedding_dim) for f in side}}
    if sorted(input_dims) != sorted(widths.values()):
        raise ValueError(f"ConcatAggregator's input_embedding_dims {sorted(input_dims)} do not match the embedder's features "
                         f"{widths}")
    if not side:
        return side, {}
    order = sorted(widths)
    side = sorted((dataclasses.replace(f, dim=widths[f.name]) for f in side), key=lambda f: f.name)
    return side, {"aggregator": "concat", "concat_item_at": order.index(item)}


def _check_side(schema, side, d: int) -> None:
    """Every side feature is summed into the d-wide input (SumAggregator): its embedding_dim must be d."""
    for f in side:
        if schema[f.name].embedding_dim != d:
            raise ValueError(f"side feature {f.name!r} has embedding_dim {schema[f.name].embedding_dim}; SumAggregator needs "
                             f"every feature at the model's embedding_dim {d}")


class _InferenceOutput(dict):
    """``InferenceOutput`` with a lazily evaluated ``hidden_states`` entry."""

    def __init__(self, logits, hidden_fn):
        super().__init__(logits=logits)
        self._hidden_fn = hidden_fn

    def __getitem__(self, k):
        if k == "hidden_states" and not super().__contains__(k):
            super().__setitem__(k, self._hidden_fn())
        return super().__getitem__(k)

    def __contains__(self, k):
        return k == "hidden_states" or super().__contains__(k)


class SasRec(torch.nn.Module):
    def __init__(self, body, loss=None, device=None, seed: int = 0):
        """``body``: a ``SasRecBody`` (the reference's constructor) or an already built ``SasRecCore``."""
        super().__init__()
        core = body.build_core(device=device, seed=seed) if isinstance(body, SasRecBody) else body
        self.core = core
        self.loss = loss if loss is not None else CE(ignore_index=core.cfg.n_items)

    @property
    def loss(self):
        """The reference's ``SasRec.loss`` attribute (model.py:181-197): assign a selector from ``replay_b200.nn.loss``
        (``CE``, ``BCE``, ``CESampled``, ``LogInCESampled``, ...) to select the fused head."""
        return self._loss

    @loss.setter
    def loss(self, spec):
        if not hasattr(spec, "kind"):
            raise NotImplementedError(f"loss {type(spec).__name__} has no fused CUDA head (supported: CE, BCE, CEWeighted, "
                                      "LogOutCE, LogOutCEWeighted, LogInCE, CESampled, CESampledWeighted, BCESampled, "
                                      "LogInCESampled)")
        self._loss = spec
        self.core.set_loss(spec.kind, **spec.engine_kwargs())

    @classmethod
    def from_params(cls, schema, embedding_dim: int = 192, num_heads: int = 4, num_blocks: int = 2,
                    max_sequence_length: int = 50, dropout: float = 0.3, excluded_features=None,
                    categorical_list_feature_aggregation_method: str = "sum", device=None, seed: int = 0) -> "SasRec":
        """replay/nn/sequential/sasrec/model.py:199-253: every schema feature except the query id, the timestamp and
        ``excluded_features`` is embedded and summed into the input (side features: csrc/rp_features.cu); ReLU FFN,
        LayerNorm(eps=1e-5) output normalisation, full CE loss."""
        name, card, pad, _ = item_feature_of(schema)
        if pad != card:
            raise ValueError("the item feature's padding_value must equal its cardinality (replay/data/nn/schema.py:89-90)")
        skip = {schema.query_id_feature_name, schema.timestamp_feature_name, *(excluded_features or [])}
        side = side_features_of(schema, skip, categorical_list_feature_aggregation_method)
        _check_side(schema, side, embedding_dim)
        cfg = EncoderConfig(n_items=card, d=embedding_dim, n_heads=num_heads, n_blocks=num_blocks,
                            max_len=max_sequence_length, dropout=dropout, variant="new", features=tuple(side))
        return cls(SasRecCore(cfg, item_feature=name, device=device, seed=seed))

    # ---- reference surface
    @property
    def item_feature_name(self) -> str:
        return self.core.item_feature

    def state_dict(self, *a, **k):
        return self.core.state_dict(*a, **k)

    def load_state_dict(self, sd, strict=True, assign=False):
        return self.core.load_state_dict(sd, strict=strict)

    def parameters(self, recurse=True):
        if self.core.flat is None:
            raise RuntimeError("no CUDA device: the parameters live in the engine's flat device buffer (replay_b200 has no CPU path)")
        return iter([self.core.flat])

    def warm_up(self, batch_size: int, seq_len: int, with_grad: bool = True):
        self.core.ensure_engine(batch_size, seq_len, with_grad)
        return self

    def get_logits(self, model_embeddings, candidates_to_score=None):
        """model.py:258-265: scores of given hidden states [*, d] against the item table (materialised, fp32)."""
        h = model_embeddings.reshape(-1, model_embeddings.shape[-1]).to(torch.bfloat16)
        h = self.core.engine.pad_features(h).contiguous()  # true hidden size -> the engine's feature slots
        tab = self.core.item_table(candidates_to_score)
        out = torch.empty(h.shape[0], tab.shape[0], device=h.device, dtype=torch.float32)
        self.core.engine._gemm(h, tab, out, h.shape[0], tab.shape[0], self.core.cfg.dp, out_mode=2)
        return out.view(*model_embeddings.shape[:-1], tab.shape[0])

    multi_positive = True   # the heads take [B, L, P] targets (TwoTower's tower compaction takes one label per position)

    def check_positives(self, positive_labels, target_padding_mask):
        """(labels, mask) of a training batch for the core: [B, L], or [B, L, P] when P > 1 positives per position reach
        a loss that trains on them (NotImplementedError / ValueError otherwise, see ``check_multi_positive``)."""
        n_pos = positive_labels.size(-1) if positive_labels.dim() == 3 else 1
        if n_pos > 1:
            if not self.multi_positive:
                raise NotImplementedError(f"The case of multi-positive labels is not supported in {type(self).__name__}")
            check_multi_positive(self._loss, n_pos)
            return positive_labels, target_padding_mask
        if positive_labels.dim() == 3:
            positive_labels = positive_labels[..., 0]
        if target_padding_mask is not None and target_padding_mask.dim() == 3:
            target_padding_mask = target_padding_mask[..., 0]
        return positive_labels, target_padding_mask

    def forward_train(self, feature_tensors, padding_mask, positive_labels, negative_labels=None, target_padding_mask=None):
        positive_labels, target_padding_mask = self.check_positives(positive_labels, target_padding_mask)
        ids = feature_tensors[self.core.item_feature]
        if self._loss.needs_negatives and negative_labels is None:
            raise ValueError(f"{type(self._loss).__name__} needs negative_labels")
        rw = self._loss.row_weights(feature_tensors, target_padding_mask) if hasattr(self._loss, "row_weights") else None
        loss = self.core.loss(ids, padding_mask, positive_labels, target_padding_mask,
                              negatives=negative_labels if self._loss.needs_negatives else None, row_weights=rw,
                              **self._side(feature_tensors))
        return {"loss": loss, "hidden_states": ()}

    def forward_inference(self, feature_tensors, padding_mask, candidates_to_score=None):
        """model.py:292-307: ``logits`` = scores of the LAST position [B, |I|] (or [B, |C|]); ``hidden_states`` = ([B, L, d],).
        The scores come from the last-position shortcut of the engine; the all-position hidden states (a second, full pass over
        the body) are only computed if that key is actually read."""
        ids, side = feature_tensors[self.core.item_feature], self._side(feature_tensors)
        logits = self.core.logits(ids, padding_mask, candidates_to_score, **side)
        return _InferenceOutput(logits, lambda: (self.core.hidden_states(ids, padding_mask, **side).float(),))

    def forward(self, feature_tensors, padding_mask, candidates_to_score=None, positive_labels=None, negative_labels=None,
                target_padding_mask=None):
        assert padding_mask.dim() == 2, "padding_mask must be [batch, sequence]"
        if self.training:
            if candidates_to_score is not None:
                warnings.warn("Variable `candidates_to_score` is not None. This will have no effect at the training stage.")
            return self.forward_train(feature_tensors, padding_mask, positive_labels, negative_labels, target_padding_mask)
        return self.forward_inference(feature_tensors, padding_mask, candidates_to_score)

    # ---- fused extras
    def predict_topk(self, feature_tensors, padding_mask, k: int, seen_ids=None, candidates_to_score=None):
        return self.core.predict_topk(feature_tensors[self.core.item_feature], padding_mask, k, seen_ids, candidates_to_score,
                                      **self._side(feature_tensors))

    def _side(self, feature_tensors) -> dict:
        """The core's ``feats`` argument: the batch's feature tensors when the model embeds side features."""
        return {"feats": feature_tensors} if getattr(self.core.cfg, "features", ()) else {}
