"""Execution engine of the SASRec hot path on H100: owns the flat parameter / gradient / optimizer buffers and the
activation workspace, and sequences the hand-written sm_90a kernels (librp_b200.so, include/rp_b200.h) for

    train step  = batch prep -> embedding -> N x [LN, QKV GEMMs, fused attention, out-proj, LN, FFN] -> final LN with
                  valid-target compaction -> fused CE head  -> full backward -> (gradient all-reduce) -> Adam
    predict     = same body without dropout -> last hidden state -> fused score + seen-mask + top-K head

It is the host-side counterpart of the reference's torch modules (replay/nn/sequential/sasrec/model.py:85-113,258-307 and
replay/models/nn/sequential/sasrec/model.py:159-180); the ``replay_b200.nn`` / ``replay_b200.models`` classes that mirror
the reference API delegate to it.  torch supplies device memory, streams, CUDA graphs and the NCCL process group only.
"""
from __future__ import annotations

import contextlib
import ctypes
import math
import os
from dataclasses import dataclass

import torch

from ._lib import (CONCAT_MAX_COLS, FEAT_BAG_MEAN, FEAT_BAG_SUM, FEAT_CAT, FEAT_IDENT, FEAT_MAX, FEAT_MAX_NUM_COLS, FEAT_NUM,
                   MAX_POSITIVES, RpFeature, SCE_ALL, SampledDesc, SceDesc, AttnBwdDesc, AttnDesc, GemmDesc, WgradPair, check, lib)


_BLOCK_PARAMS = ("ln1_w", "ln1_b", "in_w", "in_b", "out_w", "out_b", "ln2_w", "ln2_b", "w1", "b1", "w2", "b2")


def _ru(x, m):
    return (x + m - 1) // m * m


@dataclass(frozen=True)
class OptimizerConfig:
    """The optimizer of the fused step, as the reference's factories build it (models/nn/optimizer_utils/
    optimizer_factory.py:71-87, nn/lightning/optimizer.py:44-60): ``torch.optim.Adam(lr, betas, eps, weight_decay)`` or
    ``torch.optim.SGD(lr, momentum, weight_decay)``.  The learning rate is the engine's device-resident ``lr``."""

    kind: str = "adam"            # "adam" | "sgd"
    betas: tuple = (0.9, 0.98)
    eps: float = 1e-8
    weight_decay: float = 0.0
    momentum: float = 0.0

    def __post_init__(self):
        object.__setattr__(self, "betas", tuple(self.betas))

    def validate(self) -> OptimizerConfig:
        """The reference factories raise for an unknown name from ``create()``, not from their constructor: so does a step."""
        if self.kind not in _OPT_KINDS:
            raise ValueError("Unexpected optimizer")
        return self


_OPT_KINDS = {"adam": 0, "sgd": 1}   # RP_OPT_ADAM / RP_OPT_SGD


@dataclass
class BaseConfig:
    """What SASRec (EncoderConfig) and BERT4Rec (BertConfig) share: the transformer's sizes, the feature-slot geometry
    the kernels see, and the padded parameter layout with its pad kinds."""
    n_items: int
    d: int
    n_heads: int
    n_blocks: int
    max_len: int
    dropout: float = 0.0

    def __post_init__(self):
        if self.d % self.n_heads:
            raise ValueError("d must be divisible by n_heads")
        if self.d // self.n_heads > 128:
            raise ValueError("head_dim must not exceed 128 (one 128-wide tensor-core feature slot per head)")
        if self.dp not in (64, 128, 256, 512):
            raise ValueError(f"hidden size {self.d} with {self.n_heads} heads needs {self.dp} padded columns; the kernels "
                             "support 64/128/256/512 (= n_heads x 64-wide slots, or 128-wide for head_dim > 64)")

    # ---- feature slots: every head occupies one 64-wide (head_dim <= 64) or 128-wide tensor-core slot.  The reference's own
    # defaults (embedding_dim 192 / 4 heads -> head_dim 48; legacy hidden_size 50; examples d 64 / 2 heads -> 32) leave padded
    # columns, which are zero in every activation / weight / gradient (include/rp_b200.h "PADDED FEATURE SLOTS")
    @property
    def head_dim(self) -> int:
        return self.d // self.n_heads

    @property
    def head_slot(self) -> int:
        return 64 if self.head_dim <= 64 else 128

    @property
    def dp(self) -> int:
        """columns of the token-major activations / weights as the kernels see them"""
        return self.n_heads * self.head_slot

    @property
    def n_apps(self) -> int:
        """block applications of one body pass: each has its own activations and dropout sites (BertConfig repeats blocks)"""
        return self.n_blocks

    @property
    def hd_valid(self) -> int:
        """the kernels' `hd_valid` argument: real features per slot, 0 when nothing is padded"""
        return 0 if self.head_dim == self.head_slot else self.head_dim

    def feat_index(self, device=None) -> torch.Tensor:
        """padded column of every true feature: (head h, j) -> h * slot + j"""
        h = torch.arange(self.n_heads, device=device).repeat_interleave(self.head_dim)
        j = torch.arange(self.head_dim, device=device).repeat(self.n_heads)
        return h * self.head_slot + j

    # ---- padded parameter layout: (name, padded shape, (row kind, column kind)) in flat-buffer order.  Pad kinds: 'f' = a
    # feature axis (true features scattered into the head slots), 'f3' = three stacked feature axes (packed in-projection),
    # None = not padded; BertConfig adds the FFN's inner axis and the head bias, whose true entries lead.
    def param_layout(self) -> list:
        raise NotImplementedError

    def axis_sizes(self) -> dict:
        """true size of every pad kind"""
        return {"f": self.d, "f3": 3 * self.d}

    def true_shapes(self) -> dict:
        """name -> shape of the parameter in the reference model"""
        size = self.axis_sizes()
        return {name: tuple(n if k is None else size[k] for n, k in zip(shp, kinds)) for name, shp, kinds in self.param_layout()}

    def _block_layout(self, i: int, ffn: int, ffn_kind: str) -> list:
        """block ``i``'s parameters (_BLOCK_PARAMS order) with an FFN inner axis of ``ffn`` columns of kind ``ffn_kind``"""
        d, vec, mat = self.dp, ("f", None), ("f", "f")
        shapes = ((d,), (d,), (3 * d, d), (3 * d,), (d, d), (d,), (d,), (d,), (ffn, d), (ffn,), (d, ffn), (d,))
        kinds = (vec, vec, ("f3", "f"), ("f3", None), mat, vec, vec, vec, (ffn_kind, "f"), (ffn_kind, None), ("f", ffn_kind), vec)
        return [(f"b{i}.{k}", s, pk) for k, s, pk in zip(_BLOCK_PARAMS, shapes, kinds)]


@dataclass(frozen=True)
class SideFeature:
    """One side feature of the new-path SASRec input (replay/nn/embedding.py), summed into the item embedding.

    ``kind``: "cat" (Embedding), "bag_sum" / "bag_mean" (EmbeddingBag over a categorical list), "num" (Linear(tensor_dim,
    d)) or "ident" (tensor_dim == d: the values themselves).  ``cardinality`` / ``padding_value``: categorical kinds (the
    table has cardinality + 1 rows, the padding row is zero and frozen).  ``width``: tensor_dim of the numerical kinds; a
    categorical list takes its width from the batch.  ``dim``: the feature's own embedding_dim under ConcatAggregator (0:
    the model's d, as SumAggregator needs)."""
    name: str
    kind: str
    cardinality: int = 0
    padding_value: int = 0
    width: int = 1
    dim: int = 0

    @property
    def categorical(self) -> bool:
        return self.kind in ("cat", "bag_sum", "bag_mean")


_FEAT_KINDS = {"cat": FEAT_CAT, "bag_sum": FEAT_BAG_SUM, "bag_mean": FEAT_BAG_MEAN, "num": FEAT_NUM, "ident": FEAT_IDENT}


def _check_side_features(fs, d: int, kinds):
    """The checks SASRec's and BERT4Rec's side features share: at most FEAT_MAX of them with distinct names, every kind one
    of ``kinds``, positive cardinalities, and identity features as wide as the true hidden size ``d``."""
    if len(fs) > FEAT_MAX or len({f.name for f in fs}) != len(fs):
        raise ValueError(f"at most {FEAT_MAX} side features with distinct names")
    for f in fs:
        if f.kind not in kinds:
            raise ValueError(f"side feature {f.name!r}: unknown kind {f.kind!r}")
        if f.categorical and f.cardinality < 1:
            raise ValueError(f"side feature {f.name!r}: cardinality must be positive")
        if f.kind == "ident" and f.width != (f.dim or d):
            raise ValueError(f"side feature {f.name!r}: an identity feature needs tensor_dim == {f.dim or d}")


@dataclass
class EncoderConfig(BaseConfig):
    variant: str = "new"  # "new": replay.nn.sequential.SasRec ; "legacy": replay.models.nn.sequential.SasRecModel
    lnf_eps: float | None = None
    features: tuple = ()  # SideFeature, ... (new path only); empty: the item-only input of rp_embed_fwd
    # "sum": SumAggregator, every side feature at width d.  "concat": ConcatAggregator + its Linear(sum of widths, d); the
    # segments come in ``features`` order with the item's after the first ``concat_item_at`` of them (the reference sorts
    # them by name)
    aggregator: str = "sum"
    concat_item_at: int = 0
    side_pad_rows = True  # a categorical side table has cardinality + 1 rows, its padding row zero and frozen

    def __post_init__(self):
        if self.variant not in ("new", "legacy"):
            raise ValueError(f"unknown variant {self.variant}")
        if self.aggregator not in ("sum", "concat"):
            raise ValueError(f"unknown aggregator {self.aggregator!r}")
        super().__post_init__()
        if self.lnf_eps is None:
            # new: torch.nn.LayerNorm default (nn/sequential/sasrec/model.py:248); legacy: 1e-8 (sasrec/model.py:463)
            self.lnf_eps = 1e-5 if self.variant == "new" else 1e-8
        self.features = tuple(self.features)
        if self.aggregator == "concat" and not self.features:
            raise ValueError("a concatenated input needs side features (the item alone is the item-only model)")
        if self.features:
            self._check_features()

    def _check_features(self):
        fs = self.features
        if self.variant != "new":
            raise ValueError("side features exist on the new-path SASRec only")
        _check_side_features(fs, self.d, _FEAT_KINDS)
        for f in fs:
            if f.kind == "num" and f.width < 1:
                raise ValueError(f"side feature {f.name!r}: tensor_dim must be positive")
        if self.num_cols > FEAT_MAX_NUM_COLS:
            raise ValueError(f"the numerical side features' tensor_dims sum to {self.num_cols}; at most {FEAT_MAX_NUM_COLS} "
                             "are projected inside the embedding kernel")
        if self.aggregator == "sum":
            for f in fs:
                if f.dim not in (0, self.d):
                    raise ValueError(f"side feature {f.name!r} has embedding_dim {f.dim}; SumAggregator needs the model's {self.d}")
            return
        for f in fs:
            if f.dim < 1:
                raise ValueError(f"side feature {f.name!r}: ConcatAggregator needs its embedding_dim")
        if not 0 <= self.concat_item_at <= len(fs):
            raise ValueError(f"concat_item_at {self.concat_item_at} outside [0, {len(fs)}]")
        if self.concat_kp > CONCAT_MAX_COLS:
            raise ValueError(f"the concatenated embeddings are {self.concat_width} wide ({self.concat_kp} padded); the CUDA path "
                             f"projects at most {CONCAT_MAX_COLS} columns")

    @property
    def concat(self) -> bool:
        return self.aggregator == "concat"

    @property
    def concat_width(self) -> int:
        """columns of the concatenated input (ConcatAggregator): the item's d plus every side feature's embedding_dim"""
        return self.d + sum(f.dim for f in self.features)

    @property
    def concat_kp(self) -> int:
        """the concatenated input's columns padded for the tensor cores: 64, or a multiple of 128 (the weight-gradient
        kernel's column tiles, rp_wgrad_group)"""
        return 64 if self.concat_width <= 64 else _ru(self.concat_width, 128)

    def concat_columns(self):
        """(first column of the item's segment, first column of every side feature's segment) of the concatenated input"""
        col, item_col, cols = 0, 0, []
        for k, f in enumerate(self.features):
            if k == self.concat_item_at:
                item_col, col = col, col + self.d
            cols.append(col)
            col += f.dim
        if self.concat_item_at == len(self.features):
            item_col = col
        return item_col, cols

    def axis_sizes(self) -> dict:
        return {**super().axis_sizes(), "k": self.concat_width}   # 'k': the projection's input, true columns first

    @property
    def num_cols(self) -> int:
        """summed tensor_dim of the numerical (Linear) side features"""
        return sum(f.width for f in self.features if f.kind == "num")

    @property
    def pad_id(self) -> int:
        return self.n_items

    def param_layout(self) -> list:
        d, emb, vec = self.dp, (None, "f"), ("f", None)
        out = [("item_emb", (self.n_items + 1, d), emb), ("pos_emb", (self.max_len, d), emb)]
        for i in range(self.n_blocks):
            out += self._block_layout(i, d, "f")
        out += [("lnf_w", (d,), vec), ("lnf_b", (d,), vec)]
        for f in self.features:   # after every item-only parameter: an item-only model keeps its layout and seeded init
            w, k = (f.dim, None) if self.concat else (d, "f")   # concat: each at its own, unpadded width
            if f.categorical:
                out.append((f"feat.{f.name}", (f.cardinality + 1, w), (None, k)))
            elif f.kind == "num":
                out += [(f"feat.{f.name}.w", (w, f.width), (k, None)), (f"feat.{f.name}.b", (w,), (k, None))]
        if self.concat:   # ConcatAggregator.feat_projection, after every other parameter
            out += [("feat_proj.w", (d, self.concat_kp), ("f", "k")), ("feat_proj.b", (d,), vec)]
        return out


class _CountingLib:
    """Proxy over the ctypes library that counts the sm_90a kernel launches issued through it (bench.py reports them)."""

    KERNELS = {"rp_gemm": 1, "rp_attn_fwd": 1, "rp_attn_bwd": 1, "rp_attn_last": 1, "rp_attn_softmax_bwd": 1, "rp_prepare_batch": 2, "rp_embed_fwd": 1,
               "rp_embed_bwd": 2, "rp_layernorm_fwd": 1, "rp_layernorm_fwd_compact": 1, "rp_layernorm_bwd": 1, "rp_dropout_bwd": 1, "rp_colsum": 1, "rp_colsum_multi": 1,
               "rp_adam_step": 2, "rp_optimizer_step": 2, "rp_cast_bf16": 1, "rp_counter_add": 1, "rp_reduce_splits": 1, "rp_ce_head_fwd": 2, "rp_ce_head_bwd": 3,
               "rp_score_topk": 2, "rp_seen_prepare": 1, "rp_sampled_head_fwd": 4, "rp_sampled_head_bwd": 4, "rp_post_attn_fused": 1,
               "rp_post_attn_train": 1, "rp_wgrad_group": 2, "rp_ln_qkv_fused": 1, "rp_pre_attn_bwd": 1,
               "rp_post_attn_bwd": 1, "rp_row_plan": 3, "rp_embed_fwd_rows": 1, "rp_embed_bwd_rows": 2, "rp_ln_qkv_fused_rows": 1,
               "rp_post_attn_train_rows": 1, "rp_post_attn_bwd_rows": 1, "rp_pre_attn_bwd_rows": 1, "rp_wgrad_group_rows": 2,
               "rp_bert_feature_embed_fwd": 1, "rp_bert_feature_embed_bwd": 1, "rp_concat_gather": 1, "rp_concat_gather_rows": 1,
               "rp_concat_embed_fwd": 1, "rp_concat_scatter": 1, "rp_embed_pos_bwd": 1, "rp_prepare_batch_multi": 4,
               "rp_bce_head_multi_fwd": 2, "rp_bce_head_multi_bwd": 1}

    def __init__(self, L):
        self._L = L
        self.count = 0
        self._cache = {}

    def __getattr__(self, name):
        w = self._cache.get(name)
        if w is None:
            fn, k = getattr(self._L, name), self.KERNELS.get(name, 0)

            def w(*a, _fn=fn, _k=k):
                self.count += _k
                return _fn(*a)

            self._cache[name] = w
        return w


class SasRecEngine:
    def __init__(self, cfg: EncoderConfig, max_batch: int, seq_len: int, device="cuda", seed: int = 0,
                 with_grad: bool = True):
        self.cfg = cfg
        self.dev = torch.device(device)
        self.B, self.L = max_batch, seq_len
        self._check_geometry(seq_len)
        self.T = max_batch * seq_len
        self.Lp = _ru(seq_len, 64)
        self.with_grad = with_grad
        self.lib = _CountingLib(lib())
        d = cfg.dp   # padded width: what buffers and kernels use; cfg.d is the model's true hidden size
        self._feat = cfg.feat_index(self.dev)
        # ---------------------------------------------------------------- flat parameter layout
        self.layout, self._kinds, off = {}, {}, 0
        for name, shp, kinds in cfg.param_layout():
            self.layout[name], self._kinds[name] = (off, shp), kinds
            off = _ru(off + math.prod(shp), 64)
        self._true = cfg.true_shapes()
        self.features = tuple(getattr(cfg, "features", ()))
        self.concat = getattr(cfg, "concat", False)
        self._side_pad = {f"feat.{f.name}": f.padding_value for f in self.features
                          if f.categorical and cfg.side_pad_rows}
        self.n_flat = off
        f32 = dict(device=self.dev, dtype=torch.float32)
        self.p32 = torch.zeros(off, **f32)
        self.p16 = torch.zeros(off, device=self.dev, dtype=torch.bfloat16)
        self.params = {k: self.p32[o:o + math.prod(s)].view(s) for k, (o, s) in self.layout.items()}
        self.params16 = {k: self.p16[o:o + math.prod(s)].view(s) for k, (o, s) in self.layout.items()}
        if with_grad:
            self._alloc_grad_state()
        self.rng_counter = torch.zeros(1, device=self.dev, dtype=torch.int64)
        self.seed = seed & 0xFFFFFFFFFFFF
        self.training = with_grad
        # fused attention backward: head_dim 64, L <= 256; otherwise (head_dim 128, or L in (256, 512]) saved probabilities +
        # batched GEMMs
        self.fused_attn_bwd = cfg.head_slot == 64 and seq_len <= 256
        self.sampled = None       # full-catalog CE unless set_loss() selects a sampled head
        self.sce = None           # buffers of the scalable CE head (set_loss("sce", ...))
        self.bce, self.ce_row = False, None   # full-catalog BCE / per-row CE variants (set_loss)
        self._loss_args = None
        # training: out-projection + LayerNorm + FFN (+ dropouts, saved activations) in one pass for d <= 128; all weight / bias
        # gradients of a block in one grouped launch (RP_FUSED_BODY=0 restores round 1's launch-per-GEMM body for A/B runs)
        fused_body = os.environ.get("RP_FUSED_BODY", "1") != "0"
        self.fused_post_attn_train = fused_body
        self.fused_wgrad = fused_body and d <= 256          # rp_wgrad_group: at most 48 output tiles per block
        self.fused_pre_attn = fused_body and d <= 128       # LN1 + Q / KV projections in one pass (forward and backward)
        self.fused_post_attn_bwd = fused_body and d <= 128  # dropout' + FFN + LN2 + out-projection backward in one pass
        # new-path training with the fused body on each sequence's live suffix only, packed (packed_eligible).  The training
        # driver (trainer.Trainer) turns it on; direct callers keep the padded rows, whose activation buffers they may read
        self.packed_body = False
        self._packed = False      # the staged training batch runs packed (set by _prepare)
        self.fused_ce = True      # single-pass CE forward + dH (guarded on the device by a bound on |logit|)
        self.n_valid_hint = 0     # host estimate of the number of valid targets per step (load balance of the CE head only)
        self.mp_gen = 0           # bumped whenever the multi-positive buffers move (_ensure_multi)
        self._alloc_workspace()
        self.init_parameters(seed)

    # ------------------------------------------------------------------------------------------------ state that outlives a batch geometry
    def _alloc_grad_state(self):
        """Flat gradient, optimizer state, learning rate and step counter: sized by the configuration only, allocated once.
        ``adam_m`` / ``adam_v`` are Adam's moments; SGD keeps its momentum buffer in ``adam_m``."""
        f32 = dict(device=self.dev, dtype=torch.float32)
        n = self.n_flat
        # data-parallel runs on one NVLink node: the gradient lives in a symmetric (peer-mapped) allocation so that the
        # all-reduce is this repo's own in-graph kernel (replay_b200/peer.py); otherwise a plain buffer (ncclAllReduce)
        from .peer import alloc_peer_grad

        self.peer = alloc_peer_grad(n, self.dev)
        self.g32 = self.peer.g32 if self.peer is not None else torch.zeros(n, **f32)
        self.adam_m = torch.zeros(n, **f32)
        self.adam_v = torch.zeros(n, **f32)
        self.grads = {k: self.g32[o:o + math.prod(s)].view(s) for k, (o, s) in self.layout.items()}
        self.lr = torch.full((1,), 1e-3, **f32)
        self.step_count = torch.zeros(1, device=self.dev, dtype=torch.int32)
        self.opt_kind = "adam"   # the optimizer the state belongs to

    def _check_geometry(self, seq_len: int):
        cfg = self.cfg
        if seq_len > cfg.max_len:
            raise ValueError(f"sequence length {seq_len} exceeds max_len {cfg.max_len}")
        if cfg.variant == "legacy" and seq_len != cfg.max_len:
            raise ValueError("legacy SASRec needs seq_len == max_len (sasrec/model.py:528-529)")
        if seq_len > 512:
            raise ValueError("attention kernels support seq_len <= 512")

    def resize(self, max_batch: int, seq_len: int, with_grad: bool | None = None):
        """New batch geometry (a larger validation / predict batch, another sequence length): ONLY the activation workspace is
        re-allocated.  Parameters, the bf16 shadow, gradients, Adam moments, the learning rate, the step counter and the
        dropout counter keep their buffers - and their addresses, so an ``nn.Parameter`` / optimizer / CUDA pointer that
        refers to them stays valid."""
        self._check_geometry(seq_len)
        if with_grad and not self.with_grad:
            self.with_grad = True
            self._alloc_grad_state()
        self.B, self.L = max_batch, seq_len
        self.T = max_batch * seq_len
        self.Lp = _ru(seq_len, 64)
        self.fused_attn_bwd = self.cfg.head_slot == 64 and seq_len <= 256
        self._alloc_workspace()
        if self._loss_args is not None and self._loss_args[0] != "ce":  # sampled-head buffers are sized by (B, T)
            self.sampled = None
            if self.with_grad:
                self.set_loss(*self._loss_args[:1], **self._loss_args[1])
        return self

    # ------------------------------------------------------------------------------------------------ parameters
    def _pad_kind(self, name: str):
        """(row kind, column kind) of a parameter in the padded layout (BaseConfig.param_layout)."""
        return self._kinds[name]

    def _axis_index(self, kind):
        """padded position of every true entry of an axis of pad kind ``kind``"""
        if kind == "f":
            return self._feat
        if kind == "f3":
            return torch.cat([self._feat + k * self.cfg.dp for k in range(3)])
        return torch.arange(self.cfg.axis_sizes()[kind], device=self.dev)   # true entries first, zero tail

    def _true_index(self, name: str, shape):
        """(rows, cols | None): where the true entries of parameter ``name`` sit in its padded tensor"""
        idx = [self._axis_index(k) if k else torch.arange(n, device=self.dev) for n, k in zip(shape, self._kinds[name])]
        return idx[0], (idx[1] if len(idx) == 2 else None)

    def import_named(self, name: str, value: torch.Tensor, dst=None):
        """Write a TRUE-shape tensor (reference layout) into the padded parameter ``name`` (padded entries become zero)."""
        tgt = (self.params if dst is None else dst)[name]
        v = value.to(self.dev, torch.float32)
        if self._true[name] == tgt.shape:
            tgt.copy_(v.reshape(tgt.shape))
            return
        rows, cols = self._true_index(name, tgt.shape)
        tgt.zero_()
        if cols is None:
            tgt[rows] = v.reshape(-1)
        else:
            tgt[rows[:, None], cols[None, :]] = v.reshape(len(rows), len(cols))

    def export_named(self, name: str, source=None) -> torch.Tensor:
        """The TRUE-shape view (a copy) of the padded parameter / gradient / moment ``name``."""
        t = (self.params if source is None else source)[name].detach()
        if self._true[name] == t.shape:
            return t.clone()
        rows, cols = self._true_index(name, t.shape)
        return (t[rows] if cols is None else t[rows[:, None], cols[None, :]]).clone()

    def true_shape(self, name: str):
        return self._true[name]

    def init_parameters(self, seed: int = 0):
        """Reference-style init: xavier_normal_ on >=2-D tensors, LN (1, 0), FFN biases U(+-1/sqrt(fan_in)), other biases
        zero, pad row zero (SASRec new path, nn/embedding.py:198-200; BERT4Rec: bert4rec/model.py:167-170) - drawn in the
        model's TRUE shapes, then laid out in the head slots.  Weights are normally loaded from a reference state_dict instead
        (``load_canonical``)."""
        g = torch.Generator(device="cpu").manual_seed(seed)
        with torch.no_grad():
            for name in self.layout:
                shp = self.true_shape(name)
                if len(shp) == 2:
                    std = math.sqrt(2.0 / (shp[0] + shp[1]))
                    v = torch.randn(shp, generator=g) * std
                    if name == "item_emb" and self.cfg.variant == "new":
                        v[self.cfg.pad_id].zero_()
                    elif name in self._side_pad:   # CategoricalEmbedding.reset_parameters (nn/embedding.py)
                        v[self._side_pad[name]].zero_()
                elif name.startswith(("feat.", "feat_proj.")):   # Linear biases keep torch's default init
                    fan_in = self.true_shape(name[:-1] + "w")[1]
                    v = (torch.rand(shp, generator=g) * 2 - 1) / math.sqrt(fan_in)
                elif name.endswith(("ln1_w", "ln2_w", "lnf_w")):
                    v = torch.ones(shp)
                elif name.endswith((".b1", ".b2")):
                    fan_in = self.true_shape(name[:-2] + "w" + name[-1])[1]
                    v = (torch.rand(shp, generator=g) * 2 - 1) / math.sqrt(fan_in)
                else:
                    v = torch.zeros(shp)
                self.import_named(name, v)
        self.refresh_shadow()

    def refresh_shadow(self):
        check(self.lib.rp_cast_bf16(self.p32.data_ptr(), self.p16.data_ptr(), self.n_flat, self._stream()), "rp_cast_bf16")

    def load_canonical(self, P: dict):
        """Copy weights from the canonical dict used by oracle/ (true shapes; block parameters under blocks[i][...], every
        other parameter under its own name)."""
        with torch.no_grad():
            for name in self.layout:
                blk, _, leaf = name.partition(".")
                self.import_named(name, P["blocks"][int(blk[1:])][leaf] if leaf else P[name])
        self.refresh_shadow()

    def export_canonical(self, source=None) -> dict:
        P = {}
        for name in self.layout:
            v = self.export_named(name, source).cpu()
            blk, _, leaf = name.partition(".")
            if not leaf:
                P[name] = v
                continue
            blocks = P.setdefault("blocks", [])
            if int(blk[1:]) == len(blocks):
                blocks.append({})
            blocks[-1][leaf] = v
        return P

    def unpad_features(self, t: torch.Tensor) -> torch.Tensor:
        """[..., dp] activations -> [..., d] (the reference's hidden size)"""
        return t if self.cfg.hd_valid == 0 else t[..., self._feat].contiguous()

    def pad_features(self, t: torch.Tensor) -> torch.Tensor:
        if self.cfg.hd_valid == 0:
            return t
        out = torch.zeros(*t.shape[:-1], self.cfg.dp, device=t.device, dtype=t.dtype)
        out[..., self._feat] = t
        return out

    # ------------------------------------------------------------------------------------------------ workspace
    def _alloc_workspace(self):
        """Activation workspace of the current batch geometry: batch staging, hidden states, the attention core's saves,
        LayerNorm statistics and the CE head's state here; the block program's own buffers in ``_alloc_body``."""
        cfg, T, d, dev = self.cfg, self.T, self.cfg.dp, self.dev
        self._alloc_B, self._alloc_T, self._sub_last_idx = self.B, self.T, {}
        bf = dict(device=dev, dtype=torch.bfloat16)
        f32 = dict(device=dev, dtype=torch.float32)
        i32 = dict(device=dev, dtype=torch.int32)
        BH = self.B * cfg.n_heads
        self.ids32 = torch.zeros(T, **i32)
        self.in_ids = torch.zeros(T, device=dev, dtype=torch.int64)
        self.in_pad = torch.zeros(T, device=dev, dtype=torch.bool)
        self.in_labels = torch.zeros(T, device=dev, dtype=torch.int64)
        self.in_tmask = torch.zeros(T, device=dev, dtype=torch.bool)
        self.valid_idx = torch.zeros(T, **i32)
        self.labels_c = torch.zeros(T, **i32)
        self.n_valid = torch.zeros(1, **i32)
        self.prep_scratch = torch.zeros((T + 1023) // 1024 + 1, **i32)
        # row plan of a packed batch (rp_row_plan): first kept position and first packed row of every sequence, the packed row
        # count, the token of every packed row and the packed row of every valid target
        self.seq_first = torch.zeros(self.B, **i32)
        self.seq_off = torch.zeros(self.B, **i32)
        self.n_rows = torch.zeros(1, **i32)
        self.row_tok = torch.zeros(T, **i32)
        self.valid_rows = torch.zeros(T, **i32)
        # multi-positive targets of the staged batch (n_pos > 1): buffers sized by (T, n_pos), allocated by _ensure_multi
        self.n_pos, self.mp = 1, None
        # hidden states and saved activations per block APPLICATION (cfg.n_apps; the same as n_blocks unless blocks repeat)
        self.x = [torch.zeros(T, d, **bf) for _ in range(cfg.n_apps + 1)]
        self.act = []
        for _ in range(cfg.n_apps):
            a = {k: torch.zeros(T, **f32) for k in ("mean1", "rstd1", "mean2", "rstd2")}
            a["O"] = torch.zeros(T, d, **bf)
            if self.with_grad:
                if not self.fused_attn_bwd:
                    a["P"] = torch.zeros(BH, self.Lp, self.Lp, **bf)
                a["inv_sum"] = torch.zeros(BH, self.Lp, **f32)
                a["m2"] = torch.zeros(BH, self.Lp, **f32)
            self.act.append(a)
        self.hc = torch.zeros(T, d, **bf)
        self.hq = torch.zeros(self.B, d, **bf)
        self._alloc_features()
        self.last_idx = (torch.arange(self.B, device=dev, dtype=torch.int32) * self.L + (self.L - 1)).contiguous()
        if self.with_grad:
            from .ops import CEHeadState

            self.ce = CEHeadState(T, cfg.n_items, d, dev)
            self.s = {k: torch.zeros(T, d, **bf) for k in ("dhc", "dxa", "dxb", "d_o")}
            if not self.fused_attn_bwd:
                self.s["dpd"] = torch.zeros(BH, self.Lp, self.Lp, **bf)
            self.wg_ws = torch.zeros(self.n_sm * 4 * d * d, **f32)  # split-K partials of the weight-gradient GEMMs
        self._alloc_body()

    def _alloc_features(self):
        """Static staging buffers of the side features (a captured step reads the batch staged into them): int32 [T] / [T, K]
        ids, fp32 [T, tensor_dim] values; a categorical list's buffer is sized by the first batch (set_features).  With
        numerical features the backward also keeps dS bf16 [T, dp], the gathered values bf16 [T, 64] and their gradients.
        ConcatAggregator adds the concatenated input X bf16 [T, kp] and its projection fp32 [T, dp]; its backward keeps
        dY = dS and dX bf16 [T, kp], and the numerical gradients cover all kp rows of dX^T . V."""
        self.feat_in = {}
        if not self.features:
            return
        i32, f32 = dict(device=self.dev, dtype=torch.int32), dict(device=self.dev, dtype=torch.float32)
        bf = dict(device=self.dev, dtype=torch.bfloat16)
        for f in self.features:
            if f.kind == "cat":
                self.feat_in[f.name] = torch.full((self.T, 1), f.padding_value, **i32)
            elif not f.categorical:
                self.feat_in[f.name] = torch.zeros(self.T, f.width, **f32)
        has_num = any(f.kind == "num" for f in self.features)
        if self.with_grad and (has_num or self.concat):
            self.feat_ds = torch.zeros(self.T, self.cfg.dp, **bf)
        if self.with_grad and has_num:
            rows = self.cfg.concat_kp if self.concat else self.cfg.dp
            self.feat_v = torch.zeros(self.T, FEAT_MAX_NUM_COLS, **bf)
            self.feat_dw = torch.zeros(rows, FEAT_MAX_NUM_COLS, **f32)
            self.feat_db = torch.zeros(rows, **f32)
        if self.concat:
            self.cat_x = torch.zeros(self.T, self.cfg.concat_kp, **bf)
            self.cat_y = torch.zeros(self.T, self.cfg.dp, **f32)
            if self.with_grad:
                self.cat_dx = torch.zeros(self.T, self.cfg.concat_kp, **bf)

    def set_features(self, feats: dict) -> bool:
        """Stage the side features of the current batch (name -> [B, L] or [B, L, K] tensor, as the reference's
        ``feature_tensors``) into the static buffers; B * L <= T rows.  Returns True when a categorical list's buffer had to
        be (re)allocated for a new list width, which moves it: graphs captured before then read the old buffer."""
        moved = False
        for f in self.features:
            if f.name not in feats:
                raise ValueError(f"feature_tensors lacks the side feature {f.name!r}")
            v = feats[f.name]
            n = v.shape[0] * v.shape[1]
            if f.categorical:
                k = 1 if f.kind == "cat" else (v.shape[2] if v.dim() == 3 else 1)
                if f.kind == "cat" and v.dim() != 2 or f.kind != "cat" and v.dim() != 3:
                    raise ValueError(f"side feature {f.name!r}: expected {'[B, L]' if f.kind == 'cat' else '[B, L, K]'} ids, "
                                     f"got {tuple(v.shape)}")
                buf = self.feat_in.get(f.name)
                if buf is None or buf.shape[1] != k:
                    buf = self.feat_in[f.name] = torch.full((self._alloc_T, k), f.padding_value, device=self.dev,
                                                            dtype=torch.int32)
                    moved = True
            else:
                buf = self.feat_in[f.name]
                want = (v.shape[0], v.shape[1], f.width) if f.width > 1 or v.dim() == 3 else (v.shape[0], v.shape[1])
                if tuple(v.shape) != want:
                    raise ValueError(f"side feature {f.name!r}: expected values {want}, got {tuple(v.shape)}")
            if n > buf.shape[0]:
                raise ValueError(f"side feature {f.name!r}: {n} rows do not fit the engine's {buf.shape[0]}")
            buf[:n].copy_(v.reshape(n, -1), non_blocking=True)
        return moved

    def _feature_descs(self, with_grad: bool):
        """ctypes array of rp_feature for the staged side features (gradient pointers when ``with_grad``)."""
        fs = self.features
        arr = (RpFeature * len(fs))()
        col = 0
        for k, f in enumerate(fs):
            a, buf = arr[k], self.feat_in[f.name]
            a.kind, a.width, a.values = _FEAT_KINDS[f.kind], buf.shape[1], buf.data_ptr()
            if f.categorical:
                # without padding rows (BERT4Rec) every id in [0, cardinality) is a row: -1 matches no id
                a.n_rows, a.padding_value = ((f.cardinality + 1, f.padding_value) if self.cfg.side_pad_rows
                                             else (f.cardinality, -1))
                a.table = self.params16[f"feat.{f.name}"].data_ptr()
                a.d_table = self.grads[f"feat.{f.name}"].data_ptr() if with_grad else None
            elif f.kind == "num":
                a.table, a.bias = self.params[f"feat.{f.name}.w"].data_ptr(), self.params[f"feat.{f.name}.b"].data_ptr()
                a.val_col = col
                col += f.width
        return arr

    def _concat_segments(self):
        """(item_col, seg_col, seg_dim) of rp_concat_*: host int arrays in feature order"""
        item_col, cols = self.cfg.concat_columns()
        n = len(self.features)
        return item_col, (ctypes.c_int * n)(*cols), (ctypes.c_int * n)(*[f.dim for f in self.features])

    def _concat_fwd(self, drop: float, pos0: int):
        """ConcatAggregator's input stage: gather the segments into X, Y = X . W^T + b on the tensor cores (fp32 out), then
        x[0] = dropout(Y * sqrt(d) + pos) in one elementwise pass with the item-only dropout stream."""
        cfg, T, L, d, kp = self.cfg, self.T, self.L, self.cfg.dp, self.cfg.concat_kp
        fa = self._feature_descs(False)
        item_col, seg_col, seg_dim = self._concat_segments()
        item, ids = self.params16["item_emb"].data_ptr(), self.ids32.data_ptr()
        rt, nr = (self.row_tok, self.n_rows) if self._packed else (None, None)
        if self._packed:
            check(self.lib.rp_concat_gather_rows(item, ids, fa, seg_col, seg_dim, len(fa), item_col, rt.data_ptr(), nr.data_ptr(),
                                                 T, d, cfg.hd_valid, kp, self.cat_x.data_ptr(), self._stream()),
                  "rp_concat_gather_rows")
        else:
            check(self.lib.rp_concat_gather(item, ids, fa, seg_col, seg_dim, len(fa), item_col, T, d, cfg.hd_valid, kp,
                                            self.cat_x.data_ptr(), self._stream()), "rp_concat_gather")
        self._gemm(self.cat_x, self.params16["feat_proj.w"], self.cat_y, T, d, kp, bias=self.params["feat_proj.b"], out_mode=2,
                   m_limit=nr)
        check(self.lib.rp_concat_embed_fwd(self.cat_y.data_ptr(), self.params["pos_emb"].data_ptr(),
                                           None if rt is None else rt.data_ptr(), None if nr is None else nr.data_ptr(), T, L, d,
                                           pos0, math.sqrt(cfg.d), drop, self.seed, 0, self.rng_counter.data_ptr(),
                                           self.x[0].data_ptr(), self._stream()), "rp_concat_embed_fwd")

    def _concat_bwd(self, dx, drop: float, pos0: int):
        """Backward of _concat_fwd from the block input's gradient ``dx``: dY = sqrt(d) * dropout'(dx), dX = dY . W, the table
        rows (item included) from dX, dW / db of the projection and of the numerical features in fixed order, positions."""
        cfg, G, T, L, d, kp, st = self.cfg, self.grads, self.T, self.L, self.cfg.dp, self.cfg.concat_kp, self._stream
        packed = self._packed
        rows = self.n_rows.data_ptr() if packed else None
        dY, dX = self.feat_ds, self.cat_dx
        args = (cfg.hd_valid, math.sqrt(cfg.d), drop, self.seed, 0, self.rng_counter.data_ptr(), dY.data_ptr(), None, 0, st())
        if packed:
            check(self.lib.rp_feature_embed_bwd_rows(dx.data_ptr(), None, 0, self.row_tok.data_ptr(), rows, T, d, *args),
                  "rp_feature_embed_bwd_rows")
        else:
            check(self.lib.rp_feature_embed_bwd(dx.data_ptr(), None, 0, T, d, *args), "rp_feature_embed_bwd")
        self._gemm(dY, self.params16["feat_proj.w"], dX, T, kp, d, b_mn=True, m_limit=self.n_rows if packed else None)
        fa = self._feature_descs(True)
        item_col, seg_col, seg_dim = self._concat_segments()
        nc = cfg.num_cols
        check(self.lib.rp_concat_scatter(dX.data_ptr(), self.ids32.data_ptr(), G["item_emb"].data_ptr(), cfg.pad_id, fa, seg_col,
                                         seg_dim, len(fa), item_col, self.row_tok.data_ptr() if packed else None, rows, T, d,
                                         cfg.hd_valid, kp, self.feat_v.data_ptr() if nc else None, FEAT_MAX_NUM_COLS if nc else 0,
                                         st()), "rp_concat_scatter")
        # dW = dY^T . X: at most (512 / 128) x (1024 / 128) = 32 output tiles, within one rp_wgrad_group launch
        n_rows = self.n_rows if packed else None
        self._wgrad_group([(dY, self.cat_x, G["feat_proj.w"], G["feat_proj.b"])], n_rows)
        if nc:
            self.feat_dw.zero_()
            self.feat_db.zero_()
            self._wgrad_group([(dX, self.feat_v, self.feat_dw, self.feat_db)], n_rows)
            col = 0
            for f, c0 in zip(self.features, seg_col):
                if f.kind == "num":
                    G[f"feat.{f.name}.w"].add_(self.feat_dw[c0:c0 + f.dim, col:col + f.width])
                    G[f"feat.{f.name}.b"].add_(self.feat_db[c0:c0 + f.dim])
                    col += f.width
        check(self.lib.rp_embed_pos_bwd(dx.data_ptr(), self.seq_first.data_ptr() if packed else None,
                                        self.seq_off.data_ptr() if packed else None, self.B, L, d, pos0, drop, self.seed, 0,
                                        self.rng_counter.data_ptr(), G["pos_emb"].data_ptr(), st()), "rp_embed_pos_bwd")

    def _embed_fwd(self, drop: float, pos0: int):
        """x[0] = the block input: rp_embed_fwd(_rows) for an item-only model, rp_feature_embed_fwd(_rows) with side features
        summed in, _concat_fwd with ConcatAggregator."""
        cfg, T, L, d = self.cfg, self.T, self.L, self.cfg.dp
        p16, prm, pad = self.params16, self.params, self.in_pad
        legacy = cfg.variant == "legacy"
        if self.concat:
            self._concat_fwd(drop, pos0)
        elif self.features:
            fa = self._feature_descs(False)
            if self._packed:
                check(self.lib.rp_feature_embed_fwd_rows(p16["item_emb"].data_ptr(), prm["pos_emb"].data_ptr(),
                                                         self.ids32.data_ptr(), fa, len(fa), self.row_tok.data_ptr(),
                                                         self.n_rows.data_ptr(), T, L, d, cfg.hd_valid, pos0, math.sqrt(cfg.d),
                                                         drop, self.seed, 0, self.rng_counter.data_ptr(), self.x[0].data_ptr(),
                                                         self._stream()), "rp_feature_embed_fwd_rows")
            else:
                check(self.lib.rp_feature_embed_fwd(p16["item_emb"].data_ptr(), prm["pos_emb"].data_ptr(), self.ids32.data_ptr(),
                                                    fa, len(fa), T, L, d, cfg.hd_valid, pos0, math.sqrt(cfg.d), drop, self.seed,
                                                    0, self.rng_counter.data_ptr(), self.x[0].data_ptr(), self._stream()),
                      "rp_feature_embed_fwd")
        elif self._packed:
            check(self.lib.rp_embed_fwd_rows(p16["item_emb"].data_ptr(), prm["pos_emb"].data_ptr(), self.ids32.data_ptr(),
                                             pad.data_ptr(), self.row_tok.data_ptr(), self.n_rows.data_ptr(), T, L, d, pos0,
                                             math.sqrt(cfg.d), 0, drop, self.seed, 0, self.rng_counter.data_ptr(),
                                             self.x[0].data_ptr(), self._stream()), "rp_embed_fwd_rows")
        else:
            check(self.lib.rp_embed_fwd(p16["item_emb"].data_ptr(), prm["pos_emb"].data_ptr(), self.ids32.data_ptr(),
                                        pad.data_ptr(), T, L, d, pos0, math.sqrt(cfg.d), int(legacy), drop, self.seed, 0,
                                        self.rng_counter.data_ptr(), self.x[0].data_ptr(), self._stream()), "rp_embed_fwd")

    def _feature_bwd(self, dx, drop: float):
        """Side-feature gradients from the block input's gradient ``dx``: table rows by rp_feature_embed_bwd(_rows); the
        numerical Linears' dW = dS^T . V and db = colsum(dS) by one fixed-order rp_wgrad_group(_rows) over its staging."""
        cfg, G, T, d, st = self.cfg, self.grads, self.T, self.cfg.dp, self._stream
        fa = self._feature_descs(True)
        nc = cfg.num_cols
        ds, vr = (self.feat_ds.data_ptr(), self.feat_v.data_ptr()) if nc else (None, None)
        args = (cfg.hd_valid, math.sqrt(cfg.d), drop, self.seed, 0, self.rng_counter.data_ptr(), ds, vr, FEAT_MAX_NUM_COLS, st())
        if self._packed:
            check(self.lib.rp_feature_embed_bwd_rows(dx.data_ptr(), fa, len(fa), self.row_tok.data_ptr(), self.n_rows.data_ptr(),
                                                     T, d, *args), "rp_feature_embed_bwd_rows")
        else:
            check(self.lib.rp_feature_embed_bwd(dx.data_ptr(), fa, len(fa), T, d, *args), "rp_feature_embed_bwd")
        if not nc:
            return
        pair = (WgradPair * 1)()
        p = pair[0]
        p.dY, p.dy_ld, p.n_out = self.feat_ds.data_ptr(), d, d
        p.X, p.x_ld, p.n_in = self.feat_v.data_ptr(), FEAT_MAX_NUM_COLS, FEAT_MAX_NUM_COLS
        p.dW, p.dw_ld, p.db = self.feat_dw.data_ptr(), FEAT_MAX_NUM_COLS, self.feat_db.data_ptr()
        need = self.lib.rp_wgrad_group_workspace(pair, 1)
        if self._wgrad_ws is None or self._wgrad_ws.numel() < need:
            self._wgrad_ws = torch.zeros(need, device=self.dev, dtype=torch.uint8)
        if self._packed:
            check(self.lib.rp_wgrad_group_rows(pair, 1, T, 0, self.n_rows.data_ptr(), self._wgrad_ws.data_ptr(),
                                               self._wgrad_ws.numel(), st()), "rp_wgrad_group_rows")
        else:
            check(self.lib.rp_wgrad_group(pair, 1, T, 0, self._wgrad_ws.data_ptr(), self._wgrad_ws.numel(), st()), "rp_wgrad_group")
        col = 0
        for f in self.features:
            if f.kind == "num":
                G[f"feat.{f.name}.w"].add_(self.feat_dw[:, col:col + f.width])
                G[f"feat.{f.name}.b"].add_(self.feat_db)
                col += f.width

    def _alloc_body(self):
        """SASRec's block buffers: LN1 output, Q and packed [K | V], the FFN's saved activations, the predict path's last-row
        buffers and the backward's scratch."""
        T, d, dev = self.T, self.cfg.dp, self.dev
        bf = dict(device=dev, dtype=torch.bfloat16)
        for a in self.act:
            a.update({k: torch.zeros(T, d, **bf) for k in ("q_in", "Q", "h", "y", "u")})
            a["KV"] = torch.zeros(T, 2 * d, **bf)
        self.meanf = torch.zeros(T, device=dev, dtype=torch.float32)
        self.rstdf = torch.zeros(T, device=dev, dtype=torch.float32)
        self.last_buf = {k: torch.zeros(self.B, d, **bf) for k in ("q_in", "Q", "O", "h", "y", "u")}
        self.last_rows = torch.zeros(self.B, d, **bf)
        self.last_pad = torch.zeros(self.B, device=dev, dtype=torch.bool)
        if self.with_grad:
            self.s.update({k: torch.zeros(T, d, **bf) for k in ("d_t", "du", "dy", "dh", "dQ", "dq_in", "tmp")})
            self.s["dKV"] = torch.zeros(T, 2 * d, **bf)
            self._wgrad_ws = None  # workspace of rp_wgrad_group, sized on first use

    def _stream(self):
        return torch.cuda.current_stream(self.dev).cuda_stream

    @contextlib.contextmanager
    def sub_geometry(self, batch: int, seq_len: int):
        """Inference only: run a SMALLER [batch, seq_len] problem inside the allocated workspace (every activation buffer is a
        flat [T, ...] array, so a problem with batch * seq_len <= T rows uses a prefix of each).  Used by the length-bucketed
        predict (core.py): users whose whole history fits the last ``seq_len`` positions are evaluated on that window only -
        positions are right-aligned (``pos0 = max_len - L``), so the trimmed window sees the same position embeddings."""
        self._check_geometry(seq_len)
        if batch > self._alloc_B or batch * seq_len > self._alloc_T:
            raise ValueError(f"sub-geometry ({batch}, {seq_len}) exceeds the workspace ({self._alloc_B} x {self._alloc_T // self._alloc_B})")
        saved = (self.B, self.L, self.T, self.Lp, self.last_idx)
        key = (batch, seq_len)
        if key not in self._sub_last_idx:
            self._sub_last_idx[key] = (torch.arange(batch, device=self.dev, dtype=torch.int32) * seq_len + (seq_len - 1)).contiguous()
        self.B, self.L, self.T, self.Lp, self.last_idx = batch, seq_len, batch * seq_len, _ru(seq_len, 64), self._sub_last_idx[key]
        try:
            yield self
        finally:
            self.B, self.L, self.T, self.Lp, self.last_idx = saved

    # ------------------------------------------------------------------------------------------------ kernel helpers
    def _gemm(self, A, B, C, M, N, K, *, a_mn=False, b_mn=False, bias=None, act=0, residual=None, rowmask=None,
              drop_p=0.0, drop_site=0, out_mode=0, split_k=1, gate=None, gate_scale=1.0, alpha=1.0, batch=1, inner=1,
              a_off=(0, 0, 0, 0, 0, 0), b_off=(0, 0, 0, 0, 0, 0), c_geom=None, rowmask_oo=0, C2=None, gate_mode=0,
              post_drop_p=0.0, post_drop_site=0, c_split_stride=0, m_limit=None):
        g = GemmDesc()
        g.A, g.a_rows, g.a_cols, g.lda, g.a_mn = A.data_ptr(), A.shape[0], A.shape[1], A.stride(0), int(a_mn)
        g.B, g.b_rows, g.b_cols, g.ldb, g.b_mn = B.data_ptr(), B.shape[0], B.shape[1], B.stride(0), int(b_mn)
        g.M, g.N, g.K, g.batch, g.inner = M, N, K, batch, inner
        g.a_r0, g.a_ro, g.a_ri, g.a_c0, g.a_co, g.a_ci = a_off
        g.b_r0, g.b_ro, g.b_ri, g.b_c0, g.b_co, g.b_ci = b_off
        g.C = C.data_ptr()
        if c_geom is None:
            g.ldc, g.c_off0, g.c_oo, g.c_oi = C.stride(0), 0, 0, 0
        else:
            g.ldc, g.c_off0, g.c_oo, g.c_oi = c_geom
        g.out_mode = out_mode
        g.alpha = alpha
        g.bias = None if bias is None else bias.data_ptr()
        g.act = act
        g.residual = None if residual is None else residual.data_ptr()
        g.rowmask = None if rowmask is None else rowmask.data_ptr()
        g.rowmask_off0, g.rowmask_oo = 0, rowmask_oo
        g.drop_p = drop_p
        g.seed = self.seed
        g.drop_offset = drop_site << 40
        g.seed_ptr = self.rng_counter.data_ptr()
        g.split_k = split_k
        g.gate = None if gate is None else gate.data_ptr()
        g.gate_scale = gate_scale
        g.C2 = None if C2 is None else C2.data_ptr()
        g.gate_mode = gate_mode
        g.post_drop_p = post_drop_p
        g.post_drop_offset = post_drop_site << 40
        g.c_split_stride = c_split_stride
        if m_limit is not None:   # device row count: 128-row tiles at or past it are skipped
            g.m_limit_dev = m_limit.data_ptr()
        check(self.lib.rp_gemm(ctypes.byref(g), self._stream()), "rp_gemm")

    @property
    def n_sm(self) -> int:
        """Streaming multiprocessors of the engine's GPU (sizes the split-K waves of the weight gradients)."""
        return torch.cuda.get_device_properties(self.dev).multi_processor_count

    def _wgrad(self, dY, X, dW, n_out, n_in, rows=None):
        """dW[n_out, n_in] += dY[rows, n_out]^T . X[rows, n_in] (rows: T by default): both operands read MN-major in place;
        split-K over about one wave of CTAs, each storing its fp32 partial tile (no atomics: 100+ CTAs hammering the same
        16 K addresses serialise in L2), then one reduction pass adds the partials into the gradient buffer (deterministic)."""
        rows = self.T if rows is None else rows
        tiles = ((n_out + 127) // 128) * ((n_in + 127) // 128 if n_in > 64 else 1)
        chunks = (rows + 63) // 64
        n = n_out * n_in
        split = max(1, min(chunks // 8, (self.n_sm + tiles - 1) // tiles, self.wg_ws.numel() // n))
        self._gemm(dY, X, self.wg_ws, n_out, n_in, rows, a_mn=True, b_mn=True, out_mode=3, split_k=split,
                   c_geom=(n_in, 0, 0, 0), c_split_stride=n)
        check(self.lib.rp_reduce_splits(self.wg_ws.data_ptr(), split, n, n, dW.data_ptr(), 1, self._stream()), "rp_reduce_splits")

    def _wgrad_group(self, pairs, n_rows_dev=None):
        """[(dY bf16 [T, n_out], X bf16 [T, n_in], dW fp32 [n_out, n_in], db fp32 [n_out] | None), ...]: every weight and bias
        gradient of a block in one wgmma launch + one deterministic reduction launch (csrc/rp_wgrad.cu).  Gradients are
        accumulated (+=) like the un-fused path does."""
        n = len(pairs)
        arr = (WgradPair * n)()
        for k, (dY, X, dW, db) in enumerate(pairs):
            arr[k].dY, arr[k].dy_ld, arr[k].n_out = dY.data_ptr(), dY.stride(0), dW.shape[0]
            arr[k].X, arr[k].x_ld, arr[k].n_in = X.data_ptr(), X.stride(0), dW.shape[1]
            arr[k].dW, arr[k].dw_ld = dW.data_ptr(), dW.stride(0)
            arr[k].db = None if db is None else db.data_ptr()
        need = self.lib.rp_wgrad_group_workspace(arr, n)
        if need == 0:
            raise ValueError("rp_wgrad_group: unsupported gradient shapes")
        if self._wgrad_ws is None or self._wgrad_ws.numel() < need:
            self._wgrad_ws = torch.zeros(need, device=self.dev, dtype=torch.uint8)
        if n_rows_dev is not None:
            check(self.lib.rp_wgrad_group_rows(arr, n, self.T, 1, n_rows_dev.data_ptr(), self._wgrad_ws.data_ptr(),
                                               self._wgrad_ws.numel(), self._stream()), "rp_wgrad_group_rows")
            return
        check(self.lib.rp_wgrad_group(arr, n, self.T, 1, self._wgrad_ws.data_ptr(), self._wgrad_ws.numel(), self._stream()),
              "rp_wgrad_group")

    def _colsum(self, dY, db):
        check(self.lib.rp_colsum(dY.data_ptr(), dY.shape[0], dY.shape[1], dY.stride(0), db.data_ptr(), self._stream()),
              "rp_colsum")

    def _colsum_multi(self, pairs):
        """[(dY bf16 [T, cols], db fp32 [cols]), ...] (<= 6) in one launch: the bias gradients of one block."""
        n = len(pairs)
        dy = (ctypes.c_void_p * n)(*[a.data_ptr() for a, _ in pairs])
        db = (ctypes.c_void_p * n)(*[b.data_ptr() for _, b in pairs])
        cols = (ctypes.c_int * n)(*[a.shape[1] for a, _ in pairs])
        ld = (ctypes.c_longlong * n)(*[a.stride(0) for a, _ in pairs])
        check(self.lib.rp_colsum_multi(n, dy, cols, ld, db, pairs[0][0].shape[0], self._stream()), "rp_colsum_multi")

    def _ln_fwd(self, x, w, b, eps, y, mean, rstd, n_rows, gather=None, n_rows_dev=None):
        # the compaction of the valid targets for the loss heads also zeroes the rows after them up to the heads' 128-row tile
        # edge (a stale non-finite row there would reach every item's gradient)
        compact = gather is not None and n_rows_dev is not None
        fn = self.lib.rp_layernorm_fwd_compact if compact else self.lib.rp_layernorm_fwd
        check(fn(x.data_ptr(), w.data_ptr(), b.data_ptr(), eps, n_rows, self.cfg.dp,
                 None if n_rows_dev is None else n_rows_dev.data_ptr(), None if gather is None else gather.data_ptr(),
                 y.data_ptr(), mean.data_ptr(), rstd.data_ptr(), self.cfg.hd_valid, self._stream()),
              "rp_layernorm_fwd_compact" if compact else "rp_layernorm_fwd")

    def _ln_bwd(self, dy, x, w, mean, rstd, dx, dw, db, n_rows, gather=None, n_rows_dev=None, add_to=None):
        check(self.lib.rp_layernorm_bwd(dy.data_ptr(), x.data_ptr(), w.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
                                        n_rows, self.cfg.dp, None if n_rows_dev is None else n_rows_dev.data_ptr(),
                                        None if gather is None else gather.data_ptr(),
                                        None if add_to is None else add_to.data_ptr(), dx.data_ptr(), dw.data_ptr(),
                                        db.data_ptr(), self.cfg.hd_valid, self._stream()), "rp_layernorm_bwd")

    def _site(self, app, k):
        """dropout site k of block application ``app`` (offset ``site << 40``; the embedding is site 0)"""
        return 1 + app * 8 + k

    # ------------------------------------------------------------------------------------------------ forward
    # heads that take several positives per position (replay/nn/loss/base.py:49-154, bce.py:51-95)
    MULTI_POSITIVE_KINDS = ("bce", "ce_sampled", "bce_sampled", "ce_sampled_weighted")

    def set_batch(self, ids, pad_mask, labels=None, target_mask=None):
        """Stage one batch ([B, L] int64 ids, bool masks) into the engine's static input buffers (device copies).  Targets
        are [B, L] or [B, L, P] (P positives per position; P = 1 is the [B, L] batch)."""
        B, L = ids.shape
        if L != self.L or B > self.B:
            raise ValueError(f"batch shape {tuple(ids.shape)} does not fit engine ({self.B}, {self.L})")
        P = 1
        if labels is not None:
            labels, target_mask, P = self._split_positives(labels, target_mask)
        self.cur_B = B
        n = B * L
        self.in_ids[:n].copy_(ids.reshape(-1), non_blocking=True)
        self.in_pad[:n].copy_(pad_mask.reshape(-1), non_blocking=True)
        if P > 1:
            mp = self._ensure_multi(P)
            mp["labels"][:n].copy_(labels.reshape(n, P), non_blocking=True)
            mp["tmask"][:n].copy_(target_mask.reshape(n, P), non_blocking=True)
            mp["tmask"][n:].zero_()
        elif labels is not None:
            self.in_labels[:n].copy_(labels.reshape(-1), non_blocking=True)
            self.in_tmask[:n].copy_(target_mask.reshape(-1), non_blocking=True)
        self.n_pos = P
        if n < self.T:
            self.in_pad[n:].zero_()
            self.in_tmask[n:].zero_()
        if self.sce is not None:
            self.sce["n_rows"].fill_(n)

    def _split_positives(self, labels, target_mask):
        """(labels, target_mask, P) of a [B, L] or [B, L, P] target batch; [B, L, 1] is the [B, L] batch."""
        if labels.dim() != 3 or labels.shape[-1] == 1:
            if labels.dim() == 3:
                labels = labels[..., 0]
            if target_mask is not None and target_mask.dim() == 3:
                target_mask = target_mask[..., 0]
            return labels, target_mask, 1
        P = labels.shape[-1]
        if target_mask is None or target_mask.shape != labels.shape:
            raise ValueError(f"target_padding_mask must have the labels' shape {tuple(labels.shape)}")
        if P > MAX_POSITIVES:
            raise ValueError(f"at most {MAX_POSITIVES} positives per position are supported, got {P}")
        kind = self._loss_args[0] if self._loss_args is not None else "ce"
        if kind not in self.MULTI_POSITIVE_KINDS:
            raise NotImplementedError(f"multi-positive labels are not supported by the {kind!r} head")
        return labels, target_mask, P

    def _ensure_multi(self, P: int) -> dict:
        """Staging and compaction buffers of a batch with P positives per position (rp_prepare_batch_multi), and a sampled
        head's workspace large enough for P.  Reallocating bumps ``mp_gen`` (captured steps hold the old buffers)."""
        T, dev = self.T, self.dev
        if self.mp is None or self.mp["P"] != P:
            self.mp = dict(P=P, labels=torch.zeros(T, P, device=dev, dtype=torch.int64),
                           tmask=torch.zeros(T, P, device=dev, dtype=torch.bool),
                           labels_p=torch.zeros(T, P, device=dev, dtype=torch.int32),
                           slot=torch.zeros(T, P, device=dev, dtype=torch.uint8),
                           n_pairs=torch.zeros(1, device=dev, dtype=torch.int32),
                           row_sum=torch.zeros(T, device=dev, dtype=torch.float32),
                           roww=torch.ones(T, P, device=dev, dtype=torch.float32),
                           roww_c=torch.ones(T, P, device=dev, dtype=torch.float32))
            self.mp_gen += 1
        sp = self.sampled
        if sp is not None:
            need = self.lib.rp_sampled_head_workspace_multi(T, self.cfg.dp, sp["n_neg"], sp["mode"], P)
            if sp["ws_bytes"] < need:
                sp["ws"], sp["ws_bytes"] = torch.zeros(need, device=dev, dtype=torch.uint8), need
                self.mp_gen += 1
        return self.mp

    # ------------------------------------------------------------------------------------------------ sampled heads
    SAMPLED_KINDS = {"ce_sampled": 0, "bce_sampled": 1, "legacy_ce_sampled": 2, "legacy_bce_sampled": 3, "login_ce_sampled": 4,
                     "ce_sampled_weighted": 5}

    def set_loss(self, kind: str = "ce", n_neg: int = 0, neg_shape: str = "shared", ignore_index: int = -100,
                 log_eps: float = 1e-6, clamp: float = 100.0, n_buckets: int = 0, bucket_size_x: int = 0,
                 bucket_size_y: int = 0, mix_x: bool = False):
        """``"ce"`` = full-catalog CE (default).  Sampled heads (SURVEY §8 a9): ``ce_sampled`` / ``bce_sampled`` (new path,
        replay/nn/loss/ce.py:146, bce.py:98), ``login_ce_sampled`` (LogInCESampled, login_ce.py:240, with ``log_eps`` /
        ``clamp``), ``ce_sampled_weighted`` (CESampledWeighted, ce.py:252: sample weights staged with set_row_weights) and
        ``legacy_ce_sampled`` / ``legacy_bce_sampled`` (sasrec/lightning.py:310-376)
        with ``n_neg`` negatives per target, ``neg_shape`` in shared [N] / perseq [B, N] / perpos [B, L, N].
        ``"sce"``: the legacy module's scalable cross-entropy (replay/models/nn/loss/sce.py) with ``n_buckets`` buckets of
        ``bucket_size_x`` rows and ``bucket_size_y`` items (both <= 1024, the fused top-K), ``mix_x`` as the reference."""
        self._loss_args = (kind, dict(n_neg=n_neg, neg_shape=neg_shape, ignore_index=ignore_index, log_eps=log_eps, clamp=clamp,
                                      n_buckets=n_buckets, bucket_size_x=bucket_size_x, bucket_size_y=bucket_size_y,
                                      mix_x=mix_x))
        self.sce = None
        if kind == "sce":
            self.sampled, self.ce_row, self.bce = None, None, False
            self._set_sce(n_buckets, bucket_size_x, bucket_size_y, bool(mix_x))
            return
        # per-row variants of the full-catalog head (rp_ce_head_fwd_w): "ce_weighted" (LogOutCEWeighted / CEWeighted: sample
        # weights staged with set_row_weights) and "login_ce" (LogInCE); "ce" is the plain head
        self.ce_row = None
        self.bce = kind == "bce"   # full-catalog BCE (rp_bce_head_*, replay/nn/loss/bce.py:10-95) on the CE head's buffers
        if kind in ("ce", "ce_weighted", "login_ce", "bce"):
            self.sampled = None
            if kind in ("ce_weighted", "login_ce"):
                self.ce_row = dict(kind=1 if kind == "login_ce" else 0, log_eps=log_eps, clamp=clamp, weighted=(kind == "ce_weighted"))
                self._alloc_row_weights()
            return
        if kind not in self.SAMPLED_KINDS:
            raise NotImplementedError(f"Not supported loss_type {kind!r}")
        mode = {"shared": 0, "perpos": 1, "perseq": 2}[neg_shape]
        rows = {0: 1, 1: self.T, 2: self.B}[mode]
        ws_bytes = self.lib.rp_sampled_head_workspace(self.T, self.cfg.dp, n_neg, mode)
        if kind == "ce_sampled_weighted":
            self._alloc_row_weights()
        self.sampled = dict(kind=self.SAMPLED_KINDS[kind], n_neg=n_neg, mode=mode, ignore_index=ignore_index, log_eps=log_eps,
                            clamp=clamp, neg=torch.zeros(rows, n_neg, device=self.dev, dtype=torch.int64),
                            ws=torch.zeros(ws_bytes, device=self.dev, dtype=torch.uint8), ws_bytes=ws_bytes)

    def _set_sce(self, n_b: int, bsx: int, bsy: int, mix: bool):
        cfg, dev, T = self.cfg, self.dev, self.T
        if not self.with_grad:   # an inference engine has no loss buffers; resize(with_grad=True) applies the loss again
            return
        if n_b < 1 or not 1 <= bsx <= min(1024, T) or not 1 <= bsy <= min(1024, cfg.n_items):
            raise ValueError(f"SCE needs n_buckets >= 1, 1 <= bucket_size_x <= min(1024, B * L = {T}) and 1 <= bucket_size_y "
                             f"<= min(1024, n_items = {cfg.n_items}) (the fused top-K); got {n_b}, {bsx}, {bsy}")
        ws_bytes = self.lib.rp_sce_head_workspace(T, cfg.n_items, cfg.dp, n_b, bsx, bsy, int(mix))
        if ws_bytes == 0:
            raise ValueError("rp_sce_head: unsupported shape")
        i64 = dict(device=dev, dtype=torch.int64)
        sc = dict(n_buckets=n_b, bucket_size_x=bsx, bucket_size_y=bsy, mix_x=mix, draw_given=False,
                  draw=torch.zeros((T, n_b) if mix else (n_b, cfg.d), device=dev, dtype=torch.float32),
                  top_x=torch.zeros(n_b, bsx, **i64), score_x=torch.zeros(n_b, bsx, device=dev, dtype=torch.float32),
                  top_y=torch.zeros(n_b, bsy, **i64), n_rows=torch.full((1,), T, device=dev, dtype=torch.int32),
                  ws=torch.zeros(ws_bytes, device=dev, dtype=torch.uint8))
        desc = SceDesc()
        desc.hc, desc.table = self.hc.data_ptr(), self.params16["item_emb"].data_ptr()
        desc.labels, desc.pad_mask, desc.n_rows = self.in_labels.data_ptr(), self.in_pad.data_ptr(), sc["n_rows"].data_ptr()
        desc.capacity, desc.n_items, desc.d, desc.d_true, desc.hd_valid = T, cfg.n_items, cfg.dp, cfg.d, cfg.hd_valid
        desc.n_buckets, desc.bucket_size_x, desc.bucket_size_y, desc.mix_x = n_b, bsx, bsy, int(mix)
        desc.seed, desc.rng_counter, desc.draw_given = self.seed, self.rng_counter.data_ptr(), 0
        desc.draw, desc.top_x, desc.score_x, desc.top_y = (sc[k].data_ptr() for k in ("draw", "top_x", "score_x", "top_y"))
        desc.loss_out = self.ce.loss.data_ptr()
        desc.workspace, desc.workspace_bytes = sc["ws"].data_ptr(), ws_bytes
        sc["desc"] = desc
        self.sce = sc

    def set_sce_draw(self, draw: torch.Tensor | None):
        """Tests only: replace the Philox bucket draw by a fixed standard-normal draw - [n_buckets, d] (the model's true
        hidden size), or with mix_x [B * L, n_buckets] for the staged batch - so that a reference run's captured
        ``torch.randn`` can be replayed.  ``None`` returns to the Philox draw."""
        sc = self.sce
        if sc is None:
            raise RuntimeError('set_loss("sce", ...) first')
        if draw is None:
            sc["desc"].draw_given = 0
            return
        if draw.dim() != 2 or draw.shape[1] != sc["draw"].shape[1] or draw.shape[0] > sc["draw"].shape[0] or (
                not sc["mix_x"] and draw.shape[0] != sc["draw"].shape[0]):
            raise ValueError(f"draw {tuple(draw.shape)} does not fit {tuple(sc['draw'].shape)}")
        sc["draw"].zero_()
        sc["draw"][: draw.shape[0]].copy_(draw)
        sc["desc"].draw_given = 1

    def _alloc_row_weights(self):
        """Static staging buffers of the per-row sample weights: in_roww [T] by flat position, roww_c [T] in the heads'
        compacted order (filled on the stream by each forward, so a captured step reads the weights staged for its batch)."""
        if not hasattr(self, "in_roww") or self.in_roww.numel() < self.T:
            self.in_roww = torch.ones(self.T, device=self.dev, dtype=torch.float32)
            self.roww_c = torch.ones(self.T, device=self.dev, dtype=torch.float32)

    def set_row_weights(self, weights):
        """Stage the sample weights of the current batch ([B, L] float, one per position; only valid targets are read).
        A batch with P > 1 positives per position takes [B, L, P] weights, one per (position, positive) pair."""
        if getattr(self, "n_pos", 1) > 1:
            n = self.cur_B * self.L
            if weights.numel() != n * self.n_pos:
                raise ValueError(f"sample weights {tuple(weights.shape)} must have the labels' shape ({self.cur_B}, {self.L}, "
                                 f"{self.n_pos})")
            self.mp["roww"][:n].copy_(weights.reshape(n, self.n_pos).to(torch.float32), non_blocking=True)
            return
        n = weights.numel()
        self.in_roww[:n].copy_(weights.reshape(-1).to(torch.float32), non_blocking=True)

    def set_negatives(self, negative_labels):
        """Stage the negatives of the current batch ([N] | [B, N] | [B, L, N] int64, device copy)."""
        sp = self.sampled
        if sp is None:
            raise RuntimeError("set_loss(<sampled kind>, ...) first")
        neg = negative_labels.reshape(-1, sp["n_neg"])
        if neg.shape[0] > sp["neg"].shape[0]:
            raise ValueError(f"negative_labels {tuple(negative_labels.shape)} do not fit the configured shape")
        sp["neg"][: neg.shape[0]].copy_(neg, non_blocking=True)

    def _sampled_desc(self):
        sp, cfg = self.sampled, self.cfg
        sd = SampledDesc()
        sd.hc, sd.table = self.hc.data_ptr(), self.params16["item_emb"].data_ptr()
        sd.labels, sd.valid_idx, sd.negatives = self.labels_c.data_ptr(), self.valid_idx.data_ptr(), sp["neg"].data_ptr()
        sd.n_valid = self.n_valid.data_ptr()
        sd.capacity, sd.n_items, sd.d, sd.n_neg, sd.neg_mode, sd.seq_len = self.T, cfg.n_items, cfg.dp, sp["n_neg"], sp["mode"], self.L
        sd.kind, sd.ignore_index, sd.vocab_size = sp["kind"], sp["ignore_index"], cfg.n_items
        sd.log_eps, sd.clamp = sp["log_eps"], sp["clamp"]
        sd.loss_out = self.ce.loss.data_ptr()
        sd.workspace, sd.workspace_bytes = sp["ws"].data_ptr(), sp["ws_bytes"]
        if sp["kind"] == self.SAMPLED_KINDS["ce_sampled_weighted"]:
            sd.row_weight = self.roww_c.data_ptr()
        if getattr(self, "n_pos", 1) > 1:   # [B, L, P] targets staged (set_batch)
            mp = self.mp
            sd.labels, sd.num_positives = mp["labels_p"].data_ptr(), self.n_pos
            sd.slot_mask, sd.n_pairs = mp["slot"].data_ptr(), mp["n_pairs"].data_ptr()
            if sp["kind"] == self.SAMPLED_KINDS["ce_sampled_weighted"]:
                sd.row_weight = mp["roww_c"].data_ptr()
        return sd

    def _prepare(self, with_targets: bool):
        cfg = self.cfg
        if with_targets and self.n_pos > 1:
            # the live positions (a set slot with an id in the catalog) go through the single-label compaction and the row
            # plan as in_labels / in_tmask; the slots of every compacted row land in labels_p / slot
            mp = self.mp
            check(self.lib.rp_prepare_batch_multi(
                self.in_ids.data_ptr(), self.in_pad.data_ptr(), mp["labels"].data_ptr(), mp["tmask"].data_ptr(), self.T,
                self.n_pos, cfg.pad_id, cfg.n_items, self.ids32.data_ptr(), self.in_labels.data_ptr(), self.in_tmask.data_ptr(),
                self.valid_idx.data_ptr(), self.labels_c.data_ptr(), mp["labels_p"].data_ptr(), mp["slot"].data_ptr(),
                self.n_valid.data_ptr(), mp["n_pairs"].data_ptr(), self.prep_scratch.data_ptr(), self._stream()),
                "rp_prepare_batch_multi")
        else:
            check(self.lib.rp_prepare_batch(self.in_ids.data_ptr(), self.in_pad.data_ptr(),
                                            self.in_labels.data_ptr() if with_targets else None,
                                            self.in_tmask.data_ptr() if with_targets else None, self.T, cfg.pad_id,
                                            cfg.n_items, self.ids32.data_ptr(), self.valid_idx.data_ptr(),
                                            self.labels_c.data_ptr(), self.n_valid.data_ptr(), self.prep_scratch.data_ptr(),
                                            self._stream()), "rp_prepare_batch")
        self._packed = with_targets and self.packed_eligible()
        if self._packed:
            check(self.lib.rp_row_plan(self.in_pad.data_ptr(), self.in_labels.data_ptr(), self.in_tmask.data_ptr(), self.B,
                                       self.L, cfg.n_items, self.valid_idx.data_ptr(), self.n_valid.data_ptr(),
                                       self.seq_first.data_ptr(), self.seq_off.data_ptr(), self.n_rows.data_ptr(),
                                       self.row_tok.data_ptr(), self.valid_rows.data_ptr(), self._stream()), "rp_row_plan")

    def packed_eligible(self) -> bool:
        """Whether a training step runs the body on packed rows: sequence b keeps only its positions [first_b, L), from its
        first real token or valid target on (the row before the first real token is a target whose input is padding), and
        the kept rows of all sequences are stored back to back.  Exact for the new-path SASRec: pad keys are masked, a pad
        query sees nothing live, and no loss reads a row before first_b, so those rows contribute exactly zero to every
        gradient.  Not for the legacy model (its attention sees pad keys), SCE (it reads every row's hidden state), other
        encoders, or shapes outside the fused body (d <= 128, head slot 64, L <= 256)."""
        cfg = self.cfg
        return (self.packed_body and isinstance(cfg, EncoderConfig) and cfg.variant == "new" and self.with_grad
                and self.sce is None and cfg.dp <= 128 and cfg.head_slot == 64 and self.L <= 256 and self.fused_attn_bwd
                and self.fused_pre_attn and self.fused_post_attn_train and self.fused_post_attn_bwd and self.fused_wgrad)

    def _target_rows(self):
        """Rows of the body's output that hold the valid targets, in the CE head's order."""
        return self.valid_rows if self._packed else self.valid_idx

    def _body_forward(self, training: bool, last_only: bool = False):
        """``last_only`` (predict): the final block is evaluated for the LAST position of every sequence only - LN1, the Q
        projection, one-query attention, out-projection, LN2 and the FFN run on [B, d] rows; only the K/V projection of
        that block still covers all tokens.  Result rows land in ``self.last_rows`` (bf16 [B, d])."""
        cfg, T, d, L = self.cfg, self.T, self.cfg.dp, self.L
        hdv, att_scale = cfg.hd_valid, 1.0 / math.sqrt(cfg.head_dim)
        p16, prm = self.params16, self.params
        legacy = cfg.variant == "legacy"
        drop = cfg.dropout if training else 0.0
        pad = self.in_pad
        pos0 = 0 if legacy else cfg.max_len - L
        packed = self._packed
        self._embed_fwd(drop, pos0)
        H, hd = cfg.n_heads, d // cfg.n_heads
        for i in range(cfg.n_blocks):
            a, x = self.act[i], self.x[i]
            w = lambda k: p16[f"b{i}.{k}"]  # noqa: E731
            f = lambda k: prm[f"b{i}.{k}"]  # noqa: E731
            if last_only and i == cfg.n_blocks - 1:
                Bq, lb = self.B, self.last_buf
                in_w, in_b = w("in_w"), f("in_b")
                self._ln_fwd(x, f("ln1_w"), f("ln1_b"), 1e-8, lb["q_in"], self.meanf, self.rstdf, Bq, gather=self.last_idx)
                self._gemm(lb["q_in"], in_w[:d], lb["Q"], Bq, d, d, bias=in_b[:d])
                if self.fused_pre_attn:
                    # [K | V] of ALL tokens through the fused pre-attention kernel in its K | V-only mode (activations read
                    # once, both halves from one resident weight)
                    check(self.lib.rp_ln_qkv_fused(x.data_ptr(), None, None, 1e-8, in_w.data_ptr(), in_b.data_ptr(), T, d, None,
                                                   None, a["KV"].data_ptr(), None, None, hdv, self._stream()), "rp_ln_qkv_fused")
                else:
                    self._gemm(x, in_w[d:], a["KV"], T, 2 * d, d, bias=in_b[d:])
                check(self.lib.rp_attn_last(lb["Q"].data_ptr(), a["KV"].data_ptr(), a["KV"].data_ptr(), 2 * d, 2 * d, 0, d,
                                            pad.data_ptr(), Bq, H, L, hd, int(not legacy), lb["O"].data_ptr(), att_scale,
                                            self._stream()), "rp_attn_last")
                if d <= 128:
                    # out-projection + residual + LayerNorm + FFN of the B last rows in the same fused pass the full blocks
                    # use (one launch instead of GEMM, LayerNorm, GEMM, GEMM: ~10 us each on [4096, d] rows)
                    check(self.lib.rp_post_attn_fused(lb["O"].data_ptr(), lb["q_in"].data_ptr(), w("out_w").data_ptr(),
                                                      f("out_b").data_ptr(), f("ln2_w").data_ptr(), f("ln2_b").data_ptr(), 1e-8,
                                                      w("w1").data_ptr(), f("b1").data_ptr(), w("w2").data_ptr(), f("b2").data_ptr(),
                                                      self.last_pad.data_ptr() if legacy else None, Bq, d,
                                                      self.last_rows.data_ptr(), hdv, self._stream()), "rp_post_attn_fused")
                    return
                self._gemm(lb["O"], w("out_w"), lb["h"], Bq, d, d, bias=f("out_b"), residual=lb["q_in"])
                self._ln_fwd(lb["h"], f("ln2_w"), f("ln2_b"), 1e-8, lb["y"], self.meanf, self.rstdf, Bq)
                self._gemm(lb["y"], w("w1"), lb["u"], Bq, d, d, bias=f("b1"), act=1)
                self._gemm(lb["u"], w("w2"), self.last_rows, Bq, d, d, bias=f("b2"), residual=lb["y"],
                           rowmask=self.last_pad if legacy else None)
                return
            in_w, in_b = w("in_w"), f("in_b")
            if packed:
                check(self.lib.rp_ln_qkv_fused_rows(x.data_ptr(), f("ln1_w").data_ptr(), f("ln1_b").data_ptr(), 1e-8,
                                                    in_w.data_ptr(), in_b.data_ptr(), T, d, a["q_in"].data_ptr(), a["Q"].data_ptr(),
                                                    a["KV"].data_ptr(), a["mean1"].data_ptr(), a["rstd1"].data_ptr(), hdv,
                                                    self.n_rows.data_ptr(), self._stream()), "rp_ln_qkv_fused_rows")
            elif self.fused_pre_attn:
                check(self.lib.rp_ln_qkv_fused(x.data_ptr(), f("ln1_w").data_ptr(), f("ln1_b").data_ptr(), 1e-8,
                                               in_w.data_ptr(), in_b.data_ptr(), T, d, a["q_in"].data_ptr(), a["Q"].data_ptr(),
                                               a["KV"].data_ptr(), a["mean1"].data_ptr(), a["rstd1"].data_ptr(), hdv,
                                               self._stream()), "rp_ln_qkv_fused")
            else:
                self._ln_fwd(x, f("ln1_w"), f("ln1_b"), 1e-8, a["q_in"], a["mean1"], a["rstd1"], T)
                self._gemm(a["q_in"], in_w[:d], a["Q"], T, d, d, bias=in_b[:d])
                self._gemm(x, in_w[d:], a["KV"], T, 2 * d, d, bias=in_b[d:])
            self._attention_forward(i, training, (a["Q"], 0), (a["KV"], 0), (a["KV"], d), causal=True, mask_pad_keys=not legacy)
            if not training and d <= 128:
                # inference: out-projection + residual + LayerNorm + FFN in one pass over the tokens (csrc/rp_block_fused.cu)
                check(self.lib.rp_post_attn_fused(a["O"].data_ptr(), a["q_in"].data_ptr(), w("out_w").data_ptr(),
                                                  f("out_b").data_ptr(), f("ln2_w").data_ptr(), f("ln2_b").data_ptr(), 1e-8,
                                                  w("w1").data_ptr(), f("b1").data_ptr(), w("w2").data_ptr(), f("b2").data_ptr(),
                                                  pad.data_ptr() if legacy else None, T, d, self.x[i + 1].data_ptr(), hdv,
                                                  self._stream()), "rp_post_attn_fused")
                continue
            if packed:
                check(self.lib.rp_post_attn_train_rows(a["O"].data_ptr(), a["q_in"].data_ptr(), w("out_w").data_ptr(),
                                                       f("out_b").data_ptr(), f("ln2_w").data_ptr(), f("ln2_b").data_ptr(), 1e-8,
                                                       w("w1").data_ptr(), f("b1").data_ptr(), w("w2").data_ptr(),
                                                       f("b2").data_ptr(), T, d, drop, self.seed, self._site(i, 1) << 40,
                                                       self._site(i, 2) << 40, self.rng_counter.data_ptr(), a["h"].data_ptr(),
                                                       a["y"].data_ptr(), a["u"].data_ptr(), a["mean2"].data_ptr(),
                                                       a["rstd2"].data_ptr(), self.x[i + 1].data_ptr(), hdv,
                                                       self.n_rows.data_ptr(), self.row_tok.data_ptr(), self._stream()),
                      "rp_post_attn_train_rows")
                continue
            if training and d <= 128 and self.fused_post_attn_train:
                # training: the same chain in one pass, saving h / y / u and the LayerNorm statistics for the backward
                check(self.lib.rp_post_attn_train(a["O"].data_ptr(), a["q_in"].data_ptr(), w("out_w").data_ptr(),
                                                  f("out_b").data_ptr(), f("ln2_w").data_ptr(), f("ln2_b").data_ptr(), 1e-8,
                                                  w("w1").data_ptr(), f("b1").data_ptr(), w("w2").data_ptr(), f("b2").data_ptr(),
                                                  pad.data_ptr() if legacy else None, T, d, drop, self.seed,
                                                  self._site(i, 1) << 40, self._site(i, 2) << 40, self.rng_counter.data_ptr(),
                                                  a["h"].data_ptr(), a["y"].data_ptr(), a["u"].data_ptr(),
                                                  a["mean2"].data_ptr(), a["rstd2"].data_ptr(), self.x[i + 1].data_ptr(), hdv,
                                                  self._stream()), "rp_post_attn_train")
                continue
            self._gemm(a["O"], w("out_w"), a["h"], T, d, d, bias=f("out_b"), residual=a["q_in"])
            self._ln_fwd(a["h"], f("ln2_w"), f("ln2_b"), 1e-8, a["y"], a["mean2"], a["rstd2"], T)
            self._gemm(a["y"], w("w1"), a["u"], T, d, d, bias=f("b1"), act=1, drop_p=drop, drop_site=self._site(i, 1))
            self._gemm(a["u"], w("w2"), self.x[i + 1], T, d, d, bias=f("b2"), drop_p=drop, drop_site=self._site(i, 2),
                       residual=a["y"], rowmask=pad if legacy else None)

    def _attn_desc(self, desc, i, q, k, v, causal, mask_pad_keys, drop_p):
        """The fields rp_attn_fwd's and rp_attn_bwd's descriptors share, for block ``i`` (output act[i]["O"])."""
        cfg = self.cfg
        for nm, (t, c0) in zip("qkv", (q, k, v)):
            setattr(desc, nm, t.data_ptr())
            setattr(desc, nm + "_rows", self.T)
            setattr(desc, nm + "_cols", t.shape[1])
            setattr(desc, "ld" + nm, t.stride(0))
            setattr(desc, nm + "_c0", c0)
        desc.B, desc.H, desc.L, desc.head_dim = self.B, cfg.n_heads, self.L, cfg.head_slot
        desc.causal, desc.mask_pad_keys = int(causal), int(mask_pad_keys)
        desc.scale = 1.0 / math.sqrt(cfg.head_dim)
        desc.pad_mask = self.in_pad.data_ptr()
        desc.out, desc.ldo = self.act[i]["O"].data_ptr(), cfg.dp
        desc.drop_p, desc.seed, desc.drop_off, desc.seed_ptr = drop_p, self.seed, self._site(i, 0) << 40, self.rng_counter.data_ptr()
        if self._packed:   # a packed training batch (set by _prepare; predict is never packed)
            desc.seq_first, desc.seq_off = self.seq_first.data_ptr(), self.seq_off.data_ptr()
        return desc

    def _attention_forward(self, i: int, training: bool, q, k, v, causal: bool, mask_pad_keys: bool):
        """Attention core of block ``i``: act[i]["O"] = softmax(Q.K^T * scale, causal and / or pad-key mask) . V, with Q, K
        and V given as (tensor, first column) of [T, *] arrays; saves the row statistics (and P on the un-fused path) when
        training with gradients."""
        a = self.act[i]
        ad = self._attn_desc(AttnDesc(), i, q, k, v, causal, mask_pad_keys, self.cfg.dropout if training else 0.0)
        if training and self.with_grad:
            ad.p_save = None if self.fused_attn_bwd else a["P"].data_ptr()
            ad.inv_sum, ad.m_save = a["inv_sum"].data_ptr(), a["m2"].data_ptr()
        else:
            ad.p_save, ad.inv_sum, ad.m_save = None, None, None
        check(self.lib.rp_attn_fwd(ctypes.byref(ad), self._stream()), "rp_attn_fwd")

    def _attention_backward(self, i: int, q, k, v, dq, dk, dv, causal: bool, mask_pad_keys: bool):
        """dQ, dK, dV of block ``i``'s attention core into the (tensor, first column) destinations ``dq``, ``dk``, ``dv`` from
        s["d_o"] and what ``_attention_forward(i, True, q, k, v, ...)`` saved: the fused kernel for head slot 64 at L <= 256,
        otherwise (head slot 128 at any L <= 512, head slot 64 at L > 256) dPd = dO.V^T, the row-wise softmax backward over
        the saved probabilities, and three batched GEMMs."""
        cfg, T, d, L, Lp = self.cfg, self.T, self.cfg.dp, self.L, self.Lp
        a, s, drop = self.act[i], self.s, cfg.dropout
        if self.fused_attn_bwd:
            bd = self._attn_desc(AttnBwdDesc(), i, q, k, v, causal, mask_pad_keys, drop)
            bd.d_out, bd.do_rows, bd.do_cols, bd.ld_do = s["d_o"].data_ptr(), T, d, d
            bd.m_save, bd.inv_sum = a["m2"].data_ptr(), a["inv_sum"].data_ptr()
            for nm, (t, c0) in zip(("dq", "dk", "dv"), (dq, dk, dv)):
                setattr(bd, nm, t.data_ptr())
                setattr(bd, "ld_" + nm, t.stride(0))
                setattr(bd, nm + "_c0", c0)
            check(self.lib.rp_attn_bwd(ctypes.byref(bd), self._stream()), "rp_attn_bwd")
            return
        H, hd = cfg.n_heads, cfg.head_slot
        BH = self.B * H
        P, dpd = a["P"].view(BH * Lp, Lp), s["dpd"].view(BH * Lp, Lp)
        heads = dict(batch=BH, inner=H, a_off=(0, H * Lp, Lp, 0, 0, 0))   # A = dS / Pd [BH*Lp, Lp]
        out = lambda t, c0: (t.stride(0), c0, L * t.stride(0), hd)  # noqa: E731  per-head [L, hd] blocks of a [T, *] array
        # dPd = dO . V^T
        self._gemm(s["d_o"], v[0], dpd, L, L, hd, batch=BH, inner=H, a_off=(0, L, 0, 0, 0, hd), b_off=(0, L, 0, v[1], 0, hd),
                   c_geom=(Lp, 0, H * Lp * Lp, Lp * Lp))
        check(self.lib.rp_attn_softmax_bwd(P.data_ptr(), dpd.data_ptr(), a["inv_sum"].data_ptr(), BH, L,
                                           1.0 / math.sqrt(cfg.head_dim), drop, self.seed, self._site(i, 0) << 40,
                                           self.rng_counter.data_ptr(), self._stream()), "rp_attn_softmax_bwd")
        # dQ = dS . K      (A = dS K-major, B = K MN-major)
        self._gemm(dpd, k[0], dq[0], L, hd, L, b_mn=True, b_off=(0, L, 0, k[1], 0, hd), c_geom=out(*dq), **heads)
        # dK = dS^T . Q    (A = dS MN-major, B = Q MN-major)
        self._gemm(dpd, q[0], dk[0], L, hd, L, a_mn=True, b_mn=True, b_off=(0, L, 0, q[1], 0, hd), c_geom=out(*dk), **heads)
        # dV = Pd^T . dO
        self._gemm(P, s["d_o"], dv[0], L, hd, L, a_mn=True, b_mn=True, b_off=(0, L, 0, 0, 0, hd), c_geom=out(*dv), **heads)

    def forward_train(self):
        """Loss of the staged batch (device fp32 [2] view: mean CE over the valid targets, 1/n_valid)."""
        cfg, T = self.cfg, self.T
        if self.sce is not None:
            # SCE reads the final hidden state of every position, pad rows included (the mix_x buckets sum over them)
            self._prepare(False)
            self._body_forward(True)
            self._final_norm_fwd(self.x[-1], self.hc, T)
            check(self.lib.rp_sce_head_fwd(ctypes.byref(self.sce["desc"]), SCE_ALL, self._stream()), "rp_sce_head_fwd")
            return self.ce.loss
        self._prepare(True)
        self._body_forward(True)
        self._final_norm_fwd(self.x[-1], self.hc, T, gather=self._target_rows(), n_rows_dev=self.n_valid)
        if self.sampled is not None:
            if self.sampled["kind"] == self.SAMPLED_KINDS["ce_sampled_weighted"]:   # weights in the head's compacted order
                if self.n_pos > 1:
                    torch.index_select(self.mp["roww"], 0, self.valid_idx, out=self.mp["roww_c"])
                else:
                    torch.index_select(self.in_roww, 0, self.valid_idx, out=self.roww_c)
            check(self.lib.rp_sampled_head_fwd(ctypes.byref(self._sampled_desc()), self._stream()), "rp_sampled_head_fwd")
            return self.ce.loss
        return self._catalog_head_fwd(self.params16["item_emb"][: cfg.n_items])

    def _final_norm_fwd(self, x, out, n_rows, gather=None, n_rows_dev=None):
        """The body's output normalization (LayerNorm lnf_w / lnf_b) of ``n_rows`` rows of ``x`` (or of the rows ``gather``
        lists) into ``out``; its statistics land in meanf / rstdf for ``_final_norm_bwd``."""
        self._ln_fwd(x, self.params["lnf_w"], self.params["lnf_b"], self.cfg.lnf_eps, out, self.meanf, self.rstdf, n_rows,
                     gather=gather, n_rows_dev=n_rows_dev)

    def _final_norm_bwd(self, dy, x, dx, n_rows, gather=None, n_rows_dev=None):
        G = self.grads
        self._ln_bwd(dy, x, self.params["lnf_w"], self.meanf, self.rstdf, dx, G["lnf_w"], G["lnf_b"], n_rows, gather=gather,
                     n_rows_dev=n_rows_dev)

    def _catalog_head_fwd(self, table, bias=None):
        """Full-catalog CE (or its per-row variants) / BCE head over the gathered rows self.hc -> loss (device fp32 [2])."""
        from .ops import bce_head_fwd, ce_head_fwd

        self.lib.count += 2
        d_hc = self.s["dhc"] if self.fused_ce else None
        if self.bce:
            loss = bce_head_fwd(self.ce, self.hc, table, self.labels_c, self.n_valid, bias=bias, d_hc=d_hc,
                                n_valid_hint=self.n_valid_hint)
            if self.n_pos > 1:   # the rest of each row's positive set
                mp = self.mp
                check(self.lib.rp_bce_head_multi_fwd(self.hc.data_ptr(), table.data_ptr(), self.labels_c.data_ptr(),
                                                     mp["labels_p"].data_ptr(), self.n_valid.data_ptr(), self.T, self.n_pos,
                                                     self.cfg.n_items, self.cfg.dp, loss.data_ptr(), mp["row_sum"].data_ptr(),
                                                     self._stream()), "rp_bce_head_multi_fwd")
            return loss
        row = self.ce_row
        roww = None
        if row is not None and row["weighted"]:   # weights of the valid targets in the head's compacted order
            torch.index_select(self.in_roww, 0, self.valid_idx, out=self.roww_c)
            roww = self.roww_c
        return ce_head_fwd(self.ce, self.hc, table, self.labels_c, self.n_valid, bias=bias, d_hc=d_hc,
                           n_valid_hint=self.n_valid_hint, row_weight=roww, loss_kind=row["kind"] if row else 0,
                           log_eps=row["log_eps"] if row else 1e-6, clamp=row["clamp"] if row else 100.0)

    def _catalog_head_bwd(self, table, d_table, bias=None, d_bias=None, n_valid_hint=None):
        """Backward of _catalog_head_fwd: d_hc into self.s["dhc"] (unless the forward already wrote it), d_table and d_bias
        (iff bias) overwritten.  ``n_valid_hint`` None: self.n_valid_hint."""
        from .ops import bce_head_bwd, ce_head_bwd

        head_bwd = bce_head_bwd if self.bce else ce_head_bwd
        head_bwd(self.ce, self.hc, table, self.labels_c, self.n_valid, self.s["dhc"], d_table, bias=bias, d_bias=d_bias,
                 n_valid_hint=self.n_valid_hint if n_valid_hint is None else n_valid_hint)
        if self.bce and self.n_pos > 1:
            mp = self.mp
            check(self.lib.rp_bce_head_multi_bwd(self.hc.data_ptr(), table.data_ptr(), self.labels_c.data_ptr(),
                                                 mp["labels_p"].data_ptr(), self.n_valid.data_ptr(), self.T, self.n_pos,
                                                 self.cfg.n_items, self.cfg.dp, self.ce.loss.data_ptr(), self.s["dhc"].data_ptr(),
                                                 d_table.data_ptr(), self._stream()), "rp_bce_head_multi_bwd")
        self.lib.count += 3

    # ------------------------------------------------------------------------------------------------ backward
    def _head_backward(self):
        """Backward of the loss head and the output normalization: returns d(last block's output), bf16 [T, dp]."""
        cfg, T, p16, G, s, st = self.cfg, self.T, self.params16, self.grads, self.s, self._stream
        if self.sce is not None:
            G["item_emb"].zero_()  # the reference's SCE scores a detached copy of the table: only the input gather reaches it
            check(self.lib.rp_sce_head_bwd(ctypes.byref(self.sce["desc"]), s["dhc"].data_ptr(), st()), "rp_sce_head_bwd")
        elif self.sampled is not None:
            G["item_emb"].zero_()  # the sampled head accumulates sparse rows (the full-CE head overwrites the dense table)
            check(self.lib.rp_sampled_head_bwd(ctypes.byref(self._sampled_desc()), s["dhc"].data_ptr(), G["item_emb"].data_ptr(),
                                               st()), "rp_sampled_head_bwd")
        else:
            self._catalog_head_bwd(p16["item_emb"][: cfg.n_items], G["item_emb"])
        dx = s["dxa"]
        dx.zero_()
        if self.sce is not None:
            self._final_norm_bwd(s["dhc"], self.x[-1], dx, T)
        else:
            self._final_norm_bwd(s["dhc"], self.x[-1], dx, T, gather=self._target_rows(), n_rows_dev=self.n_valid)
        return dx

    def backward(self):
        cfg, T, d, L = self.cfg, self.T, self.cfg.dp, self.L
        hdv = cfg.hd_valid
        p16, prm, G, s = self.params16, self.params, self.grads, self.s
        legacy = cfg.variant == "legacy"
        drop = cfg.dropout
        ks = 1.0 / (1.0 - drop) if drop > 0 else 1.0
        st = self._stream
        packed = self._packed
        rows = self.n_rows.data_ptr() if packed else None
        dx = self._head_backward()
        other = s["dxb"]
        for i in reversed(range(cfg.n_blocks)):
            a, x = self.act[i], self.x[i]
            w = lambda k: p16[f"b{i}.{k}"]  # noqa: E731
            f = lambda k: prm[f"b{i}.{k}"]  # noqa: E731
            g = lambda k: G[f"b{i}.{k}"]  # noqa: E731
            dz = dx
            if packed:
                check(self.lib.rp_post_attn_bwd_rows(dz.data_ptr(), a["u"].data_ptr(), a["h"].data_ptr(), a["mean2"].data_ptr(),
                                                     a["rstd2"].data_ptr(), f("ln2_w").data_ptr(), w("w2").data_ptr(),
                                                     w("w1").data_ptr(), w("out_w").data_ptr(), T, d, drop, self.seed,
                                                     self._site(i, 2) << 40, self.rng_counter.data_ptr(),
                                                     s["d_t"].data_ptr() if drop > 0 else None, s["du"].data_ptr(),
                                                     s["dh"].data_ptr(), s["d_o"].data_ptr(), g("ln2_w").data_ptr(),
                                                     g("ln2_b").data_ptr(), hdv, rows, self.row_tok.data_ptr(), st()),
                      "rp_post_attn_bwd_rows")
                d_t = s["d_t"] if drop > 0 else dz
            elif self.fused_post_attn_bwd:
                # one pass: d_t, du, dh (operands of the weight gradients), d_o (into the attention backward), dLN2
                masked = legacy or drop > 0
                check(self.lib.rp_post_attn_bwd(dz.data_ptr(), a["u"].data_ptr(), a["h"].data_ptr(), a["mean2"].data_ptr(),
                                                a["rstd2"].data_ptr(), f("ln2_w").data_ptr(), w("w2").data_ptr(),
                                                w("w1").data_ptr(), w("out_w").data_ptr(),
                                                self.in_pad.data_ptr() if legacy else None, T, d, drop, self.seed,
                                                self._site(i, 2) << 40, self.rng_counter.data_ptr(),
                                                s["d_t"].data_ptr() if masked else None, s["du"].data_ptr(), s["dh"].data_ptr(),
                                                s["d_o"].data_ptr(), g("ln2_w").data_ptr(), g("ln2_b").data_ptr(), hdv, st()),
                      "rp_post_attn_bwd")
                d_t = s["d_t"] if masked else dz
            else:
                if legacy:  # x_next = (...) * pad   (sasrec/model.py:441)
                    check(self.lib.rp_dropout_bwd(dz.data_ptr(), dz.data_ptr(), T, d, self.in_pad.data_ptr(), 0.0, 0, 0, None,
                                                  st()), "rp_dropout_bwd")
                if drop > 0:
                    check(self.lib.rp_dropout_bwd(dz.data_ptr(), s["d_t"].data_ptr(), T, d, None, drop, self.seed,
                                                  self._site(i, 2) << 40, self.rng_counter.data_ptr(), st()), "rp_dropout_bwd")
                    d_t = s["d_t"]
                else:
                    d_t = dz
                # ---- FFN backward
                self._gemm(d_t, w("w2"), s["du"], T, d, d, b_mn=True, gate=a["u"], gate_scale=ks)
                self._gemm(s["du"], w("w1"), s["dy"], T, d, d, b_mn=True, residual=dz)
                self._ln_bwd(s["dy"], a["h"], f("ln2_w"), a["mean2"], a["rstd2"], s["dh"], g("ln2_w"), g("ln2_b"), T)
                # ---- out projection
                self._gemm(s["dh"], w("out_w"), s["d_o"], T, d, d, b_mn=True)
            self._attention_backward(i, (a["Q"], 0), (a["KV"], 0), (a["KV"], d), (s["dQ"], 0), (s["dKV"], 0), (s["dKV"], d),
                                     causal=True, mask_pad_keys=not legacy)
            # ---- projections
            in_w = w("in_w")
            if packed:
                check(self.lib.rp_pre_attn_bwd_rows(s["dQ"].data_ptr(), s["dKV"].data_ptr(), s["dh"].data_ptr(), x.data_ptr(),
                                                    a["mean1"].data_ptr(), a["rstd1"].data_ptr(), f("ln1_w").data_ptr(),
                                                    in_w.data_ptr(), T, d, other.data_ptr(), g("ln1_w").data_ptr(),
                                                    g("ln1_b").data_ptr(), hdv, rows, st()), "rp_pre_attn_bwd_rows")
            elif self.fused_pre_attn:
                check(self.lib.rp_pre_attn_bwd(s["dQ"].data_ptr(), s["dKV"].data_ptr(), s["dh"].data_ptr(), x.data_ptr(),
                                               a["mean1"].data_ptr(), a["rstd1"].data_ptr(), f("ln1_w").data_ptr(),
                                               in_w.data_ptr(), T, d, other.data_ptr(), g("ln1_w").data_ptr(),
                                               g("ln1_b").data_ptr(), hdv, st()), "rp_pre_attn_bwd")
            else:
                self._gemm(s["dQ"], in_w[:d], s["dq_in"], T, d, d, b_mn=True, residual=s["dh"])
                self._ln_bwd(s["dq_in"], x, f("ln1_w"), a["mean1"], a["rstd1"], s["tmp"], g("ln1_w"), g("ln1_b"), T)
                self._gemm(s["dKV"], in_w[d:], other, T, d, 2 * d, b_mn=True, residual=s["tmp"])
            # ---- the block's weight and bias gradients (dY, X, dW, db) in one dispatch: no operand is overwritten within the block
            pairs = [(d_t, a["u"], g("w2"), g("b2")), (s["du"], a["y"], g("w1"), g("b1")), (s["dh"], a["O"], g("out_w"), g("out_b")),
                     (s["dQ"], a["q_in"], g("in_w")[:d], g("in_b")[:d]), (s["dKV"], x, g("in_w")[d:], g("in_b")[d:])]
            if self.fused_wgrad:
                self._wgrad_group(pairs, self.n_rows if packed else None)
            else:
                for dY, X, dW, _ in pairs:
                    self._wgrad(dY, X, dW, *dW.shape)
                self._colsum_multi([(dY, db) for dY, _, _, db in pairs])
            dx, other = other, dx
        pos0 = 0 if legacy else cfg.max_len - L
        if self.concat:
            self._concat_bwd(dx, drop, pos0)
            return
        if self.features:
            self._feature_bwd(dx, drop)
        if packed:
            check(self.lib.rp_embed_bwd_rows(dx.data_ptr(), self.ids32.data_ptr(), self.in_pad.data_ptr(), self.row_tok.data_ptr(),
                                             rows, self.seq_first.data_ptr(), self.seq_off.data_ptr(), self.B, L, d, cfg.pad_id,
                                             pos0, math.sqrt(cfg.d), 0, drop, self.seed, 0, self.rng_counter.data_ptr(),
                                             G["item_emb"].data_ptr(), G["pos_emb"].data_ptr(), st()), "rp_embed_bwd_rows")
            return
        check(self.lib.rp_embed_bwd(dx.data_ptr(), self.ids32.data_ptr(), self.in_pad.data_ptr(), self.B, L, d, cfg.pad_id,
                                    pos0, math.sqrt(cfg.d), int(legacy), drop, self.seed, 0, self.rng_counter.data_ptr(),
                                    G["item_emb"].data_ptr(), G["pos_emb"].data_ptr(), st()), "rp_embed_bwd")

    def optimizer_step(self, grad_scale: float = 1.0, opt: OptimizerConfig = OptimizerConfig()):
        """One step of ``opt`` (default: torch.optim.Adam(lr, betas=(0.9, 0.98)), optimizer_factory.py:56-63,79-80) on the
        flat buffers; also refreshes the bf16 shadow weights and zeroes the gradients.  A step of another kind than the
        state's starts from fresh state, as a newly built torch optimizer does."""
        if opt.validate().kind != self.opt_kind:
            self.reset_optimizer_state(opt.kind)
        adam = opt.kind == "adam"
        check(self.lib.rp_optimizer_step(_OPT_KINDS[opt.kind], self.p32.data_ptr(), self.g32.data_ptr(),
                                         self.adam_m.data_ptr(), self.adam_v.data_ptr() if adam else None, self.p16.data_ptr(),
                                         self.n_flat, self.lr.data_ptr(), self.step_count.data_ptr(), opt.betas[0],
                                         opt.betas[1], opt.eps, opt.weight_decay, opt.momentum, grad_scale, None, 1,
                                         self._stream()), "rp_optimizer_step")

    def reset_optimizer_state(self, kind: str = "adam"):
        """Zero the moments (or momentum buffer) and the step counter: the state of a newly built optimizer of ``kind``."""
        self.adam_m.zero_()
        self.adam_v.zero_()
        self.step_count.zero_()
        self.opt_kind = kind

    def optimizer_state(self, opt: OptimizerConfig) -> dict:
        """The state of ``opt`` for the flat parameter in torch.optim's per-parameter format (host copies): Adam's ``step`` /
        ``exp_avg`` / ``exp_avg_sq``, SGD's ``momentum_buffer``; empty where a newly built torch optimizer's is (no step
        taken, momentum 0, or state of the other kind, which the next step discards)."""
        steps = int(self.step_count.item())
        if opt.kind != self.opt_kind or steps == 0:
            return {}
        if opt.kind == "adam":
            return {"step": torch.tensor(float(steps)), "exp_avg": self.adam_m.cpu(), "exp_avg_sq": self.adam_v.cpu()}
        return {"momentum_buffer": self.adam_m.cpu()} if opt.momentum != 0 else {}

    def load_optimizer_state(self, state: dict):
        """Restore what ``optimizer_state`` returns (or a torch Adam / SGD state of the flat parameter)."""
        if "exp_avg" in state:
            self.reset_optimizer_state("adam")
            self.adam_m.copy_(state["exp_avg"])
            self.adam_v.copy_(state["exp_avg_sq"])
            self.step_count.fill_(int(state["step"]))
        elif state.get("momentum_buffer") is not None:
            self.reset_optimizer_state("sgd")
            self.adam_m.copy_(state["momentum_buffer"])
            self.step_count.fill_(1)   # torch's SGD keeps no step count: the restored buffer stands for one or more steps
        else:
            self.reset_optimizer_state(self.opt_kind)

    def tick_rng(self):
        check(self.lib.rp_counter_add(self.rng_counter.data_ptr(), 0x9E3779B97F4A7C15 & 0xFFFFFFFFFFFF, self._stream()),
              "rp_counter_add")

    def train_step(self, all_reduce=None, opt: OptimizerConfig = OptimizerConfig()):
        """forward + backward + (optional gradient all-reduce callback on the flat fp32 gradient) + the optimizer step."""
        opt.validate()   # before the backward accumulates a gradient that no step would consume
        self.tick_rng()
        loss = self.forward_train()
        self.backward()
        scale = 1.0
        if all_reduce is not None:
            scale = all_reduce(self.g32)
        self.optimizer_step(grad_scale=scale, opt=opt)
        return loss

    # ------------------------------------------------------------------------------------------------ inference
    def forward_last_hidden(self):
        """Eval-mode body (no dropout) -> final LayerNorm of the LAST position of every sequence -> self.hq bf16 [B, d]
        (SasRec.forward_inference, nn/sequential/sasrec/model.py:292-307 ; legacy get_query_embeddings, model.py:157)."""
        self._prepare(False)
        if self.cfg.variant == "legacy":
            self.last_pad.copy_(self.in_pad.view(self.B, self.L)[:, -1])
        self._body_forward(False, last_only=True)
        self._ln_fwd(self.last_rows, self.params["lnf_w"], self.params["lnf_b"], self.cfg.lnf_eps, self.hq, self.meanf, self.rstdf,
                     self.B)
        return self.hq

    def forward_hidden_all(self):
        """Eval-mode hidden states of every position, bf16 [T, d] (for parity tests / HiddenStatesCallback)."""
        self._prepare(False)
        self._body_forward(False)
        out = torch.empty(self.T, self.cfg.dp, device=self.dev, dtype=torch.bfloat16)
        self._ln_fwd(self.x[-1], self.params["lnf_w"], self.params["lnf_b"], self.cfg.lnf_eps, out, self.meanf, self.rstdf, self.T)
        return out
