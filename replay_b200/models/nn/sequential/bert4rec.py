"""Mirror of the legacy ``replay.models.nn.sequential.bert4rec`` modules on the H100 engine: ``Bert4RecModel``
(bert4rec/model.py:10-170) and the Lightning module ``Bert4Rec`` (bert4rec/lightning.py:15-683), plus the host-side
input-layout helpers (uniform masker dataset.py:55-92, predict shift dataset.py:322-345)."""
from __future__ import annotations

import torch

from ....core import SasRecCore, _EngineLoss, dist_grad_all_reduce
from ....engine_bert import Bert4RecEngine, BertConfig
from ....schema import bert_side_features_of, item_feature_of
from .lightning_base import LegacyLightningModule

# in the order TransformerBlock registers its parameters (bert4rec/model.py:481-500)
_BLEAF = {"in_w": "attention.in_proj_weight", "in_b": "attention.in_proj_bias", "out_w": "attention.out_proj.weight",
          "out_b": "attention.out_proj.bias", "ln1_w": "attention_norm.weight", "ln1_b": "attention_norm.bias",
          "w1": "pff.w_1.weight", "b1": "pff.w_1.bias", "w2": "pff.w_2.weight", "b2": "pff.w_2.bias",
          "ln2_w": "pff_norm.weight", "ln2_b": "pff_norm.bias"}


def bert_key_map(n_blocks: int, tying: bool, item_feature: str = "item_id", positional: bool = True, features=()) -> dict:
    """engine parameter name -> reference state_dict key (SURVEY.md Appendix B), in the reference's order.  Without the
    positional embedding the reference registers no ``item_embedder.position`` module (bert4rec/model.py:236-237), so there
    is no pos_emb key.  The categorical side ``features`` follow the item table (its ``cat_embeddings``, in schema order for
    a schema that starts with the item id)."""
    m = {"item_emb": f"item_embedder.cat_embeddings.{item_feature}.weight"}
    for f in features:
        if f.kind == "cat":
            m[f"feat.{f.name}"] = f"item_embedder.cat_embeddings.{f.name}.weight"
    m["mask_emb"] = "item_embedder.mask_embedding.weight"
    if positional:
        m["pos_emb"] = "item_embedder.position.pe.weight"
    for i in range(n_blocks):
        for k, leaf in _BLEAF.items():
            m[f"b{i}.{k}"] = f"transformer_blocks.{i}." + leaf
    if tying:
        m["head_b"] = "_head.out_bias"
    else:
        m["head_w"], m["head_b"] = "_head.linear.weight", "_head.linear.bias"
    return m


def uniform_masker(pad_mask: torch.Tensor, mask_prob: float = 0.15, generator=None) -> torch.Tensor:
    """Bert4RecUniformMasker.mask (dataset.py:71-92), vectorised over rows: token_mask = (rand * pad) >= p (0 = masked);
    a row where NOTHING is masked gets its last position masked, else a row where EVERYTHING is masked gets position -2
    unmasked - literally the reference's corner cases (known answers: tests/.../test_bert4rec_dataset.py:15-41)."""
    pm = pad_mask if pad_mask.dim() == 2 else pad_mask.unsqueeze(0)
    r = torch.rand(pm.shape, dtype=torch.float32, generator=generator, device="cpu").to(pm.device)
    tok = (r * pm) >= mask_prob
    all_kept = tok.all(-1)
    none_kept = ~tok.any(-1) & ~all_kept
    tok[all_kept, -1] = False
    if pm.shape[-1] > 1:
        tok[none_kept, -2] = True
    return tok if pad_mask.dim() == 2 else tok[0]


def shift_features(ids, pad_mask, token_mask, pad_value: int = 0):
    """_shift_features (dataset.py:322-345): roll left by one; the last position becomes <MASK> with pad = True."""
    ids2 = torch.roll(ids, -1, dims=-1); ids2[..., -1] = pad_value
    pm = torch.roll(pad_mask, -1, dims=-1); pm[..., -1] = True
    tm = torch.roll(token_mask, -1, dims=-1); tm[..., -1] = False
    return ids2, pm, tm


class _BertCore(SasRecCore):
    def _key_map(self):
        return bert_key_map(self.cfg.n_blocks, self.cfg.tying, self.item_feature, self.cfg.positional, self.cfg.features)

    def _initial_seq_len(self):
        return self.cfg.max_len

    def _make_engine(self, batch, seq_len, with_grad):
        return Bert4RecEngine(self.cfg, batch, seq_len, self._device, seed=self._seed, with_grad=with_grad)

    def _to_ref(self, k, v):
        return v   # export_named already gives the reference shapes (true d, 4d inner width, n_items bias entries)

    def _from_ref(self, k, v):
        return v

    def state_dict(self, *a, destination=None, prefix="", keep_vars=False):
        src = self._export() if self.engine is not None else (self._pending_state or {})
        out = destination if destination is not None else {}
        for k in self._keymap.values():   # the reference's order
            if k in src:
                out[prefix + k] = src[k]
        if self.cfg.tying:  # the tied head registers the embedder again (Appendix B)
            for k, v in list(src.items()):
                if k.startswith("item_embedder."):
                    out[prefix + "_head._item_embedder." + k[len("item_embedder."):]] = v
        return out

    @property
    def loss_kind(self) -> str:
        """The full-catalog head chosen with ``set_loss``: "ce" (the default) or "bce"."""
        return getattr(self, "_loss_spec", ("ce", {}))[0]

    def _apply_loss(self, eng):
        kind = self.loss_kind
        if getattr(eng, "_loss_applied", None) != kind:
            eng.set_loss(kind)
            eng._loss_applied = kind
            self._drop_graphs()   # captured graphs launch the other head's kernels

    # ``feats``: the batch's feature tensors by name (its "inputs"); a model with side features stages them, an item-only
    # model ignores them
    def loss(self, ids, pad_mask, token_mask, labels, feats=None):
        eng = self.ensure_engine(*ids.shape, with_grad=True)
        self._apply_loss(eng)
        self._stage_features(eng, feats)
        eng.set_batch(ids, pad_mask, token_mask, labels)
        return _EngineLoss.apply(self.flat, self)

    def fused_step(self, ids, pad_mask, token_mask, labels, all_reduce="auto", lr=None, feats=None):
        eng = self.ensure_engine(*ids.shape, with_grad=True)
        if self._shadow_dirty:
            eng.refresh_shadow(); self._shadow_dirty = False
        self._set_lr(eng, lr)
        self._apply_loss(eng)
        self._stage_features(eng, feats)
        eng.set_batch(ids, pad_mask, token_mask, labels)
        if isinstance(all_reduce, str):
            return self._graph_trainer(eng).run()[0]
        return eng.train_step(all_reduce, opt=self.optimizer)[0]

    @torch.no_grad()
    def _query_padded(self, ids, pad_mask, token_mask, feats=None):
        """last-position hidden states at the padded width bf16 [B, dp] (pairs with the padded head)"""
        eng = self.ensure_engine(*ids.shape, with_grad=self.engine.with_grad if self.engine is not None else False)
        if self._shadow_dirty:
            eng.refresh_shadow(); self._shadow_dirty = False
        self._stage_features(eng, feats)
        eng.set_batch(ids, pad_mask, token_mask)
        return eng.forward_last_hidden()[: ids.shape[0]]

    @torch.no_grad()
    def hidden_states(self, ids, pad_mask, token_mask, feats=None):
        """eval-mode hidden states of every position at the model's true hidden size, bf16 [B, L, d]"""
        B, L = ids.shape
        eng = self.ensure_engine(B, L, with_grad=self.engine.with_grad if self.engine is not None else False)
        if self._shadow_dirty:
            eng.refresh_shadow(); self._shadow_dirty = False
        self._stage_features(eng, feats)
        eng.set_batch(ids, pad_mask, token_mask)
        return eng.unpad_features(eng.forward_hidden_all().view(eng.B, L, -1)[:B])

    @torch.no_grad()
    def head_logits(self, h, item_ids=None):
        """Biased head scores fp32 [N, |I|] (or [N, |item_ids|]) of hidden rows ``h`` [N, d] at the true hidden size."""
        eng = self.engine
        if self._shadow_dirty:
            eng.refresh_shadow(); self._shadow_dirty = False
        hp = eng.pad_features(h.to(torch.bfloat16)).contiguous()
        W, b = eng.head_for_scoring()
        b = b[: self.cfg.n_items]
        if item_ids is not None:
            W, b = W[item_ids].contiguous(), b[item_ids].contiguous()
        out = torch.empty(hp.shape[0], W.shape[0], device=hp.device, dtype=torch.float32)
        eng._gemm(hp, W, out, hp.shape[0], W.shape[0], self.cfg.dp, out_mode=2, bias=b)
        return out

    @torch.no_grad()
    def query_embeddings(self, ids, pad_mask, token_mask, feats=None):
        """bf16 [B, d] at the model's true hidden size"""
        return self.engine.unpad_features(self._query_padded(ids, pad_mask, token_mask, feats))

    @torch.no_grad()
    def logits(self, ids, pad_mask, token_mask, candidates=None, feats=None):
        hq = self._query_padded(ids, pad_mask, token_mask, feats)
        W, b = self.engine.head_for_scoring()
        b = b[: self.cfg.n_items]
        if candidates is not None:
            W, b = W[candidates].contiguous(), b[candidates].contiguous()
        out = torch.empty(hq.shape[0], W.shape[0], device=hq.device, dtype=torch.float32)
        self.engine._gemm(hq, W, out, hq.shape[0], W.shape[0], self.cfg.dp, out_mode=2, bias=b)
        return out

    @torch.no_grad()
    def predict_topk(self, ids, pad_mask, token_mask, k, seen_ids=None, candidates=None, feats=None):
        from .... import ops

        hq = self._query_padded(ids, pad_mask, token_mask, feats).contiguous()
        W, b = self.engine.head_for_scoring()
        n_items, inv = self.cfg.n_items, None
        if candidates is not None:
            inv = torch.full((n_items,), -1, device=hq.device, dtype=torch.int32)
            inv[candidates] = torch.arange(candidates.numel(), device=hq.device, dtype=torch.int32)
            W = W[candidates].contiguous()
            bb = torch.zeros((candidates.numel() + 127) // 128 * 128, device=hq.device)
            bb[: candidates.numel()] = b[candidates]
            b = bb
        seen = None if seen_ids is None else ops.seen_prepare(seen_ids.contiguous(), n_items, inv)
        return ops.score_topk(hq, W, k, seen, candidates, bias=b)


class Bert4RecModel(torch.nn.Module):
    def __init__(self, schema, max_len: int = 100, hidden_size: int = 256, num_blocks: int = 2, num_heads: int = 4,
                 num_passes_over_block: int = 1, dropout: float = 0.1, enable_positional_embedding: bool = True,
                 enable_embedding_tying: bool = False, device=None, seed: int = 0):
        super().__init__()
        name, card, pad, _ = item_feature_of(schema)
        self.schema, self.item_feature_name, self.item_count, self.max_len = schema, name, card, max_len
        self.hidden_size, self.num_blocks, self.num_heads, self.dropout = hidden_size, num_blocks, num_heads, dropout
        self.num_passes_over_block = num_passes_over_block
        self.enable_positional_embedding, self.enable_embedding_tying = enable_positional_embedding, enable_embedding_tying
        # every other categorical and numerical feature of the schema is summed into the item embedding (BertEmbedding)
        cfg = BertConfig(n_items=card, d=hidden_size, n_heads=num_heads, n_blocks=num_blocks, max_len=max_len, dropout=dropout,
                         tying=enable_embedding_tying, pad_id=pad if 0 <= pad < card else 0, passes=num_passes_over_block,
                         positional=bool(enable_positional_embedding), features=tuple(bert_side_features_of(schema)))
        self.core = _BertCore(cfg, item_feature=name, device=device, seed=seed)

    def state_dict(self, *a, **k):
        return self.core.state_dict(*a, **k)

    def load_state_dict(self, sd, strict=True, assign=False):
        return self.core.load_state_dict(sd, strict=strict)

    def get_query_embeddings(self, inputs, pad_mask, token_mask):
        return self.core.query_embeddings(inputs[self.item_feature_name], pad_mask, token_mask, inputs).float()

    # ---- inference-only restatements of the reference's forward / forward_step / get_logits (bert4rec/model.py:86-157)
    def forward_step(self, inputs, pad_mask, token_mask):
        """Hidden states of every position, fp32 [B, L, d] (eval mode: no dropout)."""
        return self.core.hidden_states(inputs[self.item_feature_name], pad_mask, token_mask, inputs).float()

    def get_logits(self, out_embeddings, item_ids=None):
        """Biased head scores of hidden states [..., d]: [..., |I|], or [..., |item_ids|]."""
        h = out_embeddings.reshape(-1, out_embeddings.shape[-1])
        out = self.core.head_logits(h, item_ids)
        return out.view(*out_embeddings.shape[:-1], out.shape[-1])

    def forward(self, inputs, pad_mask, token_mask):
        """All-position scores [B, L, |I|] - materialised; use only for small problems."""
        return self.get_logits(self.forward_step(inputs, pad_mask, token_mask))

    # ---- catalog growth
    def _weights(self) -> dict:
        """reference-keyed copies of every weight (materialises the seeded initial ones on first use)"""
        if self.core.engine is None and not self.core._pending_state:
            self.core.ensure_engine(1, self.max_len, with_grad=False)
        return {k: v.detach().clone() for k, v in self.core.state_dict().items()}

    def item_embeddings(self) -> torch.Tensor:
        """A copy of the item table [I, d] (BertEmbedding.item_embeddings, model.py:298-303)."""
        return self._weights()[f"item_embedder.cat_embeddings.{self.item_feature_name}.weight"]

    def get_all_embeddings(self) -> dict:
        """Copies of the item table [I, d], every categorical side table under its feature's name and, when it is on, the
        position table [max_len, d] (model.py:298-312).  A numerical feature has no table: KeyError, as in the reference."""
        sd = self._weights()
        out = {"item_embedding": sd[f"item_embedder.cat_embeddings.{self.item_feature_name}.weight"]}
        for name, _ in self.schema.items():
            if name != self.item_feature_name:
                key = f"item_embedder.cat_embeddings.{name}.weight"
                if key not in sd:
                    raise KeyError(name)
                out[name] = sd[key]
        if self.enable_positional_embedding:
            out["positional_embedding"] = sd["item_embedder.position.pe.weight"]
        return out

    def resize_items(self, table: torch.Tensor):
        """Rebuild for the catalog of ``table`` [I', d] (I' >= I), keeping every other weight, side tables included
        (lightning.py:612-627): the
        head keeps its first I rows and bias entries and takes fresh ones for the new items - ``Linear(hidden, I')``'s
        default initialisation untied, N(0, 0.01) bias entries tied.  The core is rebuilt for the new catalog size
        (``SasRecCore.for_catalog``); the passes and the positional setting carry over with its configuration."""
        n_new = int(table.shape[0])
        sd = {k: v.float().cpu() for k, v in self._weights().items()}
        n_old, d = self.item_count, self.hidden_size
        sd[f"item_embedder.cat_embeddings.{self.item_feature_name}.weight"] = table.detach().float().cpu()
        if self.enable_embedding_tying:
            bias = torch.empty(n_new).normal_(0, 0.01)
            bias[:n_old] = sd["_head.out_bias"]
            sd["_head.out_bias"] = bias
        else:
            lin = torch.nn.Linear(d, n_new)
            w, b = lin.weight.detach().clone(), lin.bias.detach().clone()
            w[:n_old], b[:n_old] = sd["_head.linear.weight"], sd["_head.linear.bias"]
            sd["_head.linear.weight"], sd["_head.linear.bias"] = w, b
        self.core = self.core.for_catalog(n_new, sd)
        self.item_count = n_new

    def predict(self, inputs, pad_mask, token_mask, candidates_to_score=None):
        return self.core.logits(inputs[self.item_feature_name], pad_mask, token_mask, candidates_to_score, inputs)


class Bert4Rec(LegacyLightningModule):
    def __init__(self, tensor_schema, block_count: int = 2, head_count: int = 4, hidden_size: int = 256, max_seq_len: int = 100,
                 dropout_rate: float = 0.1, pass_per_transformer_block_count: int = 1, enable_positional_embedding: bool = True,
                 enable_embedding_tying: bool = False, loss_type: str = "CE", loss_sample_count=None,
                 negative_sampling_strategy: str = "global_uniform", negatives_sharing: bool = False, optimizer_factory=None,
                 lr_scheduler_factory=None, fused_optimizer: bool = True, device=None):
        super().__init__()
        self.save_hyperparameters()
        # "CE_restricted" is the same CE over the same rows (bert4rec/lightning.py:379-391,475-489); sampled losses are not built
        kind = {"CE": "ce", "CE_restricted": "ce", "BCE": "bce"}.get(loss_type)
        if kind is None or loss_sample_count is not None:
            raise NotImplementedError("Not supported loss_type")
        self._attach(Bert4RecModel(tensor_schema, max_len=max_seq_len, hidden_size=hidden_size, num_blocks=block_count,
                                   num_heads=head_count, num_passes_over_block=pass_per_transformer_block_count,
                                   dropout=dropout_rate, enable_positional_embedding=enable_positional_embedding,
                                   enable_embedding_tying=enable_embedding_tying, device=device),
                     tensor_schema, optimizer_factory, lr_scheduler_factory, fused_optimizer)
        self._model.core.set_loss(kind)

    def training_step(self, batch: dict, batch_idx: int = 0):
        """batch keys (bert4rec/dataset.py:167-173): query_id, pad_mask, inputs, token_mask, positive_labels."""
        ids = batch["inputs"][self._model.item_feature_name]
        args = (ids, batch["pad_mask"], batch["token_mask"], batch["positive_labels"])
        core, feats = self._model.core, batch["inputs"]
        loss = core.fused_step(*args, lr=self._current_lr(), feats=feats) if self.fused_optimizer else core.loss(*args, feats)
        self.log("train_loss", loss, on_step=True, on_epoch=True, prog_bar=True, sync_dist=True)
        return loss

    def _prepared(self, batch):
        """_prepare_prediction_batch (bert4rec/lightning.py:649-683): a batch of full length is taken AS IS (the prediction
        dataset already shifted it, bert4rec/dataset.py:322-345); a shorter one is left-padded with the padding value and
        then shifted; a longer one is an error.  Every categorical side feature is padded and shifted the same way with its
        own padding value.  A short batch with a numerical side feature raises: the reference's ``view(B, L)`` of its
        [B, L, tensor_dim] values fails there.  Returns (ids, pad_mask, token_mask, feature tensors)."""
        ids, pm, tm = batch["inputs"][self._model.item_feature_name], batch["pad_mask"], batch["token_mask"]
        seq_len, max_len = pm.shape[1], self._model.max_len
        feats = batch["inputs"]
        if seq_len > max_len:
            raise ValueError("The length of the submitted sequence must not exceed the maximum length of the sequence. "
                             f"The length of the sequence is given {seq_len}, while the maximum length is {max_len}")
        if seq_len < max_len:
            side = self._model.core.cfg.features
            num = [f.name for f in side if f.kind != "cat"]
            if num:
                raise ValueError(f"a batch shorter than max_seq_len cannot carry the numerical features {num}: the reference "
                                 "cannot left-pad their [B, L, tensor_dim] values")
            item = self._schema.item_id_features
            item = item.item() if hasattr(item, "item") else item[self._schema.item_id_feature_name]
            padded = torch.nn.functional.pad(pm, (max_len - seq_len, 0), value=0)
            pads = [(self._model.item_feature_name, int(item.padding_value))] + [(f.name, f.padding_value) for f in side]
            feats = {}
            for name, pad in pads:
                v = torch.nn.functional.pad(batch["inputs"][name], (max_len - seq_len, 0), value=pad)
                feats[name], pm, tm = shift_features(v, padded, padded, pad)
            ids = feats[self._model.item_feature_name]
        return ids, pm, tm, feats

    def _model_predict(self, ids, pm, tm, candidates_to_score=None, feats=None):
        cands = self._candidates_to_score if candidates_to_score is None else candidates_to_score
        return self._model.core.logits(ids, pm, tm, cands, feats)

    def forward(self, feature_tensors, padding_mask, tokens_mask, candidates_to_score=None):
        return self._model_predict(feature_tensors[self._model.item_feature_name], padding_mask, tokens_mask, candidates_to_score,
                                   feature_tensors)

    def validation_step(self, batch: dict, batch_idx: int = 0, dataloader_idx: int = 0):
        return self._model_predict(batch["inputs"][self._model.item_feature_name], batch["pad_mask"], batch["token_mask"],
                                   feats=batch["inputs"])

    def predict_step(self, batch: dict, batch_idx: int = 0, dataloader_idx: int = 0):
        ids, pm, tm, feats = self._prepared(batch)
        return self._model_predict(ids, pm, tm, feats=feats)

    def predict(self, batch: dict, candidates_to_score=None):
        ids, pm, tm, feats = self._prepared(batch)
        return self._model_predict(ids, pm, tm, candidates_to_score, feats)

    def predict_topk(self, batch: dict, k: int, seen_ids=None, candidates_to_score=None):
        ids, pm, tm, feats = self._prepared(batch)
        cands = self._candidates_to_score if candidates_to_score is None else candidates_to_score
        return self._model.core.predict_topk(ids, pm, tm, k, seen_ids, cands, feats)

    # ---- catalog growth for fine-tuning on new items (bert4rec/lightning.py:501-628)
    def get_all_embeddings(self) -> dict:
        return self._model.get_all_embeddings()

    def _embedding_dim(self) -> int:
        dim = item_feature_of(self._model.schema)[3]
        return self._model.hidden_size if dim is None else int(dim)

    def _set_new_item_table(self, table: torch.Tensor):
        self._model.resize_items(table)
        self._item_count_changed()

    def set_item_embeddings_by_size(self, new_vocab_size: int):
        """Keep the fitted item embeddings and add xavier-normal rows (drawn over the whole new table) for the new items."""
        if new_vocab_size <= self._vocab_size:
            raise ValueError("New vocabulary size must be greater then already fitted")
        new = torch.empty(new_vocab_size, self._embedding_dim())
        torch.nn.init.xavier_normal_(new)
        new[: self._vocab_size] = self._model.item_embeddings()
        self._set_new_item_table(new)

    def set_item_embeddings_by_tensor(self, all_item_embeddings: torch.Tensor):
        """Replace the whole item table, possibly with more items."""
        if all_item_embeddings.dim() != 2:
            raise ValueError("Input tensor must have (number of all items, model hidden size) shape")
        if all_item_embeddings.shape[0] < self._vocab_size:
            raise ValueError("New vocabulary size can't be less then already fitted")
        if all_item_embeddings.shape[1] != self._embedding_dim():
            raise ValueError("Input tensor second dimension doesn't match embedding dim")
        self._set_new_item_table(all_item_embeddings.detach().float().cpu())

    def append_item_embeddings(self, item_embeddings: torch.Tensor):
        """Append rows for new items only."""
        if item_embeddings.dim() != 2:
            raise ValueError("Input tensor must have (number of all items, model hidden size) shape")
        if item_embeddings.shape[1] != self._embedding_dim():
            raise ValueError("Input tensor second dimension doesn't match embedding dim")
        new = torch.cat([self._model.item_embeddings().cpu(), item_embeddings.detach().float().cpu()])
        self._set_new_item_table(new)
