"""Mirror of the legacy ``replay.models.nn.sequential.sasrec`` modules on the H100 engine:
``SasRecModel`` (model.py:15-197) and the Lightning module ``SasRec`` (lightning.py:22-658).  Legacy semantics: causal mask
only (pad keys are NOT masked), pad rows zeroed after the embedding and after every block, final LayerNorm eps 1e-8,
sequence length must equal ``max_len`` (predict batches are left-padded up to it, lightning.py:624-658)."""
from __future__ import annotations

import torch

from ....core import SasRecCore
from ....engine import EncoderConfig
from ....engine_tisasrec import TiConfig, TiSasRecCore
from ..loss import check_sce_params
from .lightning_base import LegacyLightningModule
from ....schema import item_feature_of


def _prepare_prediction_batch(schema, max_len: int, batch: dict) -> dict:
    """lightning.py:624-658: raise if longer than max_len, left-pad (ids with 0, mask with False) if shorter."""
    seq_len = batch["padding_mask"].shape[1]
    if seq_len > max_len:
        msg = ("The length of the submitted sequence must not exceed the maximum length of the sequence. "
               f"The length of the sequence is given {seq_len}, while the maximum length is {max_len}")
        raise ValueError(msg)
    if seq_len < max_len:
        pad = (max_len - seq_len, 0)
        batch = dict(batch)
        batch["feature_tensor"] = {k: torch.nn.functional.pad(v, pad, value=0) for k, v in batch["feature_tensor"].items()}
        batch["padding_mask"] = torch.nn.functional.pad(batch["padding_mask"], pad, value=0)
    return batch


class SasRecModel(torch.nn.Module):
    def __init__(self, schema, num_blocks: int = 2, num_heads: int = 1, hidden_size: int = 50, max_len: int = 200,
                 dropout: float = 0.2, ti_modification: bool = False, time_span: int = 256, device=None, seed: int = 0):
        super().__init__()
        name, card, pad, _ = item_feature_of(schema)
        self.schema = schema
        self.item_feature_name = name
        self.item_count = card
        self.padding_idx = card
        self.max_len = max_len
        self.hidden_size, self.num_blocks, self.num_heads, self.dropout = hidden_size, num_blocks, num_heads, dropout
        self.ti_modification, self.time_span = ti_modification, time_span
        if ti_modification:   # TiSASRec (model.py:532-800): the timestamps come with the batch's feature tensors
            assert schema.timestamp_feature_name
            self.timestamp_feature_name = schema.timestamp_feature_name
            cfg = TiConfig(n_items=card, d=hidden_size, n_heads=num_heads, n_blocks=num_blocks, max_len=max_len,
                           dropout=dropout, time_span=time_span)
            self.core = TiSasRecCore(cfg, item_feature=name, timestamp_feature=self.timestamp_feature_name, device=device,
                                     seed=seed)
        else:
            cfg = EncoderConfig(n_items=card, d=hidden_size, n_heads=num_heads, n_blocks=num_blocks, max_len=max_len,
                                dropout=dropout, variant="legacy")
            self.core = SasRecCore(cfg, item_feature=name, device=device, seed=seed)

    def feats(self, feature_tensor):
        """What the core stages next to the item ids: the timestamps of TiSASRec, nothing otherwise."""
        return feature_tensor if self.ti_modification else None

    def state_dict(self, *a, **k):
        return self.core.state_dict(*a, **k)

    def load_state_dict(self, sd, strict=True, assign=False):
        return self.core.load_state_dict(sd, strict=strict)

    def item_table_fp32(self) -> torch.Tensor:
        """fp32 master copy of the item table incl. the padding row, [item_count + 1, hidden]."""
        if self.core.engine is None and not self.core._pending_state:
            self.core.ensure_engine(1, self.max_len, with_grad=False)  # materialise the seeded initial weights
        return self.core.state_dict()["item_embedder.item_emb.weight"].detach().clone()

    def replace_item_table(self, table: torch.Tensor):
        """Swap in a table for a (larger) vocabulary, keeping every other weight (lightning.py:612-621): the core is rebuilt
        for the new catalog size (``SasRecCore.for_catalog``)."""
        sd = {k: v for k, v in self.state_dict().items() if not k.startswith("_head.")}
        sd["item_embedder.item_emb.weight"] = table.detach().to(torch.float32)
        new_count = table.shape[0] - 1
        self.core = self.core.for_catalog(new_count, sd)
        self.item_count = self.padding_idx = new_count

    def forward_step(self, feature_tensor, padding_mask):
        """Hidden states [B, L, d] (model.py:159-180)."""
        return self.core.hidden_states(feature_tensor[self.item_feature_name], padding_mask, self.feats(feature_tensor)).float()

    def get_query_embeddings(self, feature_tensor, padding_mask):
        return self.core.query_embeddings(feature_tensor[self.item_feature_name], padding_mask,
                                          self.feats(feature_tensor)).float()

    def get_logits(self, out_embeddings, item_ids=None):
        h = out_embeddings.reshape(-1, out_embeddings.shape[-1]).to(torch.bfloat16)
        h = self.core.engine.pad_features(h).contiguous()  # true hidden size -> the engine's feature slots
        tab = self.core.item_table(item_ids)
        out = torch.empty(h.shape[0], tab.shape[0], device=h.device, dtype=torch.float32)
        self.core.engine._gemm(h, tab, out, h.shape[0], tab.shape[0], self.core.cfg.dp, out_mode=2)
        return out.view(*out_embeddings.shape[:-1], tab.shape[0])

    def forward(self, feature_tensor, padding_mask):
        """All-position scores [B, L, |I|] (model.py:111-125) - materialised; use only for small problems."""
        return self.get_logits(self.forward_step(feature_tensor, padding_mask))

    def predict(self, feature_tensor, padding_mask, candidates_to_score=None):
        return self.core.logits(feature_tensor[self.item_feature_name], padding_mask, candidates_to_score,
                                self.feats(feature_tensor))


class SasRec(LegacyLightningModule):
    def __init__(self, tensor_schema, block_count: int = 2, head_count: int = 1, hidden_size: int = 50,
                 max_seq_len: int = 200, dropout_rate: float = 0.2, ti_modification: bool = False, time_span: int = 256,
                 loss_type: str = "CE", loss_sample_count=None, negative_sampling_strategy: str = "global_uniform",
                 negatives_sharing: bool = False, optimizer_factory=None, lr_scheduler_factory=None, sce_params=None,
                 fused_optimizer: bool = True, device=None):
        super().__init__()
        self.save_hyperparameters()
        if loss_type == "SCE":
            assert sce_params is not None, "You should define ``sce_params`` when using SCE loss function."  # lightning.py:105-106
            check_sce_params(sce_params)
        elif loss_type not in ("CE", "BCE") or (loss_type == "BCE" and loss_sample_count is None):
            raise NotImplementedError("Not supported loss_type")  # lightning.py:485 ; full-catalog BCE: no fused head
        if negative_sampling_strategy not in {"global_uniform", "inbatch"}:
            raise AssertionError("negative_sampling_strategy must be 'global_uniform' or 'inbatch'")
        if loss_sample_count is not None and negative_sampling_strategy != "global_uniform":
            raise NotImplementedError("only the 'global_uniform' negative sampling strategy has a fused head")
        self._attach(SasRecModel(tensor_schema, num_blocks=block_count, num_heads=head_count, hidden_size=hidden_size,
                                 max_len=max_seq_len, dropout=dropout_rate, ti_modification=ti_modification,
                                 time_span=time_span, device=device),
                     tensor_schema, optimizer_factory, lr_scheduler_factory, fused_optimizer)
        self._loss_type, self._loss_sample_count = loss_type, loss_sample_count
        self._negative_sampling_strategy, self._negatives_sharing = negative_sampling_strategy, negatives_sharing
        self._sce_params = sce_params if loss_type == "SCE" else None
        if self._sce_params is not None:
            p = self._sce_params
            if p.bucket_size_y > min(1024, self._vocab_size):
                raise ValueError(f"bucket_size_y = {p.bucket_size_y} exceeds min(1024, item count = {self._vocab_size}): "
                                 "the fused top-K of the SCE head selects at most 1024 items per bucket")
            self._model.core.set_loss("sce", n_buckets=p.n_buckets, bucket_size_x=p.bucket_size_x,
                                      bucket_size_y=p.bucket_size_y, mix_x=bool(p.mix_x))
        elif loss_sample_count is not None:
            self._model.core.set_loss("legacy_ce_sampled" if loss_type == "CE" else "legacy_bce_sampled")

    def _sample_negatives(self, ids):
        """lightning.py:394-472, 'global_uniform': one shared draw without replacement (negatives_sharing) or an independent
        uniform draw per position.  Drawn on the device with torch's generator (the reference draws inside the loss too)."""
        n = min(self._loss_sample_count, self._vocab_size)
        if self._negatives_sharing:
            return torch.multinomial(torch.ones(self._vocab_size, device=ids.device), n, replacement=False)
        return torch.randint(0, self._vocab_size, (*ids.shape, n), device=ids.device, dtype=torch.long)

    def training_step(self, batch: dict, batch_idx: int = 0):
        ids = batch["feature_tensor"][self._model.item_feature_name]
        args = (ids, batch["padding_mask"], batch["positive_labels"], batch["target_padding_mask"])
        core = self._model.core
        if self._sce_params is not None and self._sce_params.bucket_size_x > min(1024, ids.numel()):
            raise ValueError(f"bucket_size_x = {self._sce_params.bucket_size_x} exceeds min(1024, B * L = {ids.numel()}): "
                             "the fused top-K of the SCE head selects at most 1024 rows per bucket")
        neg = (self._sample_negatives(ids) if self._loss_sample_count is not None and self._sce_params is None else None)
        feats = self._model.feats(batch["feature_tensor"])
        if self.fused_optimizer:
            loss = core.fused_step(*args, lr=self._current_lr(), negatives=neg, feats=feats)  # all_reduce="auto": DDP inside
        else:
            loss = core.loss(*args, negatives=neg, feats=feats)
        self.log("train_loss", loss, on_step=True, on_epoch=True, prog_bar=True, sync_dist=True)
        return loss

    def forward(self, feature_tensors, padding_mask, candidates_to_score=None):
        return self._model.predict(feature_tensors, padding_mask, candidates_to_score)

    def predict_step(self, batch: dict, batch_idx: int = 0, dataloader_idx: int = 0):
        batch = _prepare_prediction_batch(self._schema, self._model.max_len, batch)
        return self._model.predict(batch["feature_tensor"], batch["padding_mask"], self._candidates_to_score)

    def predict(self, batch: dict, candidates_to_score=None):
        batch = _prepare_prediction_batch(self._schema, self._model.max_len, batch)
        return self._model.predict(batch["feature_tensor"], batch["padding_mask"], candidates_to_score)

    def predict_topk(self, batch: dict, k: int, seen_ids=None, candidates_to_score=None):
        """Fused predict (no [B, |I|] scores): (item ids [B,k] int64, scores [B,k])."""
        batch = _prepare_prediction_batch(self._schema, self._model.max_len, batch)
        ids = batch["feature_tensor"][self._model.item_feature_name]
        return self._model.core.predict_topk(ids, batch["padding_mask"], k, seen_ids, candidates_to_score,
                                             self._model.feats(batch["feature_tensor"]))

    def validation_step(self, batch: dict, batch_idx: int = 0, dataloader_idx: int = 0):
        """lightning.py:196-220: scores of the validation batch (same computation as predict)."""
        batch = _prepare_prediction_batch(self._schema, self._model.max_len, batch)
        return self._model.predict(batch["feature_tensor"], batch["padding_mask"])

    # ---- vocabulary growth (lightning.py:493-566, 612-621)
    def _set_new_item_table(self, table: torch.Tensor):
        self._model.replace_item_table(table)
        self._item_count_changed()

    def set_item_embeddings_by_size(self, new_vocab_size: int):
        """Keep the fitted item embeddings and add xavier-normal rows for the new items."""
        old = self._model.item_table_fp32()
        old_vocab, hidden = old.shape[0] - 1, self._model.hidden_size
        if new_vocab_size <= old_vocab:
            raise ValueError("New vocabulary size must be greater then already fitted")
        new = torch.empty(new_vocab_size + 1, hidden)
        torch.nn.init.xavier_normal_(new)
        new[:old_vocab] = old[:-1].cpu()
        self._set_new_item_table(new)

    def set_item_embeddings_by_tensor(self, all_item_embeddings: torch.Tensor):
        """Replace the whole item table (possibly with more items); the padding row is zero."""
        if all_item_embeddings.dim() != 2:
            raise ValueError("Input tensor must have (number of all items, model hidden size) shape")
        old_vocab, hidden = self._model.item_count, self._model.hidden_size
        if all_item_embeddings.shape[0] < old_vocab:
            raise ValueError("New vocabulary size can't be less then already fitted")
        if all_item_embeddings.shape[1] != hidden:
            raise ValueError("Input tensor second dimension doesn't match model hidden size")
        new = torch.zeros(all_item_embeddings.shape[0] + 1, hidden)
        new[:-1] = all_item_embeddings.detach().float().cpu()
        self._set_new_item_table(new)

    def append_item_embeddings(self, item_embeddings: torch.Tensor):
        """Append rows for new items only; the padding row is zero."""
        if item_embeddings.dim() != 2:
            raise ValueError("Input tensor must have (number of new items, model hidden size) shape")
        if item_embeddings.shape[1] != self._model.hidden_size:
            raise ValueError("Input tensor second dimension doesn't match model hidden size")
        old = self._model.item_table_fp32()
        old_vocab = old.shape[0] - 1
        new = torch.zeros(old_vocab + item_embeddings.shape[0] + 1, self._model.hidden_size)
        new[:old_vocab] = old[:-1].cpu()
        new[old_vocab:-1] = item_embeddings.detach().float().cpu()
        self._set_new_item_table(new)

    def get_all_embeddings(self):
        """Copies, with the reference's keys (sasrec/model.py:374-381)."""
        sd = self._model.state_dict() if (self._model.core.engine is not None or self._model.core._pending_state) else None
        if sd is None:
            self._model.item_table_fp32()
            sd = self._model.state_dict()
        if self._model.ti_modification:   # TiSasRecEmbeddings.get_all_embeddings (model.py:633-646)
            return {"item_embedding": sd["item_embedder.item_emb.weight"][:-1].detach().clone(),
                    **{k: sd[f"item_embedder.{k}{'.pe' if k.startswith('abs') else ''}.weight"].detach().clone()
                       for k in ("abs_pos_k_emb", "abs_pos_v_emb", "time_matrix_k_emb", "time_matrix_v_emb")}}
        return {"item_embedding": sd["item_embedder.item_emb.weight"][:-1].detach().clone(),
                "positional_embedding": sd["item_embedder.pos_emb.pe.weight"].detach().clone()}
