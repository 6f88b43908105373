from __future__ import annotations

import torch

from ....compat import CallbackBase
from .postprocessors import RemoveSeenItems


def _batch_device(batch):
    """SasRec batches carry ``padding_mask``, Bert4Rec batches ``pad_mask``."""
    return (batch["padding_mask"] if "padding_mask" in batch else batch["pad_mask"]).device


class BasePredictionCallback(CallbackBase):
    """replay/models/nn/sequential/callbacks/prediction_callbacks.py:30-120.  With a ``replay_b200`` module and only
    ``RemoveSeenItems`` postprocessors and ``top_k <= ops.MAX_FUSED_K`` the scores / filter / top-K run fused on the device."""

    def __init__(self, top_k: int, query_column: str, item_column: str, rating_column: str = "rating", postprocessors=None):
        self.query_column, self.item_column, self.rating_column = query_column, item_column, rating_column
        self._top_k = top_k
        self._postprocessors = postprocessors or []
        self._query_batches, self._item_batches, self._item_scores = [], [], []

    def on_predict_epoch_start(self, trainer, pl_module):
        self._query_batches.clear(); self._item_batches.clear(); self._item_scores.clear()
        for p in self._postprocessors:
            p.candidates = pl_module.candidates_to_score

    def on_predict_batch_end(self, trainer, pl_module, outputs, batch, batch_idx, dataloader_idx=0):
        from ....ops import MAX_FUSED_K

        query_ids = batch["query_id"]
        fusable = (hasattr(pl_module, "predict_topk") and self._top_k <= MAX_FUSED_K
                   and all(isinstance(p, RemoveSeenItems) for p in self._postprocessors))
        if fusable:
            seen = self._postprocessors[0].seen_tensor(query_ids, _batch_device(batch)) if self._postprocessors else None
            ids, scores = pl_module.predict_topk(batch, self._top_k, seen, pl_module.candidates_to_score)
        else:
            scores_full = outputs
            for p in self._postprocessors:
                query_ids, scores_full = p.on_prediction(query_ids, scores_full)
            scores, ids = torch.topk(scores_full, k=self._top_k, dim=1)
        self._query_batches.append(query_ids)
        self._item_batches.append(ids)
        self._item_scores.append(scores)

    def get_result(self):
        return self._ids_to_result(torch.cat(self._query_batches), torch.cat(self._item_batches), torch.cat(self._item_scores))

    def _ids_to_result(self, q, i, s):
        raise NotImplementedError


class TorchPredictionCallback(BasePredictionCallback):
    def _ids_to_result(self, q, i, s):
        return q.flatten().cpu().long(), i.cpu().long(), s.cpu()


def _exploded(q, i, s):
    k = i.shape[1]
    return q.flatten().cpu().numpy().repeat(k), i.cpu().numpy().reshape(-1), s.cpu().numpy().reshape(-1)


class PandasPredictionCallback(BasePredictionCallback):
    """prediction_callbacks.py:130-152"""

    def _ids_to_result(self, q, i, s):
        import pandas as pd

        qq, ii, ss = _exploded(q, i, s)
        return pd.DataFrame({self.query_column: qq, self.item_column: ii, self.rating_column: ss})


class PolarsPredictionCallback(BasePredictionCallback):
    """prediction_callbacks.py:155-177"""

    def _ids_to_result(self, q, i, s):
        import polars as pl

        qq, ii, ss = _exploded(q, i, s)
        return pl.DataFrame({self.query_column: qq, self.item_column: ii, self.rating_column: ss})


class SparkPredictionCallback(BasePredictionCallback):
    """prediction_callbacks.py:180-240"""

    def __init__(self, top_k: int, query_column: str, item_column: str, rating_column: str, spark_session, postprocessors=None):
        super().__init__(top_k, query_column, item_column, rating_column, postprocessors)
        self.spark_session = spark_session

    def _ids_to_result(self, q, i, s):
        from pyspark.sql.types import DoubleType, IntegerType, StructType

        schema = (StructType().add(self.query_column, IntegerType(), False).add(self.item_column, IntegerType(), False)
                  .add(self.rating_column, DoubleType(), False))
        qq, ii, ss = _exploded(q, i, s)
        return self.spark_session.createDataFrame(data=list(zip(qq.tolist(), ii.tolist(), ss.astype("float64").tolist())),
                                                  schema=schema)


class QueryEmbeddingsPredictionCallback(CallbackBase):
    """prediction_callbacks.py:282-326: the last hidden state of every query, through the module's ``_model.get_query_embeddings``
    (SASRec: features + padding mask, BERT4Rec: + tokens mask)."""

    def __init__(self):
        self._embeddings_per_batch: list[torch.Tensor] = []

    def on_predict_epoch_start(self, trainer, pl_module):
        self._embeddings_per_batch.clear()

    def on_predict_batch_end(self, trainer, pl_module, outputs, batch, batch_idx, dataloader_idx=0):
        import inspect

        fn = pl_module._model.get_query_embeddings
        names = list(inspect.signature(fn).parameters)
        if hasattr(pl_module, "_prepare_batch"):
            batch = pl_module._prepare_batch(batch)
        alias = {"feature_tensor": ("feature_tensor", "feature_tensors", "features", "inputs"), "inputs": ("inputs", "features"),
                 "padding_mask": ("padding_mask", "pad_mask"), "pad_mask": ("pad_mask", "padding_mask"),
                 "token_mask": ("token_mask", "tokens_mask"), "tokens_mask": ("tokens_mask", "token_mask")}
        kwargs = {}
        for n in names:
            for key in alias.get(n, (n,)):
                if key in batch:
                    kwargs[n] = batch[key]
                    break
        self._embeddings_per_batch.append(fn(**kwargs))

    def get_result(self):
        return torch.cat(self._embeddings_per_batch)


class ValidationMetricsCallback(CallbackBase):
    """callbacks/validation_callback.py:37-200: ranking metrics of the validation / test stages of the LEGACY modules (the
    batch carries ``query_id``, ``ground_truth`` and - for novelty / coverage - ``train``; postprocessors have the legacy
    ``on_validation(query_ids, scores, ground_truth)`` signature).  With a ``replay_b200`` module and only ``RemoveSeenItems``
    postprocessors the top-K comes from the fused kernel instead of the dense scores."""

    def __init__(self, metrics=None, ks=None, postprocessors=None, item_count=None):
        from ....nn.lightning.metrics import DEFAULT_KS, DEFAULT_METRICS

        self._metrics = tuple(metrics or DEFAULT_METRICS)
        self._ks = tuple(ks or DEFAULT_KS)
        self._item_count = item_count
        self._postprocessors = postprocessors or []
        self._metrics_builders = []
        self.last_metrics: dict = {}

    def _start(self, trainer, attr):
        from ....nn.lightning.metrics import RankingMetrics

        sizes = getattr(trainer, attr, None) if trainer is not None else None
        n = len(sizes) if isinstance(sizes, (list, tuple)) else 1
        self._metrics_builders = [RankingMetrics(self._metrics, self._ks, self._item_count) for _ in range(max(1, n))]

    def on_validation_epoch_start(self, trainer, pl_module):
        self._start(trainer, "num_val_batches")

    def on_test_epoch_start(self, trainer, pl_module):
        self._start(trainer, "num_test_batches")

    def _batch_end(self, pl_module, outputs, batch, dataloader_idx):
        from ....ops import MAX_FUSED_K

        if not self._metrics_builders:
            self._start(None, "")
        b = self._metrics_builders[dataloader_idx]
        query_ids, gt = batch["query_id"], batch["ground_truth"]
        if (hasattr(pl_module, "predict_topk") and b.max_k <= MAX_FUSED_K
                and all(isinstance(p, RemoveSeenItems) for p in self._postprocessors)):
            seen = self._postprocessors[0].seen_tensor(query_ids, _batch_device(batch)) if self._postprocessors else None
            ids, _ = pl_module.predict_topk(batch, b.max_k, seen)
        else:
            scores = outputs
            for p in self._postprocessors:
                query_ids, scores, gt = p.on_validation(query_ids, scores, gt)
            ids = torch.topk(scores, k=b.max_k, dim=1).indices
        b.add_prediction(ids, gt, batch.get("train"))

    def on_validation_batch_end(self, trainer, pl_module, outputs, batch, batch_idx, dataloader_idx=0):
        self._batch_end(pl_module, outputs, batch, dataloader_idx)

    def on_test_batch_end(self, trainer, pl_module, outputs, batch, batch_idx, dataloader_idx=0):
        self._batch_end(pl_module, outputs, batch, dataloader_idx)

    def _epoch_end(self, trainer, pl_module):
        m = {}
        for i, b in enumerate(self._metrics_builders):
            if b._n == 0:
                continue
            suffix = "" if len(self._metrics_builders) == 1 else f"/dataloader_idx_{i}"
            m.update({k + suffix: v for k, v in b.get_metrics().items()})
        if hasattr(pl_module, "log_dict"):
            pl_module.log_dict(m, on_epoch=True, sync_dist=True)
        self.last_metrics = m
        return m

    def on_validation_epoch_end(self, trainer, pl_module):
        return self._epoch_end(trainer, pl_module)

    def on_test_epoch_end(self, trainer, pl_module):
        return self._epoch_end(trainer, pl_module)
