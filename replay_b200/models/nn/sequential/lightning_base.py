"""What the legacy Lightning modules ``SasRec`` and ``Bert4Rec`` share around their engine-backed model ``_model``:
checkpoints under the ``_model.`` prefix, the optimizer and its factory, ``candidates_to_score`` and the schema's item
cardinality after the catalog grows."""
from __future__ import annotations

import torch

from ....compat import FusedOptimizerModule


class LegacyLightningModule(FusedOptimizerModule):
    def _attach(self, model, tensor_schema, optimizer_factory, lr_scheduler_factory, fused_optimizer: bool):
        """The constructor's common tail: ``model`` has ``core`` and ``item_count``."""
        self._model, self._schema = model, tensor_schema
        self._vocab_size = model.item_count
        self._candidates_to_score = None
        self._setup_optimizer(model.core, optimizer_factory, lr_scheduler_factory, fused_optimizer)

    def state_dict(self, *a, prefix="", **k):
        return {prefix + "_model." + key: v for key, v in self._model.state_dict().items()}

    def load_state_dict(self, sd, strict=True, assign=False):
        return self._model.load_state_dict({k[len("_model."):]: v for k, v in sd.items() if k.startswith("_model.")}, strict)

    def _fused_core(self):
        return self._model.core

    def configure_optimizers(self):
        opt = self._create_optimizer([self._model.core.flat])
        if self._lr_scheduler_factory is None:
            return opt
        return [opt], [self._lr_scheduler_factory.create(opt)]

    def _item_count_changed(self):
        """After the catalog grew: the module and the schema's item feature take the model's new item count."""
        self._vocab_size = self._model.item_count
        feats = self._schema.item_id_features
        feat = feats.item() if hasattr(feats, "item") else feats[self._schema.item_id_feature_name]
        feat._set_cardinality(self._vocab_size)

    @property
    def optimizer_factory(self):
        return self._optimizer_factory

    @optimizer_factory.setter
    def optimizer_factory(self, optimizer_factory):
        # sasrec/lightning.py:575-585, bert4rec/lightning.py:614-626: an isinstance check against OptimizerFactory
        if not hasattr(optimizer_factory, "create"):
            raise ValueError(f"Expected optimizer_factory of type OptimizerFactory, got {type(optimizer_factory)}")
        self._use_optimizer_factory(optimizer_factory, self._model.core)

    @property
    def candidates_to_score(self):
        return self._candidates_to_score

    @candidates_to_score.setter
    def candidates_to_score(self, candidates=None):
        total = self._model.item_count  # sasrec/lightning.py:594-610, bert4rec/lightning.py:613-628
        if isinstance(candidates, torch.Tensor) and candidates.dtype is torch.long:
            if not (0 < candidates.shape[0] <= total):
                raise ValueError(f"Expected candidates length to be between 1 and total_item_count={total}")
        elif candidates is not None:
            raise ValueError(f"Expected candidates to be of type torch.LongTensor or None, gpt {type(candidates)}")
        self._candidates_to_score = candidates
