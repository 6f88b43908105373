from __future__ import annotations

import inspect

import torch

from ...compat import FusedOptimizerModule


class OptimizerFactory:
    """replay/nn/lightning/optimizer.py:24-60 - Adam(lr 1e-3, betas (0.9, 0.98)) by default, or SGD.  The fused step runs
    the same optimizer (``optimizer``, ``learning_rate``, ``weight_decay``, ``sgd_momentum``, ``betas``) on the GPU."""

    def __init__(self, optimizer: str = "adam", learning_rate: float = 0.001, weight_decay: float = 0.0,
                 sgd_momentum: float = 0.0, betas: tuple = (0.9, 0.98)):
        self.optimizer = optimizer
        self.learning_rate = learning_rate
        self.weight_decay = weight_decay
        self.sgd_momentum = sgd_momentum
        self.betas = betas

    def create(self, parameters):
        if self.optimizer == "adam":
            return torch.optim.Adam(parameters, lr=self.learning_rate, weight_decay=self.weight_decay, betas=self.betas)
        if self.optimizer == "sgd":
            return torch.optim.SGD(parameters, lr=self.learning_rate, weight_decay=self.weight_decay,
                                   momentum=self.sgd_momentum)
        raise ValueError("Unexpected optimizer")


class LazyInferenceOutput(dict):
    """``InferenceOutput`` (replay/nn/output.py) whose ``logits`` [B, |I|] and ``hidden_states`` are computed on first access.
    ``predict_step`` / ``validation_step`` return it, so a callback that runs the fused score + seen-filter + top-K head
    (``TopItemsCallbackBase``, ``ComputeMetricsCallback``) never makes the body run twice nor the [B, |I|] fp32 scores get
    written (8 GB per 4096 users at 500 K items); a callback that does read ``outputs["logits"]`` gets the reference's tensor."""

    def __init__(self, compute):
        super().__init__()
        self._compute = compute

    def _fill(self):
        if self._compute is not None:
            self._inner, self._compute = self._compute(), None
            super().update(self._inner)

    def __getitem__(self, k):
        self._fill()
        if not super().__contains__(k):  # the model's own output may compute entries lazily as well (hidden_states)
            super().__setitem__(k, self._inner[k])
        return super().__getitem__(k)

    def __contains__(self, k):
        return k in ("logits", "hidden_states") or super().__contains__(k)

    def get(self, k, default=None):
        self._fill()
        return super().get(k, default)

    def keys(self):
        self._fill()
        return super().keys()

    def items(self):
        self._fill()
        return super().items()

    def values(self):
        self._fill()
        return super().values()

    @property
    def materialised(self) -> bool:
        return self._compute is None


class LightningModule(FusedOptimizerModule):
    """replay/nn/lightning/module.py:13-123.  ``fused_optimizer=True`` (default) runs forward+backward+the factory's
    optimizer inside the CUDA engine (manual optimisation; under ``torch.distributed`` the flat gradient is all-reduced
    before the optimizer step, which is what Lightning's DDP does for the reference); with False the loss goes through
    autograd and the optimizer from ``optimizer_factory``.  In fused mode the learning rate of every step is read from the
    optimizer Lightning configured (so an lr scheduler takes effect), the rest comes from the factory."""

    def __init__(self, model, optimizer_factory: OptimizerFactory | None = None, lr_scheduler_factory=None,
                 fused_optimizer: bool = True):
        super().__init__()
        self.save_hyperparameters(ignore=["model"])
        self.model = model
        self._candidates_to_score = None
        self._setup_optimizer(getattr(model, "core", None), optimizer_factory or OptimizerFactory(), lr_scheduler_factory,
                              fused_optimizer)
        self._sig = set(inspect.signature(model.forward).parameters)

    def _fused_core(self):
        return getattr(self.model, "core", None)

    def forward(self, batch: dict):
        if "candidates_to_score" in self._sig and self._candidates_to_score is not None and not self.model.training:
            batch = {**batch, "candidates_to_score": self._candidates_to_score}
        return self.model(**{k: v for k, v in batch.items() if k in self._sig})

    # ---- checkpoints: the reference's keys are ``model.`` + the model's own (SURVEY Appendix B); torch's recursive loader
    # would bypass the engine-backed model's ``load_state_dict`` and find no tensors to load into
    def state_dict(self, *args, destination=None, prefix="", keep_vars=False):
        if not hasattr(self.model, "core"):
            return super().state_dict(*args, destination=destination, prefix=prefix, keep_vars=keep_vars)
        out = destination if destination is not None else {}
        for k, v in self.model.state_dict().items():
            out[prefix + "model." + k] = v
        return out

    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):
        if not hasattr(self.model, "core"):
            return super().load_state_dict(state_dict, strict=strict, assign=assign)
        inner = {k[len("model."):]: v for k, v in state_dict.items() if k.startswith("model.")}
        res = self.model.load_state_dict(inner, strict=strict)
        unexpected = sorted(k for k in state_dict if not k.startswith("model."))
        if strict and unexpected:
            raise RuntimeError(f"unexpected keys in state_dict: {unexpected[:5]}")
        missing = ["model." + k for k in getattr(res, "missing_keys", [])]
        return torch.nn.modules.module._IncompatibleKeys(missing, unexpected)

    def training_step(self, batch: dict, batch_idx: int = 0):
        if self.fused_optimizer and hasattr(self.model, "core"):
            core = self.model.core
            lab, tm = batch["positive_labels"], batch["target_padding_mask"]
            if hasattr(self.model, "check_positives"):   # [B, L, P] targets reach the heads that train on them
                lab, tm = self.model.check_positives(lab, tm)
            elif lab.dim() == 3:
                if lab.size(-1) != 1:
                    raise NotImplementedError(f"The case of multi-positive labels is not supported in {type(self.model).__name__}")
                lab, tm = lab[..., 0], (tm[..., 0] if tm.dim() == 3 else tm)
            spec = getattr(self.model, "loss", None)
            neg = batch.get("negative_labels") if getattr(spec, "needs_negatives", False) else None
            if getattr(spec, "needs_negatives", False) and neg is None:
                raise ValueError(f"{type(spec).__name__} needs `negative_labels` in the batch")
            lr = self._current_lr()
            rw = spec.row_weights(batch["feature_tensors"], tm) if hasattr(spec, "row_weights") else None
            side = {"feats": batch["feature_tensors"]} if getattr(core.cfg, "features", ()) else {}
            loss = core.fused_step(batch["feature_tensors"][core.item_feature], batch["padding_mask"], lab, tm,
                                   lr=lr, negatives=neg, row_weights=rw, **side)  # all_reduce="auto": DDP exchange inside
            self.log("learning_rate", lr, on_step=True, on_epoch=True, prog_bar=True, sync_dist=True)
        else:
            loss = self(batch)["loss"]
        self.log("train_loss", loss, on_step=True, on_epoch=True, prog_bar=True, sync_dist=True)
        return loss

    def _inference(self, batch: dict):
        self.model.eval()
        if hasattr(self.model, "core"):
            return LazyInferenceOutput(lambda: self(batch))
        return self(batch)

    def predict_step(self, batch: dict, batch_idx: int = 0, dataloader_idx: int = 0):
        return self._inference(batch)

    def validation_step(self, batch: dict, batch_idx: int = 0, dataloader_idx: int = 0):
        return self._inference(batch)

    def test_step(self, batch: dict, batch_idx: int = 0, dataloader_idx: int = 0):
        return self._inference(batch)

    def configure_optimizers(self):
        opt = self._optimizer_factory.create(self.model.parameters())
        if self._lr_scheduler_factory is None:
            return opt
        return [opt], [self._lr_scheduler_factory.create(opt)]

    @property
    def candidates_to_score(self):
        return self._candidates_to_score

    @candidates_to_score.setter
    def candidates_to_score(self, candidates):
        if candidates is not None:
            if not (isinstance(candidates, torch.Tensor) and candidates.dtype == torch.long and candidates.dim() == 1):
                raise ValueError("candidates_to_score must be a 1-D torch.LongTensor")
            if candidates.unique().numel() != candidates.numel():
                raise ValueError("candidates_to_score must contain unique item ids")  # module.py:118-123
        self._candidates_to_score = candidates
