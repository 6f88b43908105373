"""Lightning compatibility: subclass ``lightning.LightningModule`` / ``Callback`` when Lightning is importable, otherwise
minimal stand-ins exposing the hooks the reference's modules use (training_step / predict_step / configure_optimizers /
log / save_hyperparameters), so the mirrors work - and are testable - where Lightning is not installed (SURVEY.md §7.2)."""
from __future__ import annotations

import torch

try:  # pragma: no cover - depends on the environment
    import lightning as _L

    LightningModuleBase = _L.LightningModule
    CallbackBase = _L.Callback
    HAVE_LIGHTNING = True
except Exception:  # noqa: BLE001
    HAVE_LIGHTNING = False

    class _HParams(dict):
        __getattr__ = dict.get

    class LightningModuleBase(torch.nn.Module):
        def __init__(self, *a, **k):
            super().__init__()
            self._hparams = _HParams()
            self.trainer = None
            self.automatic_optimization = True
            self.logged = {}

        def save_hyperparameters(self, *names, ignore=None, **k):
            import inspect

            frame = inspect.currentframe().f_back
            loc = frame.f_locals
            ignore = set(ignore or [])
            for key, val in loc.items():
                if key in ("self", "__class__") or key in ignore:
                    continue
                self._hparams[key] = val

        @property
        def hparams(self):
            return self._hparams

        def log(self, name, value, *a, **k):
            self.logged[name] = value

        def log_dict(self, d, *a, **k):
            self.logged.update(d)

    class CallbackBase:
        pass


class FusedOptimizerModule(LightningModuleBase):
    """Optimizer plumbing of the engine-backed Lightning modules.  With ``fused_optimizer=True`` the CUDA engine runs the
    factory's Adam or SGD itself under manual optimisation: each step reads its learning rate from the optimizer Lightning
    configured, so an lr scheduler takes effect, and the schedulers are stepped here at epoch end, which Lightning leaves to
    the module under manual optimisation (the default interval of the reference's factories,
    replay/nn/lightning/scheduler.py).  Checkpoints carry the engine's optimizer state in the torch optimizer's format."""

    def _setup_optimizer(self, core, optimizer_factory, lr_scheduler_factory, fused_optimizer: bool):
        self._lr_scheduler_factory = lr_scheduler_factory
        self.fused_optimizer = fused_optimizer
        if fused_optimizer:
            self.automatic_optimization = False
        self._use_optimizer_factory(optimizer_factory, core)

    def _use_optimizer_factory(self, optimizer_factory, core):
        """``_lr``, the learning rate of a step without a trainer, is the factory's (1e-3 without one); its ``optimizer``,
        ``weight_decay``, ``sgd_momentum`` and ``betas`` become ``core``'s fused optimizer, each at the reference's default
        where the factory has none (optimizer_factory.py:56-87 / nn/lightning/optimizer.py:24-60)."""
        from .engine import OptimizerConfig

        self._optimizer_factory = optimizer_factory
        self._lr = getattr(optimizer_factory, "learning_rate", 1e-3)
        if core is not None:
            f = optimizer_factory
            core.optimizer = OptimizerConfig(kind=getattr(f, "optimizer", "adam"), betas=getattr(f, "betas", (0.9, 0.98)),
                                             weight_decay=getattr(f, "weight_decay", 0.0),
                                             momentum=getattr(f, "sgd_momentum", 0.0))

    def _fused_core(self):
        """The engine-backed core whose optimizer runs fused, or None."""
        raise NotImplementedError

    def _create_optimizer(self, params):
        """The torch optimizer of ``params``: the factory's, torch.optim.Adam(lr 1e-3, betas (0.9, 0.98)) without one."""
        if self._optimizer_factory is None:
            return torch.optim.Adam(params, lr=1e-3, betas=(0.9, 0.98))   # optimizer_factory.py:56-63
        return self._optimizer_factory.create(params)

    def on_save_checkpoint(self, checkpoint: dict):
        """Fused mode: ``optimizer_states[0]`` becomes the engine's state as the torch optimizer built by the factory for
        ``core.flat`` would save it, so the checkpoint resumes in either mode."""
        core = self._fused_core() if self.fused_optimizer else None
        if core is None or core.flat is None:
            return
        opt = self._create_optimizer([core.flat])
        opt.param_groups[0]["lr"] = self._current_lr()
        eng = core.engine
        state = eng.optimizer_state(core.optimizer) if eng.with_grad else (core._pending_opt_state or {})
        if state:
            opt.state[core.flat] = state
        states = checkpoint.setdefault("optimizer_states", [])
        states[:1] = [opt.state_dict()]

    def on_load_checkpoint(self, checkpoint: dict):
        """Fused mode: the engine takes its optimizer state from ``optimizer_states[0]`` (see ``on_save_checkpoint``)."""
        core = self._fused_core() if self.fused_optimizer else None
        states = checkpoint.get("optimizer_states")
        if core is not None and states:
            core.load_optimizer_state(states[0]["state"].get(0, {}))

    def on_train_start(self):
        """Fused mode: the optimizer Lightning configured never steps, so the state a resumed checkpoint loaded into it is
        released (the engine holds its own copy)."""
        if not self.fused_optimizer:
            return
        try:
            opts = self.optimizers()
        except Exception:  # noqa: BLE001 - no trainer attached
            return
        for o in (opts if isinstance(opts, (list, tuple)) else [opts]):
            getattr(o, "optimizer", o).state.clear()

    def _current_lr(self) -> float:
        """The learning rate Lightning's (possibly scheduled) optimizer holds right now; ``_lr`` without a trainer."""
        try:
            opt = self.optimizers()
        except Exception:  # noqa: BLE001 - no trainer attached (direct use, tests)
            opt = None
        if isinstance(opt, (list, tuple)):
            opt = opt[0] if opt else None
        if opt is not None and getattr(opt, "param_groups", None):
            return float(opt.param_groups[0]["lr"])
        return float(self._lr)

    def on_train_epoch_end(self):
        if self.fused_optimizer and self._lr_scheduler_factory is not None:
            try:
                sch = self.lr_schedulers()
            except Exception:  # noqa: BLE001 - no trainer attached
                sch = None
            for s_ in (sch if isinstance(sch, (list, tuple)) else [sch]):
                if s_ is not None:
                    s_.step()
