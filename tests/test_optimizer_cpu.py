"""The optimizer options of the fused step without a GPU: the factory's surface, the configuration the modules build from a
factory (the reference's FatOptimizerFactory fields included), and the C entry point's argument checks."""
import ctypes

import pytest
import torch

from replay_b200.engine import OptimizerConfig
from replay_b200.schema import TensorFeatureInfo, TensorSchema


class _FatFactory:
    """The fields of the reference's FatOptimizerFactory (models/nn/optimizer_utils/optimizer_factory.py)."""

    def __init__(self, optimizer="adam", learning_rate=0.001, weight_decay=0.0, sgd_momentum=0.0, betas=(0.9, 0.98)):
        self.optimizer, self.learning_rate, self.weight_decay = optimizer, learning_rate, weight_decay
        self.sgd_momentum, self.betas = sgd_momentum, betas

    def create(self, params):
        return torch.optim.SGD(params, lr=self.learning_rate)


def _schema():
    return TensorSchema(TensorFeatureInfo("item_id", 40, 40, 64))


def _module(kind, factory):
    if kind == "sasrec":
        from replay_b200.models.nn.sequential import SasRec

        return SasRec(_schema(), hidden_size=64, head_count=1, max_seq_len=8, optimizer_factory=factory, device="cpu")
    if kind == "bert4rec":
        from replay_b200.models.nn.sequential import Bert4Rec

        return Bert4Rec(_schema(), hidden_size=64, head_count=1, max_seq_len=8, optimizer_factory=factory, device="cpu")
    from replay_b200.nn.lightning import LightningModule
    from replay_b200.nn.sequential import SasRec

    return LightningModule(SasRec.from_params(_schema(), embedding_dim=64, num_heads=1, device="cpu"),
                           optimizer_factory=factory)


def _core(m):
    return m._model.core if hasattr(m, "_model") else m.model.core


def test_factory_creates_the_reference_optimizers():
    from replay_b200.nn.lightning import OptimizerFactory

    p = [torch.nn.Parameter(torch.zeros(3))]
    f = OptimizerFactory()
    assert (f.optimizer, f.learning_rate, f.weight_decay, f.sgd_momentum, f.betas) == ("adam", 1e-3, 0.0, 0.0, (0.9, 0.98))
    a = OptimizerFactory(weight_decay=1e-2, betas=(0.8, 0.9)).create(p)
    assert type(a) is torch.optim.Adam
    assert {k: a.defaults[k] for k in ("lr", "weight_decay", "betas")} == dict(lr=1e-3, weight_decay=1e-2, betas=(0.8, 0.9))
    s = OptimizerFactory("sgd", learning_rate=0.1, weight_decay=1e-4, sgd_momentum=0.9).create(p)
    assert type(s) is torch.optim.SGD
    assert {k: s.defaults[k] for k in ("lr", "weight_decay", "momentum", "dampening", "nesterov")} == dict(
        lr=0.1, weight_decay=1e-4, momentum=0.9, dampening=0, nesterov=False)
    bad = OptimizerFactory("rmsprop")   # the constructor accepts any name, as the reference's does
    with pytest.raises(ValueError, match="Unexpected optimizer"):
        bad.create(p)


@pytest.mark.parametrize("kind", ["sasrec", "bert4rec", "new_path"])
def test_modules_take_every_factory_field(kind):
    from replay_b200.nn.lightning import OptimizerFactory

    f = _FatFactory("sgd", learning_rate=0.05, weight_decay=1e-4, sgd_momentum=0.9)
    m = _module(kind, f)
    assert _core(m).optimizer == OptimizerConfig("sgd", (0.9, 0.98), 1e-8, 1e-4, 0.9)
    assert m._lr == 0.05
    m = _module(kind, OptimizerFactory(weight_decay=1e-2, betas=[0.8, 0.9]))
    assert _core(m).optimizer == OptimizerConfig("adam", (0.8, 0.9), 1e-8, 1e-2, 0.0)
    assert _core(m).adam_betas == (0.8, 0.9)

    class Bare:   # no fields at all: the reference's defaults
        def create(self, params):
            return torch.optim.Adam(params)

    assert _core(_module(kind, Bare())).optimizer == OptimizerConfig()
    m = _module(kind, _FatFactory("rmsprop"))   # accepted here, refused by the step
    with pytest.raises(ValueError, match="Unexpected optimizer"):
        _core(m).optimizer.validate()


def test_legacy_setter_replaces_the_configuration_and_growth_keeps_it():
    m = _module("sasrec", None)
    assert _core(m).optimizer == OptimizerConfig()
    m.optimizer_factory = _FatFactory("sgd", sgd_momentum=0.5)
    assert _core(m).optimizer.kind == "sgd" and _core(m).optimizer.momentum == 0.5
    core = _core(m)
    core.adam_betas = (0.7, 0.8)   # the betas alone, as before
    assert core.optimizer == OptimizerConfig("sgd", (0.7, 0.8), 1e-8, 0.0, 0.5)


def test_hooks_without_an_engine_leave_the_checkpoint_alone():
    m = _module("sasrec", _FatFactory("sgd", sgd_momentum=0.9))
    ckpt = {"optimizer_states": [{"state": {}, "param_groups": []}]}
    m.on_save_checkpoint(ckpt)
    assert ckpt == {"optimizer_states": [{"state": {}, "param_groups": []}]}
    m.on_load_checkpoint({"optimizer_states": [{"state": {0: {"momentum_buffer": torch.ones(3)}}, "param_groups": []}]})
    assert torch.equal(_core(m)._pending_opt_state["momentum_buffer"], torch.ones(3))


def test_optimizer_step_argument_checks():
    from replay_b200._lib import lib

    L = lib()
    EINVAL = -1
    buf = ctypes.create_string_buffer(64)
    p = ctypes.cast(buf, ctypes.c_void_p)
    args = lambda kind, s0, s1, n=4: (kind, p, p, s0, s1, None, n, p, p, 0.9, 0.98, 1e-8, 0.0, 0.9, 1.0, None, 1, None)  # noqa: E731
    assert L.rp_optimizer_step(*args(0, None, p)) == EINVAL        # Adam needs both moments
    assert L.rp_optimizer_step(*args(0, p, None)) == EINVAL
    assert L.rp_optimizer_step(*args(1, None, None)) == EINVAL     # SGD with momentum needs its buffer
    assert L.rp_optimizer_step(*args(2, p, p)) == EINVAL           # no such kind
    assert L.rp_optimizer_step(*args(1, p, None, n=6)) == EINVAL   # n % 4
    assert L.rp_optimizer_step(0, None, p, p, p, None, 4, p, p, 0.9, 0.98, 1e-8, 0.0, 0.0, 1.0, None, 1, None) == EINVAL


def test_train_start_releases_the_unused_torch_optimizer_state_in_fused_mode():
    for fused, kept in ((True, 0), (False, 1)):
        m = _module("sasrec", None) if fused else _module_unfused()
        p = torch.nn.Parameter(torch.zeros(3))
        opt = torch.optim.Adam([p])
        opt.state[p] = {"exp_avg": torch.ones(3)}
        m.optimizers = lambda: opt
        m.on_train_start()
        assert len(opt.state) == kept


def _module_unfused():
    from replay_b200.models.nn.sequential import SasRec

    return SasRec(_schema(), hidden_size=64, head_count=1, max_seq_len=8, fused_optimizer=False, device="cpu")
