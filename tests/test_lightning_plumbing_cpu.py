"""The optimizer plumbing the engine-backed Lightning modules share (the learning rate of a fused step, the epoch-end
scheduler step, the legacy optimizer factory) and the core rebuild of catalog growth, without a GPU.  The modules are built
with ``device="cpu"``; a loaded checkpoint stays the core's pending state, so catalog growth needs no engine."""
import pytest
import torch

from replay_b200.schema import TensorFeatureInfo, TensorSchema

MODULES = ["sasrec", "bert4rec", "new_path"]


class _Factory:
    def __init__(self, learning_rate=3e-4, betas=(0.8, 0.9)):
        self.learning_rate, self.betas = learning_rate, betas

    def create(self, params):
        return torch.optim.Adam(params, lr=self.learning_rate, betas=self.betas)


class _BareFactory:   # a factory without ``learning_rate`` / ``betas``
    def create(self, params):
        return torch.optim.Adam(params)


class _Scheduler:
    def __init__(self):
        self.steps = 0

    def step(self):
        self.steps += 1


def _schema(n_items=40, d=64, ts=False):
    return TensorSchema(TensorFeatureInfo("item_id", n_items, n_items, d), timestamp_feature_name="timestamp" if ts else None)


def _module(kind, **kw):
    if kind in ("sasrec", "tisasrec"):
        from replay_b200.models.nn.sequential import SasRec

        return SasRec(_schema(ts=kind == "tisasrec"), hidden_size=64, head_count=1, max_seq_len=8,
                      ti_modification=kind == "tisasrec", device="cpu", **kw)
    if kind == "bert4rec":
        from replay_b200.models.nn.sequential import Bert4Rec

        return Bert4Rec(_schema(), hidden_size=64, head_count=1, max_seq_len=8, device="cpu", **kw)
    from replay_b200.nn.lightning import LightningModule
    from replay_b200.nn.sequential import SasRec

    return LightningModule(SasRec.from_params(_schema(), embedding_dim=64, num_heads=1, device="cpu"), **kw)


@pytest.mark.parametrize("kind", MODULES)
def test_step_lr_is_the_trainers_optimizers_else_the_factorys(kind):
    assert _module(kind)._current_lr() == 1e-3
    assert _module(kind, optimizer_factory=_BareFactory())._current_lr() == 1e-3
    m = _module(kind, optimizer_factory=_Factory(learning_rate=3e-4))
    assert m._current_lr() == 3e-4
    opt = torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=0.5)
    opt.param_groups[0]["lr"] = 0.25   # where a scheduler leaves it
    m.optimizers = lambda: opt
    assert m._current_lr() == 0.25
    m.optimizers = lambda: [opt]
    assert m._current_lr() == 0.25


@pytest.mark.parametrize("kind", MODULES)
def test_epoch_end_steps_the_schedulers_of_a_fused_optimizer(kind):
    a, b = _Scheduler(), _Scheduler()
    m = _module(kind, lr_scheduler_factory=object())
    m.on_train_epoch_end()   # no trainer: nothing to step
    m.lr_schedulers = lambda: a
    m.on_train_epoch_end()
    assert a.steps == 1
    m.lr_schedulers = lambda: [a, b]
    m.on_train_epoch_end()
    assert (a.steps, b.steps) == (2, 1)
    for kw in ({}, {"lr_scheduler_factory": object(), "fused_optimizer": False}):
        m = _module(kind, **kw)
        m.lr_schedulers = lambda: [a, b]
        m.on_train_epoch_end()
    assert (a.steps, b.steps) == (2, 1)


def test_legacy_sasrec_optimizer_factory_property():
    m = _module("sasrec")
    assert m.optimizer_factory is None
    f = _Factory()
    m.optimizer_factory = f
    assert m.optimizer_factory is f and m._current_lr() == 3e-4 and m._model.core.adam_betas == (0.8, 0.9)
    with pytest.raises(ValueError, match="OptimizerFactory"):
        m.optimizer_factory = object()


_ITEM_TABLE = {"sasrec": "item_embedder.item_emb.weight", "tisasrec": "item_embedder.item_emb.weight",
               "bert4rec": "item_embedder.cat_embeddings.item_id.weight"}


@pytest.mark.parametrize("kind, loss", [("sasrec", dict(loss_type="BCE", loss_sample_count=8)),
                                        ("tisasrec", dict(loss_type="CE", loss_sample_count=8)),
                                        ("bert4rec", dict(loss_type="BCE"))])
def test_catalog_growth_keeps_loss_betas_device_and_seed(kind, loss):
    n, d = 40, 64
    m = _module(kind, optimizer_factory=_Factory(betas=(0.8, 0.9)), **loss)
    core0 = m._model.core
    # a checkpoint whose item table and head have their true shapes; growth only carries the other weights over
    rows = n + (kind != "bert4rec")   # the legacy SasRec table has a padding row
    shapes = {_ITEM_TABLE[kind]: (rows, d), "_head.linear.weight": (n, d), "_head.linear.bias": (n,)}
    g = torch.Generator().manual_seed(0)
    sd = {k: torch.randn(shapes.get(k, (1,)), generator=g) for k in core0._keymap.values()}
    m.load_state_dict({"_model." + k: v for k, v in sd.items()})
    core0._predict_graphs = {"captured": None}
    spec = core0._loss_spec

    m.set_item_embeddings_by_size(n + 5)
    core = m._model.core
    assert core is not core0 and type(core) is type(core0) and core.cfg.n_items == n + 5
    assert core.adam_betas == (0.8, 0.9) and core._loss_spec == spec
    assert (core._device, core._seed, core.item_feature) == (core0._device, core0._seed, core0.item_feature)
    assert core0._predict_graphs == {}
    assert getattr(core, "timestamp_feature", None) == ("timestamp" if kind == "tisasrec" else None)
    assert m._vocab_size == n + 5 and m._schema.item_id_features.item().cardinality == n + 5
    table = core.state_dict()[_ITEM_TABLE[kind]]
    assert table.shape == (rows + 5, d) and torch.equal(table[:n], sd[_ITEM_TABLE[kind]][:n])
