"""GPU tests of the full-catalog BCE head (rp_bce_head_fwd / _bwd) against a float64 restatement on the same bf16 inputs
(tests/bce_reference.py states the bounds), and of the surfaces that select it: the new-path ``SasRec`` with
``loss = BCE()`` and ``Bert4Rec(loss_type="BCE" | "CE_restricted")``.

Rows past n_valid hold finite non-zero garbage, as stale rows of an earlier, larger batch do in the engine: they must not
reach d_table / d_bias, and d_hc must stay untouched there."""
import pytest
import torch

from bce_reference import reference, worst

pytestmark = pytest.mark.gpu

SENTINEL = 3.0   # d_hc rows past n_valid must keep it


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from replay_b200 import ops as _ops

    return _ops


def _inputs(cap, n_valid, I, d, bias, *, scale_h=0.5, scale_e=0.3, shared_label=False, seed=0):
    g = torch.Generator().manual_seed(seed + 13 * cap + I + d)
    h = torch.randn(cap, d, generator=g) * scale_h
    h[n_valid:] = torch.randn(cap - n_valid, d, generator=g) * 2.0 + 1.0   # stale rows: finite, non-zero
    W = torch.randn(I, d, generator=g) * scale_e
    labels = torch.randint(0, I, (cap,), generator=g, dtype=torch.int32)
    if shared_label:
        labels[:] = min(5, I - 1)
    b = None
    if bias:
        b = torch.zeros((I + 127) // 128 * 128)
        b[:I] = torch.randn(I, generator=g) * 0.5
        b[I:] = 7.0   # padding entries are never read as a live item's bias
    dev = torch.device("cuda")
    return (h.to(dev, torch.bfloat16), W.to(dev, torch.bfloat16), None if b is None else b.to(dev), labels.to(dev),
            torch.tensor([n_valid], dtype=torch.int32, device=dev))


def _run(ops, h, W, b, labels, nv, *, fused, hint=0):
    cap, d = h.shape
    I = W.shape[0]
    st = ops.CEHeadState(cap, I, d, h.device)
    d_hc = torch.full((cap, d), SENTINEL, device=h.device, dtype=torch.bfloat16)
    d_W = torch.full((I, d), 9.0, device=h.device)
    d_b = torch.full((I,), 9.0, device=h.device) if b is not None else None
    loss = ops.bce_head_fwd(st, h, W, labels, nv, bias=b, d_hc=d_hc if fused else None, n_valid_hint=hint).clone()
    ops.bce_head_bwd(st, h, W, labels, nv, d_hc, d_W, bias=b, d_bias=d_b, n_valid_hint=hint)
    torch.cuda.synchronize()
    return loss, d_hc, d_W, d_b


def _check(ops, cap, n_valid, I, d, bias, *, fused, hint=0, rerun=True, **kw):
    h, W, b, labels, nv = _inputs(cap, n_valid, I, d, bias, **kw)
    loss, d_hc, d_W, d_b = _run(ops, h, W, b, labels, nv, fused=fused, hint=hint)
    r = reference(h, W, None if b is None else b[:I], labels, n_valid)
    assert abs(float(loss[0]) - float(r["loss"])) <= float(r["bound_loss"]), (float(loss[0]), float(r["loss"]))
    assert abs(float(loss[1]) - (1.0 / n_valid if n_valid else 0.0)) <= 2e-7 / max(n_valid, 1)   # fast-math reciprocal
    assert worst(d_hc[:n_valid], r["d_h"], r["bound_h"]) <= 1.0
    assert (d_hc[n_valid:] == SENTINEL).all(), "d_hc rows past n_valid were written"
    assert worst(d_W, r["d_W"], r["bound_W"]) <= 1.0
    if bias:
        assert worst(d_b, r["d_b"], r["bound_b"]) <= 1.0
    if rerun:   # loss and d_hc are reduced in a fixed order
        loss2, d_hc2, _, _ = _run(ops, h, W, b, labels, nv, fused=fused, hint=hint)
        assert torch.equal(loss2, loss) and torch.equal(d_hc2, d_hc)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("fused", [True, False], ids=["fused", "unfused"])
@pytest.mark.parametrize("d,bias", [(64, False), (64, True), (128, False), (128, True), (256, False), (256, True), (512, False)])
def test_head_split_over_the_catalog(ops, d, bias, fused):
    """Few row tiles: the fused pass splits the catalog over several CTAs (partials + bce_finalize_kernel)."""
    _check(ops, 384, 300, 20001, d, bias, fused=fused)


@pytest.mark.parametrize("fused", [True, False], ids=["fused", "unfused"])
@pytest.mark.parametrize("d,bias", [(64, True), (128, False), (256, True)])
def test_head_one_split(ops, d, bias, fused):
    """As many row tiles as SMs at full capacity: one split, the pass writes d_hc and the row losses itself."""
    cap = _sms() * 128
    _check(ops, cap, cap, 129, d, bias, fused=fused)


@pytest.mark.parametrize("n_items", [1, 63, 129, 50000])
@pytest.mark.parametrize("n_valid", [0, 1, 127, 128, 129])
def test_head_ragged_edges(ops, n_items, n_valid):
    """Catalogs ragged against 64 and 128 columns, and n_valid on both sides of a 128-row tile (0 = an empty batch:
    loss 0, 1/M reported as 0, zero gradients, as the CE head)."""
    _check(ops, 256, n_valid, n_items, 128, n_items > 100, fused=True, rerun=False)


@pytest.mark.parametrize("d,bias", [(64, True), (256, False)])
def test_head_large_logits_and_shared_label(ops, d, bias):
    """|x| beyond 30 in both directions (sigmoid saturates, softplus is linear) and every row sharing one label."""
    _check(ops, 256, 200, 5000, d, bias, fused=True, scale_h=4.0, scale_e=1.5)
    _check(ops, 256, 200, 5000, d, bias, fused=True, shared_label=True)
    h, W, b, labels, nv = _inputs(256, 200, 5000, d, bias, scale_h=4.0, scale_e=1.5)
    x = h[:200].double() @ W.double().T
    assert x.max() > 30 and x.min() < -30


def test_head_unfused_matches_fused(ops):
    """Both forwards compute the same loss (within the bound) and the same d_hc (same partition, same order)."""
    h, W, b, labels, nv = _inputs(512, 450, 30000, 128, True)
    lf, dhf, dWf, _ = _run(ops, h, W, b, labels, nv, fused=True)
    lu, dhu, dWu, _ = _run(ops, h, W, b, labels, nv, fused=False)
    r = reference(h, W, b[:30000], labels, 450)
    assert abs(float(lf[0]) - float(lu[0])) <= 2 * float(r["bound_loss"])
    assert torch.equal(dhf, dhu)


# ------------------------------------------------------------------------------------------------ surfaces
def test_new_path_sasrec_bce_and_switch(ops):
    """LightningModule(SasRec) with loss = BCE() trains through the fused, graph-captured step; a CE -> BCE -> CE switch on
    one module gives each head's loss, checked against the fp64 head on the engine's own hidden rows."""
    from replay_b200.nn.lightning import LightningModule, OptimizerFactory
    from replay_b200.nn.loss import BCE, CE
    from replay_b200.nn.sequential import SasRec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema
    from replay_b200.synthetic import make_sequences

    n_items, d, L, B = 2000, 64, 32, 64
    model = SasRec.from_params(TensorSchema(TensorFeatureInfo("item_id", n_items, n_items, d)), embedding_dim=d, num_heads=1,
                               num_blocks=2, max_sequence_length=L, dropout=0.0, seed=1)
    model.loss = BCE()
    lm = LightningModule(model, optimizer_factory=OptimizerFactory(learning_rate=3e-3))
    ids, pm, lab, tm = (t.cuda() for t in make_sequences(B, n_items, L, seed=5))
    batch = {"feature_tensors": {"item_id": ids}, "padding_mask": pm, "positive_labels": lab.unsqueeze(-1),
             "target_padding_mask": tm.unsqueeze(-1)}
    model.train()
    losses = [float(lm.training_step(batch, i)) for i in range(30)]
    assert losses[-1] < 0.5 * losses[0], losses[::5]
    eng = model.core.engine
    # the loss a step reports is its forward's: restate it from the hidden rows the step gathered (the update does not touch
    # them) and the bf16 item table from before the update
    for spec in (CE(), BCE(), CE()):
        W_before = eng.params16["item_emb"][:n_items].clone()
        model.loss = spec
        got = float(lm.training_step(batch, 0))
        nv = int(eng.n_valid.item())
        x = eng.hc[:nv].double() @ W_before.double().T
        y = eng.labels_c[:nv].long()
        if isinstance(spec, BCE):
            ref = float((torch.nn.functional.softplus(x).sum() - x.gather(1, y[:, None]).sum()) / nv)
        else:
            ref = float(torch.nn.functional.cross_entropy(x, y))
        assert abs(got - ref) < 2e-3 * abs(ref), (type(spec).__name__, got, ref)


def test_new_path_sasrec_bce_unfused_matches_fused(ops):
    from replay_b200.nn.loss import BCE
    from replay_b200.nn.sequential import SasRec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema
    from replay_b200.synthetic import make_sequences

    n_items, d, L, B = 3000, 128, 32, 32
    ids, pm, lab, tm = (t.cuda() for t in make_sequences(B, n_items, L, seed=3))
    out = []
    for fused in (True, False):
        model = SasRec.from_params(TensorSchema(TensorFeatureInfo("item_id", n_items, n_items, d)), embedding_dim=d,
                                   num_heads=2, num_blocks=1, max_sequence_length=L, dropout=0.0, seed=2)
        model.loss = BCE()
        model.train()
        model.core.ensure_engine(B, L, with_grad=True).fused_ce = fused
        loss = model.core.loss(ids, pm, lab, tm)
        loss.backward()
        out.append((loss.item(), model.core.flat.grad.clone()))
    assert abs(out[0][0] - out[1][0]) < 1e-4 * abs(out[0][0])
    torch.testing.assert_close(out[0][1], out[1][1], rtol=1e-3, atol=1e-6)


def _bert(tying, loss_type, n_items=1000, d=64, L=32, seed=0):
    from replay_b200.models.nn.sequential import Bert4Rec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    torch.manual_seed(seed)
    return Bert4Rec(TensorSchema(TensorFeatureInfo("item_id", n_items, 0, d)), block_count=2, head_count=1, hidden_size=d,
                    max_seq_len=L, dropout_rate=0.0, enable_embedding_tying=tying, loss_type=loss_type)


def _bert_batch(B, n_items, L, seed):
    from replay_b200.models.nn.sequential.bert4rec import uniform_masker

    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(1, n_items, (B, L), generator=g)
    pm = torch.ones(B, L, dtype=torch.bool)
    pm[: B // 2, : L // 3] = False
    tok = uniform_masker(pm, 0.2, generator=g)
    return {"query_id": torch.arange(B).view(-1, 1), "inputs": {"item_id": ids.cuda()}, "pad_mask": pm.cuda(),
            "token_mask": tok.cuda(), "positive_labels": ids.cuda()}


@pytest.mark.parametrize("tying", [False, True], ids=["untied", "tied"])
def test_bert4rec_bce_trains_and_survives_a_new_shape(ops, tying):
    m = _bert(tying, "BCE")
    core = m._model.core
    batch = _bert_batch(16, 1000, 32, 1)
    def step_checked(b, i):
        eng = core.ensure_engine(*b["inputs"]["item_id"].shape, with_grad=True)
        W_before = (eng.params16["item_emb"] if tying else eng.params16["head_w"]).clone()
        b_before = eng.params["head_b"][:1000].clone()
        loss = float(m.training_step(b, i))
        eng = core.engine
        nv = int(eng.n_valid.item())
        ref = float(reference(eng.hc, W_before, b_before, eng.labels_c, nv)["loss"])
        assert abs(loss - ref) < 2e-3 * abs(ref), (loss, ref)
        return loss

    first = step_checked(batch, 0)
    losses = [float(m.training_step(batch, i)) for i in range(1, 29)]
    last = step_checked(batch, 29)
    assert last < 0.5 * first, (first, losses[::5], last)
    # a larger batch re-allocates the engine's buffers: it must keep BCE
    step_checked(_bert_batch(40, 1000, 32, 2), 30)
    assert core.engine.bce and core.engine.B >= 40


def test_bert4rec_ce_restricted_is_ce(ops):
    batch = _bert_batch(16, 1000, 32, 4)
    losses = []
    for lt in ("CE", "CE_restricted"):
        m = _bert(False, lt, seed=3)
        losses.append([m.training_step(batch, i).clone() for i in range(3)])
    # the first step's forward runs on identical parameters: bit for bit.  Later steps follow updates whose item-table
    # gradient receives its one-hot part through atomics (summation order varies), so they agree to rounding only.
    assert torch.equal(losses[0][0], losses[1][0])
    for a, b in zip(losses[0][1:], losses[1][1:]):
        assert abs(float(a) - float(b)) <= 1e-4 * abs(float(b))
    assert not m._model.core.engine.bce
