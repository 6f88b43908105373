"""LogInCESampled and CESampledWeighted on the sampled CUDA head (rp_sampled_head_* kinds 4 and 5).

(a) the kernels through the C ABI against the float64 reference of tests/sampled_ext_reference.py, with the inputs, checks
    and tolerances of tests/test_gpu_sampled_head.py: both kinds x three negative layouts x d 64 / 128 / 256 / 512, n_valid
    0, 1, 127, 128, 129 and the capacity, N 1, 31, 33 and 2048, rows whose every negative is rejected, LogInCE clamp edges,
    zero / negative / non-uniform weights (NaN past n_valid, which the head must not read) and a NaN-filled workspace;
(b) the engine against losses and gradients of the reference's own classes (tests/golden/sampled_ext_losses.npz);
(c) the new-path SasRec with the new ``loss``: autograd forward / backward and LightningModule's fused, graph-replayed
    training step on consecutive batches with different negatives and weights, each against an eager engine; packed
    against padded body; the DiffTransformer body;
(d) identities: all-ones weights give CESampled, log_epsilon 0 with a wide clamp gives CESampled's loss.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

import sampled_ext_reference as sx
from fp64_checks import WorstErrors
from replay_b200._lib import SampledDesc, check, lib
from test_gpu_sampled_head import (MODES, N_ITEMS, SENT, TOL_TABLE_ROW, TOL_TABLE_SHARED, Case, assert_within, errors,
                                   make_inputs, preset_table, workspace)

pytestmark = pytest.mark.gpu

KINDS = {"login": sx.LOGIN_CE_SAMPLED, "cew": sx.CE_SAMPLED_WEIGHTED}

_worst = WorstErrors()


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    _worst.report()


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda")


# ----------------------------------------------------------------------------------------------------------------------
# (a) kernels against float64
# ----------------------------------------------------------------------------------------------------------------------
CASES = [
    # both kinds x three layouts x four widths
    Case("login", "shared", 128, 1200, 1200, 1000),
    Case("login", "perpos", 128, 1200, 1190, 100, ignore="pad"),
    Case("login", "perseq", 128, 1200, 129, 33, L=50),
    Case("cew", "shared", 128, 1200, 127, 257),
    Case("cew", "perpos", 128, 1200, 128, 31, ignore="none"),
    Case("cew", "perseq", 128, 1200, 1200, 100, ignore="pad"),
    Case("login", "shared", 64, 300, 290, 7),
    Case("login", "perpos", 64, 300, 300, 33, L=50),
    Case("login", "perseq", 64, 4133, 4133, 100, ignore="pad"),
    Case("cew", "shared", 64, 4133, 4123, 8, ignore="pad"),
    Case("cew", "perpos", 64, 300, 1, 100, L=50, ignore="none"),
    Case("cew", "perseq", 64, 300, 129, 31, L=50),
    Case("login", "shared", 256, 4133, 4133, 129),
    Case("login", "perpos", 256, 1200, 128, 31, ignore="none"),
    Case("login", "perseq", 256, 300, 290, 1, L=50, ignore="none"),
    Case("cew", "shared", 256, 300, 129, 64, ignore="none"),
    Case("cew", "perpos", 256, 4133, 4123, 100, L=50, ignore="pad"),
    Case("cew", "perseq", 256, 1200, 127, 33),
    Case("login", "shared", 512, 1200, 1200, 2048, ignore="pad"),
    Case("login", "perpos", 512, 4133, 4133, 100, L=50),
    Case("login", "perseq", 512, 300, 300, 33, L=50, ignore="none"),
    Case("cew", "shared", 512, 4133, 129, 1000),
    Case("cew", "perpos", 512, 300, 290, 31, L=50),
    Case("cew", "perseq", 512, 4133, 4123, 100, ignore="pad"),
    # edges: no valid row, one valid row, one shared negative (every negative of a third of the rows rejected), N 2048
    Case("login", "shared", 128, 300, 0, 65),
    Case("cew", "perpos", 128, 300, 0, 31, L=50),
    Case("login", "perpos", 128, 1200, 1, 33),
    Case("login", "shared", 64, 1200, 1200, 1),
    Case("cew", "shared", 64, 1200, 1200, 1),
    Case("cew", "shared", 128, 1200, 1190, 2048),
    Case("cew", "perpos", 128, 1200, 1200, 2048, L=50),
    # LogInCE clamps: rows on both sides of -clamp, and rows whose every logit is clamped (d_hc exactly zero)
    Case("login", "shared", 128, 1200, 1200, 257, scale=8.0, log_eps=1e-3, clamp=5.5),
    Case("login", "perpos", 128, 1200, 1190, 100, scale=8.0, log_eps=1e-3, clamp=5.5),
    Case("login", "perseq", 64, 300, 300, 33, L=50, scale=8.0, log_eps=1e-3, clamp=5.5),
]


def ext_inputs(c: Case, dev, seed=0):
    """make_inputs of test_gpu_sampled_head plus a row whose every negative is rejected (per-row layouts) and the weights:
    fp32 [capacity], non-uniform, zero on every 11th row, negative on about a quarter, NaN past n_valid."""
    x = make_inputs(c, dev, seed)
    if c.mode != "shared" and c.nv > 4:
        r = int(x["valid_idx"][4]) // (c.L if c.mode == "perseq" else 1)
        x["neg"][r] = x["labels"][4].long()
    g = torch.Generator().manual_seed(1000 + c.cap + c.nv + c.N + c.d)
    w = torch.rand(c.cap, generator=g) * 2.0 - 0.5
    w[::11] = 0.0
    w[c.nv:] = float("nan")
    x["w"] = w.to(dev)
    return x


def run(c: Case, x, ws, nv=None):
    """fwd + bwd -> (loss_out [2], d_hc [cap + 64, d] with sentinel rows, d_table [n_items + 1, d], preset)."""
    dev = ws.device
    if nv is not None:
        x["nv"].fill_(nv)
    sd = SampledDesc()
    sd.hc, sd.table, sd.labels = x["hc"].data_ptr(), x["table"].data_ptr(), x["labels"].data_ptr()
    sd.valid_idx, sd.negatives, sd.n_valid = x["valid_idx"].data_ptr(), x["neg"].data_ptr(), x["nv"].data_ptr()
    sd.capacity, sd.n_items, sd.d, sd.n_neg, sd.neg_mode, sd.seq_len = c.cap, N_ITEMS, c.d, c.N, MODES[c.mode], c.L
    sd.kind, sd.ignore_index, sd.vocab_size = KINDS[c.kind], x["ignore_index"], c.vocab
    sd.log_eps, sd.clamp = c.log_eps, c.clamp
    sd.row_weight = x["w"].data_ptr()
    loss = torch.full((2,), float("nan"), dtype=torch.float32, device=dev)
    sd.loss_out = loss.data_ptr()
    sd.workspace, sd.workspace_bytes = ws.data_ptr(), ws.numel()
    d_hc = torch.full((c.cap + 64, c.d), SENT, dtype=torch.bfloat16, device=dev)
    preset = preset_table(c, dev)
    d_table = preset.clone()
    st = torch.cuda.current_stream().cuda_stream
    L = lib()
    check(L.rp_sampled_head_fwd(ctypes.byref(sd), st), "rp_sampled_head_fwd")
    check(L.rp_sampled_head_bwd(ctypes.byref(sd), d_hc.data_ptr(), d_table.data_ptr(), st), "rp_sampled_head_bwd")
    torch.cuda.synchronize()
    return loss, d_hc, d_table, preset


def reference(c: Case, x):
    nv = int(x["nv"][0])
    return sx.reference(x["hc"], x["table"], x["labels"], x["valid_idx"], x["neg"], nv, KINDS[c.kind], MODES[c.mode], L=c.L,
                        ignore_index=x["ignore_index"], row_weight=x["w"], log_eps=c.log_eps, clamp=c.clamp)


@pytest.mark.parametrize("c", CASES, ids=lambda c: c.id)
def test_sampled_ext_head_matches_fp64(cuda, c):
    x = ext_inputs(c, cuda)
    ws = workspace(c, cuda)
    out = run(c, x, ws)
    ref = reference(c, x)
    err, bad = errors(c, c.nv, out, ref)
    for k, v in err.items():
        _worst.note(f"{c.kind} {k}", v)
    out2 = run(c, x, ws)
    if not (torch.equal(out2[0], out[0]) and torch.equal(out2[1], out[1])):
        bad.append("a second identical call gave a different loss or d_hc")
    t_gap = float(((out2[2].double() - out[2].double()).abs() / (ref["mag_table"] + out[3].double())).max())
    if t_gap > (TOL_TABLE_SHARED if c.mode == "shared" else TOL_TABLE_ROW):
        bad.append(f"d_table differs between two identical calls by {t_gap:.3g}")
    if c.clamp != 100.0 and c.mode == "perpos" and c.nv >= 2:
        for tt in (0, c.nv - 1):   # every logit of these rows is clamped: the gradient is exactly zero
            if not (out[1][tt].float() == 0).all():
                bad.append(f"d_hc row {tt}, all of whose terms are clamped, is not zero")
    if c.kind == "cew" and c.nv > 11:
        if not (out[1][0].float() == 0).all() or not (out[1][11].float() == 0).all():
            bad.append("a zero-weight row has a non-zero d_hc")
    assert_within(c, err, bad)


def test_login_clamp_is_active_on_both_sides(cuda):
    """The shared-negative clamp case above holds rows inside the clamp and rows outside it (zero gradient)."""
    c = CASES[-3]
    assert c.kind == "login" and c.mode == "shared" and c.clamp == 5.5
    per_row = reference(c, ext_inputs(c, cuda))["d_hc"].abs().sum(1)
    assert (per_row == 0).any() and (per_row > 0).any()


@pytest.mark.parametrize("kind", ["login", "cew"])
@pytest.mark.parametrize("nv", [290, 300])
def test_shared_negatives_ignore_stale_workspace(cuda, kind, nv):
    """A workspace of 0xFF bytes (NaN in fp32 and bf16) gives the result of a zeroed one; capacity 300 is not a multiple of
    64, so the dE_neg GEMM's last K chunk reaches past the capacity into the bf16 dz rows."""
    c = Case(kind, "shared", 128, 300, nv, 65)
    x = ext_inputs(c, cuda)
    out = run(c, x, workspace(c, cuda, fill=0xFF))
    err, bad = errors(c, nv, out, reference(c, x))
    assert_within(c, err, bad)
    fresh = run(c, x, workspace(c, cuda))
    assert torch.equal(out[0], fresh[0]) and torch.equal(out[1], fresh[1])


# ----------------------------------------------------------------------------------------------------------------------
# (b) the engine against the reference's classes
# ----------------------------------------------------------------------------------------------------------------------
GOLDEN = {"login": ("login_ce_sampled", {}), "login_clamped": ("login_ce_sampled", dict(log_eps=1e-3, clamp=4.37)),
          "weighted": ("ce_sampled_weighted", {})}


def _load(golden_dir):
    z = np.load(os.path.join(golden_dir, "sasrec_new_tiny.npz"))
    sd = {k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd::")}
    return z, sd, np.load(os.path.join(golden_dir, "sampled_ext_losses.npz"))


def _cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def _tiny_engine(z, sd, cuda, packed=False):
    from oracle import sasrec as osr
    from replay_b200.engine import EncoderConfig, SasRecEngine
    B, L = z["ids"].shape
    cfg = EncoderConfig(n_items=int(z["n_items"]), d=int(z["d"]), n_heads=int(z["H"]), n_blocks=int(z["n_blocks"]), max_len=L,
                        dropout=0.0, variant="new")
    eng = SasRecEngine(cfg, B, L, cuda)
    eng.load_canonical(osr.params_from_new_state_dict(sd))
    eng.packed_body = packed
    return eng


def _step(eng, z, neg, kind, w=None, **kw):
    """Stage the golden batch with ``neg`` (and weights), forward + backward: (loss, canonical gradients)."""
    eng.set_loss(kind, n_neg=neg.shape[-1], neg_shape={1: "shared", 2: "perseq", 3: "perpos"}[neg.dim()], **kw)
    eng.set_batch(*(torch.from_numpy(z[k]).cuda() for k in ("ids", "pad_mask", "labels", "target_mask")))
    eng.set_negatives(neg.cuda())
    if w is not None:
        eng.set_row_weights(w.cuda()[..., 0] if w.dim() == 3 else w.cuda())
    loss = eng.forward_train()
    eng.g32.zero_()
    eng.grads["item_emb"].fill_(3.0)   # the sampled head owns (overwrites) the table gradient
    eng.backward()
    torch.cuda.synchronize()
    return float(loss[0]), eng.export_canonical(eng.grads)


@pytest.mark.parametrize("shape", ["shared", "perseq", "perpos"])
@pytest.mark.parametrize("case", sorted(GOLDEN))
def test_engine_matches_reference_goldens(golden_dir, cuda, case, shape):
    z, sd, zx = _load(golden_dir)
    eng = _tiny_engine(z, sd, cuda)
    kind, kw = GOLDEN[case]
    w = torch.from_numpy(zx["weights"]) if kind == "ce_sampled_weighted" else None
    l, G = _step(eng, z, torch.from_numpy(zx["neg_" + shape]), kind, w, ignore_index=int(zx["ignore_index"]), **kw)
    ref = float(zx[f"{case}_{shape}_loss"])
    assert abs(l - ref) < 5e-3 * abs(ref), (l, ref)
    gE, gW = torch.from_numpy(zx[f"{case}_{shape}_gE"]), torch.from_numpy(zx[f"{case}_{shape}_gW"])
    for nm, a, b in (("item_emb", G["item_emb"].cpu(), gE), ("in_w", G["blocks"][0]["in_w"].cpu(), gW)):
        c, r = _cos(a, b), float(a.double().norm() / b.double().norm())
        assert c > 0.995 and abs(r - 1) < 0.03, (nm, c, r)
    touched = gE.abs().sum(1) > 0
    assert (G["item_emb"].cpu()[~touched] == 0).all()


# ----------------------------------------------------------------------------------------------------------------------
# (c) the public model
# ----------------------------------------------------------------------------------------------------------------------
def _batches(z, zx, n_items):
    """Two batches: the golden one with the per-sequence negatives and weights, and the same sequences with other
    negatives (an ignore-index entry and collisions included) and other weights ([B, L] this time)."""
    g = torch.Generator().manual_seed(5)
    ign = int(zx["ignore_index"])
    ids, pm = torch.from_numpy(z["ids"]).cuda(), torch.from_numpy(z["pad_mask"]).cuda()
    lab, tm = torch.from_numpy(z["labels"]).cuda(), torch.from_numpy(z["target_mask"]).cuda()
    neg2 = torch.randint(0, n_items, tuple(zx["neg_perseq"].shape), generator=g)
    neg2[:, 0] = lab[:, -1].cpu()
    neg2[0, 1] = ign
    w2 = torch.rand(*ids.shape, generator=g) * 3 - 1
    base = {"feature_tensors": {"item_id": ids}, "padding_mask": pm, "positive_labels": lab.unsqueeze(-1),
            "target_padding_mask": tm.unsqueeze(-1)}
    return [dict(base, feature_tensors={"item_id": ids, "w": torch.from_numpy(zx["weights"]).cuda()},
                 negative_labels=torch.from_numpy(zx["neg_perseq"]).cuda()),
            dict(base, feature_tensors={"item_id": ids, "w": w2.cuda()}, negative_labels=neg2.cuda())]


def _spec(case, ign):
    from replay_b200.nn.loss import CESampledWeighted, LogInCESampled
    return {"login_clamped": lambda: LogInCESampled(log_epsilon=1e-3, clamp_border=4.37, negative_labels_ignore_index=ign),
            "weighted": lambda: CESampledWeighted("w", negative_labels_ignore_index=ign)}[case]()


def _eager_loss(eng, spec, batch):
    """The loss of ``batch`` on a plain eager engine (padded body) with the given weights."""
    w = spec.row_weights(batch["feature_tensors"], batch["target_padding_mask"][..., 0]) if hasattr(spec, "row_weights") else None
    eng.set_loss(spec.kind, n_neg=batch["negative_labels"].shape[-1], neg_shape="perseq", **spec.engine_kwargs())
    eng.set_batch(batch["feature_tensors"]["item_id"], batch["padding_mask"], batch["positive_labels"][..., 0],
                  batch["target_padding_mask"][..., 0])
    eng.set_negatives(batch["negative_labels"])
    if w is not None:
        eng.set_row_weights(w)
    return eng.forward_train()


@pytest.mark.parametrize("case", ["login_clamped", "weighted"])
def test_sasrec_autograd_and_lightning_steps_match_eager(golden_dir, cuda, case):
    from oracle import sasrec as osr
    from replay_b200.nn.lightning import LightningModule, OptimizerFactory
    from replay_b200.nn.sequential import SasRec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    z, sd, zx = _load(golden_dir)
    n_items, d, H, L = int(z["n_items"]), int(z["d"]), int(z["H"]), int(z["L"])
    model = SasRec.from_params(TensorSchema(TensorFeatureInfo("item_id", n_items, n_items, d)), embedding_dim=d, num_heads=H,
                               num_blocks=int(z["n_blocks"]), max_sequence_length=L, dropout=0.0)
    model.load_state_dict(sd)
    spec = _spec(case, int(zx["ignore_index"]))
    model.loss = spec
    model.train()
    batches = _batches(z, zx, n_items)
    ref_eng = _tiny_engine(z, sd, cuda)
    # autograd: loss and flat gradient of each batch against the eager engine
    for b in batches:
        out = model(**b)
        ref = _eager_loss(ref_eng, spec, b)
        ref_eng.g32.zero_()
        ref_eng.backward()
        l_out = float(out["loss"].detach())
        assert abs(l_out - float(ref[0])) <= 1e-6 * abs(float(ref[0])), (l_out, float(ref[0]))
        out["loss"].backward()
        torch.testing.assert_close(model.core.flat.grad, ref_eng.g32, rtol=1e-4, atol=1e-7)
        model.core.flat.grad = None
    # Lightning: fused forward + backward + Adam, captured after two eager steps and replayed, batches alternating
    lm = LightningModule(model, optimizer_factory=OptimizerFactory(learning_rate=3e-3))
    losses = []
    for i in range(6):
        b = batches[i % 2]
        ref_eng.load_canonical(osr.params_from_new_state_dict(model.state_dict()))
        ref = float(_eager_loss(ref_eng, spec, b)[0])
        got = float(lm.training_step(b, i))
        assert abs(got - ref) <= 2e-5 * abs(ref), (i, got, ref)
        losses.append(got)
    assert losses[4] < losses[0] and losses[5] < losses[1], losses
    with pytest.raises(ValueError):
        lm.training_step({k: v for k, v in batches[0].items() if k != "negative_labels"}, 6)


@pytest.mark.parametrize("case", ["login_clamped", "weighted"])
def test_packed_body_matches_padded(golden_dir, cuda, case):
    z, sd, zx = _load(golden_dir)
    kind, kw = GOLDEN[case]
    w = torch.from_numpy(zx["weights"]) if kind == "ce_sampled_weighted" else None
    out = []
    for packed in (False, True):
        eng = _tiny_engine(z, sd, cuda, packed=packed)
        out.append(_step(eng, z, torch.from_numpy(zx["neg_perpos"]), kind, w, ignore_index=int(zx["ignore_index"]), **kw))
    assert abs(out[0][0] - out[1][0]) <= 1e-6 * abs(out[0][0])
    for nm in ("item_emb", "pos_emb", "lnf_w"):
        torch.testing.assert_close(out[1][1][nm], out[0][1][nm], rtol=1e-4, atol=1e-6)
    torch.testing.assert_close(out[1][1]["blocks"][0]["in_w"], out[0][1]["blocks"][0]["in_w"], rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("spec_name", ["login", "weighted"])
def test_diff_body_takes_the_new_losses(cuda, spec_name):
    """The DiffTransformer engine inherits the head: with all-ones weights / log_epsilon 0 the new losses give CESampled's
    loss, and fused steps train."""
    from replay_b200.nn.loss import CESampled, CESampledWeighted, LogInCESampled
    from test_gpu_diff_sasrec import _batch, _model

    n_items, d, H, L, B = 400, 64, 2, 50, 8
    ids, pm, labels, tm = (t.to(cuda) for t in _batch(B, L, n_items, seed=4))
    neg = torch.randint(0, n_items, (B, 32), generator=torch.Generator().manual_seed(1)).to(cuda)
    m = _model(n_items, d, H, L, 2, "layernorm", seed=3)
    m.train()
    fts = {"item_id": ids, "w": torch.ones(B, L, 1, device=cuda)}
    kw = dict(feature_tensors=fts, padding_mask=pm, positive_labels=labels, negative_labels=neg, target_padding_mask=tm)
    m.loss = CESampled()
    base = float(m(**kw)["loss"])
    m.loss = CESampledWeighted("w") if spec_name == "weighted" else LogInCESampled(log_epsilon=0.0, clamp_border=1e30)
    got = float(m(**kw)["loss"])
    assert abs(got - base) <= 1e-5 * abs(base), (got, base)
    rw = fts["w"][..., 0] if spec_name == "weighted" else None
    losses = [float(m.core.fused_step(ids, pm, labels, tm, all_reduce=None, lr=1e-2, negatives=neg, row_weights=rw))
              for _ in range(6)]
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses


# ----------------------------------------------------------------------------------------------------------------------
# (d) identities
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", ["shared", "perseq", "perpos"])
def test_identities_with_ce_sampled(golden_dir, cuda, shape):
    z, sd, zx = _load(golden_dir)
    neg = torch.from_numpy(zx["neg_" + shape])
    ign = dict(ignore_index=int(zx["ignore_index"]))
    eng = _tiny_engine(z, sd, cuda)
    l_ce, G_ce = _step(eng, z, neg, "ce_sampled", **ign)
    ones = torch.ones(z["ids"].shape)
    l_w, G_w = _step(eng, z, neg, "ce_sampled_weighted", ones, **ign)
    assert l_w == l_ce                                    # a weight of 1 leaves every row's arithmetic as it was
    for a, b in ((G_w["item_emb"], G_ce["item_emb"]), (G_w["blocks"][0]["in_w"], G_ce["blocks"][0]["in_w"])):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-8)
    l_in, G_in = _step(eng, z, neg, "login_ce_sampled", log_eps=0.0, clamp=1e30, **ign)
    assert abs(l_in - l_ce) <= 1e-6 * abs(l_ce), (l_in, l_ce)
    for a, b in ((G_in["item_emb"], G_ce["item_emb"]), (G_in["blocks"][0]["in_w"], G_ce["blocks"][0]["in_w"])):
        torch.testing.assert_close(a, b, rtol=1e-3, atol=1e-6)
