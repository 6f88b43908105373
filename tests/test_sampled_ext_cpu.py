"""LogInCESampled and CESampledWeighted without a GPU: the restatement (oracle/sampled_ext.py) against losses and gradients of the
reference's own classes (tests/golden/sampled_ext_losses.npz, written by oracle/gen_sampled_ext_golden.py), the float64
kernel reference (tests/sampled_ext_reference.py) against the restatement, the public selectors, the engine's buffers and
descriptor, the core's staging and the C ABI's argument checks."""
import ctypes
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import sampled_ext_reference as sx
from oracle import sampled as osm
from oracle import sampled_ext as osx
from oracle import sasrec as osr

SHAPES = ["shared", "perseq", "perpos"]
MODES = {"shared": 0, "perpos": 1, "perseq": 2}
GOLDEN_CASES = {"login": ("login_ce", {}), "login_clamped": ("login_ce", dict(log_eps=1e-3, clamp=4.37)),
                "weighted": ("ce_weighted", {})}

# replay/nn/loss/__init__.py: __all__ of the reference's package
REFERENCE_ALL = ["BCE", "CE", "BCESampled", "CESampled", "CESampledWeighted", "CEWeighted", "LogInCE", "LogInCESampled",
                 "LogOutCE", "LogOutCESampled", "LogOutCEWeighted", "LossProto"]


def _golden(golden_dir):
    z = np.load(os.path.join(golden_dir, "sasrec_new_tiny.npz"))
    sd = {k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd::")}
    return z, sd, np.load(os.path.join(golden_dir, "sampled_ext_losses.npz"))


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("case", sorted(GOLDEN_CASES))
def test_oracle_matches_reference_goldens(golden_dir, case, shape):
    z, sd, zx = _golden(golden_dir)
    P = osr.params_from_new_state_dict(sd)
    ids, pm = torch.from_numpy(z["ids"]), torch.from_numpy(z["pad_mask"])
    labels, tm = torch.from_numpy(z["labels"]), torch.from_numpy(z["target_mask"])
    kind, kw = GOLDEN_CASES[case]
    if kind == "ce_weighted":
        kw = dict(kw, weights=torch.from_numpy(zx["weights"]))
    l, G = osx.loss_and_grads(P, ids, pm, labels, tm, torch.from_numpy(zx["neg_" + shape]), int(z["H"]), kind,
                              ignore_index=int(zx["ignore_index"]), **kw)
    torch.testing.assert_close(l, torch.from_numpy(zx[f"{case}_{shape}_loss"]), rtol=2e-5, atol=2e-6)
    torch.testing.assert_close(G["item_emb"], torch.from_numpy(zx[f"{case}_{shape}_gE"]), rtol=1e-4, atol=2e-6)
    torch.testing.assert_close(G["blocks"][0]["in_w"], torch.from_numpy(zx[f"{case}_{shape}_gW"]), rtol=1e-4, atol=2e-6)


def test_goldens_cover_the_edges(golden_dir):
    """Each layout has an ignore-index negative and a negative equal to its row's positive; the weights hold zeros,
    negative and non-uniform values; in each layout the tight clamp is active on some rows, and no row's log(p + eps) lies
    within 0.02 of the border (bf16 logits move it by under 0.01, so the engine clamps the same rows as the reference)."""
    z, sd, zx = _golden(golden_dir)
    labels, tm = torch.from_numpy(z["labels"]), torch.from_numpy(z["target_mask"])
    ign = int(zx["ignore_index"])
    for shape in SHAPES:
        neg = torch.from_numpy(zx["neg_" + shape])
        full = {"shared": lambda: neg.expand(*labels.shape, -1), "perseq": lambda: neg[:, None, :].expand(-1, labels.shape[1], -1),
                "perpos": lambda: neg}[shape]()[tm]
        assert (full == ign).any(), shape
        assert (full == labels[tm][:, None]).any(), shape
    w = torch.from_numpy(zx["weights"])[tm[..., None]]
    assert (w == 0).any() and (w < 0).any() and w.std() > 0.1
    P = osr.params_from_new_state_dict(sd)
    h = osr.sasrec_body(P, torch.from_numpy(z["ids"]), torch.from_numpy(z["pad_mask"]), int(z["H"]), "new")
    clamp = GOLDEN_CASES["login_clamped"][1]["clamp"]
    for shape in SHAPES:
        z_pos, z_neg, pos, neg = osm.sampled_logits(h, P["item_emb"], labels, torch.from_numpy(zx["neg_" + shape]), tm)
        z_neg = osm.mask_negative_logits(z_neg, neg, pos, ign)
        lg = torch.log(torch.softmax(torch.cat((z_pos, z_neg), -1), -1)[:, 0] + 1e-3).detach()
        assert (lg < -clamp).any() and (lg > -clamp).any(), shape
        assert (lg + clamp).abs().min() > 0.02, shape


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("kind", ["login_ce", "ce_weighted"])
def test_fp64_reference_matches_oracle(kind, mode):
    """The compacted float64 reference of the kernel test against the [B, L, d] restatement, with collisions, duplicates,
    the ignore index, a row whose every negative is rejected and (LogInCE) an active clamp."""
    g = torch.Generator().manual_seed(31 + MODES[mode] + (7 if kind == "login_ce" else 0))
    B, L, d, I, N = 3, 7, 16, 40, 9
    hidden = torch.randn(B, L, d, generator=g, dtype=torch.float64) * 2
    table = torch.randn(I + 1, d, generator=g, dtype=torch.float64) * 0.7
    labels = torch.randint(0, I, (B, L), generator=g)
    tm = torch.rand(B, L, generator=g) < 0.7
    tm[0, 1] = True
    shape = {"shared": (N,), "perseq": (B, N), "perpos": (B, L, N)}[mode]
    neg = torch.randint(0, I, shape, generator=g)
    neg[..., 1] = neg[..., 0]
    neg[..., 5] = I
    if mode == "shared":
        neg[2] = labels[tm][0]
    elif mode == "perseq":
        neg[:, 2] = labels[:, -1]
    else:
        neg[..., 3] = labels
        neg[0, 1, :] = labels[0, 1]                      # every negative rejected
    w = torch.rand(B, L, 1, generator=g, dtype=torch.float64) * 2 - 0.5
    w[0, 2] = 0.0
    kw = dict(log_eps=1e-3, clamp=2.5) if kind == "login_ce" else {}
    h = hidden.clone().requires_grad_(True)
    t = table.clone().requires_grad_(True)
    if kind == "login_ce":
        l_ref = osx.login_ce_sampled(h, t, labels, neg, tm, ignore_index=I, **kw)
    else:
        l_ref = osx.ce_sampled_weighted(h, t, labels, neg, tm, w, ignore_index=I)
    l_ref.backward()
    vi = tm.reshape(-1).nonzero()[:, 0].to(torch.int32)
    hc, yc = hidden.reshape(-1, d)[vi.long()], labels.reshape(-1)[vi.long()]
    neg_c = neg.reshape(-1, N) if mode == "perpos" else neg
    r = sx.reference(hc, table, yc, vi, neg_c, len(vi), sx.LOGIN_CE_SAMPLED if kind == "login_ce" else sx.CE_SAMPLED_WEIGHTED,
                     MODES[mode], L=L, ignore_index=I, row_weight=w.reshape(-1)[vi.long()], chunk=5, **kw)
    d_hidden = torch.zeros(B * L, d, dtype=torch.float64)
    d_hidden[vi.long()] = r["d_hc"]
    for a, b in ((r["loss"], l_ref), (d_hidden.reshape(B, L, d), h.grad), (r["d_table"], t.grad)):
        torch.testing.assert_close(a, b.detach(), rtol=1e-12, atol=1e-12)
    if kind == "login_ce":
        p = torch.softmax(torch.cat(osm.sampled_logits(hidden, table, labels, neg, tm)[:2], -1), -1)[:, 0]
        assert (torch.log(p + 1e-3).abs() > 2.5).any()   # the clamp is active on some rows


def test_loss_package_exports_the_reference_names():
    from replay_b200.nn import loss as L

    for name in REFERENCE_ALL:
        assert hasattr(L, name), name
    assert sorted(L.__all__) == sorted(REFERENCE_ALL)
    from typing import Protocol
    assert issubclass(L.LossProto, Protocol)


def test_selectors():
    from replay_b200.nn import loss as L

    s = L.LogInCESampled()
    assert s.kind == "login_ce_sampled" and s.needs_negatives
    assert s.engine_kwargs() == {"ignore_index": -100, "log_eps": 1e-6, "clamp": 100.0}
    s = L.LogInCESampled(log_epsilon=1e-3, clamp_border=5.5, negative_labels_ignore_index=7)
    assert s.engine_kwargs() == {"ignore_index": 7, "log_eps": 1e-3, "clamp": 5.5}
    w = L.CESampledWeighted("w", negative_labels_ignore_index=3)
    assert w.kind == "ce_sampled_weighted" and w.needs_negatives and w.feature_name == "w"
    assert isinstance(w, L.CESampled) and w.engine_kwargs() == {"ignore_index": 3}
    tm = torch.ones(2, 5, dtype=torch.bool)
    for ft in ({"w": torch.rand(2, 5, 1)}, {"w": torch.rand(2, 5)}):
        rw = w.row_weights(ft, tm)
        assert rw.shape == (2, 5) and torch.equal(rw, ft["w"].reshape(2, 5))
    with pytest.raises(NotImplementedError):
        L.CESampledWeighted("w", label_smoothing=0.1)
    with pytest.raises(TypeError):
        L.LogInCESampled(reduction="sum")
    # the callback surface of the reference's LossProto
    s.logits_callback = len
    assert s.logits_callback is len


def test_sasrec_takes_the_new_selectors_without_a_gpu():
    from replay_b200.nn import loss as L
    from replay_b200.nn.sequential import SasRec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    m = SasRec.from_params(TensorSchema(TensorFeatureInfo("item_id", 50, 50, 64)), embedding_dim=64, num_heads=1,
                           max_sequence_length=8, device="cpu")
    m.loss = L.LogInCESampled(log_epsilon=1e-3)
    assert m.core._loss_spec == ("login_ce_sampled", {"ignore_index": -100, "log_eps": 1e-3, "clamp": 100.0})
    m.loss = L.CESampledWeighted("w")
    assert m.core._loss_spec == ("ce_sampled_weighted", {"ignore_index": -100})
    with pytest.raises(NotImplementedError, match="CESampledWeighted") as e:
        m.loss = object()
    assert "LogInCESampled" in str(e.value) and "BCE" in str(e.value)


class _StubEngine:
    """What SasRecCore._stage touches on an engine."""

    def __init__(self):
        self.sampled, self.calls = None, []

    def set_loss(self, kind, **kw):
        self.sampled = {"kind": kind} if kind.endswith(("_sampled", "_sampled_weighted")) else None
        self.calls.append(("set_loss", kind))

    def set_batch(self, *a):
        self.calls.append(("set_batch",))

    def set_negatives(self, neg):
        self.calls.append(("set_negatives",))

    def set_row_weights(self, w):
        self.calls.append(("set_row_weights", tuple(w.shape)))


def test_core_stages_the_weights_of_the_sampled_weighted_loss():
    from replay_b200.core import SasRecCore
    from replay_b200.engine import EncoderConfig

    core = SasRecCore(EncoderConfig(n_items=50, d=64, n_heads=1, n_blocks=1, max_len=8, variant="new"), device="cpu")
    ids = torch.zeros(2, 8, dtype=torch.int64)
    pm = torch.ones(2, 8, dtype=torch.bool)
    neg = torch.zeros(5, dtype=torch.int64)
    core.set_loss("ce_sampled_weighted", ignore_index=-100)
    eng = _StubEngine()
    core._stage(eng, ids, pm, ids, pm, neg, torch.ones(2, 8))
    assert eng.calls == [("set_loss", "ce_sampled_weighted"), ("set_batch",), ("set_negatives",), ("set_row_weights", (2, 8))]
    with pytest.raises(ValueError, match="sample weights"):
        core._stage(_StubEngine(), ids, pm, ids, pm, neg, None)
    core.set_loss("login_ce_sampled", ignore_index=-100, log_eps=1e-6, clamp=100.0)
    eng = _StubEngine()
    core._stage(eng, ids, pm, ids, pm, neg, None)
    assert [c[0] for c in eng.calls] == ["set_loss", "set_batch", "set_negatives"]


def _engine_stub(T=12, B=2, L=6, dp=64):
    from replay_b200._lib import lib

    f32, i32 = dict(dtype=torch.float32), dict(dtype=torch.int32)
    from replay_b200.engine import SasRecEngine

    return SimpleNamespace(SAMPLED_KINDS=SasRecEngine.SAMPLED_KINDS, T=T, B=B, L=L, dev="cpu", cfg=SimpleNamespace(dp=dp, n_items=50), lib=lib(), sce=None,
                           _loss_args=None, hc=torch.zeros(T, dp, dtype=torch.bfloat16),
                           params16={"item_emb": torch.zeros(51, dp, dtype=torch.bfloat16)}, labels_c=torch.zeros(T, **i32),
                           valid_idx=torch.zeros(T, **i32), n_valid=torch.zeros(1, **i32),
                           ce=SimpleNamespace(loss=torch.zeros(2, **f32)))


@pytest.mark.parametrize("kind,code", [("login_ce_sampled", 4), ("ce_sampled_weighted", 5)])
def test_engine_sets_up_the_new_kinds(kind, code):
    from replay_b200.engine import SasRecEngine

    e = _engine_stub()
    e._alloc_row_weights = lambda: SasRecEngine._alloc_row_weights(e)
    SasRecEngine.set_loss(e, kind, n_neg=5, neg_shape="perpos", ignore_index=7, log_eps=1e-3, clamp=5.5)
    sp = e.sampled
    assert sp["kind"] == code and sp["mode"] == 1 and sp["neg"].shape == (12, 5)
    assert (sp["ignore_index"], sp["log_eps"], sp["clamp"]) == (7, 1e-3, 5.5)
    sd = SasRecEngine._sampled_desc(e)
    assert sd.kind == code and abs(sd.log_eps - 1e-3) < 1e-9 and sd.clamp == 5.5
    if kind == "ce_sampled_weighted":
        assert e.in_roww.shape == (12,) and e.roww_c.shape == (12,)
        assert sd.row_weight == e.roww_c.data_ptr()
        SasRecEngine.set_row_weights(e, torch.full((2, 6), 0.5))
        assert (e.in_roww == 0.5).all()
    else:
        assert not sd.row_weight and not hasattr(e, "in_roww")


def test_c_abi_rejects_the_weighted_kind_without_weights():
    """Argument errors are decided before any CUDA call, so they are checked here without a GPU."""
    from replay_b200._lib import SampledDesc, lib

    L = lib()
    EINVAL = -1
    buf = torch.zeros(64, dtype=torch.float32)   # any non-null pointer: nothing is read before the checks fail
    p = buf.data_ptr()
    sd = SampledDesc()
    sd.hc = sd.table = sd.labels = sd.valid_idx = sd.negatives = sd.n_valid = sd.loss_out = sd.workspace = p
    sd.capacity, sd.n_items, sd.d, sd.n_neg, sd.neg_mode, sd.seq_len = 16, 50, 64, 5, 1, 8
    sd.workspace_bytes = 1 << 30
    sd.kind = 5
    assert L.rp_sampled_head_fwd(ctypes.byref(sd), None) == EINVAL
    assert L.rp_sampled_head_bwd(ctypes.byref(sd), p, p, None) == EINVAL
    sd.kind, sd.row_weight = 6, p
    assert L.rp_sampled_head_fwd(ctypes.byref(sd), None) == EINVAL
