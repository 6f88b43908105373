"""CPU checks of the full-catalog BCE head's reference and selectors: the float64 restatement equals torch's
BCEWithLogitsLoss (the reference's computation) and autograd, each plausible kernel mistake moves a compared quantity by at
least 10x its bound, and the selectors reach the engines without a GPU."""
import pytest
import torch

from bce_reference import reference, worst


def _inputs(cap=96, n_valid=70, I=300, d=64, seed=0):
    g = torch.Generator().manual_seed(seed)
    h = (torch.randn(cap, d, generator=g) * 0.5).bfloat16()
    h[n_valid:] = (torch.randn(cap - n_valid, d, generator=g) * 2.0 + 1.0).bfloat16()
    W = (torch.randn(I, d, generator=g) * 0.3).bfloat16()
    b = torch.randn(I, generator=g) * 0.5
    y = torch.randint(0, I, (cap,), generator=g, dtype=torch.int32)
    return h, W, b, y, n_valid


def test_reference_is_bce_with_logits_and_its_gradient():
    h, W, b, y, nv = _inputs()
    r = reference(h, W, b, y, nv)
    hh = h[:nv].double().requires_grad_()
    WW = W.double().requires_grad_()
    bb = b.double().requires_grad_()
    x = hh @ WW.T + bb
    target = torch.nn.functional.one_hot(y[:nv].long(), W.shape[0]).double()
    loss = torch.nn.BCEWithLogitsLoss(reduction="sum")(x, target) / nv
    loss.backward()
    torch.testing.assert_close(r["loss"], loss.detach(), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(r["d_h"], hh.grad, rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(r["d_W"], WW.grad, rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(r["d_b"], bb.grad, rtol=1e-10, atol=1e-12)


def test_empty_batch_reference():
    h, W, b, y, _ = _inputs()
    r = reference(h, W, b, y, 0)
    assert float(r["loss"]) == 0.0 and r["d_W"].abs().max() == 0 and r["d_b"].abs().max() == 0


def _mutants(h, W, b, y, nv):
    """quantities a kernel with each plausible mistake would report"""
    cap, I = h.shape[0], W.shape[0]
    hd, Wd, bd = h.double(), W.double(), b.double()
    out = {}
    # rows past n_valid not masked in the dE pass: every row's sigmoid reaches d_table / d_bias
    g_all = torch.sigmoid(hd @ Wd.T + bd)
    g_all[torch.arange(nv), y[:nv].long()] -= 1.0
    out["unmasked padded rows"] = dict(d_W=(g_all.T @ hd) / nv, d_b=g_all.sum(0) / nv)
    # the bias factored out of the sigmoid in the dE pass, as CE factors e^b out of the exponential
    x = hd[:nv] @ Wd.T
    g = torch.sigmoid(x) * torch.exp(bd)[None, :]
    g[torch.arange(nv), y[:nv].long()] -= 1.0
    out["bias outside the sigmoid"] = dict(d_W=(g.T @ hd[:nv]) / nv, d_b=g.sum(0) / nv)
    # the one-hot part missing
    xb = x + bd
    s = torch.sigmoid(xb) / nv
    out["one-hot part missing"] = dict(d_h=s @ Wd, d_W=s.T @ hd[:nv], d_b=s.sum(0))
    # mean over M * |I| instead of M
    r = reference(h, W, b, y, nv)
    out["divided by M |I|"] = {k: r[k] / I for k in ("loss", "d_h", "d_W", "d_b")}
    # sigmoid and softplus swapped
    sp = torch.nn.functional.softplus(xb)
    gs = sp.clone()
    gs[torch.arange(nv), y[:nv].long()] -= 1.0
    gs /= nv
    xy = xb.gather(1, y[:nv].long()[:, None]).sum()
    out["sigmoid and softplus swapped"] = dict(loss=(torch.sigmoid(xb).sum() - xy) / nv, d_h=gs @ Wd, d_W=gs.T @ hd[:nv])
    return out


def test_each_plausible_mistake_moves_a_compared_quantity_by_10x_its_bound():
    h, W, b, y, nv = _inputs()
    r = reference(h, W, b, y, nv)
    bounds = {"loss": r["bound_loss"], "d_h": r["bound_h"], "d_W": r["bound_W"], "d_b": r["bound_b"]}
    for name, q in _mutants(h, W, b, y, nv).items():
        moved = max(worst(v, r[k], bounds[k]) for k, v in q.items())
        assert moved >= 10.0, (name, moved)


def test_bounds_cover_bf16_rounding_of_the_sigmoid():
    """the bound admits what the kernel does: sigmoid rounded to bf16 as the MMA operand, fp32 sums, bf16 d_h"""
    h, W, b, y, nv = _inputs(I=5000)
    r = reference(h, W, b, y, nv)
    x = (h[:nv].float() @ W.float().T + b.float())
    s = torch.sigmoid(x).bfloat16().float()
    g = s.clone()
    g[torch.arange(nv), y[:nv].long()] -= 1.0
    d_h = ((s @ W.float() - W.float()[y[:nv].long()]) / nv).bfloat16()
    d_W = (s.T @ h[:nv].float() - torch.zeros_like(W.float()).index_add_(0, y[:nv].long(), h[:nv].float())) / nv
    assert worst(d_h, r["d_h"], r["bound_h"]) <= 1.0
    assert worst(d_W, r["d_W"], r["bound_W"]) <= 1.0


def test_selectors():
    from replay_b200.core import SasRecCore
    from replay_b200.nn.loss import BCE

    assert BCE().kind == "bce" and BCE().engine_kwargs() == {} and not BCE().needs_negatives
    with pytest.raises(NotImplementedError):
        BCE(pos_weight=torch.ones(3))
    with pytest.raises(NotImplementedError):
        BCE(weight=torch.ones(3))
    assert "bce" in SasRecCore._FULL_CATALOG


def test_sasrec_loss_setter_lists_bce():
    from replay_b200.nn.sequential import SasRec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    m = SasRec.from_params(TensorSchema(TensorFeatureInfo("item_id", 50, 50, 64)), embedding_dim=64, num_heads=1,
                           max_sequence_length=8, device="cpu")
    with pytest.raises(NotImplementedError, match="BCE"):
        m.loss = object()


def test_bert4rec_loss_types():
    from replay_b200.models.nn.sequential import Bert4Rec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    schema = TensorSchema(TensorFeatureInfo("item_id", 50, 0, 64))
    kinds = {lt: Bert4Rec(schema, hidden_size=64, head_count=1, max_seq_len=8, loss_type=lt, device="cpu")._model.core.loss_kind
             for lt in ("CE", "CE_restricted", "BCE")}
    assert kinds == {"CE": "ce", "CE_restricted": "ce", "BCE": "bce"}
    for kw in (dict(loss_type="BCE", loss_sample_count=8), dict(loss_type="CE", loss_sample_count=8),
               dict(loss_type="SCE"), dict(loss_type="CESampled")):
        with pytest.raises(NotImplementedError):
            Bert4Rec(schema, hidden_size=64, head_count=1, max_seq_len=8, device="cpu", **kw)


def test_bert_engine_rejects_sampled_kinds():
    from replay_b200.engine_bert import Bert4RecEngine

    class _E:   # set_loss only touches these attributes
        pass

    e = _E()
    for kind in ("ce", "bce"):
        Bert4RecEngine.set_loss(e, kind)
        assert e.bce == (kind == "bce") and e.sampled is None
    for kind in ("ce_sampled", "bce_sampled", "legacy_ce_sampled", "login_ce"):
        with pytest.raises(NotImplementedError):
            Bert4RecEngine.set_loss(e, kind)
