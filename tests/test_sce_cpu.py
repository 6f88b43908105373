"""CPU tests of the scalable cross-entropy loss: the restatement (oracle/sce.py) against the real reference
(tests/golden/sce_losses.npz), the SCEParams mirror and the legacy SasRec constructor's errors.  No kernel is launched."""
import dataclasses
import os

import numpy as np
import pytest
import torch

CASES = ["nomix", "mix", "bigx", "overlap", "fullcollide", "r111", "r221"]


def _legacy_tiny(golden_dir):
    z = np.load(os.path.join(golden_dir, "sasrec_legacy_tiny.npz"))
    sd = {k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd::")}
    return z, sd


def _real_rows(top, pm):
    """per bucket, the set of selected rows that are real positions (pad rows picked at -inf carry nothing)"""
    return [sorted(int(t) for t in row if pm[int(t)]) for row in top]


@pytest.mark.parametrize("case", CASES)
def test_restatement_matches_reference(golden_dir, case):
    from oracle import sasrec as osr
    from oracle import sce

    z, sd = _legacy_tiny(golden_dir)
    zs = np.load(os.path.join(golden_dir, "sce_losses.npz"))
    n_b, bsx, bsy, mix = (int(v) for v in zs[f"{case}_params"])
    P = osr.params_from_legacy_state_dict(sd)
    ids, pm = torch.from_numpy(z["ids"]), torch.from_numpy(z["pad_mask"])
    labels = torch.from_numpy(zs[f"{case}_labels"])
    draw = torch.from_numpy(zs[f"{case}_draw"])
    loss, G, tx, ty = sce.loss_and_grads(P, ids, pm, labels, int(z["H"]), draw, bsx, bsy, bool(mix))
    pmf = pm.reshape(-1)
    assert _real_rows(tx, pmf) == _real_rows(torch.from_numpy(zs[f"{case}_top_x"]), pmf)
    assert [sorted(r) for r in ty.tolist()] == [sorted(r) for r in zs[f"{case}_top_y"].tolist()]
    ref = torch.from_numpy(zs[f"{case}_loss"]).double()
    assert torch.allclose(loss.double(), ref, rtol=1e-5, atol=1e-6), (float(loss), float(ref))
    for a, b in ((G["item_emb"], zs[f"{case}_gE"]), (G["blocks"][0]["in_w"], zs[f"{case}_gW"])):
        b = torch.from_numpy(b)
        assert torch.allclose(a, b, rtol=1e-4, atol=1e-6 * max(1.0, float(b.abs().max()))), float((a - b).abs().max())


def test_golden_cases_cover_the_edges(golden_dir):
    """The golden exercises what the issue pins: both mix_x settings, bucket_size_x above the real rows, rows selected by
    several buckets (and tied maxima), label collisions including rows whose CE is exactly 0, the (1, 1, 1) and (2, 2, 1)
    shapes, and a top-k margin the bf16 inputs of the CUDA head cannot cross."""
    from oracle import sce

    z, sd = _legacy_tiny(golden_dir)
    zs = np.load(os.path.join(golden_dir, "sce_losses.npz"))
    pm = torch.from_numpy(z["pad_mask"]).reshape(-1)
    assert {int(zs[f"{c}_params"][3]) for c in CASES} == {0, 1}
    assert int(zs["bigx_params"][1]) > int(pm.sum())
    assert all(float(zs[f"{c}_margin"]) > 1 for c in CASES)
    counts = torch.bincount(torch.from_numpy(zs["overlap_top_x"]).reshape(-1), minlength=pm.numel())
    assert int(counts[pm].max()) >= 3
    lab = torch.from_numpy(zs["overlap_labels"]).reshape(-1)
    tx, ty = torch.from_numpy(zs["overlap_top_x"]), torch.from_numpy(zs["overlap_top_y"])
    assert int((lab[tx].unsqueeze(-1) == ty.unsqueeze(1)).sum()) > 10
    # bs_y = 1 with labels set to the bucket's item: some selected real rows have CE exactly 0 in every bucket
    from oracle import sasrec as osr
    P = osr.params_from_legacy_state_dict(sd)
    h = osr.sasrec_body(P, torch.from_numpy(z["ids"]), torch.from_numpy(z["pad_mask"]), int(z["H"]), "legacy")
    x = h.reshape(-1, h.shape[-1])
    lab = torch.from_numpy(zs["fullcollide_labels"]).reshape(-1)
    txf, tyf = torch.from_numpy(zs["fullcollide_top_x"]), torch.from_numpy(zs["fullcollide_top_y"])
    ce = sce.row_losses(x, lab, P["item_emb"][:-1], txf, tyf)
    per_row = torch.zeros(x.shape[0]).scatter_reduce(0, txf.reshape(-1), ce.reshape(-1), reduce="amax", include_self=False)
    assert bool(((per_row == 0) & pm & torch.isin(torch.arange(x.shape[0]), txf)).any())
    for c, shape in (("r111", (1, 1, 1)), ("r221", (2, 2, 1))):
        assert tuple(int(v) for v in zs[f"{c}_params"][:3]) == shape


def test_restatement_no_counted_row_gives_nan():
    from oracle import sce

    x = torch.randn(4, 8, dtype=torch.float64, requires_grad=True)
    w = torch.randn(5, 8, dtype=torch.float64)
    y = torch.tensor([1, 2, 3, 4])
    pm = torch.tensor([False, True, True, False])
    # one item per bucket equal to every selected row's label: every CE is exactly 0
    top_x = torch.tensor([[1, 2]])
    top_y = torch.tensor([[2]])
    y = torch.tensor([0, 2, 2, 0])
    loss, _, _ = sce.sce_loss(x, y, w, pm, torch.randn(1, 8), 2, 1, top_x=top_x, top_y=top_y)
    assert torch.isnan(loss)


def test_sce_params_mirror():
    from replay_b200.models.nn.loss import SCEParams

    p = SCEParams(n_buckets=4, bucket_size_x=8, bucket_size_y=16)
    assert p.mix_x is False and p._get_not_none_params() == [4, 8, 16]
    with pytest.raises(dataclasses.FrozenInstanceError):
        p.n_buckets = 5
    assert SCEParams(1, 2, 3, True) == SCEParams(n_buckets=1, bucket_size_x=2, bucket_size_y=3, mix_x=True)


def _schema(n=300, d=64):
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    return TensorSchema(TensorFeatureInfo("item_id", n, n, d))


def test_legacy_sasrec_sce_constructor_errors():
    from replay_b200.models.nn.loss import SCEParams
    from replay_b200.models.nn.sequential import SasRec

    with pytest.raises(AssertionError, match="sce_params"):
        SasRec(_schema(), hidden_size=64, max_seq_len=8, loss_type="SCE", device="cpu")
    with pytest.raises(AssertionError, match="n_buckets"):
        SasRec(_schema(), hidden_size=64, max_seq_len=8, loss_type="SCE", sce_params=SCEParams(None, 2, 3), device="cpu")
    with pytest.raises(ValueError, match="bucket_size_y"):
        SasRec(_schema(), hidden_size=64, max_seq_len=8, loss_type="SCE", sce_params=SCEParams(2, 2, 301), device="cpu")
    with pytest.raises(ValueError, match="bucket_size_y"):
        SasRec(_schema(5000), hidden_size=64, max_seq_len=8, loss_type="SCE", sce_params=SCEParams(2, 2, 1025), device="cpu")
    m = SasRec(_schema(), hidden_size=64, max_seq_len=8, loss_type="SCE", sce_params=SCEParams(2, 17, 300), device="cpu")
    assert m._model.core._loss_spec == ("sce", dict(n_buckets=2, bucket_size_x=17, bucket_size_y=300, mix_x=False))
    # bucket_size_x is bounded by B * L of the batch: checked at the first batch, before any kernel runs
    b = {"feature_tensor": {"item_id": torch.ones(2, 8, dtype=torch.long)}, "padding_mask": torch.ones(2, 8, dtype=torch.bool),
         "positive_labels": torch.ones(2, 8, dtype=torch.long), "target_padding_mask": torch.ones(2, 8, dtype=torch.bool)}
    with pytest.raises(ValueError, match="bucket_size_x"):
        m.training_step(b, 0)
