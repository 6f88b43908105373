"""Multi-positive targets ([B, L, P] labels and target mask) without a GPU:
(a) the plain-torch restatement (oracle/multi_positive.py) against the real reference's losses and gradients
    (tests/golden/multi_positive_losses.npz: BCE, CESampled, BCESampled, CESampledWeighted, P = 3, every negative layout);
(b) every loss that takes one positive per position raises NotImplementedError, naming itself, from SasRec.forward and from
    LightningModule.training_step alike, and so does TwoTower; more than 32 positives raise ValueError;
(c) the C ABI: the fields appended to rp_sampled_desc, their ctypes mirror and the new entry points."""
import os
import re

import numpy as np
import pytest
import torch

from oracle import multi_positive as omp
from oracle import sasrec as osr

CASES = [("bce", "none"), *[(k, s) for k in ("ce_sampled", "bce_sampled", "ce_sampled_weighted")
                            for s in ("shared", "perseq", "perpos")]]


def _load(golden_dir):
    z = np.load(os.path.join(golden_dir, "sasrec_new_tiny.npz"))
    sd = {k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd::")}
    return z, sd, np.load(os.path.join(golden_dir, "multi_positive_losses.npz"))


@pytest.mark.parametrize("kind,shape", CASES)
def test_restatement_matches_reference(golden_dir, kind, shape):
    z, sd, zm = _load(golden_dir)
    P = {k: (v.double() if torch.is_tensor(v) else [{kk: vv.double() for kk, vv in b.items()} for b in v])
         for k, v in osr.params_from_new_state_dict(sd).items()}
    ids, pm = torch.from_numpy(z["ids"]), torch.from_numpy(z["pad_mask"])
    lab, m = torch.from_numpy(zm["labels"]), torch.from_numpy(zm["target_mask"])
    kw = {}
    if kind != "bce":
        kw["ignore_index"] = int(zm["ignore_index"])
    if kind == "ce_sampled_weighted":
        kw["weights"] = torch.from_numpy(zm["weights"]).double()
    neg = torch.from_numpy(zm["neg_" + shape]) if kind != "bce" else None
    loss, G = omp.loss_and_grads(P, ids, pm, lab, m, neg, int(z["H"]), kind, **kw)
    ref = float(zm[f"{kind}_{shape}_loss"])
    assert abs(float(loss) - ref) <= 2e-5 * abs(ref), (float(loss), ref)
    torch.testing.assert_close(G["item_emb"].float(), torch.from_numpy(zm[f"{kind}_{shape}_gE"]), rtol=2e-4, atol=2e-6)
    torch.testing.assert_close(G["blocks"][0]["in_w"].float(), torch.from_numpy(zm[f"{kind}_{shape}_gW"]), rtol=2e-4,
                               atol=2e-6)


def test_golden_batch_has_the_edge_cases(golden_dir):
    _, _, zm = _load(golden_dir)
    lab, m = torch.from_numpy(zm["labels"]), torch.from_numpy(zm["target_mask"])
    live = m.any(-1)
    assert (live & ~m.all(-1)).any()                                     # padded slots inside live rows
    assert (live & (m.sum(-1) == 1)).any()                                # live positions with one set slot
    dup = (lab.unsqueeze(-1) == lab.unsqueeze(-2)) & m.unsqueeze(-1) & m.unsqueeze(-2) & ~torch.eye(3, dtype=torch.bool)
    assert dup.any()                                                      # a duplicated id within a row
    ign = int(zm["ignore_index"])
    for shape in ("shared", "perseq", "perpos"):
        neg = torch.from_numpy(zm["neg_" + shape])
        assert (neg == ign).any()
        full = neg.view(1, 1, -1) if neg.dim() == 1 else (neg.unsqueeze(1) if neg.dim() == 2 else neg)
        full = full.expand(lab.shape[0], lab.shape[1], -1)
        for k, want in ((1, True), (2, False)):   # a set non-first positive; a padded slot's value
            sel = live & (m[..., k] == want)
            assert (full[sel] == lab[..., k][sel].unsqueeze(-1)).any(), (shape, k)


# ----------------------------------------------------------------------------------------------------------------------
# (b) raising cases
# ----------------------------------------------------------------------------------------------------------------------
def _cpu_model(loss):
    from replay_b200.nn.sequential import SasRec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    m = SasRec.from_params(TensorSchema(TensorFeatureInfo("item_id", 50, 50, 64)), embedding_dim=64, num_heads=2,
                           num_blocks=1, max_sequence_length=8, dropout=0.0, device="cpu")
    m.core.set_loss = lambda *a, **k: None   # no engine on the CPU: the loss is only recorded
    m.loss = loss
    m.train()
    return m


def _batch(P, B=2, L=8):
    return {"feature_tensors": {"item_id": torch.zeros(B, L, dtype=torch.long), "w": torch.ones(B, L, P)},
            "padding_mask": torch.ones(B, L, dtype=torch.bool),
            "positive_labels": torch.zeros(B, L, P, dtype=torch.long),
            "target_padding_mask": torch.ones(B, L, P, dtype=torch.bool),
            "negative_labels": torch.zeros(4, dtype=torch.long)}


def _raising():
    from replay_b200.nn import loss as L

    return {"CE": (L.CE(), "the CE loss"), "CEWeighted": (L.CEWeighted("w"), "the CE loss"),
            "LogInCE": (L.LogInCE(50), "the LogInCE loss"), "LogInCESampled": (L.LogInCESampled(), "the LogInCESampled loss"),
            "LogOutCE": (L.LogOutCE(50), "the LogOutCE loss"),
            "LogOutCEWeighted": (L.LogOutCEWeighted(50, "w"), "the LogOutCEWeighted loss")}


@pytest.mark.parametrize("name", ["CE", "CEWeighted", "LogInCE", "LogInCESampled", "LogOutCE", "LogOutCEWeighted"])
def test_single_positive_losses_raise(name):
    from replay_b200.nn.lightning import LightningModule

    loss, msg = _raising()[name]
    m = _cpu_model(loss)
    b = _batch(3)
    with pytest.raises(NotImplementedError, match=f"multi-positive labels is not supported in {msg}"):
        m(**b)
    lm = LightningModule(m)
    with pytest.raises(NotImplementedError, match=f"multi-positive labels is not supported in {msg}"):
        lm.training_step(b, 0)


def test_reference_message_for_ce():
    m = _cpu_model(_raising()["CE"][0])
    with pytest.raises(NotImplementedError, match="^The case of multi-positive labels is not supported in the CE loss$"):
        m(**_batch(2))


def test_two_tower_raises():
    from replay_b200.nn.loss import CESampled
    from replay_b200.nn.sequential.twotower import TwoTower

    tt = TwoTower.__new__(TwoTower)
    torch.nn.Module.__init__(tt)
    tt._loss = CESampled()
    with pytest.raises(NotImplementedError, match="not supported in TwoTower"):
        tt.check_positives(torch.zeros(2, 8, 2, dtype=torch.long), torch.ones(2, 8, 2, dtype=torch.bool))
    lab, tm = tt.check_positives(torch.zeros(2, 8, 1, dtype=torch.long), torch.ones(2, 8, 1, dtype=torch.bool))
    assert lab.shape == (2, 8) and tm.shape == (2, 8)


@pytest.mark.parametrize("name", ["BCE", "CESampled", "BCESampled", "CESampledWeighted"])
def test_positive_cap(name):
    from replay_b200.nn import loss as L

    spec = {"BCE": L.BCE(), "CESampled": L.CESampled(), "BCESampled": L.BCESampled(),
            "CESampledWeighted": L.CESampledWeighted("w")}[name]
    L.check_multi_positive(spec, 32)
    with pytest.raises(ValueError, match="at most 32"):
        L.check_multi_positive(spec, 33)
    with pytest.raises(ValueError, match="at most 32"):
        _cpu_model(spec)(**_batch(33))


def test_single_slot_is_the_plain_batch():
    from replay_b200.nn.loss import CE

    m = _cpu_model(CE())
    lab, tm = m.check_positives(torch.arange(16).view(2, 8, 1), torch.ones(2, 8, 1, dtype=torch.bool))
    assert lab.shape == (2, 8) and tm.shape == (2, 8) and lab[1, 3] == 11


def test_weighted_loss_keeps_per_pair_weights():
    from replay_b200.nn.loss import CESampledWeighted

    spec = CESampledWeighted("w")
    w = torch.rand(2, 8, 3)
    assert spec.row_weights({"w": w}, torch.ones(2, 8, 3, dtype=torch.bool)) is w
    assert spec.row_weights({"w": w[..., :1]}, torch.ones(2, 8, dtype=torch.bool)).shape == (2, 8)


# ----------------------------------------------------------------------------------------------------------------------
# (c) ABI
# ----------------------------------------------------------------------------------------------------------------------
def _header():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "include", "rp_b200.h")) as fh:
        return fh.read()


def test_sampled_desc_mirror_appends_the_new_fields():
    from replay_b200._lib import MAX_POSITIVES, SampledDesc

    names = [f[0] for f in SampledDesc._fields_]
    assert names[-4:] == ["row_weight", "num_positives", "slot_mask", "n_pairs"]
    body = re.search(r"typedef struct rp_sampled_desc \{(.*?)\} rp_sampled_desc;", _header(), re.S).group(1)
    assert "int num_positives; const uint8_t* slot_mask; const int32_t* n_pairs;" in body.splitlines()[-1 if body.splitlines()[-1].strip() else -2]
    assert SampledDesc().num_positives == 0 and SampledDesc().slot_mask is None   # zero / NULL: one positive per position
    assert re.search(r"#define RP_MAX_POSITIVES (\d+)", _header()).group(1) == str(MAX_POSITIVES) == "32"


def test_new_entry_points_are_declared_and_exported():
    from replay_b200._lib import LIB_PATH, _EXTRA_SIGS

    names = ["rp_prepare_batch_multi", "rp_sampled_head_workspace_multi", "rp_bce_head_multi_fwd", "rp_bce_head_multi_bwd"]
    h = _header()
    sigs = {n for n, _, _ in _EXTRA_SIGS}
    for n in names:
        assert re.search(rf"\b{n}\(", h), n
        assert n in sigs, n
    if os.path.exists(LIB_PATH):
        from replay_b200._lib import lib

        for n in names:
            assert hasattr(lib(), n), n
