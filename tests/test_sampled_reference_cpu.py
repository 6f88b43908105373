"""Pins the float64 sampled-head reference of the kernel-level GPU test (tests/sampled_reference.py, compacted rows) against
the restatement over [B, L, d] hidden states (oracle/sampled.py) and against losses and gradients of the reference's own
classes (tests/golden/sampled_losses.npz).  CPU only."""
import os

import numpy as np
import pytest
import torch

import sampled_reference as sr
from oracle import sampled as osm
from oracle import sasrec as osr

KINDS = {"ce": sr.CE_SAMPLED, "bce": sr.BCE_SAMPLED, "legacy_ce": sr.LEGACY_CE, "legacy_bce": sr.LEGACY_BCE}
MODES = {"shared": 0, "perpos": 1, "perseq": 2}


def _compact(target_mask):
    """valid_idx: the flat b * L + l positions of the valid targets, ascending (rp_prepare_batch's order)."""
    return target_mask.reshape(-1).nonzero()[:, 0].to(torch.int32)


def _ours(hidden, table, labels, target_mask, neg, kind, mode, **kw):
    """Loss, d(hidden) [B, L, d] and d(table) of the compacted reference, from [B, L, ...] inputs."""
    B, L, d = hidden.shape
    vi = _compact(target_mask)
    hc, yc = hidden.reshape(-1, d)[vi.long()], labels.reshape(-1)[vi.long()]
    neg_c = neg.reshape(-1, neg.shape[-1]) if mode == 1 else neg
    r = sr.reference(hc, table, yc, vi, neg_c, len(vi), KINDS[kind], mode, L=L, chunk=5, **kw)
    d_hidden = torch.zeros(B * L, d, dtype=torch.float64)
    d_hidden[vi.long()] = r["d_hc"]
    return r["loss"], d_hidden.reshape(B, L, d), r["d_table"]


def _oracle(hidden, table, labels, target_mask, neg, kind, **kw):
    h = hidden.clone().requires_grad_(True)
    t = table.clone().requires_grad_(True)
    fn = {"ce": osm.ce_sampled, "bce": osm.bce_sampled, "legacy_ce": osm.legacy_ce_sampled,
          "legacy_bce": osm.legacy_bce_sampled}[kind]
    loss = fn(h, t, labels, neg, target_mask, **kw)
    loss.backward()
    return loss.detach(), h.grad, t.grad


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("kind", sorted(KINDS))
def test_reference_matches_oracle_restatement(kind, mode):
    """Random batch with collisions, duplicates and ignore_index entries; [B, L, d] oracle vs compacted reference."""
    g = torch.Generator().manual_seed(10 * sorted(KINDS).index(kind) + MODES[mode])
    B, L, d, I, N = 3, 7, 16, 40, 9
    hidden = torch.randn(B, L, d, generator=g, dtype=torch.float64)
    table = torch.randn(I + 1, d, generator=g, dtype=torch.float64) * 0.7
    labels = torch.randint(0, I, (B, L), generator=g)
    tm = torch.rand(B, L, generator=g) < 0.7
    shape = {"shared": (N,), "perseq": (B, N), "perpos": (B, L, N)}[mode]
    neg = torch.randint(0, I, shape, generator=g)
    neg[..., 1] = neg[..., 0]                                       # a duplicate in every list
    if mode == "shared":
        neg[2] = labels[tm][0]
    elif mode == "perseq":
        neg[:, 2] = labels[:, -1]
    else:
        neg[..., 3] = labels
        neg[0, 1, :] = labels[0, 1]                                 # every negative collides (legacy CE: all rejected
        neg[0, 1, 4] = (labels[0, 1] + 1) % I                       # but one)
    kw_ours, kw_or = {}, {}
    if kind in ("ce", "bce"):
        neg[..., 5] = I                                             # the pad id, masked as the ignore index
        kw_ours = kw_or = dict(ignore_index=I)
    if kind == "bce":
        kw_ours, kw_or = dict(kw_ours, log_eps=1e-3, clamp=1.5), dict(kw_or, log_eps=1e-3, clamp=1.5)
        hidden = hidden * 3                                         # logits large enough for the clamp to fire
    if kind == "legacy_ce":
        kw_ours = kw_or = dict(vocab_size=I)
    l_ref, dh_ref, dt_ref = _oracle(hidden, table, labels, tm, neg, kind, **kw_or)
    l, dh, dt = _ours(hidden, table, labels, tm, neg, kind, MODES[mode], **kw_ours)
    # legacy_ce_sampled casts its logits to float32 before the cross entropy
    tol = dict(rtol=1e-6, atol=1e-6) if kind == "legacy_ce" else dict(rtol=1e-12, atol=1e-12)
    for a, b in ((l, l_ref), (dh, dh_ref), (dt, dt_ref)):
        torch.testing.assert_close(a, b.double(), **tol)


def test_reference_legacy_ce_counts_at_most_vocab_size_negatives():
    """With more sampled negatives than the vocabulary the legacy correction divides by min(N, vocab_size) - #reject."""
    g = torch.Generator().manual_seed(4)
    B, L, d, V, N = 2, 5, 8, 6, 11
    hidden = torch.randn(B, L, d, generator=g, dtype=torch.float64)
    table = torch.randn(V + 1, d, generator=g, dtype=torch.float64)
    labels = torch.randint(0, V, (B, L), generator=g)
    tm = torch.ones(B, L, dtype=torch.bool)
    neg = torch.randint(0, V, (B, L, N), generator=g)
    neg[..., 0] = labels
    l_ref, dh_ref, dt_ref = _oracle(hidden, table, labels, tm, neg, "legacy_ce", vocab_size=V)
    l, dh, dt = _ours(hidden, table, labels, tm, neg, "legacy_ce", 1, vocab_size=V)
    for a, b in ((l, l_ref), (dh, dh_ref), (dt, dt_ref)):
        torch.testing.assert_close(a, b.double(), rtol=1e-6, atol=1e-6)


def _golden_step(P, z, neg, kind, mode, variant, **kw):
    """Body of the oracle, the compacted reference as the head, d_hc back through the body: loss, d(item_emb), d(in_w)."""
    Pg = {k: ([{kk: vv.detach().clone().requires_grad_(True) for kk, vv in b.items()} for b in v] if k == "blocks"
              else v.detach().clone().requires_grad_(True)) for k, v in P.items()}
    ids, pm = torch.from_numpy(z["ids"]), torch.from_numpy(z["pad_mask"])
    labels, tm = torch.from_numpy(z["labels"]), torch.from_numpy(z["target_mask"])
    hidden = osr.sasrec_body(Pg, ids, pm, int(z["H"]), variant)
    B, L, d = hidden.shape
    vi = _compact(tm)
    hc = hidden.reshape(-1, d)[vi.long()]
    yc = labels.reshape(-1)[vi.long()]
    r = sr.reference(hc.detach(), Pg["item_emb"].detach(), yc, vi, neg, len(vi), KINDS[kind], mode, L=L, **kw)
    hc.backward(r["d_hc"].to(hc.dtype))
    g_item = Pg["item_emb"].grad.double() + r["d_table"]
    g_item[-1] = 0.0                                               # the padding row of the reference's embedding
    return r["loss"], g_item, Pg["blocks"][0]["in_w"].grad


@pytest.mark.parametrize("loss", ["ce", "bce"])
@pytest.mark.parametrize("shape", ["shared", "perseq", "perpos"])
def test_reference_matches_golden_new_path(golden_dir, loss, shape):
    z = np.load(os.path.join(golden_dir, "sasrec_new_tiny.npz"))
    sd = {k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd::")}
    zs = np.load(os.path.join(golden_dir, "sampled_losses.npz"))
    neg = torch.from_numpy(zs["neg_" + shape])
    neg = neg.reshape(-1, neg.shape[-1]) if shape == "perpos" else neg
    l, gE, gW = _golden_step(osr.params_from_new_state_dict(sd), z, neg, loss, MODES[shape], "new",
                             ignore_index=int(zs["ignore_index"]))
    torch.testing.assert_close(l.float(), torch.from_numpy(zs[f"new_{loss}_{shape}_loss"]), rtol=2e-5, atol=2e-6)
    torch.testing.assert_close(gE.float(), torch.from_numpy(zs[f"new_{loss}_{shape}_gE"]), rtol=1e-4, atol=2e-6)
    torch.testing.assert_close(gW, torch.from_numpy(zs[f"new_{loss}_{shape}_gW"]), rtol=1e-4, atol=2e-6)


@pytest.mark.parametrize("loss", ["ce", "bce"])
def test_reference_matches_golden_legacy(golden_dir, loss):
    z = np.load(os.path.join(golden_dir, "sasrec_legacy_tiny.npz"))
    sd = {k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd::")}
    zs = np.load(os.path.join(golden_dir, "sampled_losses.npz"))
    tm = torch.from_numpy(z["target_mask"])
    nv = torch.from_numpy(zs[f"legacy_{loss}_neg"])               # [M, N] in valid-target order
    neg = torch.zeros(tm.numel(), nv.shape[1], dtype=torch.int64)
    neg[_compact(tm).long()] = nv
    kw = dict(vocab_size=int(z["n_items"])) if loss == "ce" else {}
    l, gE, gW = _golden_step(osr.params_from_legacy_state_dict(sd), z, neg, "legacy_" + loss, 1, "legacy", **kw)
    torch.testing.assert_close(l.float(), torch.from_numpy(zs[f"legacy_{loss}_loss"]), rtol=2e-5, atol=2e-6)
    torch.testing.assert_close(gE.float(), torch.from_numpy(zs[f"legacy_{loss}_gE"]), rtol=1e-4, atol=2e-6)
    torch.testing.assert_close(gW, torch.from_numpy(zs[f"legacy_{loss}_gW"]), rtol=1e-4, atol=2e-6)
