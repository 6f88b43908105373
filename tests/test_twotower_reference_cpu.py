"""tests/twotower_reference.py against oracle/twotower.py and a brute-force compaction, and every bound of
tests/test_gpu_twotower_fp64.py against a plausible mistake at that file's shapes (CPU only)."""
import math

import numpy as np
import pytest
import torch

import diff_reference as dr
import sampled_reference as sr
import twotower_reference as tr
from oracle import sasrec as osr
from oracle import twotower as ott

import test_gpu_twotower_fp64 as gt


def _sd(n, d, seed):
    g = torch.Generator().manual_seed(seed)
    sd = {ott.ITEM_KEYS[0]: torch.randn(n + 1, d, generator=g, dtype=torch.float64)}
    for layer in (1, 2):
        p = f"body.item_tower.encoder.sw{layer}."
        for k, s in (("WG.weight", (2 * d, d)), ("W1.weight", (2 * d, d)), ("W2.weight", (d, 2 * d))):
            sd[p + k] = torch.randn(s, generator=g, dtype=torch.float64) * math.sqrt(2 / (3 * d))
        for k, s in (("WG.bias", 2 * d), ("W1.bias", 2 * d), ("W2.bias", d)):
            sd[p + k] = 0.1 * torch.randn(s, generator=g, dtype=torch.float64)
        sd[f"body.item_tower.encoder.norm{layer}.weight"] = 1 + 0.1 * torch.randn(d, generator=g, dtype=torch.float64)
    sd["body.item_tower.item_reference_item_id"] = torch.arange(n)
    return sd


def _P(sd):
    P = {}
    for layer, p in ((1, "tw0."), (2, "tw1.")):
        q = f"body.item_tower.encoder.sw{layer}."
        P[p + "wgw1"] = torch.cat([sd[q + "WG.weight"], sd[q + "W1.weight"]])
        P[p + "bgb1"] = torch.cat([sd[q + "WG.bias"], sd[q + "W1.bias"]])
        P[p + "w2"], P[p + "b2"] = sd[q + "W2.weight"], sd[q + "W2.bias"]
        P[p + "norm"] = sd[f"body.item_tower.encoder.norm{layer}.weight"]
    return P


# ------------------------------------------------------------------------------------------------ restatement vs oracle
@pytest.mark.parametrize("n,d", [(7, 16), (60, 64)])
def test_tower_equals_oracle(n, d):
    sd = _sd(n, d, n + d)
    want = ott.item_tower(sd)
    got = tr.tower(sd[ott.ITEM_KEYS[0]][:n], _P(sd), 2 * d, d)
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)


def test_padded_tower_equals_true_layout():
    """the padded layout (zero columns and hidden entries) computes the true layout's tower"""
    n, d, dp, F = 9, 50, 64, 128
    sd = _sd(n, d, 3)
    P = _P(sd)
    Pp = {}
    for p in ("tw0.", "tw1."):
        w = torch.zeros(2 * F, dp, dtype=torch.float64)
        w[:2 * d, :d], w[F:F + 2 * d, :d] = P[p + "wgw1"][:2 * d], P[p + "wgw1"][2 * d:]
        b = torch.zeros(2 * F, dtype=torch.float64)
        b[:2 * d], b[F:F + 2 * d] = P[p + "bgb1"][:2 * d], P[p + "bgb1"][2 * d:]
        w2 = torch.zeros(dp, F, dtype=torch.float64)
        w2[:d, :2 * d] = P[p + "w2"]
        Pp.update({p + "wgw1": w, p + "bgb1": b, p + "w2": w2, p + "b2": torch.nn.functional.pad(P[p + "b2"], (0, dp - d)),
                   p + "norm": torch.nn.functional.pad(P[p + "norm"], (0, dp - d))})
    x = sd[ott.ITEM_KEYS[0]][:n]
    got = tr.tower(torch.nn.functional.pad(x, (0, dp - d)), Pp, F, d)
    torch.testing.assert_close(got[:, :d], tr.tower(x, P, 2 * d, d), rtol=1e-12, atol=1e-12)
    assert not got[:, d:].any()


@pytest.mark.parametrize("kind", tr.FULL_KINDS)
def test_full_head_chunked_equals_autograd(kind):
    g = torch.Generator().manual_seed(5)
    n, I, d = 37, 53, 16
    h = torch.randn(n, d, generator=g, dtype=torch.float64, requires_grad=True)
    E = torch.randn(I, d, generator=g, dtype=torch.float64, requires_grad=True)
    y = torch.randint(0, I, (n,), generator=g)
    w = torch.rand(n, generator=g, dtype=torch.float64) + 0.5
    z = h @ E.T
    if kind == "bce":
        want = ott.bce_full(h[None], E, y[None], torch.ones(1, n, dtype=torch.bool))
    elif kind == "ce":
        want = osr.ce_loss(h[None], E, y[None], torch.ones(1, n, dtype=torch.bool))
    else:
        lse = torch.logsumexp(z, -1)
        zy = z[torch.arange(n), y]
        want = (w * (lse - zy)).mean() if kind == "ce_weighted" else \
            (-torch.log(torch.exp(zy - lse) + 1e-6).clamp(-100, 100)).mean()
    want.backward()
    loss, d_h, d_E = tr.full_head_chunked(kind, h.detach(), E.detach(), y, w, rows=8)
    torch.testing.assert_close(loss, want.detach(), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(d_h, h.grad, rtol=1e-10, atol=1e-13)
    torch.testing.assert_close(d_E, E.grad, rtol=1e-10, atol=1e-13)


def _brute(n_items, labels, nv, negatives, n_neg, mode, valid_idx, ignore, cap, n_rows):
    """a plain-Python restatement: python sets, dicts"""
    ents = list(range(n_neg)) if mode == 0 else list(range(n_rows * n_neg)) if mode == 2 else \
        [int(r) * n_neg + j for r in valid_idx[:nv] for j in range(n_neg)]
    flat = list(np.asarray(negatives).reshape(-1))
    items = set()
    for v in list(labels[:nv]) + [flat[e] for e in ents if not (ignore >= 0 and flat[e] == ignore)]:
        items.add(int(v) if 0 <= v < n_items else 0)
    order = sorted(items)[:cap]
    slot = {it: s for s, it in enumerate(order)}
    remap = lambda v: cap if (ignore >= 0 and v == ignore) else slot.get(int(v), -1) if 0 <= v < n_items else cap + 1  # noqa
    return len(order), order, [slot[int(v)] if 0 <= v < n_items else cap + 1 for v in labels[:nv]], [remap(flat[e]) for e in ents]


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("nv", ["zero", "one", "part", "all"])
def test_compaction_restatement_equals_brute_force(mode, nv):
    rng = np.random.default_rng(mode * 10 + len(nv))
    n = 9000
    c = gt.make_case(n, gt._edge_items(n, rng)[:300], mode, 33, nv, (7, -100)[mode % 2], seed=mode)
    ref = tr.compact_ref(c["n_items"], c["labels"], c["n_valid"], len(c["labels"]), c["negatives"], c["n_neg"], c["mode"],
                         c["valid_idx"], c["ignore"], c["cap"], c["n_rows"])
    ns, order, lab, neg = _brute(n, c["labels"], ref["nv"], c["negatives"], c["n_neg"], mode, c["valid_idx"], c["ignore"],
                                 c["cap"], c["n_rows"])
    assert ref["n_slots"] == ns and list(ref["item_of_slot"][:ns]) == order and (ref["item_of_slot"][ns:] == -1).all()
    assert list(ref["labels_out"]) == lab and list(ref["neg_out"]) == neg


def test_make_case_poisons_unread_entries():
    """every label past n_valid and every per-position row the kernels must not read opens a new slot if read"""
    rng = np.random.default_rng(0)
    c = gt.make_case(50000, gt._edge_items(50000, rng), 1, 33, "part", 7, seed=1)
    ref = tr.compact_ref(c["n_items"], c["labels"], c["n_valid"], len(c["labels"]), c["negatives"], 33, 1, c["valid_idx"], 7,
                         c["cap"], c["n_rows"])
    slots = set(ref["item_of_slot"][:ref["n_slots"]].tolist())
    nv = c["n_valid"]
    assert nv < len(c["labels"])
    assert not slots & set(c["labels"][nv:].tolist())
    unread = np.setdiff1d(np.arange(len(c["labels"])), c["valid_idx"][:nv])
    assert unread.size and not slots & set(c["negatives"][unread].reshape(-1).tolist())
    read = c["negatives"][c["valid_idx"][:nv]].reshape(-1)
    for v in (7, -1, 50000, 1 << 40):
        assert v in read


def test_edge_items_cover_258_tiles():
    n = 1052673
    S = gt._edge_items(n, np.random.default_rng(0))
    tiles = np.unique(S // tr.TILE)
    assert -(-n // tr.TILE) == 258 and 257 in tiles and 256 in tiles and 2 not in tiles
    assert n - 1 in S and 0 in S and np.all(np.isin(np.arange(tr.TILE, 2 * tr.TILE), S))


# ------------------------------------------------------------------------------------------------ mistakes are rejected
def test_tile_local_numbering_is_rejected():
    """slots numbered per tile without the earlier tiles' prefix (the compaction compares exactly)"""
    n = 12289
    c = gt.make_case(n, gt._edge_items(n, np.random.default_rng(1)), 0, 256, "part", 7, seed=2)
    args = (c["n_items"], c["labels"], c["n_valid"], len(c["labels"]), c["negatives"], c["n_neg"], c["mode"], c["valid_idx"],
            c["ignore"], c["cap"], c["n_rows"])
    good, bad = tr.compact_ref(*args), tr.compact_ref(*args, mistake="tile_local")
    assert not np.array_equal(good["item_of_slot"], bad["item_of_slot"])
    assert not np.array_equal(good["labels_out"], bad["labels_out"])


def test_next_row_scatter_is_rejected():
    """one slot's gradient added to the next item's row: the scatter test compares bit for bit"""
    g = torch.Generator().manual_seed(3)
    n, ns, d = 50000, 22400, 32
    ios = torch.randperm(n - 1, generator=g)[:ns].sort().values
    dx = torch.randn(ns, d, generator=g).to(torch.bfloat16)
    base = torch.zeros(n + 1, d)
    good = tr.scatter_ref(base, dx, ios, ns, ns)
    bad = tr.scatter_ref(base, dx, ios, ns, ns, mistake="next_row")
    assert not torch.equal(good, bad)


def _stage_inputs(rows, d, seed):
    """the stage test's inputs at one of its shapes, on the CPU: layer 0 with tower_input rows"""
    g = torch.Generator().manual_seed(seed)
    F = 2 * d
    x = tr.tower_input(rows, d, g).to(torch.bfloat16)
    W = (torch.randn(2 * F, d, generator=g) * math.sqrt(2 / (3 * d))).to(torch.bfloat16)
    bgl = 0.1 * torch.randn(2 * F, generator=g)
    W2 = (torch.randn(d, F, generator=g) * math.sqrt(2 / (3 * d))).to(torch.bfloat16)
    b2 = 1e-3 * torch.randn(d, generator=g)
    norm = 1 + 0.1 * torch.randn(d, generator=g)
    return x, W, bgl, W2, b2, norm, F


def test_missing_residual_is_rejected():
    x, W, bgl, W2, b2, norm, F = _stage_inputs(129, 128, 0)
    GL = tr.gemm_ref(x, W, bgl)[0].to(torch.bfloat16)
    U = dr.swiglu_fwd(GL, 129, F)[0].to(torch.bfloat16)
    ref, bound = tr.gemm_ref(U, W2, b2, residual=x)
    without = tr.gemm_ref(U, W2, b2)[0].to(torch.bfloat16)
    assert dr.ratio(without, ref, bound) > 10 * gt.TOL_STAGE
    P = {}
    for p in ("tw0.", "tw1."):
        P.update({p + "wgw1": W.double(), p + "bgb1": bgl.double(), p + "w2": W2.double(), p + "b2": b2.double(),
                  p + "norm": norm.double()})
    y = tr.tower(x.double(), P, F, 128)
    assert gt._out_err(tr.tower(x.double(), P, F, 128, mistake="no_residual").to(torch.bfloat16), y) > 10 * gt.TOL_OUT


def test_rms_eps_is_rejected():
    """RMSNorm with eps 1e-5 in place of fp32 eps, on the first norm's input (z of the tower_input rows scaled by 1e-3)"""
    x, W, bgl, W2, b2, norm, F = _stage_inputs(129, 128, 1)
    GL = tr.gemm_ref(x, W, bgl)[0].to(torch.bfloat16)
    U = dr.swiglu_fwd(GL, 129, F)[0].to(torch.bfloat16)
    z = tr.gemm_ref(U, W2, b2, residual=x)[0].to(torch.bfloat16)
    y, yb, _ = dr.rmsnorm_fwd(z, norm, tr.RMS_EPS, 1.0, 129, 128, 128, 128)
    y_bad, _, _ = dr.rmsnorm_fwd(z, norm, 1e-5, 1.0, 129, 128, 128, 128)
    assert dr.ratio(y_bad.to(torch.bfloat16), y, yb) > 10 * gt.TOL_STAGE


def test_missing_silu_slope_term_is_rejected():
    x, W, bgl, W2, b2, norm, F = _stage_inputs(129, 128, 2)
    GL = tr.gemm_ref(x, W, bgl)[0].to(torch.bfloat16)
    du = torch.randn(129, F, generator=torch.Generator().manual_seed(4)).to(torch.bfloat16)
    ref, bound = dr.swiglu_bwd(du, GL, 129, F)
    bad, _ = dr.swiglu_bwd(du, GL, 129, F, with_silu_slope=False)
    assert dr.ratio(bad.to(torch.bfloat16), ref, bound) > 10 * gt.TOL_STAGE


def test_dropped_ignore_mask_is_rejected():
    """ignore_index 7 scored as a real item in the step's shared layout (3 of 256 negatives): the step's loss bound
    rejects it"""
    g = torch.Generator().manual_seed(6)
    M, R, d, N = 2000, 600, 32, 256
    hc = torch.randn(M, d, generator=g, dtype=torch.float64) * 0.3
    table = torch.randn(R, d, generator=g, dtype=torch.float64) * 0.3
    labels = torch.randint(8, R, (M,), generator=g)
    neg = torch.randint(8, R, (N,), generator=g)
    neg[:3] = 7
    vi = torch.arange(M)
    good = sr.reference(hc, table, labels, vi, neg, M, sr.CE_SAMPLED, 0, ignore_index=7)
    bad = sr.reference(hc, table, labels, vi, neg, M, sr.CE_SAMPLED, 0, ignore_index=-100)
    assert abs(float(bad["loss"] - good["loss"])) / float(good["loss"]) > gt.TOL_LOSS
