"""GPU tests of TwoTower (replay_b200/engine_twotower.py, csrc/rp_twotower.cu, the group-512 RMSNorm):

* parity with the real reference's goldens (tests/golden/twotower_*.npz) and with the fp64 oracle (oracle/twotower.py) -
  loss |rel| <= 5e-3, gradients cosine >= 0.995 and norm ratio within 3 %, as the new-path SASRec parity tests;
* every sampled loss in every negative layout against the oracle, which scores the catalog tower's rows at the candidates
  (the tower is row-wise, so that is the loss on the full-catalog tower followed by a gather);
* the item tower alone against fp64 at catalog sizes 1 .. 50 000 and d 64 .. 512;
* candidate compaction on hand-built cases, exactly;
* graph-captured against eager steps, packed against padded query rows, the inference cache, a short Lightning run."""
import os

import numpy as np
import pytest
import torch

from oracle import sasrec as osr
from oracle import twotower as ott
from oracle.diff import from_bf16_bits

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), "golden")
TAGS = ("d64h2", "d50h1", "d128h2")


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda")


class _Reader:
    def __init__(self, n):
        self.ids = torch.arange(n)

    def __getitem__(self, k):
        return self.ids

    @property
    def feature_names(self):
        return ["item_id"]


def _load(tag):
    return dict(np.load(os.path.join(GOLD, f"twotower_{tag}.npz")))


def _model(n_items, d, H, L, n_blocks, dropout=0.0, seed=0):
    from replay_b200.nn.sequential.twotower import TwoTower
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    sch = TensorSchema(TensorFeatureInfo("item_id", n_items, n_items, d))
    return TwoTower.from_params(sch, _Reader(n_items), embedding_dim=d, num_heads=H, num_blocks=n_blocks,
                                max_sequence_length=L, dropout=dropout, seed=seed)


def _golden_model(z):
    n, d, H, L, nb = (int(z[k]) for k in ("n_items", "d", "H", "L", "n_blocks"))
    sd = ott.seeded_state_dict(n, d, H, L, nb, int(z["seed"]))
    m = _model(n, d, H, L, nb)
    m.load_state_dict(sd)
    return m, sd


def _inputs(z, dev):
    return tuple(torch.from_numpy(z[k]).to(dev) for k in ("ids", "pad_mask", "labels", "target_mask"))


def _spec(kind, ignore):
    from replay_b200.nn import loss as L

    return {"ce": lambda: L.CE(ignore_index=ignore), "bce": lambda: L.BCE(),
            "ce_sampled": lambda: L.CESampled(negative_labels_ignore_index=ignore),
            "bce_sampled": lambda: L.BCESampled(negative_labels_ignore_index=ignore),
            "login_ce_sampled": lambda: L.LogInCESampled(negative_labels_ignore_index=ignore),
            "ce_sampled_weighted": lambda: L.CESampledWeighted("w", negative_labels_ignore_index=ignore)}[kind]()


def _engine_grads(model):
    """every gradient of the last backward, by reference key (the shared table under body.embedder...)"""
    from replay_b200.nn.sequential.twotower import twotower_key_map

    eng = model.core.engine
    m = twotower_key_map(model.core.cfg.n_blocks)
    return {m[k]: model.core._to_ref(k, eng.export_named(k, eng.grads)).double().cpu() for k in eng.params}


def _cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def _comparable(k, a, b, n_items):
    """the entries of gradient ``k`` worth comparing: the item table's rows without the padding row, and in_proj_bias
    without its key third, whose exact gradient is zero (softmax is invariant to the per-query constant q . b_k), so that
    both sides hold rounding noise only"""
    if k == ott.ITEM_KEYS[0]:
        return a[:n_items], b[:n_items]
    if k.endswith("in_proj_bias"):
        d = b.shape[0] // 3
        keep = torch.cat([torch.arange(d), torch.arange(2 * d, 3 * d)])
        return a[keep], b[keep]
    return a, b


def _check_grads(G, Gref, n_items, norm_tol=0.03):
    bad = []
    for k, b in Gref.items():
        a, b = _comparable(k, G[k].reshape(b.shape), b, n_items)
        if b.norm() < 1e-12:
            assert a.norm() < 1e-6, k
            continue
        c, r = _cos(a, b), float(a.norm() / b.norm())
        if c < 0.995 or abs(r - 1) > norm_tol:
            bad.append((k, round(c, 5), round(r, 4)))
    assert not bad, bad


def _train_loss(model, ids, pm, lab, tm, neg=None, w=None):
    ft = {"item_id": ids}
    if w is not None:
        ft["w"] = w
    model.train()
    model.core.flat.grad = None
    out = model(feature_tensors=ft, padding_mask=pm, positive_labels=lab, negative_labels=neg, target_padding_mask=tm)
    out["loss"].backward()
    return float(out["loss"].detach())


@pytest.mark.parametrize("tag", TAGS)
def test_ce_matches_reference_golden(cuda, tag):
    z = _load(tag)
    model, _ = _golden_model(z)
    model.loss = _spec("ce", int(z["n_items"]))
    ids, pm, lab, tm = _inputs(z, cuda)
    loss = _train_loss(model, ids, pm, lab, tm)
    ref = float(z["ce::loss"])
    assert abs(loss - ref) <= 5e-3 * abs(ref), (loss, ref)
    Gref = {k[len("ce::grad::"):]: from_bf16_bits(z[k]).double() for k in z if k.startswith("ce::grad::")}
    _check_grads(_engine_grads(model), Gref, int(z["n_items"]))


CASES = [("bce", None), ("ce_sampled", "shared"), ("ce_sampled", "perseq"), ("ce_sampled", "perpos"),
         ("bce_sampled", "perseq"), ("login_ce_sampled", "perseq"), ("login_ce_sampled", "perpos"),
         ("ce_sampled_weighted", "shared"), ("ce_sampled_weighted", "perpos")]


@pytest.mark.parametrize("tag", TAGS)
@pytest.mark.parametrize("kind, layout", CASES)
def test_losses_match_oracle(cuda, tag, kind, layout):
    """loss against the reference where the golden has the case, loss and gradients against the fp64 oracle"""
    z = _load(tag)
    model, sd = _golden_model(z)
    ign = int(z["ignore_index"])
    model.loss = _spec(kind, ign)
    ids, pm, lab, tm = _inputs(z, cuda)
    neg = None if layout is None else torch.from_numpy(z[f"neg_{layout}"])
    w = torch.from_numpy(z["weights"]) if kind == "ce_sampled_weighted" else None
    loss = _train_loss(model, ids, pm, lab, tm, None if neg is None else neg.to(cuda), None if w is None else w.to(cuda))
    gname = kind if layout is None else f"{kind}_{layout}"
    if f"{gname}::loss" in z:
        ref = float(z[f"{gname}::loss"])
        assert abs(loss - ref) <= 5e-3 * max(1.0, abs(ref)), (loss, ref)
    kw = {} if neg is None else dict(negatives=neg, ignore_index=ign)
    if w is not None:
        kw["weights"] = w.double()
    rl, Gref = ott.loss_and_grads(ott.to_dtype(sd, torch.float64), *(t.cpu() for t in _inputs(z, "cpu")), int(z["H"]), kind,
                                  **kw)
    assert abs(loss - float(rl)) <= 5e-3 * max(1.0, abs(float(rl))), (loss, float(rl))
    # a handful of targets and negatives carries each sampled gradient: bf16 rounding of the hidden states moves its
    # norm by a few per cent in the lowest block
    _check_grads(_engine_grads(model), Gref, int(z["n_items"]), norm_tol=0.03 if layout is None else 0.06)


@pytest.mark.parametrize("tag", TAGS)
def test_inference_matches_reference_golden(cuda, tag):
    z = _load(tag)
    model, _ = _golden_model(z)
    ids, pm, _, _ = _inputs(z, cuda)
    live = pm.any(1).cpu()
    model.eval()
    lo = model(feature_tensors={"item_id": ids}, padding_mask=pm)["logits"].cpu().double()
    ref = torch.from_numpy(z["eval_logits"]).double()
    assert (lo[live] - ref[live]).abs().max() <= 3e-2 * ref[live].abs().max()
    cand = torch.from_numpy(z["candidates"]).to(cuda)
    lc = model(feature_tensors={"item_id": ids}, padding_mask=pm, candidates_to_score=cand)["logits"].cpu().double()
    refc = torch.from_numpy(z["cand_logits"]).double()
    assert (lc[live] - refc[live]).abs().max() <= 3e-2 * refc[live].abs().max()
    # the reference's key list with the cache after an eval forward over the catalog
    assert list(model.state_dict()) == list(z["cache_keys"])
    # seen-filtered top-10 through the fused top-K on the cached tower, exact against the oracle on the same bf16 operands
    eng = model.core.engine
    hq = model.core.query_embeddings(ids, pm)
    seen = ids.masked_fill(~pm, int(z["n_items"]))
    got, _ = model.predict_topk({"item_id": ids}, pm, 10, seen_ids=seen)
    want, _ = osr.score_topk(eng.pad_features(hq).float().cpu(), model.core.item_table().float().cpu(), seen.cpu(), 10)
    assert torch.equal(got.cpu()[live], want[live])


def test_three_adam_steps_match_oracle(cuda):
    z = _load("d64h2")
    model, sd = _golden_model(z)
    n = int(z["n_items"])
    model.loss = _spec("ce", n)
    ids, pm, lab, tm = _inputs(z, cuda)
    P = ott.to_dtype(sd, torch.float64)
    P0 = dict(P)
    state = {}
    for step in range(1, 4):
        model.core.fused_step(ids, pm, lab, tm, all_reduce=None, lr=1e-3)
        _, G = ott.loss_and_grads(P, *(t.cpu() for t in _inputs(z, "cpu")), int(z["H"]), "ce")
        for k, g in G.items():
            m, v = state.get(k, (torch.zeros_like(g), torch.zeros_like(g)))
            p, m, v = osr.adam_step(P[k], g, m, v, step)
            P[k], state[k] = p, (m, v)
        P = ott.to_dtype(P, torch.float64)
    got = model.state_dict()
    for k, v in P.items():
        if not v.is_floating_point():
            continue
        if k in ott.ITEM_KEYS[1:]:
            continue
        # the three steps' updates (bf16 gradients: compare directions)
        a, b = _comparable(k, got[k].double().cpu() - P0[k], v - P0[k], n)
        if b.norm() < 1e-12:
            continue
        assert _cos(a, b) >= 0.98 and abs(float(a.norm() / b.norm()) - 1) <= 0.05, (k, _cos(a, b))


@pytest.mark.parametrize("n_items", [1, 127, 129, 50000])
@pytest.mark.parametrize("d", [64, 128, 256, 512])
def test_item_tower_matches_fp64(cuda, n_items, d):
    """the tower forward and backward alone (d = 512: the group-512 RMSNorm) on the engine's bf16 operands"""
    from replay_b200.engine_twotower import TOWER_LAYERS, TwoTowerConfig, TwoTowerEngine

    cfg = TwoTowerConfig(n_items=n_items, d=d, n_heads=d // 64, n_blocks=1, max_len=8)
    eng = TwoTowerEngine(cfg, 1, 8, cuda, seed=5)
    g = torch.Generator(device="cpu").manual_seed(d + n_items)
    with torch.no_grad():
        eng.params["item_emb"].copy_(torch.randn(eng.params["item_emb"].shape, generator=g))
        for p in TOWER_LAYERS:
            eng.params[p + "norm"].copy_(1 + 0.1 * torch.randn(d, generator=g))
            eng.params[p + "b2"].copy_(0.1 * torch.randn(d, generator=g))
    eng.refresh_shadow()
    eng.tower_valid = False
    out = eng.tower_table().double()
    sd = {ott.ITEM_KEYS[0]: eng.params16["item_emb"].double().clone().requires_grad_(True),
          "body.item_tower.item_reference_item_id": torch.arange(n_items, device=cuda)}
    leaves = {}
    for layer, p in enumerate(TOWER_LAYERS, start=1):
        for k, leaf in (("wg", "WG.weight"), ("bg", "WG.bias"), ("w1", "W1.weight"), ("b1", "W1.bias"), ("w2", "W2.weight"),
                        ("b2", "W2.bias")):
            src = eng.params16 if k.startswith("w") else eng.params
            leaves[p + k] = sd[f"body.item_tower.encoder.sw{layer}.{leaf}"] = src[p + k].double().clone().requires_grad_(True)
        leaves[p + "norm"] = sd[f"body.item_tower.encoder.norm{layer}.weight"] = eng.params[p + "norm"].double().clone().requires_grad_(True)
    ref = ott.item_tower(sd)
    tol = 2e-2 * float(ref.abs().max())
    assert (out - ref).abs().max() <= tol
    # backward: a random output gradient through the tower
    dY = torch.randn(n_items, d, generator=g).to(cuda)
    eng.g32.zero_()
    eng.tw["dY32"][:n_items].copy_(dY)
    eng.tower_backward(eng.params16["item_emb"], n_items)
    ref.backward(dY.double())
    dx0 = eng.tw["dxb"][:n_items].double()
    assert _cos(dx0, sd[ott.ITEM_KEYS[0]].grad[:n_items]) >= 0.995
    for name, leaf in leaves.items():
        c, r = _cos(eng.grads[name], leaf.grad), float(eng.grads[name].norm() / leaf.grad.norm())
        assert c >= 0.995 and abs(r - 1) <= 0.03, (name, c, r)


# ---------------------------------------------------------------------------------------------------------------- compaction
def _compact(cuda, n_items, labels, n_valid, negatives, mode, ignore, d=64, L=4, valid_idx=None):
    from replay_b200._lib import check, lib

    L_ = lib()
    cap_entries = len(labels) + negatives.numel()
    cap = min(n_items, cap_entries)
    table = torch.randn(n_items + 1, d, device=cuda).to(torch.bfloat16)
    lab = torch.tensor(labels, dtype=torch.int32, device=cuda)
    nv = torch.tensor([n_valid], dtype=torch.int32, device=cuda)
    neg = negatives.to(cuda, torch.int64).contiguous()
    n_neg = neg.shape[-1]
    vi = torch.as_tensor(valid_idx if valid_idx is not None else list(range(len(labels))), dtype=torch.int32, device=cuda)
    ns = torch.full((1,), -7, dtype=torch.int32, device=cuda)
    ios = torch.full((cap,), -7, dtype=torch.int32, device=cuda)
    lab_r = torch.full_like(lab, -7)
    neg_r = torch.full_like(neg, -7)
    rows = torch.full((cap, d), 3.0, device=cuda, dtype=torch.bfloat16)
    ws = torch.empty(L_.rp_tower_compact_workspace(n_items), dtype=torch.uint8, device=cuda)
    stream = torch.cuda.current_stream().cuda_stream
    check(L_.rp_tower_compact(lab.data_ptr(), nv.data_ptr(), len(labels), neg.data_ptr(), n_neg, mode,
                              neg.shape[0] if neg.dim() == 2 else 1, vi.data_ptr(), L, ignore, n_items, table.data_ptr(), d, cap,
                              ns.data_ptr(), ios.data_ptr(), lab_r.data_ptr(), neg_r.data_ptr(), rows.data_ptr(), ws.data_ptr(),
                              ws.numel(), stream), "rp_tower_compact")
    torch.cuda.synchronize()
    return cap, table, int(ns), ios.cpu(), lab_r.cpu(), neg_r.cpu(), rows


def _expected(n_items, labels, n_valid, neg_entries, ignore):
    items = set(labels[:n_valid])
    for v in neg_entries:
        if ignore >= 0 and v == ignore:
            continue
        items.add(v if 0 <= v < n_items else 0)
    return sorted(items)


@pytest.mark.parametrize("case", ["duplicates", "ignored", "no_valid", "every_item", "per_position", "per_sequence"])
def test_compaction_exact(cuda, case):
    n_items, ignore = 50, (-100 if case == "every_item" else 7)
    if case == "duplicates":
        labels, nv, neg, mode = [4, 9, 4, 30], 4, torch.tensor([9, 9, 30, 1, 1, 49]), 0
    elif case == "ignored":
        labels, nv, neg, mode = [4, 12, 3], 3, torch.tensor([7, 7, 12, 60, 0]), 0   # 60: outside the catalog -> item 0
    elif case == "no_valid":
        labels, nv, neg, mode = [4, 12, 3], 0, torch.tensor([11, 2]), 0
    elif case == "every_item":
        labels, nv, neg, mode = list(range(0, 50, 2)), 25, torch.arange(49, -1, -1), 0
    elif case == "per_sequence":
        labels, nv, neg, mode = [5, 6, 7, 8], 3, torch.tensor([[1, 7, 3], [3, 3, 49]]), 2
    else:
        labels, nv, neg, mode = [5, 6, 7], 3, torch.tensor([[1, 7, 5], [40, 41, 42], [6, 6, 2], [9, 9, 9]]), 1
    vidx = {2: [0, 4, 5], 1: [0, 2, 3]}.get(mode)
    cap, table, ns, ios, lab_r, neg_r, rows = _compact(cuda, n_items, labels, nv, neg, mode, ignore, valid_idx=vidx)
    if mode == 1:
        entries = [int(v) for r in vidx[:nv] for v in neg[r]]
    else:
        entries = [int(v) for v in neg.flatten()]
    want = _expected(n_items, labels, nv, entries, ignore)
    assert ns == len(want)
    assert ios[:ns].tolist() == want and (ios[ns:] == -1).all()
    slot = {it: s for s, it in enumerate(want)}
    assert lab_r[:nv].tolist() == [slot[v] for v in labels[:nv]]

    def remap(v):
        return cap if v == ignore else (cap + 1 if not 0 <= v < n_items else slot[v])

    if mode == 1:
        for r in vidx[:nv]:
            assert neg_r[r].tolist() == [remap(int(v)) for v in neg[r]]
    else:
        assert neg_r.flatten().tolist() == [remap(int(v)) for v in neg.flatten()]
    assert torch.equal(rows[:ns], table[torch.tensor(want, dtype=torch.long, device=cuda)]) if ns else True
    assert (rows[ns:] == 0).all()


# ---------------------------------------------------------------------------------------------------------------- training paths
def _batch(z, dev, neg_layout="shared"):
    ids, pm, lab, tm = _inputs(z, dev)
    return dict(feature_tensors={"item_id": ids}, padding_mask=pm, positive_labels=lab, target_padding_mask=tm,
                negative_labels=torch.from_numpy(z[f"neg_{neg_layout}"]).to(dev))


@pytest.mark.parametrize("kind", ["ce", "ce_sampled"])
def test_graph_captured_steps_equal_eager(cuda, kind):
    from replay_b200.nn.lightning import LightningModule, OptimizerFactory

    z = _load("d64h2")
    a, _ = _golden_model(z)
    b, _ = _golden_model(z)
    for m in (a, b):
        m.loss = _spec(kind, int(z["ignore_index"]))
        m.train()
    batch = _batch(z, cuda)
    lm = LightningModule(a, optimizer_factory=OptimizerFactory(learning_rate=1e-3))
    for i in range(5):   # two eager warm-up steps, then captured and replayed
        la = float(lm.training_step(batch, i))
        lb = float(b.core.fused_step(batch["feature_tensors"]["item_id"], batch["padding_mask"], batch["positive_labels"],
                                     batch["target_padding_mask"], all_reduce=None, lr=1e-3,
                                     negatives=batch["negative_labels"] if kind != "ce" else None))
        assert abs(la - lb) <= 2e-5 * abs(lb), (i, la, lb)
    torch.testing.assert_close(a.core.flat, b.core.flat, rtol=1e-4, atol=1e-6)   # the embedding backward adds with atomics


@pytest.mark.parametrize("kind", ["ce", "ce_sampled"])
def test_packed_query_tower_equals_padded(cuda, kind):
    z = _load("d64h2")
    out = []
    for packed in (False, True):
        m, _ = _golden_model(z)
        m.loss = _spec(kind, int(z["ignore_index"]))
        ids, pm, lab, tm = _inputs(z, cuda)
        m.core.ensure_engine(ids.shape[0], ids.shape[1], with_grad=True).packed_body = packed
        neg = torch.from_numpy(z["neg_perseq"]).to(cuda) if kind != "ce" else None
        loss = _train_loss(m, ids, pm, lab, tm, neg)
        assert m.core.engine._packed == packed
        out.append((loss, m.core.flat.grad.clone()))
    assert abs(out[0][0] - out[1][0]) <= 1e-5 * abs(out[0][0])
    assert _cos(out[0][1], out[1][1]) >= 0.9999


def test_cache_follows_training(cuda):
    z = _load("d64h2")
    model, _ = _golden_model(z)
    model.loss = _spec("ce", int(z["n_items"]))
    ids, pm, lab, tm = _inputs(z, cuda)
    model.eval()
    before = model(feature_tensors={"item_id": ids}, padding_mask=pm)["logits"].clone()
    assert "body.item_tower.cache" in model.state_dict()
    tab0 = model.core.item_table().clone()
    model.core.fused_step(ids, pm, lab, tm, all_reduce=None, lr=1e-2)
    assert "body.item_tower.cache" not in model.state_dict()
    tab1 = model.core.item_table().clone()
    assert not torch.equal(tab0, tab1)
    eng = model.core.engine
    eng.tower_valid = False   # recomputed from the updated weights: the table kept since the step must equal it
    torch.testing.assert_close(model.core.item_table(), tab1, rtol=0, atol=0)
    model.eval()
    after = model(feature_tensors={"item_id": ids}, padding_mask=pm)["logits"]
    assert not torch.allclose(before, after)
    # a loaded cache is the tower the next eval forward reads, with the reference's shape checks
    sd = model.state_dict()
    assert sd["body.item_tower.cache"].shape == (int(z["n_items"]), int(z["d"]))
    bad = dict(sd)
    bad["body.item_tower.cache"] = sd["body.item_tower.cache"][:-1]
    with pytest.raises(AssertionError):
        model.load_state_dict(bad)
    model.load_state_dict(sd)
    torch.testing.assert_close(model(feature_tensors={"item_id": ids}, padding_mask=pm)["logits"], after, rtol=0, atol=2e-2)


@pytest.mark.parametrize("kind", ["ce", "ce_sampled"])
def test_cache_follows_graph_replayed_steps(cuda, kind):
    """Lightning's fused step is captured on its third call and replayed after that, which runs no Python of the engine:
    between steps every eval path must read the tower of the current weights, never a stale or slot-ordered table."""
    from replay_b200.nn.lightning import LightningModule, OptimizerFactory

    z = _load("d64h2")
    model, _ = _golden_model(z)
    model.loss = _spec(kind, int(z["ignore_index"]))
    ids, pm, lab, tm = _inputs(z, cuda)
    batches = [_batch(z, cuda, "shared"), dict(_batch(z, cuda, "shared"), positive_labels=lab.flip(0), target_padding_mask=tm.flip(0))]
    lm = LightningModule(model, optimizer_factory=OptimizerFactory(learning_rate=3e-3))
    eng = model.core.engine
    seen = ids.masked_fill(~pm, int(z["n_items"]))
    prev = None
    for i in range(6):
        model.train()
        lm.training_step(batches[i % 2], i)
        model.eval()
        logits = model(feature_tensors={"item_id": ids}, padding_mask=pm)["logits"]
        top, _ = model.predict_topk({"item_id": ids}, pm, 10, seen_ids=seen)
        table = model.core.item_table().clone()
        eng.tower_valid = False   # force the tower from the current weights
        fresh = model.core.item_table().clone()
        torch.testing.assert_close(table, fresh, rtol=0, atol=0)
        want = model(feature_tensors={"item_id": ids}, padding_mask=pm)["logits"]
        torch.testing.assert_close(logits, want, rtol=0, atol=0)
        top_want, _ = model.predict_topk({"item_id": ids}, pm, 10, seen_ids=seen)
        assert torch.equal(top, top_want)
        if prev is not None:
            assert not torch.equal(prev, fresh)   # each step moved the tower
        prev = fresh
    assert lm.model.core._trainer._g_fb is not None   # the later steps were replays


def test_lightning_run_loss_falls(cuda):
    from replay_b200.nn.lightning import LightningModule, OptimizerFactory
    from replay_b200.synthetic import make_sequences

    n_items, d, H, L, B = 500, 64, 2, 32, 64
    model = _model(n_items, d, H, L, 2, dropout=0.1, seed=3)
    model.loss = _spec("ce_sampled", -100)
    ids, pm, lab, tm = make_sequences(B, n_items, L, seed=4)
    g = torch.Generator().manual_seed(5)
    lm = LightningModule(model, optimizer_factory=OptimizerFactory(learning_rate=3e-3))
    losses = []
    for i in range(30):
        neg = torch.randint(0, n_items, (64,), generator=g)
        batch = dict(feature_tensors={"item_id": ids.to(cuda)}, padding_mask=pm.to(cuda), positive_labels=lab.to(cuda),
                     target_padding_mask=tm.to(cuda), negative_labels=neg.to(cuda))
        losses.append(float(lm.training_step(batch, i)))
    assert np.mean(losses[-5:]) < 0.8 * np.mean(losses[:5]), losses
