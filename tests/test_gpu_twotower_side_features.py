"""TwoTower with side features on the GPU: reader item features in the item tower, sequence features in the query tower.

* the training step of every loss, eager and graph-captured, the eval / candidate logits and the seen-filtered top-10
  against the goldens of the real reference (oracle/gen_twotower_side_features_golden.py), at the tolerances of
  tests/test_gpu_twotower.py (loss |rel| <= 5e-3, gradients cosine >= 0.995 and norm ratio within 3 %);
* the state_dict: the reference's keys, shapes and dtypes, and a round trip;
* rp_item_feature_embed_fwd / _bwd against float64 with per-element bounds (tests/fp64_checks.py style) at slot counts
  0, 1 and cap with rows past *n_slots, 127 / 128 / 129 rows, a catalog pass with an item offset, padding values,
  all-padding bags, ids outside the table, a one-row table, dp > d; the full-catalog backward is bitwise reproducible."""
import os

import numpy as np
import pytest
import torch

from oracle import side_features as osf
from replay_b200._lib import FEAT_BAG_MEAN, FEAT_BAG_SUM, FEAT_CAT, FEAT_IDENT, FEAT_NUM, ItemFeaturePlan, RpFeature, check
from replay_b200._lib import lib as _lib

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TAGS = ("d64h2", "d50h1")
U_BF16 = 2.0 ** -8   # unit roundoff of bf16


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda")


# ------------------------------------------------------------------------------------------------------------ the model
class _Reader:
    def __init__(self, cols):
        self.cols = cols

    def __getitem__(self, k):
        return self.cols[k]

    @property
    def feature_names(self):
        return list(self.cols)


def _load(tag):
    return dict(np.load(os.path.join(GOLD, f"twotower_side_{tag}.npz")))


def _schema(z):
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    n, d = int(z["n_items"]), int(z["d"])
    fs = []
    for name, kind, pad, width, card in zip(z["f_name"], z["f_kind"], z["f_padding_value"], z["f_width"], z["f_cardinality"]):
        name, kind = str(name), str(kind)
        if kind in ("cat", "bag"):
            fs.append(TensorFeatureInfo(name, int(card), int(pad), d, is_list=kind == "bag"))
        else:
            fs.append(TensorFeatureInfo(name, None, 0, d, is_cat=False, tensor_dim=int(width)))
    return TensorSchema(TensorFeatureInfo("item_id", n, n, d), features=fs)


def _golden_model(z, seed=0):
    from replay_b200.nn.sequential.twotower import TwoTower

    reader = _Reader({str(k): torch.from_numpy(z["item::" + str(k)]) for k in z["reader"]})
    m = TwoTower.from_params(_schema(z), reader, embedding_dim=int(z["d"]), num_heads=int(z["H"]),
                             num_blocks=int(z["n_blocks"]), max_sequence_length=int(z["L"]), dropout=0.0,
                             categorical_list_feature_aggregation_method=str(z["method"]), seed=seed)
    sd = osf.golden_state_dict(z)
    m.load_state_dict(sd, strict=False)
    return m, sd


def _ft(z, dev, w=None):
    ft = {"item_id": torch.from_numpy(z["ids"]).to(dev)}
    ft.update({k[len("feat::"):]: torch.from_numpy(z[k]).to(dev) for k in z if k.startswith("feat::")})
    if w is not None:
        ft["sample_weight"] = w
    return ft


def _spec(kind, ignore):
    from replay_b200.nn import loss as L

    return {"ce": lambda: L.CE(ignore_index=ignore), "bce": lambda: L.BCE(),
            "ce_sampled": lambda: L.CESampled(negative_labels_ignore_index=ignore),
            "login_ce_sampled": lambda: L.LogInCESampled(negative_labels_ignore_index=ignore),
            "ce_sampled_weighted": lambda: L.CESampledWeighted("sample_weight", negative_labels_ignore_index=ignore)}[kind]()


CASES = {"ce": ("ce", None), "bce": ("bce", None), "ce_sampled_shared": ("ce_sampled", "shared"),
         "ce_sampled_perseq": ("ce_sampled", "perseq"), "ce_sampled_perpos": ("ce_sampled", "perpos"),
         "login_ce_sampled_perseq": ("login_ce_sampled", "perseq"), "ce_sampled_weighted_shared": ("ce_sampled_weighted", "shared")}


def _grads(model):
    core = model.core
    eng = core.engine
    return {core._keymap[k]: core._to_ref(k, eng.export_named(k, eng.grads)).double().cpu() for k in eng.params}


def _cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def _comparable(k, a, b, n_items):
    """as tests/test_gpu_twotower.py: the item table without its padding row, in_proj_bias without its key third"""
    if k == "body.embedder.feature_embedders.item_id.emb.weight":
        return a[:n_items], b[:n_items]
    if k.endswith("in_proj_bias"):
        d = b.shape[0] // 3
        keep = torch.cat([torch.arange(d), torch.arange(2 * d, 3 * d)])
        return a[keep], b[keep]
    return a, b


def _check_grads(G, Gref, n_items):
    bad = []
    for k, b in Gref.items():
        a, b = _comparable(k, G[k].reshape(b.shape), b, n_items)
        if b.norm() < 1e-12:
            assert a.norm() < 1e-6, k
            continue
        c, r = _cos(a, b), float(a.norm() / b.norm())
        if c < 0.995 or abs(r - 1) > 0.03:
            bad.append((k, round(c, 5), round(r, 4)))
    assert not bad, bad


def _check_case(z, name, loss, G):
    ref = float(z[f"{name}::loss"])
    assert abs(loss - ref) <= 5e-3 * abs(ref), (name, loss, ref)
    n = int(z["n_items"])
    _check_grads(G, {k.split("::")[2]: torch.from_numpy(z[k]).double() for k in z if k.startswith(f"{name}::grad::")}, n)
    bad = []
    for k in z:   # every other gradient by its norm
        if not k.startswith(f"{name}::gsum::"):
            continue
        key = k.split("::")[2]
        ref_norm = float(z[k][1])
        if key.endswith("in_proj_bias") or ref_norm < 1e-9:
            continue
        got = float(G[key].norm())
        if abs(got / ref_norm - 1) > 0.03:
            bad.append((key, got, ref_norm))
    assert not bad, (name, bad)


def _batch(z, dev, name):
    kind, layout = CASES[name]
    w = torch.from_numpy(z["weights"]).to(dev).unsqueeze(-1) if kind == "ce_sampled_weighted" else None
    neg = torch.from_numpy(z[f"neg_{layout}"]).to(dev) if layout else None
    t = lambda k: torch.from_numpy(z[k]).to(dev)  # noqa: E731
    return kind, _ft(z, dev, w), t("pad_mask"), t("labels"), t("target_mask"), neg


@pytest.mark.parametrize("tag", TAGS)
@pytest.mark.parametrize("name", list(CASES))
def test_step_matches_reference_golden(cuda, tag, name):
    z = _load(tag)
    model, _ = _golden_model(z)
    kind, ft, pm, lab, tm, neg = _batch(z, cuda, name)
    model.loss = _spec(kind, int(z["ignore_index"]) if kind != "ce" else int(z["n_items"]))
    model.train()
    out = model(feature_tensors=ft, padding_mask=pm, positive_labels=lab, negative_labels=neg, target_padding_mask=tm)
    out["loss"].backward()
    _check_case(z, name, float(out["loss"].detach()), _grads(model))


@pytest.mark.parametrize("name", ["ce", "ce_sampled_perseq", "ce_sampled_weighted_shared"])
def test_graph_captured_step_matches_reference_golden(cuda, name):
    """Four fused steps at lr 0, so the weights stay the golden ones: the third and fourth replay the captured step graph.
    Adam zeroes the gradient after each step; with the same gradient g on every step its first moment is
    (1 - beta1^4) g, which is compared with the reference's gradients."""
    z = _load("d64h2")
    model, _ = _golden_model(z)
    kind, ft, pm, lab, tm, neg = _batch(z, cuda, name)
    model.loss = _spec(kind, int(z["ignore_index"]) if kind != "ce" else int(z["n_items"]))
    model.train()
    rw = ft["sample_weight"][..., 0] if "sample_weight" in ft else None
    losses = [float(model.core.fused_step(ft["item_id"], pm, lab, tm, all_reduce=None, lr=0.0, negatives=neg,
                                          row_weights=rw, feats=ft)) for _ in range(4)]
    core = model.core
    eng = core.engine
    b1 = core.adam_betas[0]
    m = {k: eng.adam_m[o:o + int(np.prod(s))].view(s) for k, (o, s) in eng.layout.items()}
    G = {core._keymap[k]: core._to_ref(k, eng.export_named(k, m)).double().cpu() / (1 - b1 ** 4) for k in eng.params}
    for loss in losses:
        _check_case(z, name, loss, G)


def test_adam_step_matches_reference_golden(cuda):
    """one graph-step of Adam (lr 1e-3, the reference's betas) from the golden weights: the reference's checksums of the
    updated parameters.  Adam's first step moves each element by about lr on the sign of its gradient, so the sums are
    compared to a share of the total movement; in_proj_bias is left out (its key third's gradient is rounding noise)."""
    z = _load("d64h2")
    model, sd = _golden_model(z)
    kind, ft, pm, lab, tm, neg = _batch(z, cuda, "ce")
    model.loss = _spec("ce", int(z["n_items"]))
    model.train()
    model.core.fused_step(ft["item_id"], pm, lab, tm, all_reduce=None, lr=1e-3, feats=ft)
    got = model.state_dict()
    for k, (s_ref, _) in zip((str(k) for k in z["sd_keys"]), z["adam_checksum"]):
        if k.endswith("in_proj_bias"):
            continue
        p0, p1 = sd[k].double(), got[k].double().cpu().reshape(sd[k].shape)
        moved = float((p1 - p0).abs().sum())
        assert moved > 0, k
        assert abs(float(p1.sum()) - s_ref) <= 0.05 * moved + 1e-6 * abs(s_ref), k


def test_item_only_schema_builds_the_item_only_model(cuda):
    """a side-feature schema with every side feature excluded builds the item-only model: the same seeded weights bit for
    bit, the same first loss bit for bit, and the same weights after three steps up to the item table's atomic sums"""
    from replay_b200.nn.sequential.twotower import TwoTower
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    z = _load("d64h2")
    n, d, L = int(z["n_items"]), int(z["d"]), int(z["L"])
    kw = dict(embedding_dim=d, num_heads=2, num_blocks=2, max_sequence_length=L, dropout=0.2, seed=7)
    a = TwoTower.from_params(TensorSchema(TensorFeatureInfo("item_id", n, n, d)), _Reader({"item_id": torch.arange(n)}), **kw)
    side = [str(f) for f in z["f_name"]]
    b = TwoTower.from_params(_schema(z), _Reader({"item_id": torch.arange(n)}), excluded_features=side, **kw)
    assert b.core.cfg.features == () and b.core.cfg.item_features == ()
    assert torch.equal(a.core.flat.detach(), b.core.flat.detach())
    ids, pm, lab, tm = (torch.from_numpy(z[k]).to(cuda) for k in ("ids", "pad_mask", "labels", "target_mask"))
    for m in (a, b):
        m.loss = _spec("ce", n)
        m.train()
    la = [float(a.core.fused_step(ids, pm, lab, tm, all_reduce=None, lr=1e-3)) for _ in range(3)]
    lb = [float(b.core.fused_step(ids, pm, lab, tm, all_reduce=None, lr=1e-3)) for _ in range(3)]
    assert la[0] == lb[0], (la, lb)
    torch.testing.assert_close(a.core.flat, b.core.flat, rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("tag", TAGS)
def test_tower_over_the_catalog_in_passes(cuda, tag):
    """the eval tower over the catalog in passes of 16 rows (catalogs of 60 and 45 items: a short last pass) equals the
    single pass"""
    z = _load(tag)
    model, _ = _golden_model(z)
    model.eval()
    one = model.core.item_table().clone()
    eng = model.core.engine
    assert not eng.with_grad and eng._tower_rows() == int(z["n_items"])
    eng.INFER_ROWS = 16
    eng.tower_valid = False
    many = model.core.item_table()
    assert eng._tower_rows() == 16
    torch.testing.assert_close(many.float(), one.float(), rtol=0, atol=0)


@pytest.mark.parametrize("tag", TAGS)
def test_inference_matches_reference_golden(cuda, tag):
    z = _load(tag)
    model, _ = _golden_model(z)
    ft, pm = _ft(z, cuda), torch.from_numpy(z["pad_mask"]).to(cuda)
    live = pm.any(1).cpu()
    model.eval()
    cand = torch.from_numpy(z["candidates"]).to(cuda)
    # candidates before any catalog pass: the tower over the candidates' own features
    lc = model(feature_tensors=ft, padding_mask=pm, candidates_to_score=cand)["logits"].cpu().double()
    refc = torch.from_numpy(z["cand_logits_nocache"]).double()
    assert (lc[live] - refc[live]).abs().max() <= 3e-2 * refc[live].abs().max()
    lo = model(feature_tensors=ft, padding_mask=pm)["logits"].cpu().double()
    ref = torch.from_numpy(z["eval_logits"]).double()
    assert (lo[live] - ref[live]).abs().max() <= 3e-2 * ref[live].abs().max()
    lc = model(feature_tensors=ft, padding_mask=pm, candidates_to_score=cand)["logits"].cpu().double()
    refc = torch.from_numpy(z["cand_logits"]).double()
    assert (lc[live] - refc[live]).abs().max() <= 3e-2 * refc[live].abs().max()
    assert list(model.state_dict()) == [str(k) for k in z["cache_keys"]]
    # seen-filtered top-10 against the reference's, where its 10th and 11th scores are apart by more than the tolerance
    ids = ft["item_id"]
    seen = ids.masked_fill(~pm, int(z["n_items"]))
    got, _ = model.predict_topk(ft, pm, 10, seen_ids=seen)
    scores = ref.clone()
    for b in range(ids.shape[0]):
        scores[b, ids[b][pm[b]].cpu()] = -torch.inf
    top11 = torch.topk(scores, 11, dim=-1).values
    clear = live & ((top11[:, 9] - top11[:, 10]) > 6e-2 * ref.abs().max())
    want = torch.from_numpy(z["top10"])
    assert clear.sum() > 0
    assert torch.equal(got.cpu()[clear].sort(-1).values, want[clear].sort(-1).values)


@pytest.mark.parametrize("tag", TAGS)
def test_state_dict_has_reference_keys_and_round_trips(cuda, tag):
    z = _load(tag)
    model, sd = _golden_model(z)
    got = model.state_dict()
    assert list(got) == [str(k) for k in z["keys"]]
    for k, shp, dt in zip(z["keys"], z["key_shapes"], z["key_dtypes"]):
        assert "x".join(map(str, got[str(k)].shape)) == str(shp), k
        assert str(got[str(k)].dtype) == str(dt), k
    for k, v in sd.items():   # the golden weights come back (bf16-free: the fp32 master copy)
        torch.testing.assert_close(got[k].float().cpu(), v.float(), rtol=0, atol=0)
    other, _ = _golden_model(z, seed=5)
    other.load_state_dict({k: v.clone() for k, v in got.items()})
    back = other.state_dict()
    for k in got:
        assert torch.equal(back[k], got[k]), k
    bad = dict(got)
    bad["body.item_tower.item_reference_genre"] = got["body.item_tower.item_reference_genre"].flip(0)
    with pytest.raises(ValueError, match="reader"):
        other.load_state_dict(bad)


# ---------------------------------------------------------------------------------------------------------- the kernels
def _kernel_case(dev, d_true, n_items, seed=0):
    """item table, a 20-row categorical, a one-row categorical, sum and mean bags of width 4 (all-padding bags, repeated
    ids, ids outside the table), numerical features of tensor_dim 1 and 3 and an identity feature, over ``n_items``."""
    g = torch.Generator().manual_seed(seed + d_true + n_items)
    dp = d_true if d_true % 64 == 0 else 64 * ((d_true + 63) // 64)
    hd_valid = 0 if dp == d_true else d_true
    item = (torch.randn(n_items + 1, dp, generator=g) * 0.3).to(torch.bfloat16)
    spec = []
    for kind, card, K in ((FEAT_CAT, 20, 1), (FEAT_CAT, 1, 1), (FEAT_BAG_SUM, 9, 4), (FEAT_BAG_MEAN, 9, 4)):
        tab = (torch.randn(card + 1, dp, generator=g) * 0.3).to(torch.bfloat16)
        tab[card] = 0
        v = torch.randint(0, card + 1, (n_items, K), generator=g)
        if n_items > 3:
            v[0] = card                       # the padding value / an all-padding bag
            v[1, 0] = -3                      # ids outside the table
            v[2, -1] = card + 5
            if K > 1:
                v[3, 1] = v[3, 0]             # a repeated id
        spec.append(dict(kind=kind, width=K, card=card, table=tab, values=v.to(torch.int32)))
    for width in (1, 3):
        spec.append(dict(kind=FEAT_NUM, width=width, table=torch.randn(dp, width, generator=g) * 0.3,
                         bias=torch.randn(dp, generator=g) * 0.1, values=torch.randn(n_items, width, generator=g)))
    spec.append(dict(kind=FEAT_IDENT, width=d_true, values=torch.randn(n_items, d_true, generator=g)))
    if hd_valid:   # the padded feature columns of every table, weight and bias are zero, as the engine keeps them
        item[:, d_true:] = 0
        for f in spec:
            if f["kind"] == FEAT_NUM:
                f["table"][d_true:] = 0
                f["bias"][d_true:] = 0
            elif "table" in f:
                f["table"][:, d_true:] = 0
    return dict(d=d_true, dp=dp, hd_valid=hd_valid, n_items=n_items, item=item, spec=spec)


def _descs(c, dev, with_grad):
    arr = (RpFeature * len(c["spec"]))()
    col = 0
    for k, f in enumerate(c["spec"]):
        a = arr[k]
        a.kind, a.width = f["kind"], f["width"]
        f["dev_values"] = f["values"].to(dev)
        a.values = f["dev_values"].data_ptr()
        if f["kind"] in (FEAT_CAT, FEAT_BAG_SUM, FEAT_BAG_MEAN):
            a.n_rows, a.padding_value = f["card"] + 1, f["card"]
            f["dev_table"] = f["table"].to(dev)
            a.table = f["dev_table"].data_ptr()
            if with_grad:
                f["dev_grad"] = torch.full((f["card"] + 1, c["dp"]), 0.25, device=dev)   # the kernels add onto it
                a.d_table = f["dev_grad"].data_ptr()
        elif f["kind"] == FEAT_NUM:
            f["dev_table"], f["dev_bias"] = f["table"].to(dev), f["bias"].to(dev)
            a.table, a.bias, a.val_col = f["dev_table"].data_ptr(), f["dev_bias"].data_ptr(), col
            col += f["width"]
    return arr


def _pad_cols(c):
    """padded column of each true feature"""
    if not c["hd_valid"]:
        return torch.arange(c["dp"])
    return torch.tensor([(j // c["hd_valid"]) * 64 + j % c["hd_valid"] for j in range(c["d"])])


def _live(v, card):
    return (v != card) & (v >= 0) & (v <= card)


def _x0_reference(c, items):
    """float64 X0 [len(items), dp] and the per-element sum of |terms| (the bound's scale)"""
    dp = c["dp"]
    x = c["item"][items].double()
    mag = x.abs()
    for f in c["spec"]:
        v = f["values"][items]
        if f["kind"] in (FEAT_CAT, FEAT_BAG_SUM, FEAT_BAG_MEAN):
            tab = f["table"].double()
            live = _live(v, f["card"])
            rows = tab[v.clamp(0, f["card"]).long()] * live[..., None]
            s = rows.sum(1)
            if f["kind"] == FEAT_BAG_MEAN:
                s = s / live.sum(1, keepdim=True).clamp(min=1)
            x, mag = x + s, mag + rows.abs().sum(1)
        elif f["kind"] == FEAT_NUM:
            t = v.double() @ f["table"].double().T + f["bias"].double()
            x, mag = x + t, mag + (v.double().abs() @ f["table"].double().abs().T) + f["bias"].double().abs()
        else:
            t = torch.zeros(len(items), dp, dtype=torch.float64)
            t[:, _pad_cols(c)] = v.double()
            x, mag = x + t, mag + t.abs()
    return x, mag


def _check_x0(out, c, items):
    """|out - X0| <= rounding to bf16 once (u |X0|) + fp32 sums (n_terms * 2^-23 * sum|terms|)"""
    ref, mag = _x0_reference(c, items)
    n_terms = 1 + sum(f["width"] for f in c["spec"])
    bound = U_BF16 * ref.abs() + n_terms * 2.0 ** -23 * mag + 1e-30
    err = (out.double().cpu() - ref).abs()
    assert float((err / bound).max()) <= 1.0, float((err / bound).max())


@pytest.mark.parametrize("n_rows", [127, 128, 129])
@pytest.mark.parametrize("d", [64, 50, 128])
def test_item_feature_fwd_over_the_catalog(cuda, n_rows, d):
    """a catalog pass at an item offset (a catalog that is not a multiple of the pass size)"""
    c = _kernel_case(cuda, d, 300)
    fa = _descs(c, cuda, False)
    item = c["item"].to(cuda)
    item0 = 300 - n_rows
    out = torch.full((n_rows, c["dp"]), float("nan"), device=cuda, dtype=torch.bfloat16)
    check(_lib().rp_item_feature_embed_fwd(item.data_ptr(), fa, len(fa), None, None, n_rows, item0, c["dp"], c["hd_valid"],
                                        out.data_ptr(), None), "rp_item_feature_embed_fwd")
    torch.cuda.synchronize()
    _check_x0(out, c, torch.arange(item0, 300))
    if c["hd_valid"]:
        pad = torch.ones(c["dp"], dtype=torch.bool)
        pad[_pad_cols(c)] = False
        assert torch.all(out[:, pad.to(cuda)] == 0)


@pytest.mark.parametrize("n_slots", [0, 1, 40])
def test_item_feature_fwd_on_slots(cuda, n_slots):
    """compacted slots: rows from *n_slots on are zero (cap = 40, item_of_slot -1 there)"""
    cap = 40
    c = _kernel_case(cuda, 64, 200)
    fa = _descs(c, cuda, False)
    item = c["item"].to(cuda)
    items = torch.randperm(200, generator=torch.Generator().manual_seed(3))[:n_slots].sort().values
    ios = torch.full((cap,), -1, dtype=torch.int32)
    ios[:n_slots] = items.to(torch.int32)
    ios, ns = ios.to(cuda), torch.tensor([n_slots], dtype=torch.int32, device=cuda)
    out = torch.full((cap, c["dp"]), float("nan"), device=cuda, dtype=torch.bfloat16)
    check(_lib().rp_item_feature_embed_fwd(item.data_ptr(), fa, len(fa), ios.data_ptr(), ns.data_ptr(), cap, 0, c["dp"], 0,
                                        out.data_ptr(), None), "rp_item_feature_embed_fwd")
    torch.cuda.synchronize()
    if n_slots:
        _check_x0(out[:n_slots], c, items)
    assert torch.all(out[n_slots:] == 0)


def _table_grad_reference(c, f, dx, items):
    """float64 d_table of categorical feature f from dx rows (row s is item items[s]) and its magnitude"""
    v = f["values"][items]
    live = _live(v, f["card"]).double()
    w = live
    if f["kind"] == FEAT_BAG_MEAN:
        w = live / live.sum(1, keepdim=True).clamp(min=1)
    g = torch.zeros(f["card"] + 1, c["dp"], dtype=torch.float64)
    m = torch.zeros_like(g)
    idx = v.clamp(0, f["card"]).long()
    for j in range(v.shape[1]):
        g.index_add_(0, idx[:, j], dx * w[:, j:j + 1])
        m.index_add_(0, idx[:, j], dx.abs() * w[:, j:j + 1])
    return g, m


def _plan(c, dev, chunk):
    from replay_b200.engine_twotower import TwoTowerEngine

    class _Fake:   # _build_item_plan reads item_feats, dev, cfg.dp and ITEM_PLAN_CHUNK only
        ITEM_PLAN_CHUNK = chunk

    from replay_b200.engine import SideFeature

    kinds = {FEAT_CAT: "cat", FEAT_BAG_SUM: "bag_sum", FEAT_BAG_MEAN: "bag_mean", FEAT_NUM: "num", FEAT_IDENT: "ident"}
    fake = _Fake()
    fake.item_feats = tuple(SideFeature(f"f{k}", kinds[f["kind"]], f.get("card", 0), f.get("card", 0), f["width"])
                            for k, f in enumerate(c["spec"]))
    fake.item_in = {f"f{k}": f["values"] for k, f in enumerate(c["spec"])}
    fake.dev = dev
    fake.cfg = type("C", (), {"dp": c["dp"]})()
    return TwoTowerEngine._build_item_plan(fake, fake.item_in)


def _run_bwd(c, dev, dx, ios=None, ns=None, chunk=32):
    fa = _descs(c, dev, True)
    n_rows = dx.shape[0]
    v_rows = torch.full((n_rows, 64), 7.0, device=dev, dtype=torch.bfloat16)
    plan = None
    if ios is None:
        p = _plan(c, dev, chunk)
        plan = p["desc"]
    check(_lib().rp_item_feature_embed_bwd(dx.data_ptr(), fa, len(fa), None if ios is None else ios.data_ptr(),
                                        None if ns is None else ns.data_ptr(), n_rows, c["dp"], c["hd_valid"],
                                        None if plan is None else plan, v_rows.data_ptr(), 64, None),
          "rp_item_feature_embed_bwd")
    torch.cuda.synchronize()
    return {k: f["dev_grad"].cpu().clone() for k, f in enumerate(c["spec"]) if "dev_grad" in f}, v_rows.cpu()


def _check_bwd(c, grads, v_rows, dx, items, n_live_rows):
    dx64 = dx.double().cpu()[:len(items)]
    for k, f in enumerate(c["spec"]):
        if k in grads:
            ref, mag = _table_grad_reference(c, f, dx64, items)
            ref = ref + 0.25
            ref[f["card"]] = 0.25                   # the padding row is frozen
            # per table row: its live entries (each a rounded product w * dx), summed in some order onto the start value
            v = f["values"][items]
            n_add = torch.zeros(f["card"] + 1, dtype=torch.float64)
            n_add.index_add_(0, v.clamp(0, f["card"]).long().flatten(), _live(v, f["card"]).double().flatten())
            bound = (n_add[:, None] + 2) * 2.0 ** -23 * (mag + 0.25) + 1e-30
            err = (grads[k].double() - ref).abs()
            assert float((err / bound).max()) <= 1.0, (k, float((err / bound).max()))
    col = 0
    for f in c["spec"]:
        if f["kind"] == FEAT_NUM:
            want = f["values"][items].to(torch.bfloat16)
            assert torch.equal(v_rows[:n_live_rows, col:col + f["width"]], want)
            col += f["width"]
    assert torch.all(v_rows[:n_live_rows, col:] == 0)


@pytest.mark.parametrize("n_items", [1, 127, 129, 3000])
@pytest.mark.parametrize("d", [64, 50])
def test_item_feature_bwd_over_the_catalog_is_fixed_order(cuda, n_items, d):
    """the full-catalog backward against float64 (a 20-row table takes ~n/20 rows per table row; the one-row table every
    live row) and bitwise equal over two runs and over two chunk sizes' worth of re-association checks"""
    c = _kernel_case(cuda, d, n_items)
    g = torch.Generator().manual_seed(9)
    dx = (torch.randn(n_items, c["dp"], generator=g) * 0.5).to(torch.bfloat16)
    if c["hd_valid"]:
        dx[:, c["d"]:] = 0
    dx = dx.to(cuda)
    a, va = _run_bwd(c, cuda, dx)
    b, vb = _run_bwd(c, cuda, dx)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    _check_bwd(c, a, va, dx, torch.arange(n_items), n_items)
    c2, _ = _run_bwd(c, cuda, dx, chunk=5)   # another chunking: the same sums within the bound
    _check_bwd(c, c2, va, dx, torch.arange(n_items), n_items)


@pytest.mark.parametrize("n_slots", [0, 1, 40])
def test_item_feature_bwd_on_slots(cuda, n_slots):
    cap = 40
    c = _kernel_case(cuda, 64, 200)
    items = torch.randperm(200, generator=torch.Generator().manual_seed(4))[:n_slots].sort().values
    ios = torch.full((cap,), -1, dtype=torch.int32)
    ios[:n_slots] = items.to(torch.int32)
    dx = (torch.randn(cap, c["dp"], generator=torch.Generator().manual_seed(5)) * 0.5).to(torch.bfloat16)
    dx[n_slots:] = 0
    grads, v_rows = _run_bwd(c, cuda, dx.to(cuda), ios.to(cuda), torch.tensor([n_slots], dtype=torch.int32, device=cuda))
    _check_bwd(c, grads, v_rows, dx, items, n_slots)
    assert torch.all(v_rows[n_slots:] == 7.0)   # rows past the slots are not written


def test_item_feature_api_errors(cuda):
    c = _kernel_case(cuda, 64, 10)
    fa = _descs(c, cuda, False)
    out = torch.zeros(10, 64, device=cuda, dtype=torch.bfloat16)
    item = c["item"].to(cuda)
    assert _lib().rp_item_feature_embed_fwd(None, fa, len(fa), None, None, 10, 0, 64, 0, out.data_ptr(), None) != 0
    assert _lib().rp_item_feature_embed_fwd(item.data_ptr(), fa, len(fa), None, None, 10, 0, 96, 0, out.data_ptr(), None) != 0
    fg = _descs(c, cuda, True)
    assert _lib().rp_item_feature_embed_bwd(out.data_ptr(), fg, len(fg), None, None, 10, 64, 0, None, None, 64, None) != 0
    ios = torch.arange(10, device=cuda, dtype=torch.int32)
    ns = torch.tensor([10], device=cuda, dtype=torch.int32)
    assert _lib().rp_item_feature_embed_bwd(out.data_ptr(), fg, len(fg), ios.data_ptr(), ns.data_ptr(), 10, 64, 0,
                                            ItemFeaturePlan(), None, 64, None) != 0   # the slots' values need v_rows
