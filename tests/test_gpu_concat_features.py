"""The new-path SASRec with ConcatAggregator on the GPU: the gather kernel (csrc/rp_features.cu) bit for bit against a torch
gather, the engine's concat input stage forward and backward against a float64 restatement at every padded width edge,
the training step and eval logits against the goldens of the real reference (oracle/gen_concat_features_golden.py), packed
against padded rows, the item-only concat model against the item-only model, the fused steps and the fused top-K."""
import ctypes
import os

import numpy as np
import pytest
import torch

from dropout_stream import keep_draws
from oracle import concat_features as ocf
from oracle import side_features as osf
from replay_b200._lib import FEAT_BAG_MEAN, FEAT_BAG_SUM, FEAT_CAT, FEAT_IDENT, FEAT_NUM, RpFeature, check, lib
from replay_b200.engine import EncoderConfig, SasRecEngine, SideFeature
from replay_b200.nn.agg import ConcatAggregator, SumAggregator
from replay_b200.nn.embedding import SequenceEmbedding
from replay_b200.nn.mask import DefaultAttentionMask
from replay_b200.nn.sequential.sasrec import PositionAwareAggregator, SasRec, SasRecBody, SasRecTransformerLayer
from replay_b200.schema import TensorFeatureInfo, TensorSchema

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CAT_KINDS = (FEAT_CAT, FEAT_BAG_SUM, FEAT_BAG_MEAN)


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda")


# ---------------------------------------------------------------------------------------------------------------- gather
def _gather_case(dev, T, hd_valid, seed=0):
    """Odd segment widths (11, 13, 5, 7, 9), ids 0, cardinality - 1 and the padding value, bags with empty entries, a
    numerical and an identity feature; the item segment in the middle."""
    g = torch.Generator().manual_seed(seed)
    D = 64
    d_true = hd_valid or D
    n_items = 300
    item = (torch.randn(n_items + 1, D, generator=g) * 0.1)
    if hd_valid:
        item[:, d_true:] = 0
    item = item.to(torch.bfloat16)
    ids = torch.randint(0, n_items + 1, (T,), generator=g).to(torch.int32)
    ids[:3] = torch.tensor([0, n_items - 1, n_items])
    spec = []
    for kind, card, K, w in ((FEAT_CAT, 7, 1, 11), (FEAT_BAG_SUM, 9, 4, 13), (FEAT_BAG_MEAN, 5, 3, 9)):
        tab = (torch.randn(card + 1, w, generator=g) * 0.1).to(torch.bfloat16)
        v = torch.randint(0, card + 1, (T, K), generator=g).to(torch.int32)
        v[0], v[1], v[2] = 0, card - 1, card   # first row, last row, an all-padding bag
        spec.append(dict(kind=kind, width=K, card=card, dim=w, table=tab, values=v))
    spec.append(dict(kind=FEAT_NUM, width=3, dim=7, table=torch.randn(7, 3, generator=g) * 0.3,
                     bias=torch.randn(7, generator=g) * 0.1, values=torch.randn(T, 3, generator=g)))
    spec.append(dict(kind=FEAT_IDENT, width=5, dim=5, values=torch.randn(T, 5, generator=g)))
    order = [0, 1, "item", 2, 3, 4]
    col, item_col = 0, 0
    for o in order:
        if o == "item":
            item_col, col = col, col + d_true
        else:
            spec[o]["col"] = col
            col += spec[o]["dim"]
    return dict(T=T, D=D, d_true=d_true, hd_valid=hd_valid, n_items=n_items, item=item, ids=ids, spec=spec,
                item_col=item_col, width=col)


def _descs(c, dev, with_grad=False):
    n = len(c["spec"])
    arr, cols, dims = (RpFeature * n)(), (ctypes.c_int * n)(), (ctypes.c_int * n)()
    vc = 0
    for k, f in enumerate(c["spec"]):
        a = arr[k]
        a.kind, a.width = f["kind"], f["width"]
        cols[k], dims[k] = f["col"], f["dim"]
        f["dev_values"] = f["values"].to(dev).contiguous()
        a.values = f["dev_values"].data_ptr()
        if f["kind"] in CAT_KINDS:
            a.n_rows, a.padding_value = f["card"] + 1, f["card"]
            f["dev_table"] = f["table"].to(dev)
            a.table = f["dev_table"].data_ptr()
            if with_grad:
                f["dev_grad"] = torch.zeros(f["card"] + 1, f["dim"], device=dev)
                a.d_table = f["dev_grad"].data_ptr()
        elif f["kind"] == FEAT_NUM:
            f["dev_table"], f["dev_bias"] = f["table"].to(dev), f["bias"].to(dev)
            a.table, a.bias, a.val_col = f["dev_table"].data_ptr(), f["dev_bias"].data_ptr(), vc
            vc += f["width"]
    return arr, cols, dims


def _torch_gather(c, rows):
    """X bf16 [len(rows), kp-free width] from the same bf16 tables, summed in the kernel's fp32 order"""
    tok = rows.long()
    feat = torch.arange(c["d_true"])
    if c["hd_valid"]:
        feat = (feat // c["hd_valid"]) * 64 + feat % c["hd_valid"]
    X = torch.zeros(len(tok), c["width"], dtype=torch.bfloat16)
    X[:, c["item_col"]:c["item_col"] + c["d_true"]] = c["item"][c["ids"].long()[tok]][:, feat]
    for f in c["spec"]:
        sl = slice(f["col"], f["col"] + f["dim"])
        if f["kind"] in CAT_KINDS:
            v = f["values"].long()[tok]
            live = v != f["card"]
            acc = torch.zeros(len(tok), f["dim"], dtype=torch.float32)
            for i in range(v.shape[1]):
                acc = acc + torch.where(live[:, i:i + 1], f["table"][v[:, i]].float(), torch.zeros(()))
            if f["kind"] == FEAT_BAG_MEAN:
                acc = acc * (1.0 / live.sum(1, keepdim=True).clamp_min(1).float())
            X[:, sl] = acc.to(torch.bfloat16)
        elif f["kind"] == FEAT_NUM:
            X[:, sl] = (f["values"][tok].double() @ f["table"].double().T + f["bias"].double()).to(torch.bfloat16)
        else:
            X[:, sl] = f["values"][tok].to(torch.bfloat16)
    return X


@pytest.mark.parametrize("T", [65, 300])
@pytest.mark.parametrize("hd_valid", [0, 50])
@pytest.mark.parametrize("packed", [False, True])
def test_concat_gather_matches_torch_gather(cuda, T, hd_valid, packed):
    c = _gather_case(cuda, T, hd_valid)
    arr, cols, dims = _descs(c, cuda)
    kp = 128
    x = torch.full((T, kp), float("nan"), device=cuda, dtype=torch.bfloat16)
    item, ids = c["item"].to(cuda), c["ids"].to(cuda)
    st = torch.cuda.current_stream().cuda_stream
    if packed:   # a permuted subset of the tokens, as rp_row_plan would pack them
        n = T - 7
        rows = torch.randperm(T, generator=torch.Generator().manual_seed(3))[:n].to(torch.int32)
        rt, nr = rows.to(cuda), torch.tensor([n], device=cuda, dtype=torch.int32)
        check(lib().rp_concat_gather_rows(item.data_ptr(), ids.data_ptr(), arr, cols, dims, len(arr), c["item_col"],
                                          rt.data_ptr(), nr.data_ptr(), T, c["D"], hd_valid, kp, x.data_ptr(), st), "gather_rows")
    else:
        n, rows = T, torch.arange(T, dtype=torch.int32)
        check(lib().rp_concat_gather(item.data_ptr(), ids.data_ptr(), arr, cols, dims, len(arr), c["item_col"], T, c["D"],
                                     hd_valid, kp, x.data_ptr(), st), "gather")
    got = x[:n].cpu()
    ref = _torch_gather(c, rows)
    W = c["width"]
    assert (got[:, W:] == 0).all()                        # zero tail
    assert not torch.isnan(x[n:]).logical_not().any()     # rows past the packed count are not written
    exact = [slice(c["item_col"], c["item_col"] + c["d_true"])]
    exact += [slice(f["col"], f["col"] + f["dim"]) for f in c["spec"] if f["kind"] in (FEAT_CAT, FEAT_BAG_SUM, FEAT_IDENT)]
    for sl in exact:
        assert torch.equal(got[:, sl], ref[:, sl]), sl
    for f in c["spec"]:
        sl = slice(f["col"], f["col"] + f["dim"])
        if f["kind"] == FEAT_BAG_MEAN:   # 1 / count may be an approximate reciprocal under fast math: one bf16 step
            assert torch.allclose(got[:, sl].float(), ref[:, sl].float(), rtol=8e-3, atol=1e-6), sl
        elif f["kind"] == FEAT_NUM:      # fp32 FMAs against fp64, both rounded to bf16
            assert torch.allclose(got[:, sl].float(), ref[:, sl].float(), rtol=8e-3, atol=1e-3), sl


# ---------------------------------------------------------------------------------------------------------------- stage
def _stage_cfg(widths, d, heads, drop):
    """a concat config whose features are a categorical, a sum bag, a numerical and an identity feature of these widths"""
    kinds = [("c", "cat", 9, 1), ("b", "bag_sum", 6, 1), ("n", "num", 0, 3), ("v", "ident", 0, None)]
    feats = tuple(SideFeature(nm, k, card, card, w if wd is None else wd, w)
                  for (nm, k, card, wd), w in zip(kinds, widths))
    return EncoderConfig(n_items=120, d=d, n_heads=heads, n_blocks=1, max_len=16, dropout=drop, features=feats,
                         aggregator="concat", concat_item_at=2)


@pytest.mark.parametrize("widths,d,heads", [
    ((3, 4, 2, 5), 40, 1),          # 40 + 14 = 54 columns: kp 64, below the 64-column boundary
    ((3, 4, 2, 5), 50, 1),          # 64 columns: kp 64, at it
    ((3, 4, 2, 5), 64, 1),          # 78 columns: kp 128, past it
    ((250, 300, 200, 200), 64, 2),  # 1014 columns: kp 1024, the cap
])
@pytest.mark.parametrize("packed", [False, True])
def test_concat_stage_matches_fp64(cuda, widths, d, heads, packed):
    drop = 0.2
    cfg = _stage_cfg(widths, d, heads, drop)
    B, L = 5, 16
    eng = SasRecEngine(cfg, B, L, cuda, seed=7, with_grad=True)
    eng.packed_body = packed
    g = torch.Generator().manual_seed(11)
    ids = torch.randint(0, cfg.n_items, (B, L), generator=g)
    pm = torch.ones(B, L, dtype=torch.bool)
    for b in range(B):
        pm[b, : b * 3] = False
    ids[~pm] = cfg.n_items
    labels = torch.randint(0, cfg.n_items, (B, L), generator=g)
    feats = {"c": torch.randint(0, 10, (B, L), generator=g), "b": torch.randint(0, 7, (B, L, 3), generator=g),
             "n": torch.randn(B, L, 3, generator=g), "v": torch.randn(B, L, widths[3], generator=g)}
    eng.set_batch(ids.to(cuda), pm.to(cuda), labels.to(cuda), pm.to(cuda))
    eng.set_features({k: v.to(cuda) for k, v in feats.items()})
    eng.rng_counter.fill_(5)
    eng._prepare(True)
    assert eng._packed == packed
    T, dp, kp = eng.T, cfg.dp, cfg.concat_kp
    pos0 = cfg.max_len - L
    eng._embed_fwd(drop, pos0)
    n = int(eng.n_rows) if packed else T
    tok = eng.row_tok[:n].long().cpu() if packed else torch.arange(T)
    X = eng.cat_x[:n].double().cpu()
    W = eng.params16["feat_proj.w"].double().cpu()
    bias = eng.params["feat_proj.b"].double().cpu()
    P = eng.params["pos_emb"].double().cpu()
    keep = keep_draws(eng.seed + 5, 0, drop, tok.numpy(), dp).double()
    ks = 1.0 / (1.0 - drop)
    scale = cfg.d ** 0.5
    ref = ((X @ W.T + bias) * scale + P[pos0 + tok % L]) * keep * ks
    got = eng.x[0][:n].double().cpu()
    assert torch.allclose(got, ref, rtol=1e-2, atol=2e-2 * ref.abs().max().item() / 8), (got - ref).abs().max()
    # the gathered segments: the item's true features, then the side terms at their widths
    item_col, cols = cfg.concat_columns()
    feat = eng._feat.cpu()
    assert torch.equal(eng.cat_x[:n, item_col:item_col + cfg.d].cpu(), eng.params16["item_emb"][eng.ids32.long()][:, feat][tok.to(eng.dev)].cpu())
    assert (eng.cat_x[:n, cfg.concat_width:] == 0).all()
    # backward of the stage from a random block-input gradient (zero in padded feature columns)
    G = eng.grads
    eng.g32.zero_()
    dx = torch.zeros(T, dp, dtype=torch.bfloat16)
    dx[:, feat] = (torch.randn(T, cfg.d, generator=g) * 0.1).to(torch.bfloat16)
    dx_dev = dx.to(cuda)
    eng._concat_bwd(dx_dev, drop, pos0)
    dxr = dx[:n].double()
    dY = dxr * keep * ks * scale
    dX = dY @ W
    want = {"feat_proj.w": dY.T @ X, "feat_proj.b": dY.sum(0)}
    d_item = torch.zeros(cfg.n_items + 1, dp, dtype=torch.float64)
    idt = eng.ids32.long().cpu()[tok]
    live = idt != cfg.pad_id
    d_item[:, feat] = d_item[:, feat].index_add(0, idt[live], dX[live, item_col:item_col + cfg.d])
    want["item_emb"] = d_item
    d_pos = torch.zeros(cfg.max_len, dp, dtype=torch.float64)
    want["pos_emb"] = d_pos.index_add(0, pos0 + tok % L, dxr * keep * ks)
    for f, c0 in zip(cfg.features, cols):
        seg = dX[:, c0:c0 + f.dim]
        v = feats[f.name].reshape(B * L, -1)[tok]
        if f.categorical:
            tab = torch.zeros(f.cardinality + 1, f.dim, dtype=torch.float64)
            for i in range(v.shape[1]):
                ok = v[:, i] != f.padding_value
                tab.index_add_(0, v[ok, i], seg[ok])
            want[f"feat.{f.name}"] = tab
        elif f.kind == "num":
            want[f"feat.{f.name}.w"] = seg.T @ v.double()
            want[f"feat.{f.name}.b"] = seg.sum(0)
    for k, ref_g in want.items():
        got_g = G[k].double().cpu()
        tol = 2e-2 * ref_g.abs().max().item() + 1e-6
        assert torch.allclose(got_g, ref_g, rtol=2e-2, atol=tol), (k, (got_g - ref_g).abs().max().item(), tol)


# ---------------------------------------------------------------------------------------------------------------- engine
def _golden(tag):
    z = np.load(os.path.join(GOLDEN, f"sasrec_concat_{tag}.npz"))
    specs = ocf.golden_specs(z)
    return z, specs, osf.golden_state_dict(z)


def _schema(z, specs):
    feats = []
    for f in specs:
        if f["kind"] in ("cat", "bag"):
            feats.append(TensorFeatureInfo(f["name"], f["cardinality"], f["padding_value"], f["dim"], is_list=f["kind"] == "bag"))
        else:
            feats.append(TensorFeatureInfo(f["name"], None, 0, f["dim"], is_cat=False, tensor_dim=f["width"]))
    n = int(z["n_items"])
    return TensorSchema(TensorFeatureInfo(str(z["item_name"]), n, n, int(z["d"])), features=feats)


def _body(z, specs, dropout=0.0, schema=None):
    sch = schema or _schema(z, specs)
    d, H = int(z["d"]), int(z["H"])
    return SasRecBody(SequenceEmbedding(sch, categorical_list_feature_aggregation_method=str(z["method"])),
                      PositionAwareAggregator(ConcatAggregator([f.embedding_dim for _, f in sch.items()], d), int(z["L"]), dropout),
                      DefaultAttentionMask(str(z["item_name"]), H),
                      SasRecTransformerLayer(d, H, int(z["n_blocks"]), dropout, "relu"), torch.nn.LayerNorm(d))


def _batch(z, specs, dev):
    ids, pm, lab, tm, feats = ocf.batch_of(z, specs)
    return ids.to(dev), pm.to(dev), lab.to(dev), tm.to(dev), {k: v.to(dev) for k, v in feats.items()}


def _grads(core):
    eng = core.engine
    return {core._keymap[k]: core._to_ref(k, eng.export_named(k, eng.grads)).cpu() for k in eng.params}


@pytest.mark.parametrize("tag", ["d64h2", "d50h1_mean", "item_only"])
@pytest.mark.parametrize("packed", [False, True])
def test_engine_step_matches_reference_golden(cuda, tag, packed):
    z, specs, sd = _golden(tag)
    core = _body(z, specs).build_core(device=cuda, seed=1)
    assert core.cfg.concat == bool(specs)
    core.load_state_dict(sd)
    ids, pm, lab, tm, feats = _batch(z, specs, cuda)
    core.ensure_engine(*ids.shape, with_grad=True).packed_body = packed
    loss = core.loss(ids, pm, lab, tm, feats=feats)
    loss.backward()
    assert abs(float(loss) - float(z["train_loss"])) < 1e-2 * abs(float(z["train_loss"]))
    assert core.engine._packed == packed
    G = _grads(core)
    assert set(G) == {str(k) for k in z["sd_keys"] if not str(k).endswith("._weight")}
    for k in G:
        ref = torch.from_numpy(z["grad::" + k]).float()
        got = G[k].float().reshape(ref.shape)
        if ref.norm() < 1e-12:
            assert got.norm() < 1e-6, k
            continue
        cos = float((got.double() * ref.double()).sum() / (got.double().norm() * ref.double().norm()))
        ratio = float(got.double().norm() / ref.double().norm())
        assert cos > 0.995 and abs(ratio - 1) < 0.03, (k, cos, ratio)
    # users with at least one real item: a user whose window is all padding attends over no key at all, so neither side's
    # last hidden state is a prediction (the goldens keep such a row for its training target)
    real = pm.any(1).cpu()
    logits = core.logits(ids, pm, feats=feats).cpu()[real]
    ref = torch.from_numpy(z["eval_logits"])[real]
    assert (logits - ref).abs().max() < 3e-2 * ref.abs().max(), (logits - ref).abs().max()


def test_packed_step_equals_padded_step(cuda):
    z, specs, sd = _golden("d64h2")
    out = []
    for packed in (False, True):
        core = _body(z, specs, dropout=0.2).build_core(device=cuda, seed=1)
        core.load_state_dict(sd)
        ids, pm, lab, tm, feats = _batch(z, specs, cuda)
        core.ensure_engine(*ids.shape, with_grad=True).packed_body = packed
        loss = core.loss(ids, pm, lab, tm, feats=feats)
        loss.backward()
        assert core.engine._packed == packed
        out.append((float(loss), _grads(core)))
    assert abs(out[0][0] - out[1][0]) < 1e-5 * abs(out[0][0])
    for k, v in out[0][1].items():
        assert torch.allclose(v, out[1][1][k], rtol=1e-3, atol=1e-5), k


def test_item_only_concat_equals_item_only_sum_bitwise(cuda):
    z, specs, _ = _golden("item_only")
    sch = _schema(z, specs)
    d, H = int(z["d"]), int(z["H"])
    ids, pm, lab, tm, _ = _batch(z, specs, cuda)
    out = []
    for agg in (ConcatAggregator([d], d), SumAggregator(d)):
        body = SasRecBody(SequenceEmbedding(sch), PositionAwareAggregator(agg, int(z["L"]), 0.2), DefaultAttentionMask("item_id", H),
                          SasRecTransformerLayer(d, H, int(z["n_blocks"]), 0.2, "relu"), torch.nn.LayerNorm(d))
        core = body.build_core(device=cuda, seed=5)
        core.ensure_engine(*ids.shape, with_grad=True)
        loss = core.loss(ids, pm, lab, tm)
        loss.backward()
        out.append((core.cfg, core.engine.p32.clone(), loss.detach().clone(), core.engine.g32.clone()))
    (cfg_c, p_c, loss_c, g_c), (cfg_s, p_s, loss_s, g_s) = out
    assert cfg_c == cfg_s and torch.equal(p_c, p_s) and torch.equal(loss_c, loss_s)
    # the table, position and LayerNorm gradients are summed with fp32 atomics, whose order varies from run to run even for
    # one model: equal up to that order
    assert torch.allclose(g_c, g_s, rtol=1e-4, atol=1e-7)


def test_state_dict_round_trip_uses_reference_keys(cuda):
    z, specs, sd = _golden("d50h1_mean")
    core = _body(z, specs).build_core(device=cuda, seed=1)
    core.load_state_dict(sd)
    out = core.state_dict()
    assert set(out) == set(sd)
    for k, v in sd.items():
        if k.endswith("._weight"):   # IdentityEmbedding's buffer: eye(embedding_dim) whatever the checkpoint holds
            assert torch.equal(out[k], torch.eye(v.shape[0])), k
            continue
        assert torch.equal(out[k].cpu().reshape(v.shape), v), k


def _fixture_schema():
    """the reference's ConcatAggregator fixture (tests/nn/conftest.py): widths 10 .. 14, the item at 10 in a 64-wide slot"""
    return TensorSchema(TensorFeatureInfo("item_id", 15, 15, 10), features=[
        TensorFeatureInfo("cat_list_feature", 4, 4, 11, is_list=True),
        TensorFeatureInfo("num_feature", None, 0, 12, is_cat=False, tensor_dim=1),
        TensorFeatureInfo("num_list_feature", None, 0, 13, is_cat=False, tensor_dim=6),
        TensorFeatureInfo("emb_list_feature", None, 0, 14, is_cat=False, tensor_dim=14)])


@pytest.mark.parametrize("loss", ["ce", "bce", "ce_sampled"])
def test_reference_fixture_model_trains_and_predicts(cuda, loss):
    """``sasrec_parametrized`` of the reference's tests, with SasRecTransformerLayer: fused Lightning steps lower the loss, and
    the fused top-K with the seen filter equals torch.topk of the materialised scores."""
    from replay_b200.nn.lightning.module import LightningModule
    from replay_b200.nn.loss import BCE, CE, CESampled

    sch = _fixture_schema()
    body = SasRecBody(SequenceEmbedding(sch, categorical_list_feature_aggregation_method="sum"),
                      PositionAwareAggregator(ConcatAggregator([f.embedding_dim for _, f in sch.items()], 10), 7, 0.2),
                      DefaultAttentionMask("item_id", 1), SasRecTransformerLayer(10, 1, 1, 0.2, "relu"), torch.nn.LayerNorm(10))
    spec = {"ce": CE(ignore_index=15), "bce": BCE(), "ce_sampled": CESampled()}[loss]
    model = SasRec(body=body, loss=spec, device=cuda, seed=2)
    assert model.core.cfg.concat
    g = torch.Generator().manual_seed(9)
    B, L = 16, 7
    ids = torch.randint(0, 15, (B, L), generator=g)
    pm = torch.ones(B, L, dtype=torch.bool)
    pm[:4, :3] = False
    ids[~pm] = 15
    lab = torch.roll(ids, -1, 1)
    tm = pm & torch.roll(pm, -1, 1)
    tm[:, -1] = False
    ft = {"item_id": ids, "cat_list_feature": torch.randint(0, 5, (B, L, 3), generator=g),
          "num_feature": torch.randn(B, L, generator=g), "num_list_feature": torch.randn(B, L, 6, generator=g),
          "emb_list_feature": torch.randn(B, L, 14, generator=g)}
    ft = {k: v.to(cuda) for k, v in ft.items()}
    batch = {"feature_tensors": ft, "padding_mask": pm.to(cuda), "positive_labels": lab.to(cuda).unsqueeze(-1),
             "target_padding_mask": tm.to(cuda).unsqueeze(-1)}
    if loss == "ce_sampled":
        batch["negative_labels"] = torch.randint(0, 15, (6,), device=cuda)
    module = LightningModule(model)
    losses = [float(module.training_step(batch)) for _ in range(12)]
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses
    model.eval()
    logits = model(ft, batch["padding_mask"])["logits"].float()
    assert torch.isfinite(logits).all()
    seen = ft["item_id"]
    masked = logits.clone()
    for b in range(B):
        s = seen[b][seen[b] < 15]
        masked[b, s] = float("-inf")
    got_ids, got_s = model.predict_topk(ft, batch["padding_mask"], 3, seen_ids=seen)
    ref_s, _ = torch.topk(masked, 3, dim=1)
    assert torch.allclose(got_s.float(), ref_s, rtol=1e-3, atol=1e-3)
    assert torch.allclose(masked.gather(1, got_ids.long()), got_s.float(), rtol=1e-3, atol=1e-3)
