"""The new-path SASRec with side features on the GPU: the embedding kernels (csrc/rp_features.cu) against a float64
restatement at the id, bag, width, dropout and hidden-size edges, the training step and eval logits against the goldens
of the real reference (oracle/gen_side_features_golden.py), packed against padded rows, the fused steps and predict."""
import os

import numpy as np
import pytest
import torch

from dropout_stream import keep_draws
from oracle import side_features as osf
from replay_b200._lib import FEAT_BAG_MEAN, FEAT_BAG_SUM, FEAT_CAT, FEAT_IDENT, FEAT_NUM, RpFeature, check, lib
from replay_b200.core import SasRecCore
from replay_b200.engine import EncoderConfig, SideFeature

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda")


# ---------------------------------------------------------------------------------------------------------------- kernels
def _kernel_case(dev, d, drop, seed=0):
    """T tokens of L positions with every edge: ids 0, cardinality - 1 and the padding value, bag widths 1 and 5 with
    all-padding bags, a numerical feature of tensor_dim 1 and one of 7, an identity feature of width d."""
    g = torch.Generator().manual_seed(seed + d)
    B, L = 5, 13
    T = B * L
    n_items = 300
    item = (torch.randn(n_items + 1, d, generator=g) * 0.1).to(torch.bfloat16)
    item[n_items] = 0
    pos = torch.randn(L + 3, d, generator=g) * 0.1
    ids = torch.randint(0, n_items + 1, (T,), generator=g).to(torch.int32)
    spec = []
    for kind, card, K in ((FEAT_CAT, 7, 1), (FEAT_CAT, 1, 1), (FEAT_BAG_SUM, 11, 1), (FEAT_BAG_SUM, 11, 5),
                          (FEAT_BAG_MEAN, 9, 5), (FEAT_BAG_MEAN, 9, 3)):
        tab = (torch.randn(card + 1, d, generator=g) * 0.1).to(torch.bfloat16)
        v = torch.randint(0, card + 1, (T, K), generator=g).to(torch.int32)
        v[0] = 0
        v[1] = card - 1
        v[2] = card          # the padding value: zero, no gradient (an all-padding bag)
        spec.append(dict(kind=kind, width=K, card=card, table=tab, values=v))
    for width in (1, 7):
        spec.append(dict(kind=FEAT_NUM, width=width, table=torch.randn(d, width, generator=g) * 0.2,
                         bias=torch.randn(d, generator=g) * 0.1, values=torch.randn(T, width, generator=g)))
    spec.append(dict(kind=FEAT_IDENT, width=d, values=torch.randn(T, d, generator=g)))
    return dict(B=B, L=L, T=T, d=d, drop=drop, item=item, pos=pos, ids=ids, spec=spec, pos0=3, scale=d ** 0.5,
                seed=1234 + d)


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
                f["dev_grad"] = torch.zeros(f["card"] + 1, c["d"], device=dev)
                a.d_table = f["dev_grad"].data_ptr()
        elif f["kind"] == FEAT_NUM:
            f["dev_table"], f["dev_bias"] = f["table"].to(dev), f["bias"].to(dev)
            a.table, a.bias, a.val_col = f["dev_table"].data_ptr(), f["dev_bias"].data_ptr(), col
            col += f["width"]
    return arr


def _reference_s(c):
    """float64 s [T, d] (before scale / positions / dropout)."""
    s = c["item"].double()[c["ids"].long()]
    for f in c["spec"]:
        if f["kind"] in (FEAT_CAT, FEAT_BAG_SUM, FEAT_BAG_MEAN):
            v = f["values"].long()
            live = (v != f["card"]).double()
            tot = (f["table"].double()[v] * live[..., None]).sum(1)
            if f["kind"] == FEAT_BAG_MEAN:
                tot = tot / live.sum(1, keepdim=True).clamp_min(1)
            s = s + tot
        elif f["kind"] == FEAT_NUM:
            s = s + f["values"].double() @ f["table"].double().T + f["bias"].double()
        else:
            s = s + f["values"].double()
    return s


@pytest.mark.parametrize("d", [64, 128, 256, 512])
@pytest.mark.parametrize("drop", [0.0, 0.3])
def test_feature_embed_matches_fp64(cuda, d, drop):
    c = _kernel_case(cuda, d, drop)
    T, L = c["T"], c["L"]
    arr = _descs(c, cuda, True)
    item, pos, ids = c["item"].to(cuda), c["pos"].to(cuda), c["ids"].to(cuda)
    ctr = torch.tensor([77], device=cuda, dtype=torch.int64)
    out = torch.full((T, d), float("nan"), device=cuda, dtype=torch.bfloat16)
    st = torch.cuda.current_stream().cuda_stream
    L_ = lib()
    check(L_.rp_feature_embed_fwd(item.data_ptr(), pos.data_ptr(), ids.data_ptr(), arr, len(arr), T, L, d, 0, c["pos0"],
                                  c["scale"], drop, c["seed"], 0, ctr.data_ptr(), out.data_ptr(), st), "fwd")
    keep = keep_draws(c["seed"] + 77, 0, drop, np.arange(T), d).double() if drop > 0 else torch.ones(T, d, dtype=torch.float64)
    ks = 1.0 / (1.0 - drop) if drop > 0 else 1.0
    tpos = torch.arange(T) % L + c["pos0"]
    ref = (_reference_s(c) * c["scale"] + c["pos"].double()[tpos]) * keep * ks
    got = out.double().cpu()
    assert torch.allclose(got, ref, rtol=1e-2, atol=2e-2 * ref.abs().max().item() / 8), (got - ref).abs().max()
    # backward: dS = scale * dropout'(dx) into the tables (padding rows frozen, mean bags by 1 / count); d_s and v_rows
    dx = (torch.randn(T, d, generator=torch.Generator().manual_seed(5)) * 0.1).to(torch.bfloat16)
    d_s = torch.zeros(T, d, device=cuda, dtype=torch.bfloat16)
    v_rows = torch.full((T, 64), 9.0, device=cuda, dtype=torch.bfloat16)
    check(L_.rp_feature_embed_bwd(dx.to(cuda).data_ptr(), arr, len(arr), T, d, 0, c["scale"], drop, c["seed"], 0,
                                  ctr.data_ptr(), d_s.data_ptr(), v_rows.data_ptr(), 64, st), "bwd")
    dS = dx.double() * keep * ks * c["scale"]
    assert torch.allclose(d_s.double().cpu(), dS, rtol=1e-2, atol=1e-3)
    for f in c["spec"]:
        if f["kind"] in (FEAT_CAT, FEAT_BAG_SUM, FEAT_BAG_MEAN):
            v = f["values"].long()
            live = (v != f["card"]).double()
            w = live / live.sum(1, keepdim=True).clamp_min(1) if f["kind"] == FEAT_BAG_MEAN else live
            ref_g = torch.zeros(f["card"] + 1, d, dtype=torch.float64)
            ref_g.index_add_(0, v.reshape(-1), (w[..., None] * dS[:, None, :]).reshape(-1, d))
            ref_g[f["card"]] = 0
            assert torch.allclose(f["dev_grad"].double().cpu(), ref_g, rtol=1e-4, atol=1e-4)
    vals = torch.cat([f["values"] for f in c["spec"] if f["kind"] == FEAT_NUM], 1)
    n = vals.shape[1]
    assert torch.equal(v_rows[:, :n].cpu(), vals.to(torch.bfloat16))
    assert (v_rows[:, n:] == 0).all()


def test_feature_embed_argument_errors(cuda):
    c = _kernel_case(cuda, 64, 0.0)
    arr = _descs(c, cuda, False)
    item, pos, ids = c["item"].to(cuda), c["pos"].to(cuda), c["ids"].to(cuda)
    out = torch.zeros(c["T"], 64, device=cuda, dtype=torch.bfloat16)
    L_ = lib()

    def fwd(a=arr, n=len(arr), d=64, item_ptr=item.data_ptr()):
        return L_.rp_feature_embed_fwd(item_ptr, pos.data_ptr(), ids.data_ptr(), a, n, c["T"], c["L"], d, 0, 0, 8.0, 0.0, 0, 0,
                                       None, out.data_ptr(), None)

    assert fwd(d=96) == -2
    assert fwd(n=17) == -2
    assert fwd(item_ptr=None) == -1
    arr[0].kind = 9
    assert fwd() == -1
    arr[0].kind = FEAT_CAT
    arr[7].val_col = 3            # numerical columns must be consecutive
    assert fwd() == -2


# ---------------------------------------------------------------------------------------------------------------- engine
def _golden(tag):
    z = np.load(os.path.join(GOLDEN, f"sasrec_side_{tag}.npz"))
    specs = osf.golden_specs(z)
    method = str(z["method"])
    feats = tuple(SideFeature(f["name"], "bag_" + method if f["kind"] == "bag" else f["kind"], f["cardinality"],
                              f["padding_value"], f["width"]) for f in specs)
    cfg = EncoderConfig(n_items=int(z["n_items"]), d=int(z["d"]), n_heads=int(z["H"]), n_blocks=int(z["n_blocks"]),
                        max_len=int(z["L"]), dropout=0.0, variant="new", features=feats)
    return z, specs, cfg, osf.golden_state_dict(z)


def _batch(z, specs, dev):
    t = lambda k: torch.from_numpy(z[k]).to(dev)  # noqa: E731
    feats = {f["name"]: torch.from_numpy(z["feat::" + f["name"]]).to(dev) for f in specs}
    return t("ids"), t("pad_mask"), t("labels"), t("target_mask"), feats


def _grads(core):
    eng = core.engine
    return {core._keymap[k]: core._to_ref(k, eng.export_named(k, eng.grads)).cpu() for k in eng.params}


@pytest.mark.parametrize("tag", ["d64h2_sum", "d50h1_mean"])
@pytest.mark.parametrize("packed", [False, True])
def test_engine_step_matches_reference_golden(cuda, tag, packed):
    z, specs, cfg, sd = _golden(tag)
    core = SasRecCore(cfg, device=cuda, seed=1)
    core.load_state_dict(sd)
    ids, pm, lab, tm, feats = _batch(z, specs, cuda)
    core.ensure_engine(*ids.shape, with_grad=True).packed_body = packed
    loss = core.loss(ids, pm, lab, tm, feats=feats)
    loss.backward()
    assert abs(float(loss) - float(z["train_loss"])) < 1e-2 * abs(float(z["train_loss"]))
    assert core.engine._packed == packed
    G = _grads(core)
    for k in G:
        ref = torch.from_numpy(z["grad::" + k]).float()
        got = G[k].float().reshape(ref.shape)
        if ref.norm() < 1e-12:
            assert got.norm() < 1e-6, k
            continue
        # the criterion of test_gpu_engine.py's golden step: direction and size of every gradient, at bf16 activations
        cos = float((got.double() * ref.double()).sum() / (got.double().norm() * ref.double().norm()))
        ratio = float(got.double().norm() / ref.double().norm())
        assert cos > 0.995 and abs(ratio - 1) < 0.03, (k, cos, ratio)
    logits = core.logits(ids, pm, feats=feats).cpu()
    ref = torch.from_numpy(z["eval_logits"])
    assert (logits - ref).abs().max() < 3e-2 * ref.abs().max(), (logits - ref).abs().max()


def test_packed_step_equals_padded_step(cuda):
    z, specs, cfg, sd = _golden("d64h2_sum")
    cfg = EncoderConfig(**{**cfg.__dict__, "dropout": 0.2})
    out = []
    for packed in (False, True):
        core = SasRecCore(cfg, device=cuda, seed=1)
        core.load_state_dict(sd)
        ids, pm, lab, tm, feats = _batch(z, specs, cuda)
        core.ensure_engine(*ids.shape, with_grad=True).packed_body = packed
        loss = core.loss(ids, pm, lab, tm, feats=feats)
        loss.backward()
        out.append((float(loss), _grads(core)))
    assert abs(out[0][0] - out[1][0]) < 1e-5 * abs(out[0][0])
    for k, v in out[0][1].items():
        assert torch.allclose(v, out[1][1][k], rtol=1e-3, atol=1e-5), k


def test_state_dict_round_trip_uses_reference_keys(cuda):
    z, specs, cfg, sd = _golden("d50h1_mean")
    core = SasRecCore(cfg, device=cuda, seed=1)
    core.load_state_dict(sd)
    out = core.state_dict()
    assert set(out) == set(sd)
    for k, v in sd.items():
        if k.endswith("._weight"):   # IdentityEmbedding's buffer: eye(d) whatever the checkpoint holds
            assert torch.equal(out[k], torch.eye(cfg.d)), k
            continue
        assert torch.equal(out[k].cpu().reshape(v.shape), v), k


@pytest.mark.parametrize("loss", ["ce", "ce_sampled"])
def test_fused_step_and_topk(cuda, loss):
    from replay_b200.nn.lightning.module import LightningModule
    from replay_b200.nn.loss import CE, CESampled
    from replay_b200.nn.sequential.sasrec import SasRec

    z, specs, cfg, sd = _golden("d64h2_sum")
    model = SasRec(SasRecCore(cfg, device=cuda, seed=1))
    model.loss = CE(ignore_index=cfg.n_items) if loss == "ce" else CESampled()
    model.load_state_dict(sd)
    ids, pm, lab, tm, feats = _batch(z, specs, cuda)
    batch = {"feature_tensors": {"item_id": ids, **feats}, "padding_mask": pm, "positive_labels": lab.unsqueeze(-1),
             "target_padding_mask": tm.unsqueeze(-1)}
    if loss != "ce":
        batch["negative_labels"] = torch.randint(0, cfg.n_items, (20,), device=cuda)
    module = LightningModule(model)
    losses = [float(module.training_step(batch)) for _ in range(6)]
    assert all(np.isfinite(losses)) and losses[-1] < losses[0]
    model.eval()
    logits = model(batch["feature_tensors"], pm)["logits"]
    got_ids, got_s = model.predict_topk(batch["feature_tensors"], pm, 10)
    ref_s, _ = torch.topk(logits, 10, dim=1)
    assert torch.allclose(got_s.float(), ref_s, rtol=1e-3, atol=1e-3)
