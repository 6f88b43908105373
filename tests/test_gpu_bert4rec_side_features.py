"""GPU tests of the legacy BERT4Rec's side features: the BERT form of the side-feature kernels (rp_bert_feature_embed_fwd /
_bwd) against float64, the item-only equivalence of zero side features, the engine step against the reference's goldens,
captured against eager steps, catalog growth and the Lightning surface."""
import os

import numpy as np
import pytest
import torch

from dropout_stream import keep_draws

pytestmark = pytest.mark.gpu

CASES = ["d64h2", "d300h4", "d96h2_tied_bce"]
SEED = 0x5EED1234ABC


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda")


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ----------------------------------------------------------------------------------------------------------------------
# the kernel pair against float64
# ----------------------------------------------------------------------------------------------------------------------
def _inputs(d, H, B=6, L=40, I=500, seed=0):
    """Item / mask / position tables and two categoricals (cardinality 7 and 1) plus an identity feature of width d, in the
    padded layout of ``d`` / ``H`` heads.  Row 5 of the 7-row table appears at masked and pad tokens only."""
    from replay_b200.engine_bert import BertConfig

    cfg = BertConfig(n_items=I, d=d, n_heads=H, n_blocks=1, max_len=L)
    dp, fi = cfg.dp, cfg.feat_index()
    g = torch.Generator().manual_seed(seed)
    T = B * L

    def padded(rows, scale=0.5):
        t = torch.zeros(rows, dp)
        t[:, fi] = torch.randn(rows, d, generator=g) * scale
        return t

    lens = torch.tensor([L, L, 17, 9, 1, 30])[:B]
    pad = torch.arange(L)[None, :] >= (L - lens)[:, None]
    tok = (torch.rand(B, L, generator=g) > 0.25) & pad
    ids = torch.randint(0, I, (B, L), generator=g)
    genre = torch.randint(0, 7, (B, L), generator=g)
    genre[0, :4] = torch.tensor([0, 6, 0, 6])
    live = pad & tok
    genre[live & (genre == 5)] = 4
    genre[~live & (torch.rand(B, L, generator=g) < 0.5)] = 5
    flag = torch.zeros(B, L, dtype=torch.int64)
    ident = torch.randn(B, L, d, generator=g)
    c = lambda t: t.cuda()  # noqa: E731
    return dict(cfg=cfg, dp=dp, fi=fi, B=B, L=L, T=T, item=c(padded(I)), mask=c(padded(1)), pos=c(padded(L, 0.3)),
                ids=c(ids), pad=c(pad), tok=c(tok), genre=c(genre), flag=c(flag), ident=c(ident),
                tabs={"genre": c(padded(7)), "flag": c(padded(1))})


def _descs(x, tabs, d_tabs=None, kinds=None):
    from replay_b200 import _lib

    arr = (_lib.RpFeature * 3)()
    x["_keep"] = []   # the staged values must outlive the call
    for k, name in enumerate(("genre", "flag")):
        v = x[name].reshape(-1).to(torch.int32).contiguous()
        x["_keep"].append(v)
        a = arr[k]
        a.kind, a.width, a.n_rows, a.padding_value = _lib.FEAT_CAT, 1, tabs[name].shape[0], -1
        a.values, a.table = v.data_ptr(), tabs[name].data_ptr()
        a.d_table = d_tabs[name].data_ptr() if d_tabs is not None else None
    v = x["ident"].reshape(x["T"], -1).contiguous()
    x["_keep"].append(v)
    arr[2].kind, arr[2].width, arr[2].values = _lib.FEAT_IDENT, v.shape[1], v.data_ptr()
    for k, kind in (kinds or {}).items():
        arr[k].kind = kind
    return arr


def _fwd(x, tabs16, p, positional, arr=None):
    from replay_b200 import _lib

    out = torch.empty(x["T"], x["dp"], device="cuda", dtype=torch.bfloat16)
    arr = _descs(x, tabs16) if arr is None else arr
    rc = _lib.lib().rp_bert_feature_embed_fwd(
        x["item16"].data_ptr(), x["mask16"].data_ptr(), x["pos"].data_ptr() if positional else None, x["ids32"].data_ptr(),
        x["tok"].data_ptr(), arr, len(arr), x["T"], x["L"], x["dp"], x["cfg"].hd_valid, p, SEED, 0, None, out.data_ptr(),
        _stream())
    return rc, out


def _ref_fwd(x, tabs, p, positional):
    """float64 [T, dp]: where(tok, item + genre + flag + ident, mask) + pos, dropout with the embedding site's keep mask"""
    T, dp = x["T"], x["dp"]
    s = x["item"].double()[x["ids"]] + tabs["genre"].double()[x["genre"]] + tabs["flag"].double()[x["flag"]]
    s[..., x["fi"]] += x["ident"].double()
    s = torch.where(x["tok"][..., None], s, x["mask"].double().expand_as(s))
    if positional:
        s = s + x["pos"].double()[None]
    s = s.reshape(T, dp)
    if p > 0:
        s = s * keep_draws(SEED, 0, p, np.arange(T), dp).cuda().double() / (1.0 - float(np.float32(p)))
    return s


def _bf16(x, tabs):
    x["item16"], x["mask16"] = x["item"].to(torch.bfloat16), x["mask"].to(torch.bfloat16)
    x["ids32"] = x["ids"].reshape(-1).to(torch.int32).contiguous()
    return {k: v.to(torch.bfloat16) for k, v in tabs.items()}


SHAPES = [(64, 1), (128, 2), (256, 4), (512, 8), (300, 4)]


@pytest.mark.parametrize("d,H", SHAPES)
@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("positional", [True, False])
def test_kernel_pair_matches_fp64(cuda, d, H, p, positional):
    from replay_b200 import _lib

    x = _inputs(d, H)
    tabs16 = _bf16(x, x["tabs"])
    tabs = {k: v.float() for k, v in tabs16.items()}   # the values the kernel reads
    x["item"], x["mask"] = x["item16"].float(), x["mask16"].float()
    rc, out = _fwd(x, tabs16, p, positional)
    assert rc == 0
    torch.cuda.synchronize()
    ref = _ref_fwd(x, tabs, p, positional)
    err = (out.double() - ref).abs()
    assert bool((err <= ref.abs() * 2.0 ** -8 + 1e-6).all()), float(err.max())
    pad_cols = torch.ones(x["dp"], dtype=torch.bool, device="cuda")
    pad_cols[x["fi"]] = False
    assert not out[:, pad_cols].any()   # padded columns stay zero

    # backward: dS = dropout'(dx) into the categorical tables at the real, unmasked tokens
    g = torch.Generator(device="cuda").manual_seed(7)
    dx = torch.zeros(x["T"], x["dp"], device="cuda")
    dx[:, x["fi"]] = torch.randn(x["T"], d, device="cuda", generator=g)
    dx = dx.to(torch.bfloat16)
    d_tabs = {k: torch.zeros(v.shape, device="cuda") for k, v in tabs16.items()}
    arr = _descs(x, tabs16, d_tabs)
    rc = _lib.lib().rp_bert_feature_embed_bwd(dx.data_ptr(), x["pad"].data_ptr(), x["tok"].data_ptr(), arr, len(arr), x["T"],
                                              x["dp"], x["cfg"].hd_valid, p, SEED, 0, None, _stream())
    assert rc == 0
    torch.cuda.synchronize()
    gs = dx.double()
    if p > 0:
        gs = gs * keep_draws(SEED, 0, p, np.arange(x["T"]), x["dp"]).cuda().double() / (1.0 - float(np.float32(p)))
    live = (x["pad"] & x["tok"]).reshape(-1)
    for name in ("genre", "flag"):
        rows = x[name].reshape(-1)
        ref_d = torch.zeros(d_tabs[name].shape, dtype=torch.float64, device="cuda").index_add_(0, rows[live], gs[live])
        got = d_tabs[name].double()
        assert float((got - ref_d).abs().max()) <= 1e-5 * max(1.0, float(ref_d.abs().max())), name
        untouched = torch.ones(ref_d.shape[0], dtype=torch.bool, device="cuda")
        untouched[rows[live]] = False
        assert not got[untouched].any(), name   # rows only masked or pad tokens carry: exactly zero
    assert not d_tabs["genre"][5].any() and d_tabs["genre"][0].any() and d_tabs["genre"][6].any()


def test_kernel_argument_errors(cuda):
    from replay_b200 import _lib

    L_ = _lib.lib()
    x = _inputs(64, 1)
    tabs16 = _bf16(x, x["tabs"])
    d_tabs = {k: torch.zeros(v.shape, device="cuda") for k, v in tabs16.items()}
    out = torch.empty(x["T"], x["dp"], device="cuda", dtype=torch.bfloat16)
    base = [x["item16"].data_ptr(), x["mask16"].data_ptr(), None, x["ids32"].data_ptr(), x["tok"].data_ptr()]
    for i in (0, 1, 3, 4):   # item, mask_emb, ids, tok_mask
        a = list(base)
        a[i] = None
        arr = _descs(x, tabs16)
        assert L_.rp_bert_feature_embed_fwd(*a, arr, 3, x["T"], x["L"], 64, 0, 0.0, SEED, 0, None, out.data_ptr(), _stream()) == -1
    for kind in (_lib.FEAT_BAG_SUM, _lib.FEAT_BAG_MEAN, _lib.FEAT_NUM):
        arr = _descs(x, tabs16, d_tabs, kinds={0: kind})
        assert L_.rp_bert_feature_embed_fwd(*base, arr, 3, x["T"], x["L"], 64, 0, 0.0, SEED, 0, None, out.data_ptr(), _stream()) == -1
        assert L_.rp_bert_feature_embed_bwd(out.data_ptr(), x["pad"].data_ptr(), x["tok"].data_ptr(), arr, 3, x["T"], 64, 0, 0.0,
                                            SEED, 0, None, _stream()) == -1
    arr = _descs(x, tabs16)   # no gradient tables
    assert L_.rp_bert_feature_embed_bwd(out.data_ptr(), x["pad"].data_ptr(), x["tok"].data_ptr(), arr, 3, x["T"], 64, 0, 0.0, SEED,
                                        0, None, _stream()) == -1
    arr = _descs(x, tabs16, d_tabs)
    assert L_.rp_bert_feature_embed_bwd(out.data_ptr(), None, x["tok"].data_ptr(), arr, 3, x["T"], 64, 0, 0.0, SEED, 0, None,
                                        _stream()) == -1
    arr[0].values = None
    assert L_.rp_bert_feature_embed_fwd(*base, arr, 3, x["T"], x["L"], 64, 0, 0.0, SEED, 0, None, out.data_ptr(), _stream()) == -1
    arr = _descs(x, tabs16)
    assert L_.rp_bert_feature_embed_fwd(*base, arr, 3, x["T"], x["L"], 96, 0, 0.0, SEED, 0, None, out.data_ptr(), _stream()) == -2


# ----------------------------------------------------------------------------------------------------------------------
# zero side features = the item-only model
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("positional", [True, False])
def test_zero_side_features_give_the_item_only_embedding(cuda, p, positional):
    """Same dropout stream, same fp32 sum (item row + 0), one rounding: bitwise the output of rp_bert_embed_fwd."""
    from replay_b200 import _lib

    x = _inputs(128, 2)
    tabs16 = _bf16(x, {k: torch.zeros_like(v) for k, v in x["tabs"].items()})
    x["ident"] = torch.zeros_like(x["ident"])
    rc, out = _fwd(x, tabs16, p, positional)
    assert rc == 0
    ref = torch.empty_like(out)
    assert _lib.lib().rp_bert_embed_fwd(x["item16"].data_ptr(), x["mask16"].data_ptr(), x["pos"].data_ptr() if positional else None,
                                        x["ids32"].data_ptr(), x["tok"].data_ptr(), x["T"], x["L"], x["dp"], p, SEED, 0, None,
                                        ref.data_ptr(), _stream()) == 0
    torch.cuda.synchronize()
    assert torch.equal(out, ref)


def test_zero_side_features_give_the_item_only_loss(cuda):
    from replay_b200.engine import SideFeature
    from replay_b200.engine_bert import BertConfig
    from replay_b200.models.nn.sequential.bert4rec import _BertCore

    base = dict(n_items=700, d=128, n_heads=2, n_blocks=2, max_len=32, dropout=0.1)
    fs = (SideFeature("genre", "cat", 9, 0, 1), SideFeature("vec", "ident", 0, 0, 128))
    a, b = _BertCore(BertConfig(**base), device=cuda), _BertCore(BertConfig(**base, features=fs), device=cuda)
    sd = a.state_dict()
    sd["item_embedder.cat_embeddings.genre.weight"] = torch.zeros(9, 128)
    b.load_state_dict(sd)
    batch = _train_batch(16, 32, 700, seed=3, fs=fs)
    args = (batch["inputs"]["item_id"], batch["pad_mask"], batch["token_mask"], batch["positive_labels"])
    feats = dict(batch["inputs"], vec=torch.zeros_like(batch["inputs"]["vec"]))
    la, lb = float(a.loss(*args)), float(b.loss(*args, feats))
    assert torch.equal(a.engine.x[0], b.engine.x[0])
    assert la == lb, (la, lb)


# ----------------------------------------------------------------------------------------------------------------------
# the engine step against the reference's goldens
# ----------------------------------------------------------------------------------------------------------------------
def _golden(golden_dir, tag):
    from oracle import bert4rec_passes as op

    z = np.load(os.path.join(golden_dir, f"bert4rec_side_{tag}.npz"))
    return z, op.golden_state_dict(z)


def _schema_of(z):
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    d, fs = int(z["d"]), []
    for n, k, c, p in zip(z["f_name"], z["f_kind"], z["f_card"], z["f_pad"]):
        if str(k) == "cat":
            fs.append(TensorFeatureInfo(str(n), int(c), int(p), d))
        else:
            fs.append(TensorFeatureInfo(str(n), None, 0, d, is_cat=False, is_list=str(k) == "num_list", tensor_dim=d))
    return TensorSchema(TensorFeatureInfo("item_id", int(z["n_items"]), 0, d), features=fs)


def _mirror(z, dropout=0.0, schema=None):
    from replay_b200.models.nn.sequential import Bert4Rec

    return Bert4Rec(schema or _schema_of(z), block_count=int(z["n_blocks"]), head_count=int(z["H"]), hidden_size=int(z["d"]),
                    max_seq_len=int(z["L"]), dropout_rate=dropout, pass_per_transformer_block_count=int(z["passes"]),
                    enable_positional_embedding=bool(int(z["positional"])), enable_embedding_tying=bool(int(z["tying"])),
                    loss_type=str(z["loss"]))


def _cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


@pytest.mark.parametrize("tag", CASES)
def test_engine_step_matches_reference(golden_dir, cuda, tag):
    """Loss, every gradient (side tables included), predict's logits on the shifted window and the fused top-K."""
    z, sd = _golden(golden_dir, tag)
    m = _mirror(z)
    m.load_state_dict({"_model." + k: v for k, v in sd.items()})
    core = m._model.core
    t = lambda k: torch.from_numpy(z[k]).cuda()  # noqa: E731
    names = [str(n) for n in z["f_name"]]
    feats = {"item_id": t("ids"), **{n: t("feat::" + n) for n in names}}
    B, L = z["ids"].shape
    eng = core.ensure_engine(B, L, with_grad=True)
    core._apply_loss(eng)
    core._stage_features(eng, feats)
    eng.set_batch(t("ids"), t("pad_mask"), t("token_mask"), t("labels"))
    eng.refresh_shadow()
    core._shadow_dirty = False
    loss = float(eng.forward_train()[0])
    ref_loss = float(z["train_loss"])
    assert abs(loss - ref_loss) < 5e-3 * ref_loss, (loss, ref_loss)
    eng.g32.zero_()
    eng.backward()
    torch.cuda.synchronize()
    assert sorted(core._keymap[k] for k in eng.layout) == sorted(k[6:] for k in z.files if k.startswith("grad::"))
    bad = []
    for k in eng.layout:
        a, b = eng.export_named(k, eng.grads).cpu(), torch.from_numpy(z["grad::" + core._keymap[k]])
        if b.norm() < 1e-12:
            if a.norm() >= 1e-6:
                bad.append((k, "nonzero"))
            continue
        c, r = _cos(a, b), float(a.double().norm() / b.double().norm())
        if c < 0.995 or abs(r - 1) > 0.03:
            bad.append((k, round(c, 5), round(r, 4)))
    assert not bad, bad
    # a side-table row that no real, unmasked token reads has an exactly zero gradient
    for n in names:
        if f"feat.{n}" in eng.grads:
            ref = torch.from_numpy(z[f"grad::item_embedder.cat_embeddings.{n}.weight"])
            zero = ref.abs().sum(1) == 0
            assert not eng.export_named(f"feat.{n}", eng.grads).cpu()[zero].any(), n

    pfeats = {k: t("pfeat::" + k) for k in ["item_id"] + names}
    pm, tok = t("p_pad_mask"), t("p_token_mask")
    ref = torch.from_numpy(z["eval_logits"])
    tol = 0.05 * max(1.0, float(ref.abs().max()))
    scores = m._model.predict(pfeats, pm, tok)
    assert float((scores.cpu() - ref).abs().max()) < tol
    batch = {"query_id": torch.arange(B), "inputs": pfeats, "pad_mask": pm, "token_mask": tok}
    top, sc = m.predict_topk(batch, 10)
    top, sc = top.cpu(), sc.cpu()
    assert float((ref.gather(1, top) - sc).abs().max()) < tol
    assert bool((ref.topk(10).values[:, -1] <= sc[:, 0] + tol).all())


# ----------------------------------------------------------------------------------------------------------------------
# the mirror: captured steps, catalog growth, the Lightning surface
# ----------------------------------------------------------------------------------------------------------------------
def _train_batch(B, L, n_items, seed, fs, lo=0, hi=None, side_seed=None):
    """A left-padded training batch with uniform-masker token masks; the side values come from ``side_seed``"""
    from replay_b200.models.nn.sequential.bert4rec import uniform_masker

    g = torch.Generator().manual_seed(seed)
    hi = n_items if hi is None else hi
    lens = torch.randint(L // 4, L + 1, (B,), generator=g)
    pad = torch.arange(L)[None, :] >= (L - lens)[:, None]
    items = torch.randint(lo, hi, (B, L), generator=g)
    tok = uniform_masker(pad, 0.2, g)
    ids = torch.where(pad, items, torch.zeros_like(items))
    labels = torch.where(pad & ~tok, items, torch.zeros_like(items))
    gs = torch.Generator().manual_seed(seed if side_seed is None else side_seed)
    inputs = {"item_id": ids}
    for f in fs:
        inputs[f.name] = (torch.randint(0, f.cardinality, (B, L), generator=gs) if f.kind == "cat"
                          else torch.randn(B, L, f.width, generator=gs))
    return {"query_id": torch.arange(B), "inputs": {k: v.cuda() for k, v in inputs.items()}, "pad_mask": pad.cuda(),
            "token_mask": tok.cuda(), "positive_labels": labels.cuda()}


def _side_schema(n_items, d, numerical=True):
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    fs = [TensorFeatureInfo("genre", 20, 0, d), TensorFeatureInfo("flag", 1, 0, d)]
    if numerical:
        fs.append(TensorFeatureInfo("vec", None, 0, d, is_cat=False, tensor_dim=d))
    return TensorSchema(TensorFeatureInfo("item_id", n_items, 0, d), features=fs)


def _lm(n_items, d=64, L=32, dropout=0.1, numerical=True, **kw):
    from replay_b200.models.nn.sequential import Bert4Rec

    return Bert4Rec(_side_schema(n_items, d, numerical), block_count=2, head_count=2, hidden_size=d, max_seq_len=L,
                    dropout_rate=dropout, **kw)


def test_captured_step_equals_eager_step_with_changing_side_values(cuda):
    """Three fused steps with dropout replayed from the captured graphs against the same steps launched eagerly; the
    batches share ids and masks and differ in their side values only."""
    ms = [_lm(500) for _ in range(2)]
    ms[1].load_state_dict(ms[0].state_dict())
    fs = ms[0]._model.core.cfg.features
    batches = [_train_batch(16, 32, 500, seed=1, fs=fs, side_seed=s) for s in range(3)]
    args = lambda b: (b["inputs"]["item_id"], b["pad_mask"], b["token_mask"], b["positive_labels"])  # noqa: E731
    l_eager = [float(ms[0]._model.core.fused_step(*args(b), all_reduce=None, feats=b["inputs"])) for b in batches]
    l_graph = [float(ms[1]._model.core.fused_step(*args(b), feats=b["inputs"])) for b in batches]
    assert ms[1]._model.core._trainer.use_graph
    np.testing.assert_allclose(l_eager, l_graph, rtol=1e-4)
    assert len(set(l_eager)) == 3
    s0, s1 = ms[0].state_dict(), ms[1].state_dict()
    for k in s0:
        diff = (s0[k] - s1[k]).abs()
        assert float(diff.max()) <= 3 * 1e-3 + 1e-6, k
        assert float((diff > 1e-4).double().mean()) < 0.01, k


@pytest.mark.parametrize("op", ["by_size", "by_tensor", "append"])
def test_catalog_growth_keeps_side_tables(cuda, op):
    n_items, d, L = 40, 64, 16
    m = _lm(n_items, d, L)
    m._lr = 5e-3
    fs = m._model.core.cfg.features
    for s in range(3):
        m.training_step(_train_batch(32, L, n_items, seed=s, fs=fs), s)
    side = ("item_embedder.cat_embeddings.genre.weight", "item_embedder.cat_embeddings.flag.weight")
    old = {k: m._model.state_dict()[k].cpu() for k in side}
    arg = {"by_size": 47, "by_tensor": torch.rand(45, d), "append": torch.rand(3, d)}[op]
    getattr(m, {"by_size": "set_item_embeddings_by_size", "by_tensor": "set_item_embeddings_by_tensor",
                "append": "append_item_embeddings"}[op])(arg)
    n_new = {"by_size": 47, "by_tensor": 45, "append": 43}[op]
    assert m._model.item_count == n_new and m._model.core.cfg.features == fs
    sd = m._model.state_dict()
    for k in side:
        assert torch.equal(sd[k].cpu(), old[k]), k
    with pytest.raises(KeyError):   # the numerical "vec" has no table, as in the reference
        m.get_all_embeddings()
    batch = _train_batch(32, L, n_new, seed=11, fs=fs, lo=n_items, hi=n_new)
    first = float(m.training_step(batch, 0))
    for i in range(1, 40):
        last = float(m.training_step(batch, i))
    assert last < 0.7 * first, (first, last)


def test_unfused_gradients_equal_the_fused_step(cuda):
    """fused_optimizer=False: autograd reads the engine's gradient, side tables included.  The fused step's first Adam
    update moves each element by about -lr * sign(gradient), and leaves elements with a zero gradient where they are."""
    a, b = _lm(300, dropout=0.0, fused_optimizer=False), _lm(300, dropout=0.0)
    b.load_state_dict(a.state_dict())
    fs = a._model.core.cfg.features
    batch = _train_batch(16, 32, 300, seed=5, fs=fs)
    la = a.training_step(batch, 0)
    la.backward()
    core_a, core_b = a._model.core, b._model.core
    before = core_b.engine.p32.clone()
    lb = float(b.training_step(batch, 0))
    assert abs(float(la) - lb) <= 1e-5 * lb
    off, shp = core_a.engine.layout["feat.genre"]
    n = int(np.prod(shp))
    ga = core_a.flat.grad[off:off + n]
    delta = (core_b.engine.p32 - before)[off:off + n]
    assert ga.abs().max() > 0
    big = ga.abs() > 1e-5 * float(ga.abs().max())
    assert float((torch.sign(delta[big]) == -torch.sign(ga[big])).double().mean()) > 0.99
    assert not delta[ga == 0].any()


def test_surface_predicts_short_batches_and_learns(cuda):
    m = _lm(200, L=24, dropout=0.0, numerical=False)
    fs = m._model.core.cfg.features
    batch = _train_batch(8, 20, 200, seed=2, fs=fs)
    pb = {"query_id": batch["query_id"], "inputs": batch["inputs"], "pad_mask": batch["pad_mask"],
          "token_mask": batch["pad_mask"]}
    out = m.predict_step(pb, 0)
    assert out.shape == (8, 200) and bool(torch.isfinite(out).all())
    top, _ = m.predict_topk(pb, 5)
    assert top.shape == (8, 5)
    # the side values change the prediction
    pb2 = dict(pb, inputs=dict(pb["inputs"], genre=(pb["inputs"]["genre"] + 1) % 20))
    assert not torch.equal(m.predict_step(pb2, 0), out)
    m._lr = 1e-2
    train = _train_batch(32, 24, 200, seed=3, fs=fs)
    losses = [float(m.training_step(train, i)) for i in range(40)]
    assert losses[-1] < 0.5 * losses[0], losses[::10]
    # an item-only device batch lacks the side features
    with pytest.raises(ValueError, match="lacks the side feature"):
        m.training_step(dict(train, inputs={"item_id": train["inputs"]["item_id"]}), 0)
