"""GPU tests of the device sequence store's feature columns (rp_build_batch_features): every builder bit-exact against the
reference's own batches (tests/golden/device_batch_features.npz), bit-exact against the loop restatement
(oracle/device_batch_features.py) on a random store at B 512, L 200, item-only outputs unchanged, no host synchronisation,
the new-path loader's shards, and models trained and served from store batches exactly as from host-built batches."""
import os

import numpy as np
import pytest
import torch

from oracle import dataset as od
from oracle import device_batch_features as of

pytestmark = pytest.mark.gpu

NAMES = ["item_id", "cat", "num", "vec", "ts"]


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda")


def _np(t):
    return t.cpu().numpy()


def _same(got, want, what):
    got = _np(got) if isinstance(got, torch.Tensor) else got
    assert got.dtype == want.dtype, (what, got.dtype, want.dtype)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    if got.dtype.kind == "f":  # bitwise
        assert np.array_equal(got.view(f"u{got.itemsize}"), want.view(f"u{want.itemsize}")), what
    else:
        assert np.array_equal(got, want), what


def _golden(golden_dir):
    z = dict(np.load(os.path.join(golden_dir, "device_batch_features.npz")))
    off = np.concatenate([[0], np.cumsum(z["lengths"])])
    n = len(z["lengths"])
    seqs = {k: [z[f"col_{k}"][off[i]:off[i + 1]] for i in range(n)] for k in NAMES}
    loff = np.concatenate([[0], np.cumsum(z["lst_lengths"])])
    events = [z["lst_values"][loff[e]:loff[e + 1]] for e in range(len(z["lst_lengths"]))]
    seqs["lst"] = [events[off[i]:off[i + 1]] for i in range(n)]
    pads = dict(zip(NAMES + ["lst"], (int(p) for p in z["pads"])))
    return z, seqs, pads


def _golden_store(z, seqs, pads, with_list, device="cuda"):
    from replay_b200.device_data import DeviceSequenceStore
    names = ["cat", "num", "vec", "ts"] + (["lst"] if with_list else [])
    return DeviceSequenceStore(seqs["item_id"], query_ids=z["query_ids"], device=device,
                               features={n: seqs[n] for n in names}, padding_values=pads, list_widths={"lst": int(z["K"])})


def test_every_builder_matches_the_reference_batches(golden_dir, cuda):
    from replay_b200.device_data import window_index
    z, seqs, pads = _golden(golden_dir)
    L, step, prob, pad = int(z["L"]), int(z["step"]), float(z["mask_prob"]), pads["item_id"]
    st = _golden_store(z, seqs, pads, with_list=False)
    n = len(seqs["item_id"])
    for tag, sw in (("slide", step), ("last", None)):
        s, o = window_index(st.lengths, L + 1, sw)
        b = st.sasrec_training_batch(s, L, pad, seq_offset=o)
        for k in NAMES:
            _same(b["feature_tensor"][k], z[f"sas_{tag}_{k}"], ("sas", tag, k))
        _same(b["padding_mask"], z[f"sas_{tag}_pad"], "pad")
        _same(b["positive_labels"], z[f"sas_{tag}_labels"], "labels")
        _same(b["target_padding_mask"], z[f"sas_{tag}_tmask"], "tmask")
        s, o = window_index(st.lengths, L, sw)
        bb = st.bert4rec_training_batch(s, L, pad, prob, seq_offset=o, uniforms=z[f"bert_{tag}_uniforms"])
        for k in NAMES:
            _same(bb["inputs"][k], z[f"bert_{tag}_{k}"], ("bert", tag, k))
        for k, g in (("pad_mask", "pad"), ("token_mask", "tok"), ("positive_labels", "labels")):
            _same(bb[k], z[f"bert_{tag}_{g}"], ("bert", tag, k))
    p = st.sasrec_prediction_batch(np.arange(n), L, pad)
    for k in NAMES:
        _same(p["feature_tensor"][k], z[f"pred_{k}"], ("pred", k))
    _same(p["padding_mask"], z["pred_pad"], "pred pad")
    bp = st.bert4rec_prediction_batch(np.arange(n), L, pad)
    for k in NAMES:
        _same(bp["inputs"][k], z[f"bertpred_{k}"], ("bertpred", k))
    _same(bp["pad_mask"], z["bertpred_pad"], "bertpred pad")
    _same(bp["token_mask"], z["bertpred_tok"], "bertpred tok")
    # new path, list column included
    st = _golden_store(z, seqs, pads, with_list=True)
    nb = st.sasrec_new_path_batch(z["new_order"], L, pad)
    for k in NAMES + ["lst"]:
        _same(nb["feature_tensors"][k], z[f"new_train_{k}"], ("new train", k))
    _same(nb["padding_mask"], z["new_train_pad"], "new pad")
    _same(nb["positive_labels"], z["new_train_labels"], "new labels")
    _same(nb["target_padding_mask"], z["new_train_tmask"], "new tmask")
    npb = st.sasrec_new_path_prediction_batch(z["new_order"], L, pad)
    for k in NAMES + ["lst"]:
        _same(npb["feature_tensors"][k], z[f"new_predict_{k}"], ("new predict", k))
    _same(npb["padding_mask"], z["new_predict_pad"], "new predict pad")
    assert torch.equal(npb["seen_ids"], npb["feature_tensors"]["item_id"])
    # the legacy builders cannot carry ragged lists, as the reference's datasets cannot stack them
    with pytest.raises(ValueError, match="list features"):
        st.sasrec_training_batch(np.arange(n), L, pad)


def _random_store(L, with_lists, seed=0):
    from replay_b200.device_data import DeviceSequenceStore
    rng = np.random.default_rng(seed)
    U = 700
    lens = np.clip(np.round(np.exp(rng.normal(4.56, 0.95, U))), 1, 900).astype(np.int64)
    lens[:4] = [1, L - 1, L, L + 1]
    seqs = [rng.integers(0, 100_000, n) for n in lens]
    f = {"cat64": [rng.integers(2 ** 33, 2 ** 40, n) for n in lens],                       # 64-bit ids
         "ts": [3_000_000_000 + np.cumsum(rng.integers(0, 1000, n)) for n in lens],      # 64-bit timestamps
         "cat32": [rng.integers(0, 1000, n).astype(np.int32) for n in lens],
         "f64": [rng.normal(0, 1, n) / 3.0 for n in lens],
         "v64": [rng.normal(0, 1, (n, 5)) / 3.0 for n in lens],
         "v32": [rng.normal(0, 1, (n, 8)).astype(np.float32) for n in lens]}
    pads = {"cat64": 2 ** 41, "ts": 0, "cat32": 1000, "f64": -2.5, "v64": 0.25, "v32": 0, "l1": 7, "l4": 8, "l33": 9}
    widths = {"l1": 1, "l4": 4, "l33": 33}
    if with_lists:
        for k in widths:
            f[k] = [[rng.integers(0, 500, int(m)) for m in rng.integers(0, 41, n)] for n in lens]
    st = DeviceSequenceStore(seqs, features=f, padding_values=pads, list_widths=widths)
    return st, lens, seqs, f, pads, widths


def _host_new_path(seqs, f, pads, widths, s, o, L, train):
    out = {}
    for k, col in f.items():
        rows = []
        for r in range(len(s)):
            seq = col[s[r]]
            if train:
                rows.append(of.newpath_feature_at(seq, int(o[r]), L, pads[k], dtype=np.asarray(seq).dtype
                                                  if k not in widths else None, width=widths.get(k)))
            else:
                rows.append(of.newpath_feature(seq, L, pads[k], train=False, width=widths.get(k),
                                               dtype=None if k in widths else np.asarray(seq).dtype))
        out[k] = np.stack(rows)
    for k in ("cat64", "ts", "cat32"):
        out[k] = out[k].astype(np.int64)
    return out


def test_random_store_against_restatement(cuda):
    """B 512, L 200: list widths 1, 4 and 33, float64 columns, 64-bit ids and timestamps, every builder."""
    from replay_b200.device_data import window_index
    L, B = 200, 512
    st, lens, seqs, f, pads, widths = _random_store(L, with_lists=True)
    rng = np.random.default_rng(1)
    s_all, o_all = window_index(lens, L + 1, 37)
    pick = rng.choice(len(s_all), B, replace=False)
    s, o = s_all[pick], o_all[pick]
    check = rng.choice(B, 96, replace=False)  # rows restated by the Python loops
    b = st.sasrec_new_path_batch(s, L, 100_000, seq_offset=o)
    want = _host_new_path(seqs, f, pads, widths, s[check], o[check], L, train=True)
    for k, w in want.items():
        _same(b["feature_tensors"][k][torch.as_tensor(check, device=cuda)], w, ("new train", k))
    ref = [od.sasrec_training_sample(seqs[s[r]], int(o[r]), L, 100_000) for r in check]
    _same(b["feature_tensors"]["item_id"][torch.as_tensor(check, device=cuda)], np.stack([x["item_id"] for x in ref]), "ids")
    p = st.sasrec_new_path_prediction_batch(s, L, 100_000)
    want = _host_new_path(seqs, f, pads, widths, s[check], None, L, train=False)
    for k, w in want.items():
        _same(p["feature_tensors"][k][torch.as_tensor(check, device=cuda)], w, ("new predict", k))
    # legacy modes on the same columns without the lists
    st, lens, seqs, f, pads, widths = _random_store(L, with_lists=False)
    rows = torch.as_tensor(check, device=cuda)
    b = st.sasrec_training_batch(s, L, 100_000, seq_offset=o)
    for k in f:
        w = np.stack([of.sasrec_training_feature(f[k][s[r]], int(o[r]), L, pads[k]) for r in check])
        _same(b["feature_tensor"][k][rows], w, ("sas train", k))
    s2, o2 = window_index(lens, L, 37)
    pick2 = rng.choice(len(s2), B, replace=False)
    s2, o2 = s2[pick2], o2[pick2]
    bb = st.bert4rec_training_batch(s2, L, 100_000, 0.15, seq_offset=o2, seed=3)
    for k in f:
        w = np.stack([of.bert_training_feature(f[k][s2[r]], int(o2[r]), L, pads[k]) for r in check])
        _same(bb["inputs"][k][rows], w, ("bert train", k))
    for name, fn, builder in (("pred", of.prediction_feature, st.sasrec_prediction_batch),
                              ("bertpred", of.bert_prediction_feature, st.bert4rec_prediction_batch)):
        out = builder(s, L, 100_000)
        group = out["feature_tensor"] if "feature_tensor" in out else out["inputs"]
        for k in f:
            w = np.stack([fn(f[k][s[r]], L, pads[k]) for r in check])
            _same(group[k][rows], w, (name, k))


def test_item_only_outputs_unchanged(cuda):
    """The item outputs of a feature store equal an item-only store's, which runs the item-only launch."""
    from replay_b200.device_data import DeviceSequenceStore, window_index
    L = 200
    st, lens, seqs, f, pads, widths = _random_store(L, with_lists=True)
    plain = DeviceSequenceStore(seqs)
    assert plain.columns == []
    s, o = window_index(lens, L + 1, 50)
    for a, b in ((st.sasrec_new_path_batch(s, L, 7, seq_offset=o), plain.sasrec_new_path_batch(s, L, 7, seq_offset=o)),
                 (st.sasrec_new_path_prediction_batch(s, L, 7), plain.sasrec_new_path_prediction_batch(s, L, 7))):
        assert set(a) == set(b) and set(b["feature_tensors"]) == {"item_id"}
        for k in b:
            if k == "feature_tensors":
                assert torch.equal(a[k]["item_id"], b[k]["item_id"])
            else:
                assert torch.equal(a[k], b[k]), k
    st, lens, seqs, f, pads, widths = _random_store(L, with_lists=False)
    s, o = window_index(lens, L, 50)
    a = st.bert4rec_training_batch(s, L, 7, 0.2, seq_offset=o, seed=4, draw0=9)
    b = plain.bert4rec_training_batch(s, L, 7, 0.2, seq_offset=o, seed=4, draw0=9)
    for k in ("pad_mask", "token_mask", "positive_labels", "query_id"):
        assert torch.equal(a[k], b[k]), k
    assert torch.equal(a["inputs"]["item_id"], b["inputs"]["item_id"])


def test_batches_build_without_host_synchronisation(cuda):
    from replay_b200.device_data import window_index
    L = 200
    st, lens, *_ = _random_store(L, with_lists=True)
    st2, *_ = _random_store(L, with_lists=False)
    s, o = window_index(lens, L + 1, 50)
    s, o = torch.as_tensor(s[:512], device=cuda), torch.as_tensor(o[:512], device=cuda)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        outs = [st.sasrec_new_path_batch(s, L, 7, seq_offset=o), st.sasrec_new_path_prediction_batch(s, L, 7),
                st2.sasrec_training_batch(s, L, 7, seq_offset=o), st2.sasrec_prediction_batch(s, L, 7),
                st2.bert4rec_training_batch(s, L, 7, seq_offset=o, seed=1), st2.bert4rec_prediction_batch(s, L, 7)]
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert all(o is not None for o in outs)


def test_new_path_loader_shards_cover_every_window(cuda):
    from replay_b200.device_data import DeviceBatchLoader
    L = 24
    st, lens, seqs, f, pads, widths = _random_store(L, with_lists=True, seed=5)

    def rows(b):
        ft = b["feature_tensors"]
        parts = [b["query_id"], ft["item_id"], b["positive_labels"][:, -1], ft["ts"], ft["l4"].flatten(1),
                 ft["f64"].view(torch.int64)]
        return torch.cat(parts, 1).cpu()

    seen = []
    for rank in range(2):
        ld = DeviceBatchLoader(st, L, 256, 100_000, kind="sasrec_new", sliding_window_step=16, seed=3, rank=rank,
                               world_size=2)
        ld.set_epoch(2)
        seen += [rows(b) for b in ld]
    seen = torch.cat(seen)
    full = DeviceBatchLoader(st, L, 10 ** 6, 100_000, kind="sasrec_new", sliding_window_step=16, shuffle=False)
    allw = rows(next(iter(full)))
    assert len(seen) in (len(allw), len(allw) + 1)
    assert {tuple(r) for r in seen.tolist()} == {tuple(r) for r in allw.tolist()}
    # one loader batch against the restatement
    b = next(iter(DeviceBatchLoader(st, L, 64, 100_000, kind="sasrec_new", sliding_window_step=16, seed=1)))
    assert set(b) >= {"feature_tensors", "padding_mask", "positive_labels", "target_padding_mask"}
    assert b["positive_labels"].shape == (64, L, 1) and b["feature_tensors"]["l33"].shape == (64, L, 33)


# -------------------------------------------------------------------------------------------------------- end to end
def _e2e_histories(n_items, U=96, L=32, seed=0):
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, 2 * L, U)
    lens[:3] = [1, L, L + 1]
    return lens, [rng.integers(0, n_items, n) for n in lens], rng


def _to(batch, dev):
    return {k: (_to(v, dev) if isinstance(v, dict) else torch.as_tensor(v).to(dev)) for k, v in batch.items()}


def _host_new_train(seqs, cols, pads, widths, idx, L, pad):
    """What the reference's new path yields for these rows (oracle restatement, pinned by the golden), copied to the GPU."""
    ref = [od.sasrec_training_sample(seqs[i], max(0, len(seqs[i]) - L - 1), L, pad) for i in idx]
    ft = {"item_id": np.stack([r["item_id"] for r in ref])}
    for k, c in cols.items():
        ft[k] = np.stack([of.newpath_feature(c[i], L, pads[k], train=True, width=widths.get(k),
                                             dtype=None if k in widths else np.asarray(c[i]).dtype) for i in idx])
        if k not in widths and ft[k].dtype.kind in "iu":
            ft[k] = ft[k].astype(np.int64)
    return {"query_id": np.asarray(idx)[:, None], "feature_tensors": ft,
            "padding_mask": np.stack([r["padding_mask"] for r in ref]),
            "positive_labels": np.stack([r["positive_labels"] for r in ref])[..., None],
            "target_padding_mask": np.stack([r["target_padding_mask"] for r in ref])[..., None]}


def _host_new_predict(seqs, cols, pads, widths, idx, L, pad):
    ref = [od.prediction_sample(seqs[i], L, pad) for i in idx]
    ft = {"item_id": np.stack([r["item_id"] for r in ref])}
    for k, c in cols.items():
        ft[k] = np.stack([of.newpath_feature(c[i], L, pads[k], train=False, width=widths.get(k),
                                             dtype=None if k in widths else np.asarray(c[i]).dtype) for i in idx])
        if k not in widths and ft[k].dtype.kind in "iu":
            ft[k] = ft[k].astype(np.int64)
    return {"feature_tensors": ft, "padding_mask": np.stack([r["padding_mask"] for r in ref])}


def _assert_batches_equal(a, b, path=""):
    assert set(b) <= set(a), (path, set(b) - set(a))
    for k in b:
        if isinstance(b[k], dict):
            _assert_batches_equal(a[k], b[k], path + k + ".")
        else:
            _same(a[k], _np(b[k]), path + k)


def _losses_match(step, x, y):
    """The first step runs on equal parameters: equal loss bits.  Later steps start from parameters that may differ in
    the last bits (see _params_close), so their losses agree to float32 rounding."""
    x, y = torch.as_tensor(x).detach().float().cpu(), torch.as_tensor(y).detach().float().cpu()
    if step == 0:
        assert torch.equal(x, y), (float(x), float(y))
    else:
        assert torch.allclose(x, y, rtol=1e-5, atol=0), (float(x), float(y))


def _params_close(m1, m2, lr=1e-3, steps=3):
    """The two models saw bitwise-equal batches; their parameters agree up to the order of the atomic adds in the
    gradient reductions, which Adam can amplify on near-zero gradients: every element within the steps' Adam bound and
    every tensor to a relative norm of 1e-3."""
    s1, s2 = m1.state_dict(), m2.state_dict()
    assert set(s1) == set(s2)
    for k in s1:
        if isinstance(s1[k], torch.Tensor) and s1[k].is_floating_point():
            a, b = s1[k].double(), s2[k].double()
            assert float((a - b).abs().max()) <= 2 * steps * lr, k
            assert float((a - b).norm()) <= 1e-3 * float(a.norm()) + 1e-9, k


def _new_path_case(kind, cuda):
    from replay_b200.nn.agg import ConcatAggregator
    from replay_b200.nn.embedding import SequenceEmbedding
    from replay_b200.nn.mask import DefaultAttentionMask
    from replay_b200.nn.sequential.sasrec import PositionAwareAggregator, SasRec, SasRecBody, SasRecTransformerLayer
    from replay_b200.nn.sequential.twotower import TwoTower
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    n_items, d, L = 300, 64, 32
    lens, seqs, rng = _e2e_histories(n_items, L=L)
    cols = {"genre": [rng.integers(0, 20, n) for n in lens],
            "tags": [[rng.integers(0, 9, int(m)) for m in rng.integers(0, 6, n)] for n in lens],
            "price": [rng.normal(0, 1, (n, 4)).astype(np.float32) for n in lens]}
    pads, widths = {"genre": 20, "tags": 9, "price": 0}, {"tags": 3}
    dims = {"sum": (d, d, d), "concat": (16, 32, 8), "twotower": (d, d, d)}[kind]
    schema = TensorSchema(TensorFeatureInfo("item_id", n_items, n_items, d if kind != "concat" else 64), features=[
        TensorFeatureInfo("genre", 20, 20, dims[0]), TensorFeatureInfo("tags", 9, 9, dims[1], is_list=True),
        TensorFeatureInfo("price", None, 0, dims[2], is_cat=False, tensor_dim=4)])

    def make():
        if kind == "twotower":
            class Reader:
                feature_names = ["item_id"]

                def __getitem__(self, k):
                    return torch.arange(n_items)
            return TwoTower.from_params(schema, Reader(), embedding_dim=d, num_heads=2, num_blocks=1, max_sequence_length=L,
                                        dropout=0.0, device=cuda, seed=4)
        if kind == "sum":
            return SasRec.from_params(schema, embedding_dim=d, num_heads=2, num_blocks=1, max_sequence_length=L,
                                      dropout=0.0, device=cuda, seed=4)
        body = SasRecBody(SequenceEmbedding(schema, categorical_list_feature_aggregation_method="sum"),
                          PositionAwareAggregator(ConcatAggregator([64, *dims], d), L, 0.0),
                          DefaultAttentionMask("item_id", 2), SasRecTransformerLayer(d, 2, 1, 0.0, "relu"),
                          torch.nn.LayerNorm(d))
        return SasRec(body=body, device=cuda, seed=4)
    return n_items, L, lens, seqs, cols, pads, widths, make


@pytest.mark.parametrize("kind", ["sum", "concat", "twotower"])
def test_new_path_models_train_and_predict_from_store_batches(cuda, kind):
    from replay_b200.device_data import DeviceSequenceStore
    from replay_b200.nn.lightning.module import LightningModule

    n_items, L, lens, seqs, cols, pads, widths, make = _new_path_case(kind, cuda)
    st = DeviceSequenceStore(seqs, features=cols, padding_values=pads, list_widths=widths)
    rng = np.random.default_rng(2)
    steps = [rng.choice(len(seqs), 32, replace=False) for _ in range(3)]
    ma, mb = make(), make()
    la, lb = LightningModule(ma), LightningModule(mb)
    for i, idx in enumerate(steps):
        sb = st.sasrec_new_path_batch(idx, L, n_items, with_seen=False)
        hb = _to(_host_new_train(seqs, cols, pads, widths, idx, L, n_items), cuda)
        _assert_batches_equal(sb, hb)
        _losses_match(i, la.training_step(sb), lb.training_step(hb))
    _params_close(ma, mb)
    ma.eval()
    idx = np.arange(40)
    sp = st.sasrec_new_path_prediction_batch(idx, L, n_items)
    hp = _to(_host_new_predict(seqs, cols, pads, widths, idx, L, n_items), cuda)
    _assert_batches_equal(sp, hp)
    ia, sa = ma.predict_topk(sp["feature_tensors"], sp["padding_mask"], 10, seen_ids=sp["seen_ids"])
    ib, sb_ = ma.predict_topk(hp["feature_tensors"], hp["padding_mask"], 10, seen_ids=hp["feature_tensors"]["item_id"])
    assert torch.equal(ia, ib) and torch.equal(sa, sb_)


def test_legacy_bert4rec_with_side_features_from_store_batches(cuda):
    from replay_b200.device_data import DeviceSequenceStore
    from replay_b200.models.nn.sequential import Bert4Rec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    n_items, d, L = 300, 64, 32
    lens, seqs, rng = _e2e_histories(n_items, L=L, seed=3)
    cols = {"genre": [rng.integers(0, 20, n) for n in lens], "vec": [rng.normal(0, 1, (n, d)) for n in lens]}
    pads = {"genre": 0, "vec": 0}
    schema = TensorSchema(TensorFeatureInfo("item_id", n_items, 0, d), features=[
        TensorFeatureInfo("genre", 20, 0, d), TensorFeatureInfo("vec", None, 0, d, is_cat=False, tensor_dim=d)])
    st = DeviceSequenceStore(seqs, features=cols, padding_values=pads)

    def make():
        torch.manual_seed(0)
        return Bert4Rec(schema, block_count=2, head_count=2, hidden_size=d, max_seq_len=L, dropout_rate=0.0)

    ma, mb = make(), make()
    mb.load_state_dict(ma.state_dict())
    g = np.random.default_rng(4)
    for i in range(3):
        idx = g.choice(len(seqs), 32, replace=False)
        u = g.random((32, L), dtype=np.float32)
        sb = st.bert4rec_training_batch(idx, L, 0, 0.2, uniforms=u)
        ref = [od.bert_training_sample(seqs[j], max(0, len(seqs[j]) - L), L, 0, u[r], 0.2) for r, j in enumerate(idx)]
        hb = {"query_id": np.asarray(idx)[:, None],
              "inputs": {"item_id": np.stack([r["item_id"] for r in ref]),
                         **{k: np.stack([of.bert_training_feature(cols[k][j], max(0, len(seqs[j]) - L), L, pads[k])
                                         for j in idx]) for k in cols}},
              "pad_mask": np.stack([r["pad_mask"] for r in ref]), "token_mask": np.stack([r["token_mask"] for r in ref]),
              "positive_labels": np.stack([r["positive_labels"] for r in ref])}
        hb = _to(hb, cuda)
        _assert_batches_equal(sb, hb)
        _losses_match(i, ma.training_step(sb, i), mb.training_step(hb, i))
    _params_close(ma, mb)
    idx = np.arange(40)
    sp = st.bert4rec_prediction_batch(idx, L, 0)
    ref = [od.bert_prediction_sample(seqs[j], L, 0) for j in idx]
    hp = _to({"query_id": idx[:, None], "inputs": {"item_id": np.stack([r["item_id"] for r in ref]),
                                                   **{k: np.stack([of.bert_prediction_feature(cols[k][j], L, pads[k])
                                                                   for j in idx]) for k in cols}},
              "pad_mask": np.stack([r["pad_mask"] for r in ref]), "token_mask": np.stack([r["token_mask"] for r in ref])},
             cuda)
    _assert_batches_equal(sp, hp)
    ia, sa = ma.predict_topk(sp, 10)
    ib, sb_ = ma.predict_topk(hp, 10)
    assert torch.equal(ia, ib) and torch.equal(sa, sb_)


def test_tisasrec_from_store_batches(cuda):
    from replay_b200.device_data import DeviceSequenceStore
    from replay_b200.models.nn.sequential import SasRec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    n_items, d, L = 300, 64, 32
    lens, seqs, rng = _e2e_histories(n_items, L=L, seed=6)
    ts = {"timestamp": [3_000_000_000 + np.cumsum(rng.integers(0, 300, n)) for n in lens]}
    st = DeviceSequenceStore(seqs, features=ts)
    schema = TensorSchema(TensorFeatureInfo("item_id", n_items, n_items, d), timestamp_feature_name="timestamp")

    def make():
        return SasRec(schema, block_count=2, head_count=2, hidden_size=d, max_seq_len=L, dropout_rate=0.0,
                      ti_modification=True, time_span=64, device=cuda)

    ma, mb = make(), make()
    mb.load_state_dict(ma.state_dict())
    g = np.random.default_rng(7)
    for i in range(3):
        idx = g.choice(len(seqs), 32, replace=False)
        sb = st.sasrec_training_batch(idx, L, n_items)
        offs = [max(0, len(seqs[j]) - L - 1) for j in idx]
        ref = [od.sasrec_training_sample(seqs[j], o, L, n_items) for j, o in zip(idx, offs)]
        hb = _to({"query_id": np.asarray(idx)[:, None],
                  "feature_tensor": {"item_id": np.stack([r["item_id"] for r in ref]),
                                     "timestamp": np.stack([of.sasrec_training_feature(ts["timestamp"][j], o, L, 0)
                                                            for j, o in zip(idx, offs)])},
                  "padding_mask": np.stack([r["padding_mask"] for r in ref]),
                  "positive_labels": np.stack([r["positive_labels"] for r in ref]),
                  "target_padding_mask": np.stack([r["target_padding_mask"] for r in ref])}, cuda)
        _assert_batches_equal(sb, hb)
        _losses_match(i, ma.training_step(sb, i), mb.training_step(hb, i))
    _params_close(ma, mb)
    idx = np.arange(40)
    sp = st.sasrec_prediction_batch(idx, L, n_items)
    ref = [od.prediction_sample(seqs[j], L, n_items) for j in idx]
    hp = _to({"query_id": idx[:, None], "padding_mask": np.stack([r["padding_mask"] for r in ref]),
              "feature_tensor": {"item_id": np.stack([r["item_id"] for r in ref]),
                                 "timestamp": np.stack([of.prediction_feature(ts["timestamp"][j], L, 0) for j in idx])}},
             cuda)
    _assert_batches_equal(sp, hp)
    ia, sa = ma.predict_topk(sp, 10)
    ib, sb_ = ma.predict_topk(hp, 10)
    assert torch.equal(ia, ib) and torch.equal(sa, sb_)
