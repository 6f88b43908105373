"""GPU tests of the device sequence store's query lists and validation builders (RP_BATCH_COL_QUERY_LIST[_LAST] in
rp_build_batch_features): every validation builder bit-exact against the reference's own batches
(tests/golden/device_validation_batches.npz), against the loop restatement (oracle/device_validation_batches.py) on
thousands of MovieLens-shaped histories with 16 columns in one launch, per-event outputs unchanged when query lists ride
along, no host synchronisation, the validation loader's coverage under 1, 2 and 8 ranks, and identical metrics from
device-built and host-built validation batches for three models."""
import os

import numpy as np
import pytest
import torch

from oracle import device_validation_batches as ov

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda")


def _flat(prefix, batch, out):
    for k, v in batch.items():
        if isinstance(v, dict):
            _flat(f"{prefix}_{k}", v, out)
        else:
            out[f"{prefix}_{k}"] = v.cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)
    return out


def _assert_same(got: dict, want: dict, what):
    g, w = _flat("", got, {}), _flat("", want, {})
    assert set(g) == set(w), (what, sorted(set(g) ^ set(w)))
    for k in g:
        assert g[k].dtype == w[k].dtype and g[k].shape == w[k].shape, (what, k, g[k].dtype, w[k].dtype, g[k].shape,
                                                                       w[k].shape)
        assert np.array_equal(g[k], w[k]), (what, k)


def _golden(golden_dir):
    z = dict(np.load(os.path.join(golden_dir, "device_validation_batches.npz")))
    return (z, *ov.golden_inputs(z))


def test_validation_builders_match_the_reference_batches(golden_dir, cuda):
    from replay_b200.device_data import DeviceSequenceStore
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    z, seqs, pads, gt, tr = _golden(golden_dir)
    L, n, item_pad = int(z["L"]), len(z["lengths"]), pads["item_id"]
    lab = TensorSchema(TensorFeatureInfo("item_id", 40, 40, 8))
    seq = ov.SequentialStub(TensorSchema(TensorFeatureInfo("item_id", 40, 40, 8), features=[TensorFeatureInfo("cat", 7, 7, 8)]),
                            z["query_ids"], {"item_id": seqs["item_id"], "cat": seqs["cat"]})
    st = DeviceSequenceStore.from_sequential_dataset(seq, device=cuda, ground_truth=ov.SequentialStub(lab, gt[0], {"item_id": gt[1]}),
                                                     train=ov.SequentialStub(lab, tr[0], {"item_id": tr[1]}))
    assert st.columns[0].padding_value == pads["cat"]
    rows = np.arange(n)
    for tag, b in (("sas", st.sasrec_validation_batch(rows, L, item_pad)),
                   ("bert", st.bert4rec_validation_batch(rows, L, item_pad))):
        got = _flat(tag, b, {})
        assert set(got) == {k for k in z if k.startswith(tag + "_")}, tag
        for k, v in got.items():
            assert v.dtype == z[k].dtype and v.shape == z[k].shape and np.array_equal(v, z[k]), k
    # new path: the reader's widths and paddings of the three list columns
    joined = {"ground_truth": [ov.lookup(*gt, q) for q in z["query_ids"]], "train": [ov.lookup(*tr, q) for q in z["query_ids"]]}
    joined["seen_ids"] = joined["train"]
    sn = DeviceSequenceStore(seqs["item_id"], query_ids=z["query_ids"], device=cuda,
                             features={"cat": seqs["cat"], "lst": seqs["lst"]}, query_lists=joined,
                             padding_values={**pads, "ground_truth": -1, "train": -2, "seen_ids": item_pad},
                             list_widths={"lst": int(z["K"]), "ground_truth": int(z["G_W"]), "train": int(z["T_W"]),
                                          "seen_ids": int(z["T_W"])})
    got = _flat("new", sn.sasrec_new_path_validation_batch(z["new_order"], L, item_pad), {})
    masks = {f"new_{k}" for k in z["new_keys"] if k.endswith("_mask") and k != "padding_mask"}
    assert set(got) == {k for k in z if k.startswith("new_")} - masks - {"new_order", "new_keys"}
    for k, v in got.items():
        assert v.dtype == z[k].dtype and v.shape == z[k].shape and np.array_equal(v, z[k]), k


def _synthetic_store(cuda, n_users=3000, seed=0):
    """MovieLens-shaped histories with 12 per-event columns and 4 query lists (16 columns in one launch), int32 and
    int64 list storage, list lengths 0 .. past every width."""
    from replay_b200.synthetic import make_histories

    offsets, items = make_histories(n_users, 5000, seed=seed)
    off = offsets.numpy()
    seqs = [items.numpy()[off[i]:off[i + 1]] for i in range(n_users)]
    rng = np.random.default_rng(seed)
    lens = np.diff(off)
    feats = {f"c{i}": [rng.integers(0, 50 + i, n) for n in lens] for i in range(8)}
    feats["big"] = [rng.integers(2 ** 33, 2 ** 34, n) for n in lens]
    feats["f32"] = [rng.normal(0, 1, n).astype(np.float32) for n in lens]
    feats["f64"] = [rng.normal(0, 1, n) / 3 for n in lens]
    feats["vec"] = [rng.normal(0, 1, (n, 3)).astype(np.float32) for n in lens]
    lists = {"ground_truth": [rng.integers(0, 5000, rng.integers(0, 14)) for _ in lens],
             "train": [s[: max(0, len(s) - 10)] for s in seqs],
             "big_list": [rng.integers(2 ** 40, 2 ** 41, rng.integers(0, 5)) for _ in lens],
             "seen_ids": [s[-rng.integers(0, 300):] if len(s) else s for s in seqs]}
    pads = {f"c{i}": 50 + i for i in range(8)}
    pads.update({"big": -5, "f32": -1.5, "f64": 0.25, "vec": 0, "big_list": -3, "seen_ids": 5000})
    widths = {"ground_truth": 10, "train": 200, "big_list": 3, "seen_ids": 256}
    return seqs, feats, lists, pads, widths


def test_validation_builders_match_restatement_on_synthetic_histories(cuda):
    from replay_b200.device_data import DeviceBatchLoader, DeviceSequenceStore

    seqs, feats, lists, pads, widths = _synthetic_store(cuda)
    n, L, B = len(seqs), 50, 700                                     # 3000 / 700: a partial last batch of 200
    st = DeviceSequenceStore(seqs, device=cuda, features=feats, query_lists=lists, padding_values=pads,
                             list_widths=widths)
    plain = DeviceSequenceStore(seqs, device=cuda, features=feats, padding_values=pads)
    assert len(st.columns) + len(st.query_lists) == 16
    dt = {c.name: c.values.dtype for c in st.query_lists}
    assert dt["ground_truth"] == torch.int32 and dt["big_list"] == torch.int64
    for kind in ("sasrec_validate", "bert4rec_validate", "sasrec_new_validate"):
        loader = DeviceBatchLoader(st, L, B, 5000, kind=kind)
        assert len(loader) == 5
        lo = 0
        for b in loader:
            rows = np.arange(lo, lo + (B if lo + B <= n else n - lo))
            lo += len(rows)
            # per-event outputs: the same bits as the builders without query lists
            if kind == "sasrec_validate":
                ref = plain.sasrec_prediction_batch(rows, L, 5000)
                _assert_same({k: b[k] for k in ref}, ref, kind)
            elif kind == "bert4rec_validate":
                ref = plain.bert4rec_prediction_batch(rows, L, 5000)
                _assert_same({k: b[k] for k in ref}, ref, kind)
            else:
                ref = plain.sasrec_new_path_prediction_batch(rows, L, 5000)
                ref["query_id"] = ref["query_id"].view(-1)
                _assert_same({k: b[k] for k in ("query_id", "feature_tensors", "padding_mask")},
                             {k: ref[k] for k in ("query_id", "feature_tensors", "padding_mask")}, kind)
            # query lists: the restatement
            for name, x in lists.items():
                w = widths[name]
                pad = st.query_lists[st.query_list_names.index(name)].padding_value
                cut = ov.newpath_list if kind == "sasrec_new_validate" else ov.legacy_list
                want = np.stack([cut(np.asarray(x[r], dtype=np.int64), w, pad) for r in rows])
                got = b[name].cpu().numpy()
                assert got.dtype == np.int64 and np.array_equal(got, want), (kind, name)
            assert set(b) - {"query_id", "feature_tensor", "feature_tensors", "inputs", "padding_mask", "pad_mask",
                             "token_mask"} == set(lists)
        assert lo == n


def test_legacy_width_and_padding_defaults(cuda):
    from replay_b200.device_data import DeviceSequenceStore

    st = DeviceSequenceStore([np.arange(3), np.arange(2)], device=cuda,
                             query_lists={"ground_truth": [[4], [5, 6, 7]], "train": [[], [1]]})
    b = st.sasrec_validation_batch([1, 0], 4, 9)
    assert b["ground_truth"].tolist() == [[5, 6, 7], [4, -1, -1]] and b["train"].tolist() == [[1], [-2]]
    nb = st.sasrec_new_path_validation_batch([1, 0], 4, 9, seen_list="ground_truth")
    assert nb["seen_ids"] is nb["ground_truth"] and nb["query_id"].tolist() == [1, 0]
    assert torch.equal(st.sasrec_new_path_validation_batch([1, 0], 4, 9, seen_list=None)["seen_ids"],
                       nb["feature_tensors"]["item_id"])
    with pytest.raises(ValueError, match="'ground_truth' and 'train'"):
        DeviceSequenceStore([np.arange(3)], device=cuda, query_lists={"ground_truth": [[1]]}).sasrec_validation_batch([0], 4, 9)


def test_validation_batches_do_not_synchronise(cuda):
    from replay_b200.device_data import DeviceSequenceStore

    seqs, feats, lists, pads, widths = _synthetic_store(cuda, n_users=600, seed=1)
    st = DeviceSequenceStore(seqs, device=cuda, features={"c0": feats["c0"]}, query_lists=lists, padding_values=pads,
                             list_widths=widths)
    rows = torch.arange(100, 600, device=cuda, dtype=torch.int32)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        st.sasrec_validation_batch(rows, 50, 5000)
        st.bert4rec_validation_batch(rows, 50, 5000)
        st.sasrec_new_path_validation_batch(rows, 50, 5000)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


@pytest.mark.parametrize("world", [1, 2, 8])
def test_validation_loader_visits_every_query_once(cuda, world):
    from replay_b200.device_data import DeviceBatchLoader, DeviceSequenceStore

    n = 1003
    q = np.arange(n) * 3 + 11
    st = DeviceSequenceStore([np.arange(1 + i % 7) for i in range(n)], query_ids=q, device=cuda,
                             query_lists={"ground_truth": [[i] for i in range(n)], "train": [[] for _ in range(n)]})
    for kind in ("sasrec_validate", "bert4rec_validate", "sasrec_new_validate"):
        got = []
        for r in range(world):
            for b in DeviceBatchLoader(st, 8, 64, 0, kind=kind, rank=r, world_size=world):
                got.append(b["query_id"].view(-1).cpu())
                assert torch.equal(b["ground_truth"][:, -1].cpu(), (got[-1] - 11) // 3)   # the lists follow the rows
        got = torch.cat(got).numpy()
        assert len(got) == n and np.array_equal(np.sort(got), q), (kind, world)
        if world == 1:
            assert np.array_equal(got, q)                              # store order


# ----------------------------------------------------------------------------------------------------------------------
# end to end: the metrics callbacks on device-built and on reference-layout host-built batches of the same users
# ----------------------------------------------------------------------------------------------------------------------
METRICS, KS = ("recall", "ndcg", "map", "mrr", "novelty", "coverage"), (1, 5, 10)


def _e2e_data(n_items=300, n_users=333, seed=7):
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, 60, n_users)
    seqs = [rng.integers(0, n_items, n) for n in lens]
    qid = np.arange(n_users) * 2 + 100
    gt = (list(qid[1:]), [rng.integers(0, n_items, rng.integers(0, 6)) for _ in qid[1:]])       # the first user absent
    tr = (list(qid[:-1]), [s[: max(1, len(s) - 3)] for s in seqs[:-1]])                          # the last user absent
    return n_items, seqs, qid, gt, tr, rng


def _to(b, dev):
    return {k: _to(v, dev) if isinstance(v, dict) else torch.as_tensor(v).to(dev) for k, v in b.items()}


class _Seen:
    """The ``sequential`` RemoveSeenItems reads: each query's train items."""

    def __init__(self, tr, n_items):
        from replay_b200.schema import TensorFeatureInfo, TensorSchema
        self.schema = TensorSchema(TensorFeatureInfo("item_id", n_items, n_items, 8))
        self._tr = tr

    def get_sequence_by_query_id(self, query_ids, feature):
        return [ov.lookup(*self._tr, q) for q in query_ids]


@pytest.mark.parametrize("model", ["sasrec", "bert4rec"])
def test_legacy_validation_metrics_equal_from_device_and_host_batches(cuda, model):
    from replay_b200.device_data import DeviceBatchLoader, DeviceSequenceStore
    from replay_b200.models.nn.sequential import Bert4Rec, RemoveSeenItems, SasRec, ValidationMetricsCallback
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    n_items, seqs, qid, gt, tr, _ = _e2e_data()
    L, d, B = 32, 64, 128
    schema = TensorSchema(TensorFeatureInfo("item_id", n_items, n_items, d))
    torch.manual_seed(0)
    if model == "sasrec":
        m = SasRec(schema, block_count=2, head_count=1, hidden_size=d, max_seq_len=L, dropout_rate=0.0)
        host_fn, kind = ov.sasrec_validation_batch, "sasrec_validate"
    else:
        m = Bert4Rec(schema, block_count=2, head_count=2, hidden_size=d, max_seq_len=L, dropout_rate=0.0)
        host_fn, kind = ov.bert4rec_validation_batch, "bert4rec_validate"
    m.eval()
    joined = {"ground_truth": [ov.lookup(*gt, q) for q in qid], "train": [ov.lookup(*tr, q) for q in qid]}
    gw, tw = max(len(x) for x in gt[1]), max(len(x) for x in tr[1])
    st = DeviceSequenceStore(seqs, query_ids=qid, device=cuda, query_lists=joined,
                             list_widths={"ground_truth": gw, "train": tw})
    cbs = [ValidationMetricsCallback(metrics=METRICS, ks=KS, postprocessors=[RemoveSeenItems(_Seen(tr, n_items))],
                                     item_count=n_items) for _ in range(2)]
    for cb in cbs:
        cb.on_validation_epoch_start(None, m)
    for i, db in enumerate(DeviceBatchLoader(st, L, B, n_items, kind=kind)):
        rows = list(range(i * B, min((i + 1) * B, len(seqs))))
        hb = _to(host_fn({"item_id": seqs}, qid, rows, L, {"item_id": n_items}, gt, tr, gw, tw), cuda)
        _assert_same(db, hb, (model, i))
        cbs[0].on_validation_batch_end(None, m, None, db, i)
        cbs[1].on_validation_batch_end(None, m, None, hb, i)
    a, b = (cb.on_validation_epoch_end(None, m) for cb in cbs)
    assert set(a) == {f"{mm}@{k}" for mm in METRICS for k in KS} and a == b


def test_new_path_validation_metrics_equal_from_device_and_host_batches(cuda):
    from replay_b200.device_data import DeviceBatchLoader, DeviceSequenceStore
    from replay_b200.nn.lightning import ComputeMetricsCallback, LightningModule, SeenItemsFilter
    from replay_b200.nn.sequential import SasRec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    n_items, seqs, qid, gt, tr, rng = _e2e_data(seed=8)
    L, d, B = 32, 64, 100
    cols = {"genre": [rng.integers(0, 20, len(s)) for s in seqs],
            "tags": [[rng.integers(0, 9, int(k)) for k in rng.integers(0, 6, len(s))] for s in seqs]}
    pads = {"item_id": n_items, "genre": 20, "tags": 9}
    schema = TensorSchema(TensorFeatureInfo("item_id", n_items, n_items, d), features=[
        TensorFeatureInfo("genre", 20, 20, d), TensorFeatureInfo("tags", 9, 9, d, is_list=True)])
    model = SasRec.from_params(schema, embedding_dim=d, num_heads=2, num_blocks=1, max_sequence_length=L, dropout=0.0,
                               device=cuda, seed=4)
    model.eval()
    lm = LightningModule(model)
    lists = {"ground_truth": [ov.lookup(*gt, q) for q in qid], "train": [ov.lookup(*tr, q) for q in qid]}
    widths, lpads = {"ground_truth": 4, "train": 64}, {"ground_truth": -1, "train": -2}
    st = DeviceSequenceStore(seqs, query_ids=qid, device=cuda, features=cols, query_lists=lists,
                             padding_values={**pads, **lpads}, list_widths={"tags": 3, **widths})
    cbs = [ComputeMetricsCallback(metrics=METRICS, ks=KS, item_count=n_items,
                                  postprocessors=[SeenItemsFilter(n_items, "seen_ids")]) for _ in range(2)]
    for cb in cbs:
        cb.on_validation_epoch_start(None, lm)
    for i, db in enumerate(DeviceBatchLoader(st, L, B, n_items, kind="sasrec_new_validate")):
        rows = list(range(i * B, min((i + 1) * B, len(seqs))))
        hb = ov.newpath_validation_batch({"item_id": seqs, **cols}, qid, rows, L, pads, lists, widths, lpads,
                                         list_widths={"tags": 3})
        hb["seen_ids"] = hb["train"]
        hb = _to(hb, cuda)
        _assert_same(db, hb, ("new", i))
        for cb, b in zip(cbs, (db, hb)):
            cb.on_validation_batch_end(None, lm, lm.predict_step(b, 0), b, i)
    a, b = (cb.on_validation_epoch_end(None, lm) for cb in cbs)
    assert set(a) == {f"{mm}@{k}" for mm in METRICS for k in KS} and a == b
