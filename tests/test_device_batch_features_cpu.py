"""Feature columns of the device sequence store without a GPU: construction from raw sequences, a duck-typed
SequentialDataset and pyarrow tables on ``device="cpu"``, every rejected input, and the loop restatement of the reference's
feature producers (oracle/device_batch_features.py) against the reference's own batches
(tests/golden/device_batch_features.npz, oracle/gen_device_batch_features_golden.py)."""
import os

import numpy as np
import pytest
import torch

from oracle import dataset as od
from oracle import device_batch_features as of
from replay_b200.device_data import DeviceSequenceStore

NAMES = ["item_id", "cat", "num", "vec", "ts"]


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


def _stack(rows):
    return np.stack(rows)


def test_restatement_equals_reference_legacy_batches(golden_dir):
    z, seqs, pads = _golden(golden_dir)
    L, step = int(z["L"]), int(z["step"])
    lens = z["lengths"]
    for tag, sw in (("slide", step), ("last", None)):
        idx = od.window_index(lens, L + 1, sw)
        assert np.array_equal(np.asarray(idx), z[f"sas_{tag}_index"])
        for n in NAMES:
            got = _stack([of.sasrec_training_feature(seqs[n][s], o, L, pads[n]) for s, o in idx])
            assert got.dtype == z[f"sas_{tag}_{n}"].dtype and np.array_equal(got, z[f"sas_{tag}_{n}"]), (tag, n)
        idx = od.window_index(lens, L, sw)
        assert np.array_equal(np.asarray(idx), z[f"bert_{tag}_index"])
        for n in NAMES:
            got = _stack([of.bert_training_feature(seqs[n][s], o, L, pads[n]) for s, o in idx])
            assert got.dtype == z[f"bert_{tag}_{n}"].dtype and np.array_equal(got, z[f"bert_{tag}_{n}"]), (tag, n)
    for n in NAMES:
        got = _stack([of.prediction_feature(s, L, pads[n]) for s in seqs[n]])
        assert got.dtype == z[f"pred_{n}"].dtype and np.array_equal(got, z[f"pred_{n}"]), n
        got = _stack([of.bert_prediction_feature(s, L, pads[n]) for s in seqs[n]])
        assert got.dtype == z[f"bertpred_{n}"].dtype and np.array_equal(got, z[f"bertpred_{n}"]), n
    # float64 values really round on the legacy path
    assert not np.array_equal(z["col_num"].astype(np.float32).astype(np.float64), z["col_num"])
    assert z["col_ts"].max() > 2 ** 31


def test_restatement_equals_reference_new_path_batches(golden_dir):
    z, seqs, pads = _golden(golden_dir)
    L, K = int(z["L"]), int(z["K"])
    assert {len(e) for s in seqs["lst"] for e in s} >= {0, 1, K, K + 2}
    for split in ("train", "predict"):
        for n in NAMES + ["lst"]:
            rows = [of.newpath_feature(seqs[n][i], L, pads[n], train=split == "train", width=K if n == "lst" else None)
                    for i in z["new_order"]]
            got, want = _stack(rows), z[f"new_{split}_{n}"]
            assert got.dtype == want.dtype and np.array_equal(got, want), (split, n)


def test_store_from_sequences_on_cpu(golden_dir):
    z, seqs, pads = _golden(golden_dir)
    st = DeviceSequenceStore(seqs["item_id"], device="cpu", features={n: seqs[n] for n in ["cat", "num", "vec", "ts", "lst"]},
                             padding_values=pads, list_widths={"lst": 3})
    cols = {c.name: c for c in st.columns}
    assert st.feature_names == ["cat", "num", "vec", "ts", "lst"]
    assert cols["cat"].kind == "int" and cols["cat"].values.dtype == torch.int32            # narrowed: every value fits
    assert cols["ts"].kind == "int" and cols["ts"].values.dtype == torch.int64              # above 2^31
    assert cols["num"].kind == "float" and cols["num"].values.dtype == torch.float64 and cols["num"].tail == ()
    assert cols["vec"].kind == "float" and cols["vec"].values.dtype == torch.float32 and cols["vec"].tail == (3,)
    assert cols["lst"].kind == "list" and cols["lst"].tail == (3,) and cols["lst"].padding_value == 9
    assert np.array_equal(cols["ts"].values.numpy(), z["col_ts"])
    assert np.array_equal(cols["num"].values.numpy(), z["col_num"])
    assert np.array_equal(cols["vec"].values.numpy(), z["col_vec"].reshape(-1))
    assert np.array_equal(cols["lst"].values.numpy(), z["lst_values"])
    assert np.array_equal(np.diff(cols["lst"].list_offsets.numpy()), z["lst_lengths"])
    # default list width: the longest list
    assert DeviceSequenceStore(seqs["item_id"], device="cpu", features={"lst": seqs["lst"]}).columns[0].tail == (5,)
    # an item-only store has no columns
    assert DeviceSequenceStore(seqs["item_id"], device="cpu").columns == []


def test_store_from_sequential_dataset_on_cpu(golden_dir):
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    z, seqs, pads = _golden(golden_dir)
    schema = TensorSchema(TensorFeatureInfo("item_id", 40, 40, 8), features=[
        TensorFeatureInfo("cat", 7, 7, 8), TensorFeatureInfo("num", None, -1, 8, is_cat=False, tensor_dim=1),
        TensorFeatureInfo("vec", None, 0, 8, is_cat=False, tensor_dim=3),
        TensorFeatureInfo("lst", 9, 9, 8, is_list=True), TensorFeatureInfo("user_age", 5, 0, 8, is_seq=False)])

    class Seq:
        def __init__(self):
            self.schema = schema

        def __len__(self):
            return len(seqs["item_id"])

        def get_query_id(self, i):
            return 10 + i

        def get_sequence(self, i, name):
            return seqs[name][i]

    st = DeviceSequenceStore.from_sequential_dataset(Seq(), device="cpu", list_widths={"lst": 2})
    assert st.feature_names == ["cat", "num", "vec", "lst"]                 # per-query features are not read
    cols = {c.name: c for c in st.columns}
    assert cols["cat"].padding_value == 7 and cols["num"].padding_value == -1.0 and cols["lst"].tail == (2,)
    assert np.array_equal(st.query_ids.numpy(), 10 + np.arange(len(seqs["item_id"])))


def test_store_from_arrow_on_cpu(golden_dir):
    pa = pytest.importorskip("pyarrow")
    z, seqs, pads = _golden(golden_dir)
    n = len(seqs["item_id"])
    table = pa.table({
        "item_id": pa.array([s.tolist() for s in seqs["item_id"]], pa.list_(pa.int64())),
        "user": pa.array(np.arange(n) + 3),
        "cat": pa.array([s.tolist() for s in seqs["cat"]], pa.list_(pa.int32())),
        "num": pa.array([s.tolist() for s in seqs["num"]], pa.list_(pa.float64())),
        "vec": pa.array([s.tolist() for s in seqs["vec"]], pa.list_(pa.list_(pa.float32()))),
        "ts": pa.array([s.tolist() for s in seqs["ts"]], pa.list_(pa.int64())),
        "lst": pa.array([[e.tolist() for e in s] for s in seqs["lst"]], pa.list_(pa.list_(pa.int64()))),
    })
    st = DeviceSequenceStore.from_parquet(table, query_column="user", device="cpu",
                                          feature_columns=["cat", "num", "vec", "ts", "lst"], padding_values=pads,
                                          list_widths={"lst": 3})
    ref = DeviceSequenceStore(seqs["item_id"], device="cpu", features={k: seqs[k] for k in ["cat", "num", "vec", "ts", "lst"]},
                              padding_values=pads, list_widths={"lst": 3})
    for a, b in zip(st.columns, ref.columns):
        assert (a.name, a.kind, a.tail, a.padding_value) == (b.name, b.kind, b.tail, b.padding_value)
        assert a.values.dtype == b.values.dtype and torch.equal(a.values, b.values), a.name
        assert (a.list_offsets is None) == (b.list_offsets is None)
        if a.list_offsets is not None:
            assert torch.equal(a.list_offsets, b.list_offsets)
    # fixed-size inner lists are vectors too
    fixed = pa.table({"item_id": table["item_id"],
                      "vec": pa.array([s.tolist() for s in seqs["vec"]], pa.list_(pa.list_(pa.float32(), 3)))})
    c = DeviceSequenceStore.from_parquet(fixed, device="cpu", feature_columns=["vec"]).columns[0]
    assert c.tail == (3,) and torch.equal(c.values, ref.columns[2].values)


def test_rejected_columns():
    seqs = [np.array([1, 2, 3]), np.array([4])]
    with pytest.raises(ValueError, match="lengths differ"):
        DeviceSequenceStore(seqs, device="cpu", features={"c": [np.array([1, 2]), np.array([4])]})
    with pytest.raises(ValueError, match="lengths differ"):
        DeviceSequenceStore(seqs, device="cpu", features={"c": [[[1], [2], [3]], [[4], [5]]]})
    with pytest.raises(ValueError, match="sequences"):
        DeviceSequenceStore(seqs, device="cpu", features={"c": [np.array([1, 2, 3])]})
    with pytest.raises(ValueError, match="ragged vectors"):
        DeviceSequenceStore(seqs, device="cpu", features={"v": [[[0.5, 1.0], [1.0, 2.0], [0.0]], [[1.0, 1.0]]]})
    with pytest.raises(ValueError, match="ragged vectors"):
        DeviceSequenceStore(seqs, device="cpu", features={"v": [np.zeros((3, 2)), np.zeros((1, 4))]})
    with pytest.raises(ValueError, match="null"):
        DeviceSequenceStore(seqs, device="cpu", features={"c": [[1, None, 3], [4]]})
    with pytest.raises(ValueError, match="null"):
        DeviceSequenceStore(seqs, device="cpu", features={"l": [[[1], None, [3, 4]], [[4]]]})
    with pytest.raises(ValueError, match="null"):
        DeviceSequenceStore(seqs, device="cpu", features={"l": [[[1], [None], [3, 4]], [[4]]]})
    with pytest.raises(ValueError, match="K must be >= 1"):
        DeviceSequenceStore(seqs, device="cpu", features={"l": [[[1], [2], [3, 4]], [[4]]]}, list_widths={"l": 0})
    with pytest.raises(ValueError, match="at most 16"):
        DeviceSequenceStore(seqs, device="cpu", features={f"c{i}": [np.zeros(3, int), np.zeros(1, int)] for i in range(17)})
    # sixteen columns are fine
    st = DeviceSequenceStore(seqs, device="cpu", features={f"c{i}": [np.zeros(3, int), np.zeros(1, int)] for i in range(16)})
    assert len(st.columns) == 16


def test_rejected_arrow_columns():
    pa = pytest.importorskip("pyarrow")
    items = pa.array([[1, 2, 3], [4]], pa.list_(pa.int64()))

    def store(col, **kw):
        return DeviceSequenceStore.from_parquet(pa.table({"item_id": items, "f": col}), device="cpu", feature_columns=["f"],
                                                **kw)

    with pytest.raises(ValueError, match="lengths differ"):
        store(pa.array([[1, 2], [4]], pa.list_(pa.int64())))
    with pytest.raises(ValueError, match="null"):
        store(pa.array([[1, None, 3], [4]], pa.list_(pa.int64())))
    with pytest.raises(ValueError, match="null"):
        store(pa.array([[[1], None, [3]], [[4]]], pa.list_(pa.list_(pa.int64()))))
    with pytest.raises(ValueError, match="null"):
        store(pa.array([[[1.0], [None], [3.0]], [[4.0]]], pa.list_(pa.list_(pa.float32()))))
    with pytest.raises(ValueError, match="ragged vectors"):
        store(pa.array([[[1.0], [2.0, 3.0], [3.0]], [[4.0]]], pa.list_(pa.list_(pa.float32()))))
    with pytest.raises(ValueError, match="K must be >= 1"):
        store(pa.array([[[1], [2, 3], [3]], [[4]]], pa.list_(pa.list_(pa.int64()))), list_widths={"f": 0})
    with pytest.raises(ValueError, match="list column"):
        store(pa.array([1, 2], pa.int64()))
    with pytest.raises(ValueError, match="at most 16"):
        DeviceSequenceStore.from_parquet(pa.table({"item_id": items}), device="cpu", feature_columns=[f"c{i}" for i in range(17)])
