"""Query lists of the device sequence store without a GPU: the loop restatement of the reference's validation producers
(oracle/device_validation_batches.py) against the reference's own batches (tests/golden/device_validation_batches.npz,
oracle/gen_device_validation_golden.py), the store's query lists built on ``device="cpu"`` from a SequentialDataset join,
raw lists and pyarrow tables, every rejected input, and the validation loader's shards."""
import os

import numpy as np
import pytest
import torch

from oracle import device_validation_batches as ov
from replay_b200.device_data import DeviceBatchLoader, DeviceSequenceStore
from replay_b200.schema import TensorFeatureInfo, TensorSchema


def _golden(golden_dir):
    z = dict(np.load(os.path.join(golden_dir, "device_validation_batches.npz")))
    return (z, *ov.golden_inputs(z))


def _flat(prefix, batch, out):
    for k, v in batch.items():
        if isinstance(v, dict):
            _flat(f"{prefix}_{k}", v, out)
        else:
            out[f"{prefix}_{k}"] = v
    return out


def _assert_golden(z, prefix, batch, skip=()):
    got = _flat(prefix, batch, {})
    want = {k for k in z if k.startswith(prefix + "_") and k not in skip}
    assert set(got) == want, (prefix, sorted(set(got) ^ want))
    for k, v in got.items():
        v = np.asarray(v)
        assert v.dtype == z[k].dtype and v.shape == z[k].shape and np.array_equal(v, z[k]), k


def test_restatement_equals_reference_validation_batches(golden_dir):
    z, seqs, pads, gt, tr = _golden(golden_dir)
    L, n = int(z["L"]), len(z["lengths"])
    legacy = {k: seqs[k] for k in ("item_id", "cat")}
    gw, tw = max(len(x) for x in gt[1]), max(len(x) for x in tr[1])
    assert gw == z["sas_ground_truth"].shape[1] and tw == z["sas_train"].shape[1]
    # the legacy width is the label DATASET's longest list: here a user the store does not hold
    joined = [ov.lookup(*gt, q) for q in z["query_ids"]]
    assert max(len(x) for x in joined) < gw
    assert {len(x) for x in joined} >= {0, 1, int(z["G_W"]) + 1}
    assert any(q not in gt[0] for q in z["query_ids"]) and any(q not in tr[0] for q in z["query_ids"])
    rows = list(range(n))
    _assert_golden(z, "sas", ov.sasrec_validation_batch(legacy, z["query_ids"], rows, L, pads, gt, tr, gw, tw))
    _assert_golden(z, "bert", ov.bert4rec_validation_batch(legacy, z["query_ids"], rows, L, pads, gt, tr, gw, tw))
    lists = {"ground_truth": joined, "train": [ov.lookup(*tr, q) for q in z["query_ids"]]}
    lists["seen_ids"] = lists["train"]
    widths = {"ground_truth": int(z["G_W"]), "train": int(z["T_W"]), "seen_ids": int(z["T_W"])}
    list_pads = {"ground_truth": -1, "train": -2, "seen_ids": pads["item_id"]}
    nb = ov.newpath_validation_batch(seqs, z["query_ids"], list(z["new_order"]), L, pads, lists, widths, list_pads,
                                     list_widths={"lst": int(z["K"])})
    # the reader also returns every column's own mask; nothing downstream of the validate transforms reads them
    masks = {f"new_{k}" for k in z["new_keys"] if k.endswith("_mask") and k != "padding_mask"}
    _assert_golden(z, "new", nb, skip=masks | {"new_order", "new_keys"})
    assert set(z["new_keys"]) - {k[4:] for k in masks} == set(nb) - {"feature_tensors"}


def _datasets(z, seqs, gt, tr, *, n_items=40):
    item = TensorFeatureInfo("item_id", n_items, n_items, 8)
    schema = TensorSchema(item, features=[TensorFeatureInfo("cat", 7, 7, 8)])
    seq = ov.SequentialStub(schema, z["query_ids"], {k: seqs[k] for k in ("item_id", "cat")})
    lab = TensorSchema(TensorFeatureInfo("item_id", n_items, n_items, 8))
    return seq, ov.SequentialStub(lab, gt[0], {"item_id": gt[1]}), ov.SequentialStub(lab, tr[0], {"item_id": tr[1]})


def test_store_joins_validation_datasets_by_query_id(golden_dir):
    z, seqs, pads, gt, tr = _golden(golden_dir)
    seq, g, t = _datasets(z, seqs, gt, tr)
    st = DeviceSequenceStore.from_sequential_dataset(seq, device="cpu", ground_truth=g, train=t)
    assert st.feature_names == ["cat"] and st.query_list_names == ["ground_truth", "train"]
    ql = {c.name: c for c in st.query_lists}
    assert (ql["ground_truth"].width, ql["train"].width) == (z["sas_ground_truth"].shape[1], z["sas_train"].shape[1])
    assert (ql["ground_truth"].padding_value, ql["train"].padding_value) == (-1, -2)
    for name, ds in (("ground_truth", gt), ("train", tr)):
        c = ql[name]
        assert c.values.dtype == torch.int32 and c.offsets.dtype == torch.int64
        off = c.offsets.numpy()
        for i, q in enumerate(z["query_ids"]):
            assert np.array_equal(c.values.numpy()[off[i]:off[i + 1]], ov.lookup(*ds, q)), (name, q)


def test_store_raises_the_reference_checks(golden_dir):
    z, seqs, pads, gt, tr = _golden(golden_dir)
    seq, g, t = _datasets(z, seqs, gt, tr)
    msgs = [str(m) for m in z["error_messages"]]
    bad_name = ov.SequentialStub(TensorSchema(TensorFeatureInfo("item", 40, 40, 8)), gt[0], {"item": gt[1]})
    _, bad_card, _ = _datasets(z, seqs, gt, tr, n_items=41)
    no_overlap = ov.SequentialStub(g.schema, [1], {"item_id": [gt[1][1]]})
    cases = [dict(ground_truth=bad_name, train=t), dict(ground_truth=bad_card, train=t),
             dict(ground_truth=no_overlap, train=t), dict(ground_truth=g, train=t, label_feature_name="nope")]
    for kw, msg in zip(cases, msgs):
        with pytest.raises(ValueError, match=msg):
            DeviceSequenceStore.from_sequential_dataset(seq, device="cpu", **kw)
    not_cat = ov.SequentialStub(TensorSchema(TensorFeatureInfo("item_id", 40, 40, 8, is_cat=False)), gt[0],
                                {"item_id": gt[1]})
    with pytest.raises(ValueError, match="Label feature must be categorical"):
        DeviceSequenceStore.from_sequential_dataset(seq, device="cpu", ground_truth=not_cat, train=t,
                                                    label_feature_name="item_id")
    not_seq = ov.SequentialStub(TensorSchema(TensorFeatureInfo("item_id", 40, 40, 8, is_seq=False)), gt[0],
                                {"item_id": gt[1]})
    with pytest.raises(ValueError, match="Label feature must be sequential"):
        DeviceSequenceStore.from_sequential_dataset(seq, device="cpu", ground_truth=not_seq, train=t,
                                                    label_feature_name="item_id")


def test_store_query_lists_from_raw_lists_and_parquet():
    import pyarrow as pa

    seqs = [np.arange(3), np.arange(5), np.arange(1)]
    gt = [[7, 8], [], [2 ** 40]]
    st = DeviceSequenceStore(seqs, device="cpu", query_lists={"ground_truth": gt, "seen": [[1], [2, 3], []]},
                             padding_values={"seen": 99}, list_widths={"seen": 4})
    ql = {c.name: c for c in st.query_lists}
    assert ql["ground_truth"].values.dtype == torch.int64 and ql["ground_truth"].width == 2       # 2^40: int64
    assert ql["ground_truth"].padding_value == -1 and ql["seen"].padding_value == 99 and ql["seen"].width == 4
    assert ql["seen"].values.dtype == torch.int32 and ql["seen"].offsets.tolist() == [0, 1, 3, 3]
    table = pa.table({"item_id": pa.array([list(s) for s in seqs], pa.list_(pa.int64())),
                      "ground_truth": pa.array([[7, 8], None, [3]], pa.list_(pa.int32()))})
    sp = DeviceSequenceStore.from_parquet(table, device="cpu", query_list_columns=["ground_truth"],
                                          list_widths={"ground_truth": 5}, padding_values={"ground_truth": -7})
    c = sp.query_lists[0]
    assert (c.name, c.width, c.padding_value) == ("ground_truth", 5, -7)
    assert c.values[:3].tolist() == [7, 8, 3] and c.offsets.tolist() == [0, 2, 2, 3]                # null row: empty
    with pytest.raises(ValueError, match="list<int>"):
        DeviceSequenceStore.from_parquet(table.append_column("f", pa.array([[1.0]] * 3)), device="cpu",
                                         query_list_columns=["f"])
    with pytest.raises(ValueError, match="null values"):
        DeviceSequenceStore.from_parquet(table.set_column(1, "ground_truth", pa.array([[1, None], [], []])),
                                         device="cpu", query_list_columns=["ground_truth"])


def test_store_rejects_bad_query_lists():
    seqs = [np.arange(3), np.arange(5)]
    with pytest.raises(ValueError, match="2 sequences"):
        DeviceSequenceStore(seqs, device="cpu", query_lists={"ground_truth": [[1]]})
    with pytest.raises(ValueError, match="1-D integer"):
        DeviceSequenceStore(seqs, device="cpu", query_lists={"ground_truth": [[1.5], [2.0]]})
    with pytest.raises(ValueError, match="width must be >= 1"):
        DeviceSequenceStore(seqs, device="cpu", query_lists={"ground_truth": [[1], [2]]}, list_widths={"ground_truth": 0})
    with pytest.raises(ValueError, match="both feature columns and query lists"):
        DeviceSequenceStore(seqs, device="cpu", features={"x": [np.arange(3), np.arange(5)]},
                            query_lists={"x": [[1], [2]]})
    feats = {f"f{i}": [np.arange(3), np.arange(5)] for i in range(15)}
    DeviceSequenceStore(seqs, device="cpu", features=feats, query_lists={"ground_truth": [[1], [2]]})   # 16: one launch
    with pytest.raises(ValueError, match="at most 16"):
        DeviceSequenceStore(seqs, device="cpu", features=feats, query_lists={"ground_truth": [[1], [2]], "train": [[], []]})


@pytest.mark.parametrize("world", [1, 2, 8])
def test_validation_loader_shards_every_query_once(world):
    st = DeviceSequenceStore([np.arange(1 + i % 4) for i in range(1003)], device="cpu",
                             query_lists={"ground_truth": [[i] for i in range(1003)], "train": [[] for _ in range(1003)]})
    seen = []
    for kind in ("sasrec_validate", "bert4rec_validate", "sasrec_new_validate"):
        spans = []
        for r in range(world):
            ld = DeviceBatchLoader(st, 8, 64, 0, kind=kind, rank=r, world_size=world)
            assert len(ld) == -(-ld.n // 64)
            spans.append((ld.lo, ld.lo + ld.n))
        assert spans[0][0] == 0 and spans[-1][1] == 1003 and all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
        assert max(b - a for a, b in spans) - min(b - a for a, b in spans) <= 1
        seen.append(spans)
    assert seen[0] == seen[1] == seen[2]
