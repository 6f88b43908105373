"""Generate tests/golden/device_validation_batches.npz FROM THE REAL REFERENCE (build container only).  TEST INFRASTRUCTURE.

    PYTHONPATH=oracle/shim:/root/reference python oracle/gen_device_validation_golden.py

Validation and test batches, cut by the reference's own producers from a tiny store:
  * nine histories (lengths 1, L - 1, L, L + 1, 3L, ...) with a categorical side feature ``cat`` and, on the new path, a
    categorical list ``lst`` (the legacy datasets cannot stack ragged lists);
  * a ground-truth dataset whose lists have lengths 0, 1, 2 and more than the new path's width G_W, which lacks one
    stored user and holds one user the store lacks, with the longest list of all (the legacy width is the ground-truth
    DATASET's longest list, not the longest joined one);
  * a train dataset that lacks another stored user.
Legacy: SasRecValidationDataset and Bert4RecValidationDataset over PandasSequentialDataset, every sample through
torch's default collate.  New path: the parquet column classes at their metadata's shape on a fixed row order (the
validate split is not shuffled), then make_default_sasrec_transforms(schema)["validate"].  Every key of every batch is
recorded, and so are the messages of the reference's checks on mismatched validation datasets.
"""
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "shim"))
sys.path.insert(1, "/root/reference")
warnings.filterwarnings("ignore")

import pandas as pd  # noqa: E402
from replay.data import FeatureHint, FeatureSource, FeatureType  # noqa: E402
from replay.data.nn import TensorFeatureInfo, TensorFeatureSource, TensorSchema  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "device_validation_batches.npz")

N_ITEMS, L, K, G_W, T_W = 40, 6, 3, 3, 8
PADS = {"item_id": N_ITEMS, "cat": 7, "lst": 9, "ground_truth": -1, "train": -2, "seen_ids": N_ITEMS}
QID = [500 + 7 * i for i in range(9)]


def _info(name, ftype, is_seq=True, **kw):
    return TensorFeatureInfo(name=name, feature_type=ftype, is_seq=is_seq,
                             feature_sources=[TensorFeatureSource(FeatureSource.INTERACTIONS, name)],
                             padding_value=PADS.get(name, 0), **kw)


def _item(cardinality=N_ITEMS, name="item_id"):
    return _info(name, FeatureType.CATEGORICAL, cardinality=cardinality, embedding_dim=8, feature_hint=FeatureHint.ITEM_ID)


def make_data():
    rng = np.random.default_rng(5)
    lens = [1, L - 1, L, L + 1, 3 * L, 2, L + 3, 1, 3 * L]
    seqs = {"item_id": [], "cat": [], "lst": []}
    for i, n in enumerate(lens):
        seqs["item_id"].append(rng.integers(0, N_ITEMS, n).astype(np.int64))
        seqs["cat"].append(rng.integers(0, 7, n).astype(np.int64))
        seqs["lst"].append([rng.integers(0, 9, (0, 1, K, K + 2)[(i + e) % 4]).astype(np.int64) for e in range(n)])
    # ground truth: QID[2] absent, 999 only here (and longest); lengths 0, 1, 2 and > G_W
    gt_len = {QID[0]: 0, QID[1]: 1, QID[3]: 2, QID[4]: G_W + 2, QID[5]: 1, QID[6]: G_W, QID[7]: 0, QID[8]: G_W + 1,
              999: G_W + 4}
    gt = {q: rng.integers(0, N_ITEMS, n).astype(np.int64) for q, n in gt_len.items()}
    # train: QID[6] absent; lengths 0 .. > T_W
    tr_len = {QID[0]: 0, QID[1]: 3, QID[2]: T_W + 3, QID[3]: 1, QID[4]: T_W, QID[5]: 2, QID[7]: 5, QID[8]: T_W + 1}
    tr = {q: rng.integers(0, N_ITEMS, n).astype(np.int64) for q, n in tr_len.items()}
    return lens, seqs, gt, tr


def main():
    from torch.utils.data import default_collate

    from replay.data.nn.parquet.impl.array_1d_column import Array1DColumn
    from replay.data.nn.parquet.impl.array_2d_column import Array2DColumn
    from replay.data.nn.sequential_dataset import PandasSequentialDataset
    from replay.models.nn.sequential.bert4rec.dataset import Bert4RecValidationDataset
    from replay.models.nn.sequential.sasrec.dataset import SasRecValidationDataset
    from replay.nn.transform.template.sasrec import make_default_sasrec_transforms

    lens, seqs, gt, tr = make_data()
    seq_schema = TensorSchema([_item(), _info("cat", FeatureType.CATEGORICAL, cardinality=7, embedding_dim=8)])
    seq_df = pd.DataFrame({"user_id": QID, "item_id": seqs["item_id"], "cat": seqs["cat"]})
    sequential = PandasSequentialDataset(seq_schema, "user_id", "item_id", seq_df)

    def labels(d, schema=None):
        schema = schema or TensorSchema([_item()])
        name = schema.item_id_feature_name
        return PandasSequentialDataset(schema, "user_id", name, pd.DataFrame({"user_id": list(d), name: list(d.values())}))

    ground_truth, train = labels(gt), labels(tr)
    out = {"lengths": np.asarray(lens), "L": L, "K": K, "G_W": G_W, "T_W": T_W, "query_ids": np.asarray(QID),
           "col_item_id": np.concatenate(seqs["item_id"]), "col_cat": np.concatenate(seqs["cat"]),
           "lst_lengths": np.asarray([len(e) for s in seqs["lst"] for e in s], dtype=np.int64),
           "lst_values": np.concatenate([e for s in seqs["lst"] for e in s]).astype(np.int64),
           "pads": np.asarray([PADS[n] for n in ("item_id", "cat", "lst")]),
           "gt_ids": np.asarray(list(gt)), "gt_lengths": np.asarray([len(v) for v in gt.values()]),
           "gt_values": np.concatenate(list(gt.values())),
           "tr_ids": np.asarray(list(tr)), "tr_lengths": np.asarray([len(v) for v in tr.values()]),
           "tr_values": np.concatenate(list(tr.values()))}

    def flat(prefix, batch):
        for k, v in batch.items():
            if isinstance(v, dict):
                flat(f"{prefix}_{k}", v)
            else:
                out[f"{prefix}_{k}"] = v.numpy()

    # ---- legacy: every sample, then the default collate
    for tag, cls in (("sas", SasRecValidationDataset), ("bert", Bert4RecValidationDataset)):
        ds = cls(sequential, ground_truth, train, max_sequence_length=L, padding_value=N_ITEMS)
        flat(tag, default_collate([ds[i] for i in range(len(ds))]))

    # ---- the reference's checks and their messages
    msgs = []
    bad = [
        (labels(gt, TensorSchema([_item(name="item")])), train, None),                   # item feature name
        (labels(gt, TensorSchema([_item(cardinality=N_ITEMS + 1)])), train, None),       # cardinality
        (labels({1: gt[QID[1]]}), train, None),                                          # no shared query id
        (ground_truth, train, "nope"),                                                   # label not in the schema
    ]
    for g, t, lab in bad:
        try:
            SasRecValidationDataset(sequential, g, t, max_sequence_length=L, label_feature_name=lab)
        except ValueError as e:
            msgs.append(str(e))
        else:
            raise AssertionError("the reference accepted a bad validation dataset")
    out["error_messages"] = np.asarray(msgs)

    # ---- new path: the reader's columns of the validate split, then the template's validate transforms
    new_schema = TensorSchema([_item(), _info("cat", FeatureType.CATEGORICAL, cardinality=7, embedding_dim=8),
                               _info("lst", FeatureType.CATEGORICAL_LIST, cardinality=9, embedding_dim=8)])
    order = torch.tensor([3, 0, 8, 4, 1, 7, 2, 6, 5])
    lengths = torch.tensor(lens, dtype=torch.int64)
    gtl = [gt.get(q, np.zeros(0, np.int64)) for q in QID]
    trl = [tr.get(q, np.zeros(0, np.int64)) for q in QID]

    def col1(values, lens_, shape, pad):
        return Array1DColumn(data=torch.from_numpy(np.concatenate(values).astype(np.int64)),
                             lengths=torch.tensor(lens_, dtype=torch.int64), shape=shape, padding=pad)

    cols = {n: col1(seqs[n], lens, L, PADS[n]) for n in ("item_id", "cat")}
    cols["lst"] = Array2DColumn(data=torch.from_numpy(out["lst_values"]), outer_lengths=lengths,
                                inner_lengths=torch.from_numpy(out["lst_lengths"]), shape=[L, K], padding=PADS["lst"])
    cols["ground_truth"] = col1(gtl, [len(x) for x in gtl], G_W, PADS["ground_truth"])
    cols["train"] = col1(trl, [len(x) for x in trl], T_W, PADS["train"])
    cols["seen_ids"] = col1(trl, [len(x) for x in trl], T_W, PADS["seen_ids"])
    batch = {"query_id": torch.tensor(QID, dtype=torch.int64)[order]}
    for n, c in cols.items():
        mask, vals = c[order]
        batch[n], batch[f"{n}_mask"] = vals, mask
    for t in make_default_sasrec_transforms(new_schema)["validate"]:
        batch = t(batch)
    flat("new", batch)
    out["new_order"] = order.numpy()
    out["new_keys"] = np.asarray(sorted(k for k in batch if k != "feature_tensors"))
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, {k: (v.shape, v.dtype) for k, v in out.items() if k.startswith(("sas_", "bert_", "new_"))})
    print(msgs)


if __name__ == "__main__":
    main()
