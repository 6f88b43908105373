"""Generate tests/golden/device_batch_features.npz FROM THE REAL REFERENCE (build container only).  TEST INFRASTRUCTURE.

    PYTHONPATH=oracle/shim:/root/reference python oracle/gen_device_batch_features_golden.py

A tiny history store with sequence features next to the item id, cut by the reference's own producers:
  * ``cat``  categorical, cardinality 7, padding 7 (= cardinality);
  * ``num``  float64 numerical, padding -1 (legacy batches round it to float32, the new path keeps float64);
  * ``vec``  float32 numerical of tensor_dim 3;
  * ``ts``   integer timestamps above 2^31, padding 0;
  * ``lst``  (new path only: the legacy datasets cannot stack ragged lists) a categorical list of lengths 0, 1, K and
    more than K, K = 3, padding 9.
Histories have lengths 1, L - 1, L, L + 1 and 3L (and a few more).  Modes: SasRecTrainingDataset (sliding windows and
last windows), SasRecPredictionDataset, Bert4RecTrainingDataset with a seeded masker (its uniforms stored the way
gen_golden.py::gen_dataset_layout stores them), Bert4RecPredictionDataset, and the new path's column classes followed by
the default SASRec template's train and predict transforms.
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

from replay.data import FeatureHint, FeatureSource, FeatureType  # noqa: E402
from replay.data.nn import TensorFeatureInfo, TensorFeatureSource, TensorSchema  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "device_batch_features.npz")

N_ITEMS, L, STEP, PROB, K = 40, 6, 2, 0.3, 3
PADS = {"item_id": N_ITEMS, "cat": 7, "num": -1, "vec": 0, "ts": 0, "lst": 9}


def _info(name, ftype, **kw):
    return TensorFeatureInfo(name=name, feature_type=ftype, is_seq=True,
                             feature_sources=[TensorFeatureSource(FeatureSource.INTERACTIONS, name)],
                             padding_value=PADS[name], **kw)


def make_schema(with_list: bool):
    feats = [
        _info("item_id", FeatureType.CATEGORICAL, cardinality=N_ITEMS, embedding_dim=8, feature_hint=FeatureHint.ITEM_ID),
        _info("cat", FeatureType.CATEGORICAL, cardinality=7, embedding_dim=8),
        _info("num", FeatureType.NUMERICAL, tensor_dim=1, embedding_dim=8),
        _info("vec", FeatureType.NUMERICAL, tensor_dim=3, embedding_dim=8),
        _info("ts", FeatureType.NUMERICAL, tensor_dim=1, embedding_dim=8, feature_hint=FeatureHint.TIMESTAMP),
    ]
    if with_list:
        feats.append(_info("lst", FeatureType.CATEGORICAL_LIST, cardinality=9, embedding_dim=8))
    return TensorSchema(feats)


def make_histories():
    rng = np.random.default_rng(11)
    lens = [1, L - 1, L, L + 1, 3 * L, 2, L + 3, 1, 3 * L]
    seqs = {"item_id": [], "cat": [], "num": [], "vec": [], "ts": [], "lst": []}
    list_lens = [0, 1, K, K + 2]  # every kind of list event occurs in every long history
    for i, n in enumerate(lens):
        seqs["item_id"].append(rng.integers(0, N_ITEMS, n).astype(np.int64))
        seqs["cat"].append(rng.integers(0, 7, n).astype(np.int64))
        seqs["num"].append(rng.normal(0, 1, n).astype(np.float64) / 3.0)  # float64 values that round in float32
        seqs["vec"].append(rng.normal(0, 1, (n, 3)).astype(np.float32))
        seqs["ts"].append((3_000_000_000 + np.cumsum(rng.integers(1, 10_000, n))).astype(np.int64))
        seqs["lst"].append([rng.integers(0, 9, list_lens[(i + e) % 4]).astype(np.int64) for e in range(n)])
    return lens, seqs


def main():
    from replay.data.nn.parquet.impl.array_1d_column import Array1DColumn
    from replay.data.nn.parquet.impl.array_2d_column import Array2DColumn
    from replay.models.nn.sequential.bert4rec.dataset import (Bert4RecPredictionDataset, Bert4RecTrainingDataset,
                                                              Bert4RecUniformMasker)
    from replay.models.nn.sequential.sasrec.dataset import SasRecPredictionDataset, SasRecTrainingDataset
    from replay.nn.transform.template.sasrec import make_default_sasrec_transforms

    lens, seqs = make_histories()
    legacy_names = ["item_id", "cat", "num", "vec", "ts"]
    sch = make_schema(with_list=False)

    class Store:
        schema = sch

        def __len__(self):
            return len(lens)

        def get_query_id(self, i):
            return 500 + 7 * i

        def get_sequence_length(self, i):
            return lens[i]

        def get_sequence(self, i, name):
            return seqs[name][i]

        def get_max_sequence_length(self):
            return max(lens)

    ds = Store()
    lst_len = np.asarray([len(e) for s in seqs["lst"] for e in s], dtype=np.int64)
    out = {"lengths": np.asarray(lens), "L": L, "step": STEP, "mask_prob": PROB, "K": K,
           "query_ids": np.asarray([500 + 7 * i for i in range(len(lens))]),
           "pads": np.asarray([PADS[n] for n in ["item_id", "cat", "num", "vec", "ts", "lst"]]),
           "lst_lengths": lst_len, "lst_values": np.concatenate([e for s in seqs["lst"] for e in s]).astype(np.int64)}
    for n in legacy_names:
        out[f"col_{n}"] = np.concatenate(seqs[n])

    def stack(samples, *path):
        def get(s):
            for k in path:
                s = s[k]
            return s.numpy()
        return np.stack([get(s) for s in samples])

    def put(prefix, samples, group):
        for n in legacy_names:
            out[f"{prefix}_{n}"] = stack(samples, group, n)

    for tag, st in (("slide", STEP), ("last", None)):
        t = SasRecTrainingDataset(ds, max_sequence_length=L, sliding_window_step=st)
        smp = [t[i] for i in range(len(t))]
        out[f"sas_{tag}_index"] = np.asarray(t._inner._index2sequence_map)
        put(f"sas_{tag}", smp, "feature_tensor")
        out[f"sas_{tag}_pad"] = stack(smp, "padding_mask")
        out[f"sas_{tag}_labels"] = stack(smp, "positive_labels")
        out[f"sas_{tag}_tmask"] = stack(smp, "target_padding_mask")
    p = SasRecPredictionDataset(ds, max_sequence_length=L)
    smp = [p[i] for i in range(len(p))]
    put("pred", smp, "feature_tensor")
    out["pred_pad"] = stack(smp, "padding_mask")
    for tag, st in (("slide", STEP), ("last", None)):
        bt = Bert4RecTrainingDataset(ds, L, sliding_window_step=st,
                                     custom_masker=Bert4RecUniformMasker(PROB, torch.Generator().manual_seed(21)))
        smp = [bt[i] for i in range(len(bt))]
        g2 = torch.Generator().manual_seed(21)
        out[f"bert_{tag}_uniforms"] = np.stack([torch.rand(L, dtype=torch.float32, generator=g2).numpy() for _ in smp])
        out[f"bert_{tag}_index"] = np.asarray(bt._inner._index2sequence_map)
        put(f"bert_{tag}", smp, "inputs")
        out[f"bert_{tag}_pad"] = stack(smp, "pad_mask")
        out[f"bert_{tag}_tok"] = stack(smp, "token_mask")
        out[f"bert_{tag}_labels"] = stack(smp, "positive_labels")
    bp = Bert4RecPredictionDataset(ds, L)
    smp = [bp[i] for i in range(len(bp))]
    put("bertpred", smp, "inputs")
    out["bertpred_pad"] = stack(smp, "pad_mask")
    out["bertpred_tok"] = stack(smp, "token_mask")

    # ---- new path: the parquet column classes on an arbitrary (repeating) row order, then the template transforms
    schema_new = make_schema(with_list=True)
    tr = make_default_sasrec_transforms(schema_new)
    order = torch.tensor([3, 0, 8, 4, 4, 1, 7, 2, 6, 5])
    lengths = torch.tensor(lens, dtype=torch.int64)

    def columns(window):
        cols = {n: Array1DColumn(data=torch.from_numpy(np.concatenate(seqs[n])), lengths=lengths, shape=window,
                                 padding=PADS[n]) for n in ("item_id", "cat", "num", "ts")}
        cols["vec"] = Array2DColumn(data=torch.from_numpy(np.concatenate(seqs["vec"]).reshape(-1)), outer_lengths=lengths,
                                    inner_lengths=torch.full((sum(lens),), 3, dtype=torch.int64), shape=[window, 3],
                                    padding=PADS["vec"])
        cols["lst"] = Array2DColumn(data=torch.from_numpy(out["lst_values"]), outer_lengths=lengths,
                                    inner_lengths=torch.from_numpy(lst_len), shape=[window, K], padding=PADS["lst"])
        return cols

    for split, window in (("train", L + 1), ("predict", L)):
        batch = {"query_id": order.clone()}
        for n, c in columns(window).items():
            mask, vals = c[order]
            batch[n], batch[f"{n}_mask"] = vals, mask
        for t in tr[split]:
            batch = t(batch)
        out[f"new_{split}_pad"] = batch["padding_mask"].numpy()
        for n in ["item_id", "cat", "num", "vec", "ts", "lst"]:
            out[f"new_{split}_{n}"] = batch["feature_tensors"][n].numpy()
        if split == "train":
            out["new_train_labels"] = batch["positive_labels"].numpy()
            out["new_train_tmask"] = batch["target_padding_mask"].numpy()
    out["new_order"] = order.numpy()
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, {k: (v.shape, v.dtype) for k, v in out.items() if k.startswith(("new_", "sas_last", "bertpred"))})


if __name__ == "__main__":
    main()
