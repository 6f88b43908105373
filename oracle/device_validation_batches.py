"""TEST INFRASTRUCTURE - CPU restatement of how the reference's per-sample producers build VALIDATION and TEST batches,
one user at a time.  Pinned against the real reference classes by ``oracle/gen_device_validation_golden.py`` ->
``tests/golden/device_validation_batches.npz``; the device store's query lists (replay_b200/device_data.py,
csrc/rp_batch.cu) are checked against both.

Legacy (TorchSequentialValidationDataset, replay/data/nn/torch_sequential_dataset.py:183-285): the model window is the
prediction window (SasRecValidationDataset) or its BERT shift (Bert4RecValidationDataset, bert4rec/dataset.py:264-320);
``ground_truth`` / ``train`` are the label sequence of the user's query id in the ground-truth / train dataset (empty
when the id is absent: get_sequence_by_query_id), copied into a placeholder as long as the DATASET's longest sequence and
filled with -1 / -2 past the copy.
New path (Array1DColumn.__getitem__ + raw_get_mask, replay/data/nn/parquet/impl/array_1d_column.py:70-84,
indexing.py:42-78): a per-user list column keeps its last ``width`` entries, left-padded with the metadata's padding.
"""
from __future__ import annotations

import numpy as np

from . import device_batch_features as of

GROUND_TRUTH_PADDING, TRAIN_PADDING = -1, -2


def lookup(ids, lists, query_id):
    """get_sequence_by_query_id: the list of ``query_id``, or an empty one."""
    for q, x in zip(ids, lists):
        if q == query_id:
            return np.asarray(x, dtype=np.int64)
    return np.zeros(0, np.int64)


def legacy_list(seq, width: int, padding_value: int):
    """_get_ground_truth / _get_train: the list right-padded to ``width``."""
    out = np.full(width, padding_value, dtype=np.int64)
    for j in range(min(len(seq), width)):
        out[j] = seq[j]
    return out


def newpath_list(seq, width: int, padding_value: int):
    """Array1DColumn: the last ``width`` entries, left-padded."""
    out = np.full(width, padding_value, dtype=np.int64)
    m = min(len(seq), width)
    for j in range(m):
        out[width - m + j] = seq[len(seq) - m + j]
    return out


def window_mask(n: int, window: int):
    """_generate_padding_mask / raw_get_mask: True at the window's last min(n, window) positions."""
    out = np.zeros(window, dtype=bool)
    for p in range(window - min(n, window), window):
        out[p] = True
    return out


def sasrec_validation_batch(seqs, query_ids, rows, max_len, pads, gt, train, gt_width, train_width):
    """``seqs``: {name: per-user sequence}; ``gt`` / ``train``: (ids, lists) of the label datasets; ``rows``: the users."""
    item = seqs["item_id"]
    return {"query_id": np.asarray([[query_ids[r]] for r in rows], dtype=np.int64),
            "padding_mask": np.stack([window_mask(len(item[r]), max_len) for r in rows]),
            "feature_tensor": {n: np.stack([of.prediction_feature(s[r], max_len, pads[n]) for r in rows])
                               for n, s in seqs.items()},
            "ground_truth": np.stack([legacy_list(lookup(*gt, query_ids[r]), gt_width, GROUND_TRUTH_PADDING) for r in rows]),
            "train": np.stack([legacy_list(lookup(*train, query_ids[r]), train_width, TRAIN_PADDING) for r in rows])}


def bert4rec_validation_batch(seqs, query_ids, rows, max_len, pads, gt, train, gt_width, train_width):
    b = sasrec_validation_batch(seqs, query_ids, rows, max_len, pads, gt, train, gt_width, train_width)
    tok = np.roll(b["padding_mask"], -1, axis=1)  # _shift_features: rolled left, the last slot False
    tok[:, -1] = False
    pad = tok.copy()
    pad[:, -1] = True
    return {"query_id": b["query_id"], "pad_mask": pad,
            "inputs": {n: np.stack([of.bert_prediction_feature(s[r], max_len, pads[n]) for r in rows])
                       for n, s in seqs.items()},
            "token_mask": tok, "ground_truth": b["ground_truth"], "train": b["train"]}


def newpath_validation_batch(seqs, query_ids, rows, max_len, pads, lists, widths, list_pads, list_widths=None):
    """``seqs``: {name: per-user sequence}, a list feature named in ``list_widths`` ({name: K}) holding one list per
    event; ``lists``: {name: per-user list} cut at ``widths[name]`` with ``list_pads[name]``."""
    item, list_widths = seqs["item_id"], dict(list_widths or {})
    feats = {n: np.stack([of.newpath_feature(s[r], max_len, pads[n], train=False, width=list_widths.get(n), dtype=np.int64)
                          for r in rows]) for n, s in seqs.items()}
    out = {"query_id": np.asarray([query_ids[r] for r in rows], dtype=np.int64), "feature_tensors": feats,
           "padding_mask": np.stack([window_mask(len(item[r]), max_len) for r in rows])}
    for n, x in lists.items():
        out[n] = np.stack([newpath_list(np.asarray(x[r]), widths[n], list_pads[n]) for r in rows])
    return out


class SequentialStub:
    """A duck-typed SequentialDataset (replay/data/nn/sequential_dataset.py:18-105) over per-row sequences."""

    def __init__(self, schema, query_ids, sequences: dict):
        self.schema, self._ids, self._seqs = schema, list(query_ids), sequences
        self._item = schema.item_id_feature_name

    def __len__(self):
        return len(self._ids)

    def get_query_id(self, i):
        return self._ids[i]

    def get_all_query_ids(self):
        return np.asarray(self._ids)

    def get_sequence(self, i, name):
        return np.asarray(self._seqs[name][i])

    def get_sequence_length(self, i):
        return len(self._seqs[self._item][i])

    def get_max_sequence_length(self):
        return max(len(s) for s in self._seqs[self._item])

    def get_sequence_by_query_id(self, query_id, name):
        return lookup(self._ids, self._seqs[name], query_id)


def golden_inputs(z):
    """The histories, side features and label datasets of tests/golden/device_validation_batches.npz:
    (seqs {item_id, cat, lst}, pads, gt (ids, lists), train (ids, lists))."""
    off = np.concatenate([[0], np.cumsum(z["lengths"])])
    n = len(z["lengths"])
    seqs = {k: [z[f"col_{k}"][off[i]:off[i + 1]] for i in range(n)] for k in ("item_id", "cat")}
    loff = np.concatenate([[0], np.cumsum(z["lst_lengths"])])
    events = [z["lst_values"][loff[e]:loff[e + 1]] for e in range(len(z["lst_lengths"]))]
    seqs["lst"] = [events[off[i]:off[i + 1]] for i in range(n)]
    pads = dict(zip(("item_id", "cat", "lst"), (int(p) for p in z["pads"])))

    def split(tag):
        o = np.concatenate([[0], np.cumsum(z[f"{tag}_lengths"])])
        return list(z[f"{tag}_ids"]), [z[f"{tag}_values"][o[i]:o[i + 1]] for i in range(len(o) - 1)]

    return seqs, pads, split("gt"), split("tr")
