"""TEST INFRASTRUCTURE - CPU restatement of how the reference's per-sample producers cut SEQUENCE FEATURES (every schema
feature with is_seq next to the item id), one sample and one event at a time.  Pinned against the real reference classes
by ``oracle/gen_device_batch_features_golden.py`` -> ``tests/golden/device_batch_features.npz``; the device store's
feature columns (replay_b200/device_data.py, csrc/rp_batch.cu) are checked against both.

A feature's history ``seq`` is one entry per event: a scalar, a ``dim``-vector (``[n, dim]`` array) or, on the new path
only, a list of integers of any length.  Window offsets are the item ids' (oracle/dataset.py::window_index).

Legacy (TorchSequentialDataset._generate_tensor_feature / _pad_sequence / _get_tensor_dtype,
replay/data/nn/torch_sequential_dataset.py:69-136): seq[offset:offset + window] left-padded with the feature's own
padding value; integers become int64, floats float32.
  * SasRecTrainingDataset (sasrec/dataset.py:104-126): window L + 1, positions [0, L) kept.
  * SasRecPredictionDataset / Bert4RecTrainingDataset: window L.
  * Bert4RecPredictionDataset (_shift_features / _shift_seq, bert4rec/dataset.py:322-351): window L rolled left by one,
    the padding value written into the whole last slot.
New path (Array1DColumn / Array2DColumn.__getitem__, replay/data/nn/parquet/impl/array_1d_column.py:70-84,
array_2d_column.py:72-92, indexing.py:42-78; the default SASRec template, replay/nn/transform/template/sasrec.py): the
LAST ``window`` events left-padded, dtypes kept (integers here are int64); training reads L + 1 and NextTokenTransform
drops the last position, prediction reads L.  A list event keeps its last K entries left-padded to K; a padded event is
all padding.
"""
from __future__ import annotations

import numpy as np


def _legacy_dtype(seq):
    return np.int64 if np.issubdtype(np.asarray(seq).dtype, np.integer) else np.float32


def legacy_window(seq, offset: int, window: int, padding_value):
    """TorchSequentialDataset._generate_tensor_feature for one is_seq feature: [window(, dim)]."""
    seq = np.asarray(seq)
    dt = _legacy_dtype(seq)
    cut = seq[offset:offset + window].astype(dt)
    out = np.full((window,) + seq.shape[1:], padding_value, dtype=dt)
    for k in range(len(cut)):
        out[window - len(cut) + k] = cut[k]
    return out


def sasrec_training_feature(seq, offset: int, max_len: int, padding_value):
    return legacy_window(seq, offset, max_len + 1, padding_value)[:-1]


def prediction_feature(seq, max_len: int, padding_value):
    return legacy_window(seq, max(0, len(seq) - max_len), max_len, padding_value)


def bert_training_feature(seq, offset: int, max_len: int, padding_value):
    return legacy_window(seq, offset, max_len, padding_value)


def bert_prediction_feature(seq, max_len: int, padding_value):
    x = prediction_feature(seq, max_len, padding_value)
    out = np.empty_like(x)
    for p in range(max_len - 1):
        out[p] = x[p + 1]
    out[max_len - 1] = padding_value
    return out


def newpath_window(seq, window: int, padding_value, dtype):
    """Array1DColumn (scalars) / Array2DColumn with a fixed inner length (vectors): the last ``window`` events."""
    seq = np.asarray(seq)
    n = min(len(seq), window)
    out = np.full((window,) + seq.shape[1:], padding_value, dtype=dtype)
    for k in range(n):
        out[window - n + k] = seq[len(seq) - n + k]
    return out


def newpath_list_window(seq, window: int, width: int, padding_value):
    """Array2DColumn for a list column: [window, width] int64, each event's last ``width`` entries left-padded."""
    out = np.full((window, width), padding_value, dtype=np.int64)
    n = min(len(seq), window)
    for k in range(n):
        ev = list(seq[len(seq) - n + k])
        m = min(len(ev), width)
        for j in range(m):
            out[window - n + k, width - m + j] = ev[len(ev) - m + j]
    return out


def newpath_feature(seq, max_len: int, padding_value, *, train: bool, dtype=None, width=None):
    """One feature of a new-path sample: training reads max_len + 1 events and drops the last position."""
    window = max_len + (1 if train else 0)
    if width is not None:
        out = newpath_list_window(seq, window, width, padding_value)
    else:
        out = newpath_window(seq, window, padding_value, dtype if dtype is not None else np.asarray(seq).dtype)
    return out[:max_len]


def newpath_feature_at(seq, offset: int, max_len: int, padding_value, *, dtype=None, width=None):
    """A new-path training feature of the window starting at ``offset`` (sliding windows of the device loader): the
    events seq[offset:offset + max_len + 1], then the last position dropped."""
    return newpath_feature(seq[offset:offset + max_len + 1], max_len, padding_value, train=True, dtype=dtype, width=width)
