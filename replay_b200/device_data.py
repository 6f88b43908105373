"""Device-resident sequence store and batch construction (SURVEY.md §8 f.1).

All user histories are uploaded ONCE as a CSR store (offsets int64 + item ids int32); every batch is then cut, left-padded,
shifted and masked by one CUDA launch (``rp_build_batch``, csrc/rp_batch.cu) instead of the reference's per-sample host
path (``TorchSequentialDataset.__getitem__`` -> ``SasRecTrainingDataset.__getitem__`` / ``Bert4RecTrainingDataset`` ->
default collate -> H2D copy; replay/data/nn/torch_sequential_dataset.py:69-171, sasrec/dataset.py:104-126,
bert4rec/dataset.py:71-92,163-177,322-351).  The produced batch dictionaries carry the reference's key names, dtypes and
shapes, so they feed ``training_step`` / ``predict_step`` of the modules in ``replay_b200.models`` / ``replay_b200.nn``
unchanged.  There is no CPU fallback: building a batch needs the CUDA library.

Next to the item ids the store holds sequence feature columns, one entry per event and aligned with the item history,
cut in the same launch (``rp_build_batch_features``) through the same window, offset and shift as the ids, each left-padded
with its own padding value.  Four kinds: an integer scalar (stored as int32 when every value fits, else int64), a float
scalar (stored in its source dtype, float32 or float64), a float vector of one ``dim`` for every event (``[n_events,
dim]``) and an integer list of any length per event (a second level of offsets plus flat values; output width ``K``).
Legacy builders emit every integer as int64 and every float as float32 (TorchSequentialDataset._get_tensor_dtype); the
new-path builders emit integers as int64 and keep each float column's dtype.

Query lists hold one integer list per stored sequence instead of one entry per event: the ground-truth and train items of
a validation or test user (``TorchSequentialValidationDataset``, replay/data/nn/torch_sequential_dataset.py:183-285).
They are stored as CSR (int64 offsets, int32 values when every value fits, else int64) and cut in the same launch as
int64 ``[B, width]``: the legacy validation builders take each list's first ``width`` entries right-padded (``width`` is
the dataset-wide longest list, as the reference's placeholders are), the new path's take its last ``width`` entries
left-padded (Array1DColumn.__getitem__, replay/data/nn/parquet/impl/array_1d_column.py:70-84)."""
from __future__ import annotations

import numpy as np
import torch

from ._lib import (BATCH_COL_FLOAT, BATCH_COL_INT, BATCH_COL_LIST, BATCH_COL_QUERY_LIST, BATCH_COL_QUERY_LIST_LAST,
                   BATCH_MAX_COLUMNS, BatchColumn, check, lib)

SASREC_TRAIN, PREDICT, BERT_TRAIN, BERT_PREDICT = 0, 1, 2, 3
_INT32 = np.iinfo(np.int32)
# DEFAULT_GROUND_TRUTH_PADDING_VALUE / DEFAULT_TRAIN_PADDING_VALUE (torch_sequential_dataset.py:179-180); other query
# lists default to -1, which no item id, metric or seen filter takes for an item
QUERY_LIST_PADDING = {"ground_truth": -1, "train": -2}


class FeatureColumn:
    """One sequence feature of a ``DeviceSequenceStore`` on the store's device.  ``kind``: ``"int"``, ``"float"`` or
    ``"list"``; ``tail``: the per-event output shape (``()`` for a scalar, ``(dim,)`` for a vector, ``(K,)`` for a list);
    ``values``: the flat event values; ``list_offsets``: ``[n_events + 1]`` for a list column, else None."""

    def __init__(self, name, kind, values, tail, padding_value, list_offsets=None):
        self.name, self.kind, self.tail, self.list_offsets = name, kind, tuple(tail), list_offsets
        self.values = values
        self.padding_value = padding_value
        self.width = int(np.prod(self.tail)) if self.tail else 1


class QueryList:
    """One integer list per stored sequence of a ``DeviceSequenceStore``: ``offsets`` int64 ``[n_seq + 1]`` into
    ``values`` (int32 or int64) on the store's device; ``width``: the output width; ``padding_value``: the pad of both
    layouts."""

    def __init__(self, name, values, offsets, width, padding_value):
        self.name, self.values, self.offsets = name, values, offsets
        self.width, self.padding_value = int(width), int(padding_value)


def _make_query_list(name, values, lengths, n_seq, width, padding_value, device):
    """``values``: the lists concatenated; ``lengths``: entries per stored sequence.  ``width`` None: the longest list."""
    lengths = np.asarray(lengths, dtype=np.int64)
    if len(lengths) != n_seq:
        raise ValueError(f"query list {name!r}: {len(lengths)} lists, the store has {n_seq} sequences")
    if width is None:
        width = max(1, int(lengths.max())) if len(lengths) else 1
    if int(width) < 1:
        raise ValueError(f"query list {name!r}: width must be >= 1, got {width}")
    if padding_value is None:
        padding_value = QUERY_LIST_PADDING.get(name, -1)
    dev = torch.device(device)
    offs = np.zeros(n_seq + 1, dtype=np.int64)
    np.cumsum(lengths, out=offs[1:])
    t = torch.from_numpy(np.require(_narrow_int(values), requirements=["C", "W"])).to(dev)
    if t.numel() == 0:  # keep a valid pointer
        t = torch.zeros(1, dtype=t.dtype, device=dev)
    return QueryList(name, t, torch.from_numpy(offs).to(dev), width, padding_value)


def _query_list_from_sequences(name, lists, n_seq, width, padding_value, device):
    parts = []
    for x in lists:
        a = np.asarray(x)
        if a.ndim != 1 or (len(a) and a.dtype.kind not in "biu"):
            raise ValueError(f"query list {name!r}: every entry must be a 1-D integer array, got {a.dtype} {a.shape}")
        parts.append(a.astype(np.int64))
    values = np.concatenate(parts) if parts else np.zeros(0, np.int64)
    return _make_query_list(name, values, [len(a) for a in parts], n_seq, width, padding_value, device)


def _narrow_int(values: np.ndarray) -> np.ndarray:
    values = np.asarray(values, dtype=np.int64)
    if len(values) == 0 or (values.min() >= _INT32.min and values.max() <= _INT32.max):
        return values.astype(np.int32)
    return values


def _float_dtype(dtypes) -> np.dtype:
    return np.dtype(np.float64) if any(np.dtype(d) == np.float64 for d in dtypes) else np.dtype(np.float32)


def _make_column(name, kind, values, seq_lengths, item_lengths, padding_value, *, dim=None, event_lengths=None,
                 list_width=None, device="cuda"):
    """Checks one column against the item history and moves it to the device.  ``values``: flat event values (float
    vectors flattened row-major, list entries concatenated); ``seq_lengths``: events per sequence; ``event_lengths``: entries
    per event of a list column."""
    seq_lengths = np.asarray(seq_lengths, dtype=np.int64)
    if len(seq_lengths) != len(item_lengths) or np.any(seq_lengths != item_lengths):
        bad = np.flatnonzero(seq_lengths != item_lengths)[:1] if len(seq_lengths) == len(item_lengths) else []
        where = f" (sequence {int(bad[0])}: {int(seq_lengths[bad[0]])} events, {int(item_lengths[bad[0]])} items)" if len(bad) \
            else f" ({len(seq_lengths)} sequences, {len(item_lengths)} histories)"
        raise ValueError(f"feature {name!r}: per-sequence lengths differ from the item column's{where}")
    dev = torch.device(device)
    list_offsets = None
    if kind == "int":
        vals, tail = _narrow_int(values), ()
        pad = int(padding_value)
    elif kind == "float":
        vals = np.asarray(values)
        vals = vals.astype(_float_dtype([vals.dtype]))
        tail = () if dim is None else (int(dim),)
        pad = float(padding_value)
    else:
        k = list_width
        if k is None:
            k = max(1, int(np.max(event_lengths))) if len(event_lengths) else 1
        if int(k) < 1:
            raise ValueError(f"feature {name!r}: list width K must be >= 1, got {k}")
        vals, tail = _narrow_int(values), (int(k),)
        pad = int(padding_value)
        offs = np.zeros(len(event_lengths) + 1, dtype=np.int64)
        np.cumsum(event_lengths, out=offs[1:])
        list_offsets = torch.from_numpy(offs).to(dev)
    t = torch.from_numpy(np.require(vals, requirements=["C", "W"])).to(dev)
    if t.numel() == 0:  # keep a valid pointer
        t = torch.zeros(1, dtype=t.dtype, device=dev)
    return FeatureColumn(name, kind, t, tail, pad, list_offsets)


def _column_from_sequences(name, col, item_lengths, padding_value, list_width, device):
    """One raw column: a per-sequence list of 1-D integer / float arrays (scalars), ``[n, dim]`` float arrays (vectors)
    or lists of integer lists (lists; ``[n, k]`` integer arrays count as lists of k entries)."""
    if len(col) != len(item_lengths):
        raise ValueError(f"feature {name!r}: {len(col)} sequences, the store has {len(item_lengths)}")
    seq_lengths, parts, nested = [], [], False
    for x in col:
        try:
            a = np.asarray(x)
        except ValueError:  # ragged nested lists
            a = None
        if a is None or a.dtype == object:
            nested = True
            a = list(x)
        seq_lengths.append(len(a))
        parts.append(a)
    if not nested:
        live = [a for a in parts if len(a)]
        kinds = {a.dtype.kind for a in live}
        if kinds - set("biuf"):
            raise ValueError(f"feature {name!r}: unsupported dtype {sorted(kinds)}")
        ndims = {a.ndim for a in live}
        if len(ndims) > 1 or (ndims and ndims.pop() > 2):
            raise ValueError(f"feature {name!r}: events must all be scalars or all be vectors")
        two_d = bool(live) and live[0].ndim == 2
        is_float = "f" in kinds
        if not two_d:
            values = np.concatenate(live) if live else np.zeros(0, np.float32 if is_float else np.int64)
            if is_float:
                values = values.astype(_float_dtype(a.dtype for a in live if a.dtype.kind == "f"))
                return _make_column(name, "float", values, seq_lengths, item_lengths, padding_value, device=device)
            return _make_column(name, "int", values.astype(np.int64), seq_lengths, item_lengths, padding_value,
                                device=device)
        dims = {a.shape[1] for a in live}
        if is_float:
            if len(dims) > 1:
                raise ValueError(f"feature {name!r}: ragged vectors (dims {sorted(dims)})")
            values = np.concatenate([a.reshape(-1) for a in live])
            values = values.astype(_float_dtype(a.dtype for a in live if a.dtype.kind == "f"))
            return _make_column(name, "float", values, seq_lengths, item_lengths, padding_value, dim=dims.pop(),
                                device=device)
        ev_len = np.concatenate([np.full(len(a), a.shape[1], np.int64) for a in live])
        return _make_column(name, "list", np.concatenate([a.reshape(-1) for a in live]), seq_lengths, item_lengths,
                            padding_value, event_lengths=ev_len, list_width=list_width, device=device)
    # nested: one list per event
    ev_len, flat, is_float, scalar_events = [], [], False, False
    for a in parts:
        for e in a:
            ev = None if e is None else np.asarray(e)
            if ev is None or ev.dtype == object:
                raise ValueError(f"feature {name!r} holds null values")
            if ev.ndim != 1:
                scalar_events = True
                continue
            if len(ev) and ev.dtype.kind not in "biuf":
                raise ValueError(f"feature {name!r}: unsupported dtype {ev.dtype}")
            is_float |= len(ev) > 0 and ev.dtype.kind == "f"
            ev_len.append(len(ev))
            flat.append(ev)
    if scalar_events:
        raise ValueError(f"feature {name!r}: mixes scalar and list events")
    ev_len = np.asarray(ev_len, dtype=np.int64)
    if is_float:
        if len(set(ev_len.tolist())) > 1:
            raise ValueError(f"feature {name!r}: ragged vectors (dims {sorted(set(ev_len.tolist()))})")
        values = np.concatenate(flat).astype(_float_dtype(f.dtype for f in flat if len(f)))
        return _make_column(name, "float", values, seq_lengths, item_lengths, padding_value, dim=int(ev_len[0]),
                            device=device)
    values = np.concatenate(flat).astype(np.int64) if flat else np.zeros(0, np.int64)
    return _make_column(name, "list", values, seq_lengths, item_lengths, padding_value, event_lengths=ev_len,
                        list_width=list_width, device=device)


def _column_from_arrow(name, col, item_lengths, padding_value, list_width, device):
    """A ``list<T>`` (scalars) or ``list<list<T>>`` / ``list<fixed_size_list<T>>`` (float vectors, integer lists) arrow
    column, read with pyarrow compute: null rows count as empty like the item column's, null events or values raise."""
    import pyarrow as pa
    import pyarrow.compute as pc

    if not (pa.types.is_list(col.type) or pa.types.is_large_list(col.type)):
        raise ValueError(f"column {name!r} must be a list column, got {col.type}")
    seq_lengths = pc.fill_null(pc.list_value_length(col), 0).to_numpy(zero_copy_only=False).astype(np.int64)
    events = pc.list_flatten(col)
    if events.null_count:
        raise ValueError(f"column {name!r} holds null values")
    t = events.type
    nested = pa.types.is_list(t) or pa.types.is_large_list(t) or pa.types.is_fixed_size_list(t)
    if nested:
        ev_len = pc.list_value_length(events).to_numpy(zero_copy_only=False).astype(np.int64)
        values = pc.list_flatten(events)
        t = values.type
    else:
        values = events
    if values.null_count:
        raise ValueError(f"column {name!r} holds null values")
    if not (pa.types.is_integer(t) or pa.types.is_floating(t)):
        raise ValueError(f"column {name!r}: unsupported value type {t}")
    vals = values.to_numpy(zero_copy_only=False)
    if pa.types.is_floating(t):
        vals = vals.astype(_float_dtype([vals.dtype]))
        dim = None
        if nested:
            dims = np.unique(ev_len)
            if len(dims) > 1:
                raise ValueError(f"column {name!r}: ragged vectors (dims {dims.tolist()})")
            dim = int(dims[0]) if len(dims) else (events.type.list_size if pa.types.is_fixed_size_list(events.type) else 1)
        return _make_column(name, "float", vals, seq_lengths, item_lengths, padding_value, dim=dim, device=device)
    if nested:
        return _make_column(name, "list", vals, seq_lengths, item_lengths, padding_value, event_lengths=ev_len,
                            list_width=list_width, device=device)
    return _make_column(name, "int", vals, seq_lengths, item_lengths, padding_value, device=device)


def _check_validation_datasets(sequential, given, label_feature_name):
    """TorchSequentialValidationDataset.__init__ / _check_if_schema_match (torch_sequential_dataset.py:211-233,
    288-302), with its messages."""
    seq_item = sequential.schema.item_id_features.item()
    for ds in given.values():
        other = ds.schema.item_id_features.item()
        if seq_item.name != other.name:
            raise ValueError("Schema mismatch: item feature name does not match ground truth")
        if seq_item.cardinality != other.cardinality:
            raise ValueError("Schema mismatch: item feature cardinality does not match ground truth")
    gt = given.get("ground_truth")
    if label_feature_name:
        for k, ds in given.items():
            if label_feature_name not in dict(ds.schema.items()):
                raise ValueError(f"Label feature name not found in {k.replace('_', ' ')} schema")
        if gt is not None:
            if not gt.schema[label_feature_name].is_cat:
                raise ValueError("Label feature must be categorical")
            if not gt.schema[label_feature_name].is_seq:
                raise ValueError("Label feature must be sequential")
    if gt is not None and len(np.intersect1d(sequential.get_all_query_ids(), gt.get_all_query_ids())) == 0:
        raise ValueError("Sequential data and ground truth must contain the same query IDs")


def _join_by_query_id(ds, query_ids, label):
    """The label sequence of every query id in ``ds`` (empty when absent), looked up once per dataset row."""
    row = {q: i for i, q in enumerate(np.asarray(ds.get_all_query_ids()).tolist())}
    empty = np.zeros(0, np.int64)
    return [np.asarray(ds.get_sequence(row[q], label)) if q in row else empty
            for q in np.asarray(query_ids).tolist()]


def window_index(lengths, window: int, sliding_window_step: int | None = None):
    """(sequence_index int32 [n], offset int32 [n]) in the reference's iteration order
    (TorchSequentialDataset._iter_with_window, torch_sequential_dataset.py:154-171), vectorised: without a step one
    window per history at offset max(0, len - window); with a step the offsets len-window, len-window-step, ... (> 0)
    followed by 0."""
    lengths = np.asarray(lengths, dtype=np.int64)
    left = lengths - window
    if sliding_window_step is None:
        return np.arange(len(lengths), dtype=np.int32), np.maximum(left, 0).astype(np.int32)
    step = int(sliding_window_step)
    if step <= 0:
        raise ValueError("sliding_window_step must be positive")
    extra = np.where(left > 0, (left + step - 1) // step, 0)  # windows with a positive offset
    counts = extra + 1
    seq = np.repeat(np.arange(len(lengths), dtype=np.int64), counts)
    starts = np.cumsum(counts) - counts
    k = np.arange(counts.sum(), dtype=np.int64) - np.repeat(starts, counts)  # 0.. within one history
    off = np.repeat(left, counts) - k * step
    off = np.where(k == np.repeat(extra, counts), 0, off)  # the closing (i, 0) window
    return seq.astype(np.int32), off.astype(np.int32)


class DeviceSequenceStore:
    """CSR store of item-id histories in HBM.  ``sequences``: list of 1-D integer arrays (one per query, item ids already
    label-encoded to 0..|I|-1 as the reference's SequenceTokenizer does), or pass ``offsets``/``items`` directly.

    ``features``: ``{name: column}``, each column one entry per sequence with one entry per event of that sequence: a
    1-D integer or float array (scalars), an ``[n, dim]`` float array or list of equal-length float lists (vectors), or a
    list of integer lists of any length (lists).  ``padding_values``: ``{name: value}`` (default 0); ``list_widths``:
    ``{name: K}``, the output width of a list column (default: its longest list).

    ``query_lists``: ``{name: lists}``, one 1-D integer array per sequence (e.g. ``ground_truth`` and ``train``), emitted
    by the validation builders.  ``padding_values`` / ``list_widths`` apply to them too; their padding defaults to -1 for
    ``ground_truth``, -2 for ``train`` (the reference's) and -1 otherwise, their width to the longest list.

    ValueError for a column whose per-sequence lengths differ from the item column's, ragged vectors, null values,
    ``K < 1``, a query list whose count differs from the store's, or more than ``BATCH_MAX_COLUMNS`` (16) feature columns
    and query lists together."""

    def __init__(self, sequences=None, *, offsets=None, items=None, query_ids=None, device="cuda", features=None,
                 padding_values=None, list_widths=None, query_lists=None):
        if sequences is not None:
            lens = np.fromiter((len(s) for s in sequences), dtype=np.int64, count=len(sequences))
            offsets = np.zeros(len(lens) + 1, dtype=np.int64)
            np.cumsum(lens, out=offsets[1:])
            items = np.concatenate([np.asarray(s, dtype=np.int64) for s in sequences]) if len(lens) else np.zeros(0, np.int64)
        offsets = np.asarray(offsets, dtype=np.int64)
        items = np.asarray(items)
        if offsets.ndim != 1 or len(offsets) < 2 or offsets[0] != 0 or offsets[-1] != len(items) or np.any(np.diff(offsets) < 0):
            raise ValueError("offsets must be a non-decreasing CSR row pointer starting at 0 and ending at len(items)")
        if len(items) and (items.min() < 0 or items.max() >= 2 ** 31 - 1):
            raise ValueError("item ids must fit int32")
        self.device = torch.device(device)
        self.lengths = np.diff(offsets)
        self.n_seq = len(self.lengths)
        self.offsets = torch.from_numpy(np.array(offsets, dtype=np.int64)).to(self.device)
        self.items = torch.from_numpy(items.astype(np.int32)).to(self.device)
        if len(items) == 0:  # keep a valid pointer
            self.items = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.query_ids = None if query_ids is None else torch.from_numpy(np.array(query_ids, dtype=np.int64)).to(self.device)
        features, query_lists = dict(features or {}), dict(query_lists or {})
        self._check_column_count(len(features) + len(query_lists))
        both = set(features) & set(query_lists)
        if both:
            raise ValueError(f"{sorted(both)} are both feature columns and query lists")
        padding_values, list_widths = dict(padding_values or {}), dict(list_widths or {})
        self.columns = [c if isinstance(c, FeatureColumn) else
                        _column_from_sequences(n, c, self.lengths, padding_values.get(n, 0), list_widths.get(n), self.device)
                        for n, c in features.items()]
        self.query_lists = [c if isinstance(c, QueryList) else
                            _query_list_from_sequences(n, c, self.n_seq, list_widths.get(n), padding_values.get(n),
                                                       self.device)
                            for n, c in query_lists.items()]

    @staticmethod
    def _check_column_count(n):
        if n > BATCH_MAX_COLUMNS:
            raise ValueError(f"{n} feature columns and query lists: one batch launch takes at most {BATCH_MAX_COLUMNS}")

    @property
    def feature_names(self):
        return [c.name for c in self.columns]

    @property
    def query_list_names(self):
        return [c.name for c in self.query_lists]

    @classmethod
    def from_sequential_dataset(cls, sequential, feature_name: str | None = None, device="cuda", list_widths=None,
                                ground_truth=None, train=None, label_feature_name: str | None = None):
        """Duck-typed ``SequentialDataset`` (replay/data/nn/sequential_dataset.py:18-105): ``__len__``, ``get_query_id``,
        ``get_sequence`` and ``schema``.  Every other ``is_seq`` feature of the schema becomes a feature column with the
        schema's ``padding_value``; per-query (non-sequential) features are not model inputs and are not read.

        ``ground_truth`` / ``train``: the validation datasets of ``TorchSequentialValidationDataset``
        (torch_sequential_dataset.py:183-285), joined by query id once, here: each stored query gets the label feature's
        sequence of its query id as the query list ``ground_truth`` / ``train`` (an empty list when the id is absent, as
        ``get_sequence_by_query_id`` gives), padded -1 / -2 to the dataset's ``get_max_sequence_length()``.  ValueError,
        with the reference's messages, for an item feature whose name or cardinality differs from ``sequential``'s, a
        label feature missing from either schema or not categorical and sequential, and no query id shared with
        ``ground_truth``."""
        schema = sequential.schema
        name = feature_name or schema.item_id_feature_name
        n = len(sequential)
        side = [(k, f) for k, f in schema.items() if k != name and getattr(f, "is_seq", True)]
        qids = [sequential.get_query_id(i) for i in range(n)]
        lists, widths = {}, dict(list_widths or {})
        given = {k: v for k, v in (("ground_truth", ground_truth), ("train", train)) if v is not None}
        if given:
            _check_validation_datasets(sequential, given, label_feature_name)
            label = label_feature_name or next(iter(given.values())).schema.item_id_feature_name
            for k, ds in given.items():
                lists[k] = _join_by_query_id(ds, qids, label)
                widths[k] = int(ds.get_max_sequence_length())
        return cls([np.asarray(sequential.get_sequence(i, name)) for i in range(n)], query_ids=qids, device=device,
                   features={k: [sequential.get_sequence(i, k) for i in range(n)] for k, _ in side},
                   padding_values={k: getattr(f, "padding_value", 0) for k, f in side}, list_widths=widths,
                   query_lists=lists)

    @classmethod
    def from_parquet(cls, source, item_column: str = "item_id", query_column: str | None = None, device="cuda",
                     feature_columns=(), padding_values=None, list_widths=None, query_list_columns=()):
        """Sequence-per-row parquet (the layout the reference's ParquetDataset / ParquetModule reads: one row per query, the
        item ids in a list<int> column; replay/data/nn/parquet/impl/array_1d_column.py:87-140): the list column's offsets and
        flat values become the CSR store without a Python loop (null lists count as empty).  ``source``: a path, a list of
        paths or a ``pyarrow.Table``.  ``feature_columns``: ``list<T>`` (scalars) and ``list<list<T>>`` (float vectors,
        integer lists) columns read the same way, with ``padding_values`` / ``list_widths`` as in the constructor.
        ``query_list_columns``: ``list<int>`` columns held as query lists (one list per row: ground truth, train or seen
        items), with the width and padding of the reader's metadata given in ``list_widths`` / ``padding_values``."""
        import pyarrow as pa
        import pyarrow.compute as pc
        import pyarrow.parquet as pq

        feature_columns, query_list_columns = list(feature_columns), list(query_list_columns)
        cls._check_column_count(len(feature_columns) + len(query_list_columns))
        cols = [item_column] + ([query_column] if query_column else []) + feature_columns + query_list_columns
        if isinstance(source, pa.Table):
            table = source.select(cols)
        elif isinstance(source, (list, tuple)):
            table = pa.concat_tables([pq.read_table(p, columns=cols) for p in source])
        else:
            table = pq.read_table(source, columns=cols)
        col = table.column(item_column).combine_chunks()
        if not (pa.types.is_list(col.type) or pa.types.is_large_list(col.type)):
            raise ValueError(f"column {item_column!r} must be a list column, got {col.type}")
        lengths = pc.fill_null(pc.list_value_length(col), 0).to_numpy(zero_copy_only=False).astype(np.int64)
        values = pc.list_flatten(col)
        if values.null_count:
            raise ValueError(f"column {item_column!r} holds null item ids")
        offsets = np.zeros(len(lengths) + 1, dtype=np.int64)
        np.cumsum(lengths, out=offsets[1:])
        q = table.column(query_column).combine_chunks().to_numpy(zero_copy_only=False) if query_column else None
        padding_values, list_widths = dict(padding_values or {}), dict(list_widths or {})
        feats = {n: _column_from_arrow(n, table.column(n).combine_chunks(), lengths, padding_values.get(n, 0),
                                       list_widths.get(n), device) for n in feature_columns}
        lists = {}
        for n in query_list_columns:
            c = table.column(n).combine_chunks()
            if not ((pa.types.is_list(c.type) or pa.types.is_large_list(c.type)) and pa.types.is_integer(c.type.value_type)):
                raise ValueError(f"query list column {n!r} must be a list<int> column, got {c.type}")
            flat = pc.list_flatten(c)
            if flat.null_count:
                raise ValueError(f"query list column {n!r} holds null values")
            lists[n] = _make_query_list(n, flat.to_numpy(zero_copy_only=False),
                                        pc.fill_null(pc.list_value_length(c), 0).to_numpy(zero_copy_only=False),
                                        len(lengths), list_widths.get(n), padding_values.get(n), device)
        return cls(offsets=offsets, items=values.to_numpy(zero_copy_only=False), query_ids=q, device=device, features=feats,
                   query_lists=lists)

    def __len__(self):
        return self.n_seq

    # --------------------------------------------------------------------------------------------- batch builders
    def _build(self, mode, seq_index, seq_offset, L, pad_value, *, mask_prob=0.0, uniforms=None, seed=0, draw0=0,
               with_labels=False, with_aux=False, new_path=False, feature_name="item_id", query_layout=None):
        """ids, pad, labels, aux, query [B, 1], ``{name: tensor}`` of the feature columns and ``{name: [B, width]}`` of the
        query lists (empty unless ``query_layout`` is ``"first"`` (legacy) or ``"last"`` (new path)).  With neither, the
        item-only launch runs."""
        dev = self.device
        seq_index = torch.as_tensor(seq_index, device=dev).to(torch.int32).contiguous()
        B = seq_index.numel()
        if seq_offset is not None:
            seq_offset = torch.as_tensor(seq_offset, device=dev).to(torch.int32).contiguous()
            if seq_offset.numel() != B:
                raise ValueError("seq_offset must have one entry per batch row")
        ids = torch.empty(B, L, dtype=torch.int64, device=dev)
        pad = torch.empty(B, L, dtype=torch.bool, device=dev)
        labels = torch.empty(B, L, dtype=torch.int64, device=dev) if with_labels else None
        aux = torch.empty(B, L, dtype=torch.bool, device=dev) if with_aux else None
        q = torch.empty(B, dtype=torch.int64, device=dev)
        if uniforms is not None:
            uniforms = torch.as_tensor(uniforms, device=dev, dtype=torch.float32).contiguous()
            if tuple(uniforms.shape) != (B, L):
                raise ValueError("uniforms must be [B, L]")
        p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        args = (self.offsets.data_ptr(), self.items.data_ptr(), self.n_seq, seq_index.data_ptr(), p(seq_offset), B, L, mode,
                int(pad_value), float(mask_prob), p(uniforms), int(seed), int(draw0), p(self.query_ids), ids.data_ptr(),
                pad.data_ptr(), p(labels), p(aux), q.data_ptr())
        stream = torch.cuda.current_stream().cuda_stream
        if not self.columns and query_layout is None:
            check(lib().rp_build_batch(*args, stream), "rp_build_batch")
            return ids, pad, labels, aux, q.view(-1, 1), {}, {}
        feats, desc = self._feature_outputs(B, L, new_path, feature_name)
        lists, ldesc = self._query_list_outputs(B, query_layout)
        desc = (BatchColumn * (len(desc) + len(ldesc)))(*desc, *ldesc)
        check(lib().rp_build_batch_features(*args, desc, len(desc), stream), "rp_build_batch_features")
        return ids, pad, labels, aux, q.view(-1, 1), feats, lists

    def _query_list_outputs(self, B, layout):
        if layout is None:
            return {}, []
        kind = {"first": BATCH_COL_QUERY_LIST, "last": BATCH_COL_QUERY_LIST_LAST}[layout]
        lists, desc = {}, []
        for c in self.query_lists:
            out = lists[c.name] = torch.empty(B, c.width, dtype=torch.int64, device=self.device)
            desc.append(BatchColumn(kind=kind, in_bytes=c.values.element_size(), out_bytes=8, width=c.width,
                                    values=c.values.data_ptr(), list_offsets=c.offsets.data_ptr(), out=out.data_ptr(),
                                    pad_int=c.padding_value))
        return lists, desc

    def _feature_outputs(self, B, L, new_path, feature_name):
        if feature_name in self.feature_names:
            raise ValueError(f"feature column {feature_name!r} has the item feature's name")
        if not new_path:
            lists = [c.name for c in self.columns if c.kind == "list"]
            if lists:
                raise ValueError(f"list features {lists} need the new-path builders: the legacy datasets stack one tensor "
                                 "per feature and cannot stack ragged lists")
        feats, desc = {}, (BatchColumn * len(self.columns))()
        for c, d in zip(self.columns, desc):
            if c.kind == "float":
                dt = c.values.dtype if new_path else torch.float32
            else:
                dt = torch.int64
            out = torch.empty((B, L, *c.tail), dtype=dt, device=self.device)
            feats[c.name] = out
            d.kind = {"int": BATCH_COL_INT, "float": BATCH_COL_FLOAT, "list": BATCH_COL_LIST}[c.kind]
            d.in_bytes, d.out_bytes, d.width = c.values.element_size(), out.element_size(), c.width
            d.values, d.out = c.values.data_ptr(), out.data_ptr()
            d.list_offsets = None if c.list_offsets is None else c.list_offsets.data_ptr()
            if c.kind == "float":
                d.pad_float = float(c.padding_value)
            else:
                d.pad_int = int(c.padding_value)
        return feats, desc

    def sasrec_training_batch(self, seq_index, max_len: int, pad_value: int, seq_offset=None, feature_name="item_id"):
        """Reference keys (sasrec/dataset.py:120-126): query_id [B,1], feature_tensor{item_id [B,L], features...},
        padding_mask, positive_labels, target_padding_mask - all on the device."""
        ids, pad, labels, tmask, q, feats, _ = self._build(SASREC_TRAIN, seq_index, seq_offset, max_len, pad_value,
                                                        with_labels=True, with_aux=True, feature_name=feature_name)
        return {"query_id": q, "feature_tensor": {feature_name: ids, **feats}, "padding_mask": pad, "positive_labels": labels,
                "target_padding_mask": tmask}

    def sasrec_new_path_batch(self, seq_index, max_len: int, pad_value: int, feature_name="item_id", with_seen: bool = True,
                              seq_offset=None):
        """The new path's model inputs: Array1DColumn.__getitem__ with shape max_len + 1 (left-padded gather of the last
        elements, parquet/impl/indexing.py:42-78; Array2DColumn.__getitem__ for lists, array_2d_column.py:72-92) +
        NextTokenTransform(shift=1) (nn/transform/next_token.py:65-96) + the unsqueeze of the default SASRec transform
        template -> feature_tensors{item_id, features...}, padding_mask, positive_labels [B,L,1], target_padding_mask
        [B,L,1] (+ seen_ids = the window).  ``seq_offset``: window starts (default: the last L + 1 events)."""
        ids, pad, labels, tmask, q, feats, _ = self._build(SASREC_TRAIN, seq_index, seq_offset, max_len, pad_value,
                                                        with_labels=True, with_aux=True, new_path=True,
                                                        feature_name=feature_name)
        out = {"query_id": q, "feature_tensors": {feature_name: ids, **feats}, "padding_mask": pad,
               "positive_labels": labels.unsqueeze(-1), "target_padding_mask": tmask.unsqueeze(-1)}
        if with_seen:
            out["seen_ids"] = ids
        return out

    def sasrec_new_path_prediction_batch(self, seq_index, max_len: int, pad_value: int, feature_name="item_id",
                                         with_seen: bool = True):
        """The predict transforms of the default SASRec template (nn/transform/template/sasrec.py): every column read at
        max_len (the last events, left-padded), no shift -> query_id, feature_tensors{item_id, features...}, padding_mask
        (+ seen_ids = the window)."""
        ids, pad, _, _, q, feats, _ = self._build(PREDICT, seq_index, None, max_len, pad_value, new_path=True,
                                               feature_name=feature_name)
        out = {"query_id": q, "feature_tensors": {feature_name: ids, **feats}, "padding_mask": pad}
        if with_seen:
            out["seen_ids"] = ids
        return out

    def sasrec_prediction_batch(self, seq_index, max_len: int, pad_value: int, feature_name="item_id"):
        ids, pad, _, _, q, feats, _ = self._build(PREDICT, seq_index, None, max_len, pad_value, feature_name=feature_name)
        return {"query_id": q, "padding_mask": pad, "feature_tensor": {feature_name: ids, **feats}}

    def bert4rec_training_batch(self, seq_index, max_len: int, pad_value: int, mask_prob: float = 0.15, seq_offset=None,
                                seed: int = 0, draw0: int = 0, uniforms=None, feature_name="item_id"):
        """Reference keys (bert4rec/dataset.py:167-173), the feature columns unmasked under ``inputs``.  ``token_mask``
        False = masked.  Random draws: Philox keyed by (seed, draw0 + row); pass ``uniforms`` [B, L] to reproduce a given
        masker stream exactly."""
        ids, pad, labels, tok, q, feats, _ = self._build(BERT_TRAIN, seq_index, seq_offset, max_len, pad_value,
                                                      mask_prob=mask_prob, uniforms=uniforms, seed=seed, draw0=draw0,
                                                      with_labels=True, with_aux=True, feature_name=feature_name)
        return {"query_id": q, "pad_mask": pad, "inputs": {feature_name: ids, **feats}, "token_mask": tok,
                "positive_labels": labels}

    def bert4rec_prediction_batch(self, seq_index, max_len: int, pad_value: int, feature_name="item_id"):
        """_shift_features (bert4rec/dataset.py:322-351): every column shifted left, its padding value in the last slot."""
        ids, pad, _, tok, q, feats, _ = self._build(BERT_PREDICT, seq_index, None, max_len, pad_value, with_aux=True,
                                                 feature_name=feature_name)
        return {"query_id": q, "pad_mask": pad, "inputs": {feature_name: ids, **feats}, "token_mask": tok}

    # ------------------------------------------------------------------------------------ validation / test builders
    def _legacy_lists(self, lists):
        missing = [k for k in ("ground_truth", "train") if k not in lists]
        if missing:
            raise ValueError(f"the legacy validation batches need the query lists 'ground_truth' and 'train'; the store "
                             f"lacks {missing}")
        return lists

    def sasrec_validation_batch(self, seq_index, max_len: int, pad_value: int, feature_name="item_id"):
        """SasRecValidationDataset.__getitem__ + default collate (sasrec/dataset.py:218-268): the prediction window and
        every query list, first entries right-padded -> query_id, padding_mask, feature_tensor, ground_truth, train."""
        ids, pad, _, _, q, feats, lists = self._build(PREDICT, seq_index, None, max_len, pad_value,
                                                      feature_name=feature_name, query_layout="first")
        return {"query_id": q, "padding_mask": pad, "feature_tensor": {feature_name: ids, **feats},
                **self._legacy_lists(lists)}

    def bert4rec_validation_batch(self, seq_index, max_len: int, pad_value: int, feature_name="item_id"):
        """Bert4RecValidationDataset.__getitem__ + default collate (bert4rec/dataset.py:264-320): the shifted prediction
        window and every query list, first entries right-padded -> query_id, pad_mask, inputs, token_mask, ground_truth,
        train."""
        ids, pad, _, tok, q, feats, lists = self._build(BERT_PREDICT, seq_index, None, max_len, pad_value, with_aux=True,
                                                        feature_name=feature_name, query_layout="first")
        return {"query_id": q, "pad_mask": pad, "inputs": {feature_name: ids, **feats}, "token_mask": tok,
                **self._legacy_lists(lists)}

    def sasrec_new_path_validation_batch(self, seq_index, max_len: int, pad_value: int, feature_name="item_id",
                                         seen_list: str | None = "train"):
        """The validate / test transforms of the default SASRec template (nn/transform/template/sasrec.py:27-31) on the
        columns the reader cuts at their metadata's shape: every column read at max_len, no shift, and every query list's
        last ``width`` entries left-padded -> query_id [B] (the reader's query column), feature_tensors, padding_mask,
        the query lists under their names
        and ``seen_ids`` for ``SeenItemsFilter``: the query list named ``seen_ids`` when the store has one, else the
        list ``seen_list`` (None: the window, as the prediction batch)."""
        ids, pad, _, _, q, feats, lists = self._build(PREDICT, seq_index, None, max_len, pad_value, new_path=True,
                                                      feature_name=feature_name, query_layout="last")
        out = {"query_id": q.view(-1), "feature_tensors": {feature_name: ids, **feats}, "padding_mask": pad, **lists}
        if "seen_ids" not in out:
            if seen_list is not None and seen_list not in lists:
                raise ValueError(f"seen_list {seen_list!r} is not a query list of the store {self.query_list_names}")
            out["seen_ids"] = ids if seen_list is None else lists[seen_list]
        return out


VALIDATION_KINDS = ("sasrec_validate", "bert4rec_validate", "sasrec_new_validate")


class DeviceBatchLoader:
    """Iterates device-built training batches the way ``DataLoader(SasRecTrainingDataset(...), shuffle=True)`` +
    ``DistributedSampler`` would: the window index is built once (host, vectorised), permuted per epoch with a seeded
    generator shared by all ranks, padded by wrap-around to a multiple of the world size (DistributedSampler semantics) and
    strided over the ranks; every batch is then one kernel launch on HBM-resident data.  ``kind``: ``"sasrec"`` (the
    legacy SasRec's batches), ``"sasrec_new"`` (new-path training batches for ``LightningModule(SasRec | TwoTower)``) or
    ``"bert4rec"``.

    The validation / test kinds ``"sasrec_validate"``, ``"bert4rec_validate"`` and ``"sasrec_new_validate"`` yield the
    store's validation batches instead: every stored query exactly once, in store order, the last batch kept partial.
    Under ``world_size > 1`` each rank takes its contiguous shard of ``trainer.user_shard``, so the ranks together visit
    every query once with no wrap-around duplicates; ``shuffle``, ``drop_last``, ``sliding_window_step`` and
    ``partitioning`` do not apply."""

    def __init__(self, store: DeviceSequenceStore, max_len: int, batch_size: int, pad_value: int, kind: str = "sasrec",
                 sliding_window_step: int | None = None, shuffle: bool = True, drop_last: bool = False, seed: int = 0,
                 rank: int = 0, world_size: int = 1, mask_prob: float = 0.15, partitioning: str = "sampler"):
        if kind not in ("sasrec", "sasrec_new", "bert4rec") + VALIDATION_KINDS:
            raise ValueError(f"unknown kind {kind!r}")
        if partitioning not in ("sampler", "replay"):
            raise ValueError(f"unknown partitioning {partitioning!r}")
        self.partitioning = partitioning
        self.store, self.L, self.bs, self.pad, self.kind = store, int(max_len), int(batch_size), int(pad_value), kind
        self.rank, self.world, self.epoch = rank, world_size, 0
        if kind in VALIDATION_KINDS:
            from .trainer import user_shard

            self.lo, hi = user_shard(store.n_seq, rank, world_size)
            self.n = self.per_rank = hi - self.lo
            self.drop_last = False
            return
        window = self.L + (1 if kind in ("sasrec", "sasrec_new") else 0)
        seq, off = window_index(store.lengths, window, sliding_window_step)
        self.win_seq = torch.from_numpy(seq).to(store.device)
        self.win_off = torch.from_numpy(off).to(store.device)
        self.n = len(seq)
        self.shuffle, self.drop_last, self.seed, self.rank, self.world = shuffle, drop_last, int(seed), rank, world_size
        self.mask_prob = float(mask_prob)
        self.epoch = 0
        self.per_rank = -(-self.n // world_size)

    def set_epoch(self, epoch: int):
        self.epoch = int(epoch)

    def __len__(self):
        return self.per_rank // self.bs if self.drop_last else -(-self.per_rank // self.bs)

    def epoch_indices(self) -> torch.Tensor:
        """This rank's window indices for the current epoch (on the store's device): seeded permutation shared by all ranks,
        wrap-around padding to a multiple of the world size, strided over the ranks (DistributedSampler semantics).
        ``partitioning="replay"``: the reference parquet reader's assignment instead (``replay_b200.data.replica_partition`` =
        ``Partitioning.generate``, replay/data/nn/parquet/info/partitioning.py:64-122: permutation of the PADDED range, modulo)."""
        dev = self.store.device
        if getattr(self, "partitioning", "sampler") == "replay":
            from .data import replica_partition

            g = torch.Generator(device="cpu").manual_seed(self.seed + self.epoch) if self.shuffle else None
            return replica_partition(self.n, self.rank, self.world, generator=g, device=dev)
        if self.shuffle:
            g = torch.Generator(device="cpu").manual_seed(self.seed + self.epoch)
            order = torch.randperm(self.n, generator=g).to(dev)
        else:
            order = torch.arange(self.n, device=dev)
        total = self.per_rank * self.world
        if total > self.n:  # wrap-around padding
            order = torch.cat([order, order[: total - self.n]])
        return order[self.rank: total: self.world]

    def __iter__(self):
        if self.kind in VALIDATION_KINDS:
            build = {"sasrec_validate": self.store.sasrec_validation_batch,
                     "bert4rec_validate": self.store.bert4rec_validation_batch,
                     "sasrec_new_validate": self.store.sasrec_new_path_validation_batch}[self.kind]
            for i in range(len(self)):
                lo = self.lo + i * self.bs
                s = torch.arange(lo, min(lo + self.bs, self.lo + self.n), dtype=torch.int32, device=self.store.device)
                yield build(s, self.L, self.pad)
            return
        mine = self.epoch_indices()
        for i in range(len(self)):
            idx = mine[i * self.bs: (i + 1) * self.bs]
            s, o = self.win_seq[idx], self.win_off[idx]
            if self.kind == "sasrec":
                yield self.store.sasrec_training_batch(s, self.L, self.pad, seq_offset=o)
            elif self.kind == "sasrec_new":
                yield self.store.sasrec_new_path_batch(s, self.L, self.pad, seq_offset=o)
            else:
                draw0 = (self.epoch * self.per_rank * self.world) + self.rank * self.per_rank + i * self.bs
                yield self.store.bert4rec_training_batch(s, self.L, self.pad, self.mask_prob, seq_offset=o,
                                                         seed=self.seed, draw0=draw0)
