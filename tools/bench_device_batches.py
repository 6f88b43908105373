"""Cost of producing training batches with sequence features: the device sequence store against host-built batches.

    python tools/bench_device_batches.py [--iters N] [--steps S] [--rounds R]

Config 2 shape: 512 windows of L 200 from 20 000 synthetic histories (lognormal lengths, 2 .. 2000 events), |I| 50 K.
Features as in tools/bench_side_features.py: two categoricals (|C| 1 K and 20), a categorical list of width 4 (lists of
0 .. 8 entries), a numerical feature of tensor_dim 8; and, for TiSASRec, int64 timestamps.

1. Build time per batch (CUDA events around ``--iters`` builds, after a warm-up):
   * the item-only store and the feature store (new-path training batches; the legacy TiSASRec batch with timestamps);
   * the per-sample host path of the reference's legacy datasets (one torch.tensor per feature per sample, left-padding,
     default collate, H2D copy), for the features it can stack (no list) and for TiSASRec's timestamps;
   * the new path's torch-op column gathers on the same GPU (the left-padded gather of indexing.get_mask with its host
     checks, the 2-D gather of Array2DColumn for the list and the vector, then the NextToken slice).
2. Bandwidth of the store's launch: the bytes it has to move (the windows' live values and list entries read, every output
   written) over its build time, as a share of the H100 SXM's 3.35 TB/s.
3. End to end: training sequences/s of the side-feature SasRec (new path, LightningModule) and of TiSASRec (legacy SasRec,
   ti_modification=True), fed by the store, by batches built on the host every step, and by pre-built pinned host batches
   copied each step; the three feeds alternate for ``--rounds`` rounds and the median is reported.
The card's name, power limit and max SM clock are printed first and stored in the JSON line printed last."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from torch.utils.data import default_collate

from replay_b200.device_data import DeviceSequenceStore

B, L, D, H, I, U = 512, 200, 128, 2, 50_000, 20_000
PADS = {"c1": 1000, "c2": 20, "tags": 30, "num": 0, "timestamp": 0}
HBM_BYTES_PER_S = 3.35e12


def histories(seed=0):
    rng = np.random.default_rng(seed)
    lens = np.clip(np.round(np.exp(rng.normal(4.6, 1.0, U))), 2, 2000).astype(np.int64)
    seqs = [rng.integers(0, I, n) for n in lens]
    n_ev = int(lens.sum())
    tag_len = rng.integers(0, 9, n_ev)
    flat = {"c1": rng.integers(0, 1000, n_ev), "c2": rng.integers(0, 20, n_ev),
            "num": rng.normal(0, 1, (n_ev, 8)).astype(np.float32),
            "timestamp": 1_600_000_000 + np.cumsum(rng.integers(0, 3600, n_ev)),
            "tags_len": tag_len, "tags": rng.integers(0, 30, int(tag_len.sum()))}
    return lens, seqs, flat


def per_seq(lens, flat):
    """The flat scalar and vector columns cut back into per-sequence arrays (what the legacy per-sample path reads)."""
    off = np.concatenate([[0], np.cumsum(lens)])
    cols = {k: [flat[k][off[i]:off[i + 1]] for i in range(len(lens))] for k in ("c1", "c2", "num", "timestamp")}
    return cols


def store_from_flat(lens, seqs, flat, names, dev):
    """The store built from arrow-like flat columns (the from_parquet route, no per-row Python)."""
    import pyarrow as pa

    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    cols = {"item_id": pa.ListArray.from_arrays(pa.array(off), pa.array(np.concatenate(seqs)))}
    for n in names:
        if n == "tags":
            inner = pa.ListArray.from_arrays(pa.array(np.concatenate([[0], np.cumsum(flat["tags_len"])]).astype(np.int32)),
                                             pa.array(flat["tags"]))
            cols[n] = pa.ListArray.from_arrays(pa.array(off), inner)
        elif n == "num":
            inner = pa.FixedSizeListArray.from_arrays(pa.array(flat["num"].reshape(-1)), 8)
            cols[n] = pa.ListArray.from_arrays(pa.array(off), inner)
        else:
            cols[n] = pa.ListArray.from_arrays(pa.array(off), pa.array(flat[n]))
    return DeviceSequenceStore.from_parquet(pa.table(cols), device=dev, feature_columns=list(names), padding_values=PADS,
                                            list_widths={"tags": 4})


# ---------------------------------------------------------------------------------------------- host-built batches
def host_sample(seqs, cols, i, off, window, names):
    """One sample of the reference's legacy per-sample path: slice, torch.tensor, left-pad with the feature's padding."""
    out = {}
    for n, seq in [("item_id", seqs[i]), *((n, cols[n][i]) for n in names)]:
        cut = seq[off:off + window]
        t = torch.tensor(cut, dtype=torch.long if np.issubdtype(cut.dtype, np.integer) else torch.float32)
        if len(t) < window:
            full = torch.full((window, *t.shape[1:]), PADS.get(n, I), dtype=t.dtype)
            full[window - len(t):] = t
            t = full
        out[n] = t
    mask = torch.ones(window, dtype=torch.bool)
    if len(seqs[i]) < window:
        mask[:window - len(seqs[i])] = False
    return {"feature_tensor": {k: v[:-1] for k, v in out.items()}, "padding_mask": mask[:-1],
            "positive_labels": out["item_id"][1:], "target_padding_mask": mask[1:], "query_id": torch.tensor([i])}


def host_batch(seqs, cols, idx, names, dev, pin=False):
    smp = [host_sample(seqs, cols, int(i), max(0, len(seqs[i]) - L - 1), L + 1, names) for i in idx]
    b = default_collate(smp)
    if pin:
        return b
    return to_dev(b, dev)


def to_dev(b, dev):
    return {k: (to_dev(v, dev) if isinstance(v, dict) else v.to(dev, non_blocking=True)) for k, v in b.items()}


def pin(b):
    return {k: (pin(v) if isinstance(v, dict) else v.contiguous().pin_memory()) for k, v in b.items()}


def _gather_last(offsets, rows, width):
    """Left-padded gather of the last ``width`` entries of each row, with the host-side checks the new path runs on every
    call (the index bounds, the offsets' order and the mask sums are each read back to the host)."""
    assert rows.numel() > 0 and int(rows.min().cpu()) >= 0 and int(rows.max().cpu()) < offsets.numel()
    assert bool((offsets[1:] >= offsets[:-1]).all().cpu())
    lo, hi = offsets[rows], offsets[rows + 1]
    pos = (hi - width)[:, None] + torch.arange(width, device=rows.device)[None, :]
    mask = (pos >= lo[:, None]) & (pos < hi[:, None])
    assert bool((mask.sum(-1) == torch.clamp(hi - lo, max=width)).all().cpu())
    idx = torch.where(mask, pos, 0)
    assert bool(((idx.max(-1).values < hi) | (hi == lo)).all().cpu())
    return mask, idx


class TorchOpColumns:
    """The new path's column gathers on the GPU with torch ops: 1-D columns and the 2-D columns (vector, list)."""

    def __init__(self, lens, seqs, flat, dev):
        def t(x):
            return torch.as_tensor(np.ascontiguousarray(x), device=dev)
        self.off = t(np.concatenate([[0], np.cumsum(lens)]))
        self.data = {"item_id": t(np.concatenate(seqs)), "c1": t(flat["c1"]), "c2": t(flat["c2"]),
                     "timestamp": t(flat["timestamp"]), "num": t(flat["num"].reshape(-1)), "tags": t(flat["tags"])}
        self.inner = {"num": t(np.arange(0, 8 * len(flat["c1"]) + 1, 8)),
                      "tags": t(np.concatenate([[0], np.cumsum(flat["tags_len"])]))}
        self.width = {"num": 8, "tags": 4}

    def batch(self, rows, names):
        out = {}
        for n in ["item_id", *names]:
            mask, idx = _gather_last(self.off, rows, L + 1)
            if n in self.inner:  # 2-D column: a second gather over the events' inner offsets
                lo = int(idx.min().cpu())
                hi = int(idx.max().cpu())
                ev = torch.arange(lo, hi + 1, device=rows.device)
                imask, iidx = _gather_last(self.inner[n], ev, self.width[n])
                vals = torch.take(self.data[n], iidx[idx - lo])
                m = imask[idx - lo] & mask[..., None]
                vals = torch.where(m, vals, torch.as_tensor(PADS[n], dtype=vals.dtype, device=vals.device))
            else:
                vals = torch.where(mask, torch.take(self.data[n], idx), PADS.get(n, I))
            out[n], out[n + "_mask"] = vals, mask
        return {"feature_tensors": {n: out[n][:, :-1] for n in ["item_id", *names]}, "padding_mask": out["item_id_mask"][:, :-1],
                "positive_labels": out["item_id"][:, 1:, None], "target_padding_mask": out["item_id_mask"][:, 1:, None]}


# -------------------------------------------------------------------------------------------------------- timing
def events_ms(fn, n):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def store_bytes(st, lens, idx, names, flat):
    """Bytes one new-path training build moves: per row the CSR pair, the window's live item ids and feature values (list
    offsets and kept entries included) read, and every output written."""
    live = np.minimum(lens[idx], L + 1)
    ev = int(live.sum())
    rd = len(idx) * (16 + 4 + 8) + ev * 4
    wr = len(idx) * L * (8 + 1 + 8 + 1) + len(idx) * 8
    cols = {c.name: c for c in st.columns}
    off = np.concatenate([[0], np.cumsum(lens)])
    for n in names:
        c = cols[n]
        if c.kind == "list":
            kept = sum(int(np.minimum(flat["tags_len"][off[i + 1] - m: off[i + 1]], 4).sum()) for i, m in zip(idx, live))
            rd += ev * 16 + kept * c.values.element_size()
            wr += len(idx) * L * 4 * 8
        else:
            rd += ev * c.width * c.values.element_size()
            wr += len(idx) * L * c.width * (8 if c.kind == "int" else c.values.element_size())
    return rd + wr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the result JSON to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(card)
    dev = torch.device("cuda")
    lens, seqs, flat = histories()
    cols = per_seq(lens, flat)
    side = ["c1", "c2", "tags", "num"]
    item_only = store_from_flat(lens, seqs, flat, [], dev)
    feat = store_from_flat(lens, seqs, flat, side, dev)
    ti = store_from_flat(lens, seqs, flat, ["timestamp"], dev)
    tops = TorchOpColumns(lens, seqs, flat, dev)
    rng = np.random.default_rng(1)
    idx = rng.choice(U, B, replace=False)
    idx_d = torch.as_tensor(idx, device=dev)
    res = {"card": card, "shape": f"B {B} x L {L}, {U} histories"}

    # ---- 1. build time per batch
    build = {
        "store_item_only": events_ms(lambda: item_only.sasrec_new_path_batch(idx_d, L, I), a.iters),
        "store_features": events_ms(lambda: feat.sasrec_new_path_batch(idx_d, L, I), a.iters),
        "store_tisasrec_timestamps": events_ms(lambda: ti.sasrec_training_batch(idx_d, L, I), a.iters),
        "torch_op_gathers_features": events_ms(lambda: tops.batch(idx_d, side), max(5, a.iters // 5)),
        "torch_op_gathers_item_only": events_ms(lambda: tops.batch(idx_d, []), max(5, a.iters // 5)),
        "host_per_sample_features_no_list": events_ms(lambda: host_batch(seqs, cols, idx, ["c1", "c2", "num"], dev), 3),
        "host_per_sample_tisasrec": events_ms(lambda: host_batch(seqs, cols, idx, ["timestamp"], dev), 3),
        "store_features_no_list": None,
    }
    nolist = store_from_flat(lens, seqs, flat, ["c1", "c2", "num"], dev)
    build["store_features_no_list"] = events_ms(lambda: nolist.sasrec_training_batch(idx_d, L, I), a.iters)
    res["build_ms_per_batch"] = {k: round(v, 4) for k, v in build.items()}
    nbytes = store_bytes(feat, lens, idx, side, flat)
    res["store_features_bytes"] = nbytes
    res["store_features_share_of_3.35TBps"] = round(nbytes / (build["store_features"] * 1e-3) / HBM_BYTES_PER_S, 4)
    nbytes0 = store_bytes(item_only, lens, idx, [], flat)
    res["store_item_only_share_of_3.35TBps"] = round(nbytes0 / (build["store_item_only"] * 1e-3) / HBM_BYTES_PER_S, 4)
    print(json.dumps(res))

    # ---- 3. end to end
    from replay_b200.models.nn.sequential import SasRec as LegacySasRec
    from replay_b200.nn.lightning.module import LightningModule
    from replay_b200.nn.sequential.sasrec import SasRec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    schema = TensorSchema(TensorFeatureInfo("item_id", I, I, D), features=[
        TensorFeatureInfo("c1", 1000, 1000, D), TensorFeatureInfo("c2", 20, 20, D),
        TensorFeatureInfo("tags", 30, 30, D, is_list=True), TensorFeatureInfo("num", None, 0, D, is_cat=False, tensor_dim=8)])
    side_module = LightningModule(SasRec.from_params(schema, embedding_dim=D, num_heads=H, num_blocks=2,
                                                     max_sequence_length=L, dropout=0.2, device=dev, seed=0))
    ti_model = LegacySasRec(TensorSchema(TensorFeatureInfo("item_id", I, I, D), timestamp_feature_name="timestamp"),
                            block_count=2, head_count=H, hidden_size=D, max_seq_len=L, dropout_rate=0.2,
                            ti_modification=True, time_span=256, device=dev)
    steps = [rng.choice(U, B, replace=False) for _ in range(a.steps)]
    steps_d = [torch.as_tensor(s, device=dev) for s in steps]

    def new_host(s):  # the new path's host side: the same torch-op gathers on CPU tensors, then an H2D copy
        return to_dev(cpu_tops.batch(torch.as_tensor(s), side), dev)

    cpu_tops = TorchOpColumns(lens, seqs, flat, torch.device("cpu"))
    feeds = {
        "side_sasrec": {
            "store": lambda i: feat.sasrec_new_path_batch(steps_d[i], L, I, with_seen=False),
            "host_per_step": lambda i: new_host(steps[i]),
            "pinned_prebuilt": None,
        },
        "tisasrec": {
            "store": lambda i: ti.sasrec_training_batch(steps_d[i], L, I),
            "host_per_step": lambda i: host_batch(seqs, cols, steps[i], ["timestamp"], dev),
            "pinned_prebuilt": None,
        },
    }
    pinned_side = [pin(cpu_tops.batch(torch.as_tensor(s), side)) for s in steps]
    pinned_ti = [pin(host_batch(seqs, cols, s, ["timestamp"], dev, pin=True)) for s in steps]
    feeds["side_sasrec"]["pinned_prebuilt"] = lambda i: to_dev(pinned_side[i], dev)
    feeds["tisasrec"]["pinned_prebuilt"] = lambda i: to_dev(pinned_ti[i], dev)
    run = {"side_sasrec": lambda b: side_module.training_step(b), "tisasrec": lambda b: ti_model.training_step(b)}
    e2e = {}
    for model, fs in feeds.items():
        for f in fs.values():  # warm-up: every shape once
            run[model](f(0))
        torch.cuda.synchronize()
        rates = {k: [] for k in fs}
        for _ in range(a.rounds):
            for name, f in fs.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for i in range(a.steps):
                    run[model](f(i))
                torch.cuda.synchronize()
                rates[name].append(B * a.steps / (time.perf_counter() - t0))
        e2e[model] = {k: round(float(np.median(v)), 1) for k, v in rates.items()}
    res["train_seq_per_s"] = e2e
    res["note"] = ("host_per_step: side_sasrec = the new path's torch-op gathers on CPU + H2D; tisasrec = the legacy "
                   "per-sample dataset + default collate + H2D")
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
