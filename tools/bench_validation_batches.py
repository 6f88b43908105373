"""Cost of producing validation batches: the device sequence store's query lists against the reference's per-sample path.

    python tools/bench_validation_batches.py [--users N] [--iters N] [--out FILE]

Config 4 shape: L 200, every user with a 200-item train list and a 10-item ground truth, |I| 500 K, histories with
MovieLens-shaped (lognormal) lengths of 20 .. 2314 events.

1. Build time per 4096-user batch: the store's three validation builders (CUDA events around ``--iters`` builds after a
   warm-up) against the reference's per-sample path restated (TorchSequentialValidationDataset.__getitem__: the left-padded
   window and its mask, then ground_truth and train each looked up by query id in a pandas Series, as
   PandasSequentialDataset.get_sequence_by_query_id does, and copied into a -1 / -2 placeholder; default collate; H2D
   copy), timed with a host clock around whole batches ending in a device synchronise.
2. One validation epoch over ``--users`` users (default 1 M): the new-path SasRec of config 4 (d 128, 2 heads, 2 blocks)
   with ComputeMetricsCallback (recall, ndcg, map, mrr, novelty, coverage @10) and SeenItemsFilter over the train list,
   fed by DeviceBatchLoader(kind="sasrec_new_validate") and, separately, by the per-sample host batches of the same users.
   Users/s is the epoch's users over its wall time, ending in a device synchronise; both feeds' metrics must agree.
The card's name, power limit and max SM clock are read in the same run, printed first and stored in the JSON line printed
last."""
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

from replay_b200.device_data import DeviceBatchLoader, DeviceSequenceStore

L, I, D, H, G, T, BATCH = 200, 500_000, 128, 2, 10, 200, 4096


def data(n_users, seed=0):
    rng = np.random.default_rng(seed)
    lens = np.clip(np.round(np.exp(rng.normal(4.56, 0.95, n_users))), 20, 2314).astype(np.int64)
    off = np.concatenate([[0], np.cumsum(lens)])
    items = rng.integers(0, I, int(off[-1]))
    gt = rng.integers(0, I, (n_users, G))
    train = rng.integers(0, I, (n_users, T))
    qid = np.arange(n_users, dtype=np.int64) * 3 + 7
    return lens, off, items, gt, train, qid


class HostValidation:
    """The reference's per-sample validation path, restated: one window and two query-id lookups per user."""

    def __init__(self, off, items, gt, train, qid):
        import pandas as pd

        self.off, self.items, self.qid = off, items, qid
        self.gt = pd.Series(list(gt), index=qid)
        self.train = pd.Series(list(train), index=qid)
        self.g_w, self.t_w = gt.shape[1], train.shape[1]

    def sample(self, i):
        seq = self.items[self.off[i]:self.off[i + 1]]
        cut = torch.tensor(seq[max(0, len(seq) - L):], dtype=torch.long)
        ids = torch.full((L,), I, dtype=torch.long)
        ids[L - len(cut):] = cut
        mask = torch.zeros(L, dtype=torch.bool)
        mask[L - len(cut):] = True
        q = int(self.qid[i])
        out = {"query_id": torch.tensor([q]), "padding_mask": mask, "feature_tensor": {"item_id": ids}}
        for name, s, w, pad in (("ground_truth", self.gt, self.g_w, -1), ("train", self.train, self.t_w, -2)):
            x = np.array(s.loc[q])
            ph = np.full(w, pad, dtype=np.int64)
            np.copyto(ph[:len(x)], x)
            out[name] = torch.LongTensor(ph)
        return out

    def batch(self, rows, dev):
        b = default_collate([self.sample(int(i)) for i in rows])
        return {"query_id": b["query_id"].to(dev, non_blocking=True), "padding_mask": b["padding_mask"].to(dev),
                "feature_tensors": {"item_id": b["feature_tensor"]["item_id"].to(dev)},
                "ground_truth": b["ground_truth"].to(dev), "train": b["train"].to(dev), "seen_ids": b["train"].to(dev)}


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


def epoch(lm, batches, metrics_cb):
    metrics_cb.on_validation_epoch_start(None, lm)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n = 0
    for i, b in enumerate(batches):
        metrics_cb.on_validation_batch_end(None, lm, lm.predict_step(b, 0), b, i)
        n += b["padding_mask"].shape[0]
    m = metrics_cb.on_validation_epoch_end(None, lm)
    torch.cuda.synchronize()
    return n, time.perf_counter() - t0, m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=1_000_000)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--host-batches", type=int, default=3, help="4096-user batches timed on the per-sample path")
    ap.add_argument("--out", default=None, help="also write the result JSON to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(card, flush=True)
    dev = torch.device("cuda")
    lens, off, items, gt, train, qid = data(a.users)
    t0 = time.perf_counter()
    st = DeviceSequenceStore(offsets=off, items=items, query_ids=qid, device=dev,
                             query_lists={"ground_truth": list(gt), "train": list(train)},
                             list_widths={"ground_truth": G, "train": T})
    torch.cuda.synchronize()
    res = {"card": card, "users": a.users, "L": L, "items": I, "batch": BATCH, "gt": G, "train": T,
           "store_build_s": round(time.perf_counter() - t0, 2), "events": int(off[-1])}
    host = HostValidation(off, items, gt, train, qid)

    # ---- 1. one 4096-user batch
    rows = torch.arange(BATCH, dtype=torch.int32, device=dev)
    for name, fn in (("sasrec", st.sasrec_validation_batch), ("bert4rec", st.bert4rec_validation_batch),
                     ("sasrec_new", st.sasrec_new_path_validation_batch)):
        res[f"device_{name}_ms"] = round(events_ms(lambda: fn(rows, L, I), a.iters), 4)
    host.batch(range(BATCH), dev)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for k in range(a.host_batches):
        host.batch(range(k * BATCH, (k + 1) * BATCH), dev)
    torch.cuda.synchronize()
    res["host_per_sample_ms"] = round((time.perf_counter() - t0) * 1e3 / a.host_batches, 2)
    print(json.dumps(res), flush=True)

    # ---- 2. one validation epoch, metrics @10 with the seen filter
    from replay_b200.nn.lightning import ComputeMetricsCallback, LightningModule, SeenItemsFilter
    from replay_b200.nn.sequential import SasRec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    model = SasRec.from_params(TensorSchema(TensorFeatureInfo("item_id", I, I, D)), embedding_dim=D, num_heads=H,
                               num_blocks=2, max_sequence_length=L, dropout=0.0, device=dev, seed=1)
    model.eval()
    lm = LightningModule(model)

    def cb():
        return ComputeMetricsCallback(metrics=("recall", "ndcg", "map", "mrr", "novelty", "coverage"), ks=(10,),
                                      item_count=I, postprocessors=[SeenItemsFilter(I, "train")])

    loader = DeviceBatchLoader(st, L, BATCH, I, kind="sasrec_new_validate")
    epoch(lm, [next(iter(loader))], cb())                                   # warm-up: modules, workspaces
    n, dt, m_dev = epoch(lm, loader, cb())
    res.update({"device_epoch_s": round(dt, 3), "device_users_per_s": round(n / dt)})
    print(json.dumps(res), flush=True)
    host_batches = (host.batch(range(lo, min(lo + BATCH, a.users)), dev) for lo in range(0, a.users, BATCH))
    n_h, dt_h, m_host = epoch(lm, host_batches, cb())
    assert n_h == n
    res.update({"host_epoch_s": round(dt_h, 3), "host_users_per_s": round(n_h / dt_h),
                "metrics_equal": m_dev == m_host, "metrics": m_dev})
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
