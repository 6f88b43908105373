"""TwoTower with and without side features: training ms/step, the item tower's feature kernels, predict.

    python tools/bench_twotower_side_features.py [--steps 20] [--rounds 3]

Config 2 (L 200, d 128, 2 heads, |I| 50 K, 512 sequences, dropout 0.2, packed query rows).  The side features are those
of tools/bench_side_features.py (categoricals of cardinality 1000 and 20, a sum bag of width 4, a numerical feature of
tensor_dim 8) in the query tower; the item features reader holds the two categoricals and the bag.  CE and CESampled
(256 shared negatives), each with and without features, are timed alternately in rounds on one card through the
graph-captured fused step (TwoTowerCore.fused_step), medians reported.  Also: rp_item_feature_embed_fwd over the catalog
and rp_item_feature_embed_bwd over the catalog (fixed-order) and over the sampled loss's slots (atomics), and predict
users/s for a seen-filtered top-10 at 4096 users per call.  The card's name, power limit and max SM clock come first."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from replay_b200.engine import SideFeature
from replay_b200.engine_twotower import TwoTowerConfig
from replay_b200.nn.sequential.twotower import TwoTowerCore
from replay_b200.synthetic import make_sequences

B, L, D, H, I, PB = 512, 200, 128, 2, 50_000, 4096
SIDE = (SideFeature("c1", "cat", 1000, 1000), SideFeature("c2", "cat", 20, 20), SideFeature("tags", "bag_sum", 30, 30),
        SideFeature("num", "num", width=8))
READER = ("c1", "c2", "tags")


def timed(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def side_batch(n, g):
    return {"c1": torch.randint(0, 1001, (n, L), generator=g), "c2": torch.randint(0, 21, (n, L), generator=g),
            "tags": torch.randint(0, 31, (n, L, 4), generator=g), "num": torch.randn(n, L, 8, generator=g)}


def item_columns(g):
    return {"c1": torch.randint(0, 1001, (I,), generator=g), "c2": torch.randint(0, 21, (I,), generator=g),
            "tags": torch.randint(0, 31, (I, 4), generator=g)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(0)
    ids, pm, lab, tm = (t.to(dev) for t in make_sequences(B, I, L, seed=1234))
    feats = {k: v.to(dev) for k, v in side_batch(B, g).items()}
    pids, ppm, _, _ = (t.to(dev) for t in make_sequences(PB, I, L, seed=99))
    pfeats = {k: v.to(dev) for k, v in side_batch(PB, g).items()}
    cols = item_columns(g)
    neg = torch.randint(0, I, (256,), generator=g).to(dev)
    cores = {}
    for kind in ("ce", "ce_sampled"):
        for name, fs, it in (("item_only", (), ()), ("features", SIDE, READER)):
            cfg = TwoTowerConfig(n_items=I, d=D, n_heads=H, n_blocks=2, max_len=L, dropout=0.2, variant="new", features=fs,
                                 item_features=it)
            core = TwoTowerCore(cfg, device=dev, seed=1, item_values=cols)
            if kind == "ce_sampled":
                core.set_loss("ce_sampled", n_neg=256, neg_shape="shared")
            core.ensure_engine(B, L, with_grad=True).packed_body = True
            cores[(kind, name)] = core
    res = {f"{k}/{n}": {"ms_step": []} for k, n in cores}

    def step(key):
        kind, name = key
        return cores[key].fused_step(ids, pm, lab, tm, all_reduce=None, lr=1e-3, negatives=neg if kind != "ce" else None,
                                     feats=feats if name == "features" else None)

    for key in cores:   # warm-up: lazy loads and the graph capture of the fused step
        for _ in range(4):
            step(key)
    torch.cuda.synchronize()
    for _ in range(a.rounds):
        for key in cores:
            res[f"{key[0]}/{key[1]}"]["ms_step"].append(timed(lambda: step(key), a.steps))
    for r in res.values():
        r["ms_step_all"] = r["ms_step"]
        r["ms_step"] = sorted(r["ms_step"])[len(r["ms_step"]) // 2]
        r["seq_s"] = B / r["ms_step"] * 1e3
    # the item tower's feature kernels alone
    eng = cores[("ce", "features")].engine
    x0 = eng.tw["x0"]
    res["item_feature_fwd_catalog_ms"] = timed(lambda: eng._item_x0(x0, I), 50)
    res["item_feature_bwd_catalog_ms"] = timed(lambda: eng._item_feature_bwd(I), 50)
    seng = cores[("ce_sampled", "features")].engine
    rows = seng.sampled["cap"]
    res["item_feature_bwd_slots_ms"] = timed(lambda: seng._item_feature_bwd(rows, seng.tw["item_of_slot"], seng.tw["n_slots"]), 50)
    res["slots"] = {"cap": rows, "n_slots": int(seng.tw["n_slots"])}
    # predict: a seen-filtered top-10 at PB users per call (the tower over the catalog is cached after the first call)
    for name in ("item_only", "features"):
        c = cores[("ce", name)]
        f = pfeats if name == "features" else None
        for _ in range(3):
            c.predict_topk(pids, ppm, 10, seen_ids=pids, feats=f)
        res[f"predict/{name}_ms"] = timed(lambda: c.predict_topk(pids, ppm, 10, seen_ids=pids, feats=f), a.steps)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
