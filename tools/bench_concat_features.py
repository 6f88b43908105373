"""Cost of ConcatAggregator in the new-path SASRec (CUDA events), against the SumAggregator model on the same features and
the item-only model, in the same call.

    python tools/bench_concat_features.py [--steps N] [--rounds R]

Config 2: L 200, d 128, 2 heads, |I| 50 K, 512 sequences per step, dropout 0.2, packed rows, full-catalog CE.  Features
(tools/bench_side_features.py's): two categoricals (|C| 1 K and 20), a categorical list of width 4 summed, a numerical
feature of tensor_dim 8.  The Sum model embeds every one at 128; the concat model keeps the item at 128 and puts them at
32, 16, 32 and 16 (224 concatenated columns, 256 padded).  The models alternate for ``--rounds`` rounds.  Reports ms per
fused training step, predict users/s for a seen-filtered top-10 over 4096 users per call, and the concat input stage's
parts alone on the padded rows: the gather, the projection GEMM, the whole forward and the whole backward.  The card's
name, power limit and max SM clock are printed first."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from replay_b200.core import SasRecCore
from replay_b200.engine import EncoderConfig, SideFeature
from replay_b200.synthetic import make_sequences

B, L, D, H, I, PB = 512, 200, 128, 2, 50_000, 4096
SUM = (SideFeature("c1", "cat", 1000, 1000), SideFeature("c2", "cat", 20, 20), SideFeature("tags", "bag_sum", 30, 30),
       SideFeature("num", "num", width=8))
# ConcatAggregator's order is by name: c1, c2, item_id, num, tags
CONCAT = (SideFeature("c1", "cat", 1000, 1000, dim=32), SideFeature("c2", "cat", 20, 20, dim=16),
          SideFeature("num", "num", width=8, dim=16), SideFeature("tags", "bag_sum", 30, 30, dim=32))


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
    cores = {}
    for name, fs, kw in (("item_only", (), {}), ("sum", SUM, {}), ("concat", CONCAT, dict(aggregator="concat", concat_item_at=2))):
        cfg = EncoderConfig(n_items=I, d=D, n_heads=H, n_blocks=2, max_len=L, dropout=0.2, variant="new", features=fs, **kw)
        core = SasRecCore(cfg, device=dev, seed=1)
        core.ensure_engine(B, L, with_grad=True).packed_body = True
        cores[name] = core
    res = {k: {"ms_step": [], "predict_users_s": []} for k in cores}

    def step(name):
        return cores[name].fused_step(ids, pm, lab, tm, lr=1e-3, feats=None if name == "item_only" else feats)

    def predict(name):
        return cores[name].predict_topk(pids, ppm, 10, seen_ids=pids, feats=None if name == "item_only" else pfeats)

    for name in cores:   # warm-up: lazy loads, graph capture of the fused step and of predict
        for _ in range(4):
            step(name)
            predict(name)
    torch.cuda.synchronize()
    for _ in range(a.rounds):
        for name in cores:
            res[name]["ms_step"].append(timed(lambda: step(name), a.steps))
            res[name]["predict_users_s"].append(PB / (timed(lambda: predict(name), a.steps) / 1e3))
    for r in res.values():
        r["ms_step"] = sorted(r["ms_step"])[len(r["ms_step"]) // 2]
        r["predict_users_s"] = sorted(r["predict_users_s"])[len(r["predict_users_s"]) // 2]
    # the concat input stage alone, on the padded rows of the staged batch
    c = cores["concat"]
    eng, cfg = c.engine, c.cfg
    eng.packed_body = False
    step("concat")
    eng._prepare(True)
    pos0 = cfg.max_len - L
    fa = eng._feature_descs(False)
    item_col, seg_col, seg_dim = eng._concat_segments()

    def gather():
        eng.lib.rp_concat_gather(eng.params16["item_emb"].data_ptr(), eng.ids32.data_ptr(), fa, seg_col, seg_dim, len(fa),
                                 item_col, eng.T, cfg.dp, cfg.hd_valid, cfg.concat_kp, eng.cat_x.data_ptr(), eng._stream())

    def project():
        eng._gemm(eng.cat_x, eng.params16["feat_proj.w"], eng.cat_y, eng.T, cfg.dp, cfg.concat_kp,
                  bias=eng.params["feat_proj.b"], out_mode=2)

    dx = (torch.randn(eng.T, cfg.dp, device=dev) * 0.01).to(torch.bfloat16)
    parts = {"gather": gather, "projection": project, "forward": lambda: eng._embed_fwd(0.2, pos0),
             "backward": lambda: eng._concat_bwd(dx, 0.2, pos0)}
    for fn in parts.values():
        for _ in range(3):
            fn()
    res["concat"].update({f"{k}_ms": timed(fn, 50) for k, fn in parts.items()})
    eng.g32.zero_()
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
