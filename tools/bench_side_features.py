"""Cost of side features in the new-path SASRec (CUDA events, eager launches), against the item-only model in the same call.

    python tools/bench_side_features.py [--steps N] [--rounds R]

Config 2: L 200, d 128, 2 heads, |I| 50 K, 512 sequences per step, full-catalog CE.  Side features: two categoricals
(|C| 1 K and 20), one categorical list of width 4 summed, one numerical feature of tensor_dim 8.  The two models alternate
for ``--rounds`` rounds.  Reports ms per training step of each, the side-feature embedding forward and backward kernels
alone (rp_feature_embed_fwd / _bwd with the numerical weight-gradient GEMM) next to rp_embed_fwd / _bwd, and predict
users/s for a seen-filtered top-10 over 4096 users.  The card's name, power limit and max SM clock are printed first."""
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
SIDE = (SideFeature("c1", "cat", 1000, 1000), SideFeature("c2", "cat", 20, 20), SideFeature("tags", "bag_sum", 30, 30),
        SideFeature("num", "num", width=8))


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
    for name, fs in (("item_only", ()), ("side", SIDE)):
        cfg = EncoderConfig(n_items=I, d=D, n_heads=H, n_blocks=2, max_len=L, dropout=0.2, variant="new", features=fs)
        core = SasRecCore(cfg, device=dev, seed=1)
        eng = core.ensure_engine(B, L, with_grad=True)
        eng.packed_body = True
        cores[name] = core
    res = {k: {"ms_step": [], "predict_users_s": []} for k in cores}

    def step(name):
        c = cores[name]
        return c.fused_step(ids, pm, lab, tm, lr=1e-3, feats=feats if name == "side" else None)

    def predict(name):
        c = cores[name]
        return c.predict_topk(pids, ppm, 10, seen_ids=pids, feats=pfeats if name == "side" else None)

    for name in cores:   # warm-up: lazy loads, graph capture of the fused step and of predict
        for _ in range(4):
            step(name)
            predict(name)
    torch.cuda.synchronize()
    for _ in range(a.rounds):
        for name in cores:
            res[name]["ms_step"].append(timed(lambda: step(name), a.steps))
            res[name]["predict_users_s"].append(PB / (timed(lambda: predict(name), a.steps) / 1e3))
    # the embedding stage alone, on the padded rows of the staged batch
    for name, c in cores.items():
        eng = c.engine
        eng.packed_body = False
        step(name)
        eng._prepare(True)
        pos0 = c.cfg.max_len - L
        fwd = lambda: eng._embed_fwd(0.2, pos0)  # noqa: E731
        dx = torch.randn(eng.T, c.cfg.dp, device=dev).to(torch.bfloat16)

        def bwd(eng=eng, c=c, dx=dx):
            if eng.features:
                eng._feature_bwd(dx, 0.2)
            eng.lib.rp_embed_bwd(dx.data_ptr(), eng.ids32.data_ptr(), eng.in_pad.data_ptr(), eng.B, L, c.cfg.dp, c.cfg.pad_id,
                                 pos0, D ** 0.5, 0, 0.2, eng.seed, 0, eng.rng_counter.data_ptr(), eng.grads["item_emb"].data_ptr(),
                                 eng.grads["pos_emb"].data_ptr(), eng._stream())

        for _ in range(3):
            fwd()
            bwd()
        res[name]["embed_fwd_ms"] = timed(fwd, 50)
        res[name]["embed_bwd_ms"] = timed(bwd, 50)
    for name, r in res.items():
        r["ms_step"] = sorted(r["ms_step"])[len(r["ms_step"]) // 2]
        r["predict_users_s"] = sorted(r["predict_users_s"])[len(r["predict_users_s"]) // 2]
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
