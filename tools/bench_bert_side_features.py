"""Cost of side features in the legacy BERT4Rec (CUDA events), against the item-only model in the same call.

    python tools/bench_bert_side_features.py [--steps N] [--rounds R]

Config 3: L 200, d 256, 4 heads, 2 blocks, |I| 100 K, 256 sequences per step, dropout 0.1, full-catalog CE.  Side features:
two categoricals (|C| 1 K and 20) and one identity numerical of tensor_dim 256.  The two models alternate for ``--rounds``
rounds of the captured fused step.  Reports the median ms per training step of each, the embedding forward and backward
alone (rp_bert_embed_fwd / _bwd, plus rp_bert_feature_embed_fwd / _bwd for the side-feature model), and predict users/s
for a seen-filtered top-10 over 4096 users.  The card's name, power limit and max SM clock are printed first."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from replay_b200.engine import SideFeature
from replay_b200.engine_bert import BertConfig
from replay_b200.models.nn.sequential.bert4rec import _BertCore, uniform_masker

B, L, D, H, I, PB, P = 256, 200, 256, 4, 100_000, 4096, 0.1
SIDE = (SideFeature("c1", "cat", 1000, 0), SideFeature("c2", "cat", 20, 0), SideFeature("num", "ident", width=D))


def timed(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def batch(n, g, dev):
    lens = torch.randint(20, L + 1, (n,), generator=g)
    pad = torch.arange(L)[None, :] >= (L - lens)[:, None]
    ids = torch.where(pad, torch.randint(0, I, (n, L), generator=g), torch.zeros(n, L, dtype=torch.int64))
    tok = uniform_masker(pad, 0.2, g)
    feats = {"item_id": ids, "c1": torch.randint(0, 1000, (n, L), generator=g), "c2": torch.randint(0, 20, (n, L), generator=g),
             "num": torch.randn(n, L, D, generator=g)}
    return ids.to(dev), pad.to(dev), tok.to(dev), {k: v.to(dev) for k, v in feats.items()}


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
    ids, pm, tm, feats = batch(B, g, dev)
    pids, ppm, _, pfeats = batch(PB, g, dev)
    ptm = ppm.clone()
    ptm[:, -1] = False   # the prediction window: the last position is <MASK>
    cores = {}
    for name, fs in (("item_only", ()), ("side", SIDE)):
        cfg = BertConfig(n_items=I, d=D, n_heads=H, n_blocks=2, max_len=L, dropout=P, features=fs)
        cores[name] = _BertCore(cfg, device=dev, seed=1)
    res = {k: {"ms_step": [], "predict_users_s": []} for k in cores}

    def step(name):
        return cores[name].fused_step(ids, pm, tm, ids, lr=1e-3, feats=feats)

    def predict(name):
        return cores[name].predict_topk(pids, ppm, ptm, 10, seen_ids=pids, feats=pfeats)

    for name in cores:   # warm-up: lazy loads, the fused step's graph capture
        for _ in range(4):
            step(name)
            predict(name)
    torch.cuda.synchronize()
    for _ in range(a.rounds):
        for name in cores:
            res[name]["ms_step"].append(timed(lambda: step(name), a.steps))
            res[name]["predict_users_s"].append(PB / (timed(lambda: predict(name), a.steps) / 1e3))
    # the embedding stage alone, on the staged training batch: the item-only pair, and the new pair on its own
    for name, c in cores.items():
        step(name)
        eng = c.ensure_engine(B, L, with_grad=True)
        eng._prepare(True)
        dx = torch.randn(eng.T, c.cfg.dp, device=dev).to(torch.bfloat16)
        st, rng, G, p16 = eng._stream, eng.rng_counter.data_ptr(), eng.grads, eng.params16

        def item_fwd():
            return eng.lib.rp_bert_embed_fwd(p16["item_emb"].data_ptr(), p16["mask_emb"].data_ptr(),
                                             eng.params["pos_emb"].data_ptr(),
                                             eng.ids32.data_ptr(), eng.in_tok.data_ptr(), eng.T, L, c.cfg.dp, P, eng.seed, 0,
                                             rng, eng.x[0].data_ptr(), st())

        def item_bwd():
            return eng.lib.rp_bert_embed_bwd(dx.data_ptr(), eng.ids32.data_ptr(), eng.in_pad.data_ptr(), eng.in_tok.data_ptr(),
                                             eng.B, L, c.cfg.dp, P, eng.seed, 0, rng, G["item_emb"].data_ptr(),
                                             G["mask_emb"].data_ptr(), G["pos_emb"].data_ptr(), st())

        runs = {"bert_embed_fwd_ms": item_fwd, "bert_embed_bwd_ms": item_bwd}
        if eng.features:
            fa, fg = eng._feature_descs(False), eng._feature_descs(True)
            runs["bert_feature_embed_fwd_ms"] = lambda: eng.lib.rp_bert_feature_embed_fwd(
                p16["item_emb"].data_ptr(), p16["mask_emb"].data_ptr(), eng.params["pos_emb"].data_ptr(), eng.ids32.data_ptr(),
                eng.in_tok.data_ptr(), fa, len(fa), eng.T, L, c.cfg.dp, c.cfg.hd_valid, P, eng.seed, 0, rng,
                eng.x[0].data_ptr(), st())
            runs["bert_feature_embed_bwd_ms"] = lambda: eng.lib.rp_bert_feature_embed_bwd(
                dx.data_ptr(), eng.in_pad.data_ptr(), eng.in_tok.data_ptr(), fg, len(fg), eng.T, c.cfg.dp, c.cfg.hd_valid, P,
                eng.seed, 0, rng, st())
        for k, fn in runs.items():
            for _ in range(3):
                assert fn() == 0, k
            res[name][k] = timed(fn, 50)
    for name, r in res.items():
        r["ms_step"] = sorted(r["ms_step"])[len(r["ms_step"]) // 2]
        r["predict_users_s"] = sorted(r["predict_users_s"])[len(r["predict_users_s"]) // 2]
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
