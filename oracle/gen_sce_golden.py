"""Generate tests/golden/sce_losses.npz FROM THE REAL REFERENCE (run where the reference is importable; it is not on the GPU
box).  TEST INFRASTRUCTURE.

    PYTHONPATH=oracle/shim:/root/reference python oracle/gen_sce_golden.py

The legacy SasRec's _compute_loss_scalable_ce (replay/models/nn/sequential/sasrec/lightning.py:383-392, loss
replay/models/nn/loss/sce.py) on the weights and batch of sasrec_legacy_tiny, labels clamped below |I| (the reference reads
w[y] for pad rows too).  torch.randn and torch.topk are captured, so a test can replay the draw and compare selections.
Stored per case: loss, item-table gradient, block-0 in_proj_weight gradient, draw, top_x, top_y, labels.
"""
import os

import numpy as np
import torch

from gen_golden import OUT, schema  # noqa: E402  (puts the shim and the reference on sys.path)

# bucket scores at every top-k boundary must differ by more than this fraction of the bucket's score spread, so that the
# bf16 inputs of the CUDA head select the same rows and items as the fp32 reference.  Row scores carry the bf16 body's
# error in the hidden rows (~1 % relative); item scores only the bf16 rounding of the draw and the table (~0.2 %), unless
# mix_x makes the buckets themselves depend on the hidden rows.
MARGIN_X, MARGIN_Y, MARGIN_Y_MIX = 0.03, 0.008, 0.02

# name: (n_buckets, bucket_size_x, bucket_size_y, mix_x, collide)
CASES = {
    "nomix": (4, 16, 32, False, None),
    "mix": (4, 16, 32, True, None),
    "bigx": (3, 64, 16, False, None),        # bucket_size_x above the 44 real rows: pad rows come back at -inf
    "overlap": (5, 40, 24, False, "partial"),  # rows picked by several buckets; labels colliding with bucket items
    "fullcollide": (2, 12, 1, False, "full"),  # bs_y = 1 and labels equal to the bucket's item: CE exactly 0
    "r111": (1, 1, 1, False, None),
    "r221": (2, 2, 1, False, None),
}


def _model(z, sdl, p):
    from replay.models.nn.loss import SCEParams
    from replay.models.nn.sequential.sasrec.lightning import SasRec as LegacySasRec

    n_items, d, H, L, nb = int(z["n_items"]), int(z["d"]), int(z["H"]), int(z["L"]), int(z["n_blocks"])
    mod = LegacySasRec(schema(n_items, d, n_items), block_count=nb, head_count=H, hidden_size=d, max_seq_len=L,
                       dropout_rate=0.0, loss_type="SCE", sce_params=SCEParams(*p))
    mod._model.load_state_dict(sdl)
    mod.train()
    return mod


def _run(mod, ids, labels, pm, tm, seed):
    rec = {"randn": [], "topk": []}
    orig_randn, orig_topk = torch.randn, torch.topk

    def randn(*a, **k):
        r = orig_randn(*a, **k)
        rec["randn"].append(r.clone())
        return r

    def topk(*a, **k):
        r = orig_topk(*a, **k)
        rec["topk"].append(r.indices.clone())
        return r

    torch.manual_seed(seed)
    torch.randn, torch.topk = randn, topk
    try:
        loss = mod._compute_loss_scalable_ce({"item_id": ids}, labels, pm, tm)
    finally:
        torch.randn, torch.topk = orig_randn, orig_topk
    return loss, rec


def _margin_ok(x, w, pm, draw, p):
    """Relative gap at each top-k boundary (fp64 scores of the fp32 reference inputs)."""
    n_b, bsx, bsy, mix = p
    x, w, draw = x.double(), w.double(), draw.double()
    scale = x.shape[1] ** -0.25
    b = (draw * scale).T @ x if mix else draw * scale
    worst = float("inf")
    for s, k, need in ((b @ x[pm].T, bsx, MARGIN_X), (b @ w.T, bsy, MARGIN_Y_MIX if mix else MARGIN_Y)):
        srt = s.sort(dim=1, descending=True).values
        if k >= srt.shape[1]:
            continue
        gap = (srt[:, k - 1] - srt[:, k]) / srt.std(dim=1)
        worst = min(worst, float(gap.min()) / need)
    return worst   # > 1: every boundary keeps its margin


def gen_sce_losses():
    zl = np.load(os.path.join(OUT, "sasrec_legacy_tiny.npz"))
    sdl = {k[4:]: torch.from_numpy(zl[k]) for k in zl.files if k.startswith("sd::")}
    n_items = int(zl["n_items"])
    ids, pm = torch.from_numpy(zl["ids"]), torch.from_numpy(zl["pad_mask"])
    labels0, tm = torch.from_numpy(zl["labels"]).clamp(max=n_items - 1), torch.from_numpy(zl["target_mask"])
    out = {}
    for name, (n_b, bsx, bsy, mix, collide) in CASES.items():
        p = (n_b, bsx, bsy, mix)
        mod = _model(zl, sdl, p)
        with torch.no_grad():
            x = mod._model.forward_step({"item_id": ids}, pm).reshape(-1, int(zl["d"]))
        w = mod.get_all_embeddings()["item_embedding"]
        for seed in range(3000):
            _, rec = _run(mod, ids, labels0, pm, tm, seed)
            m = _margin_ok(x, w, pm.reshape(-1), rec["randn"][0], p)
            if m > 1:
                break
        else:
            raise RuntimeError(f"{name}: no seed keeps the top-k margins")
        labels = labels0.clone()
        if collide is not None:   # selections do not depend on the labels: set labels to items of the selecting buckets
            top_x, top_y = rec["topk"][0], rec["topk"][1]
            flat = labels.view(-1)
            for b in range(n_b):
                for i in range(0, bsx, 3 if collide == "partial" else 1):
                    t = int(top_x[b, i])
                    if pm.view(-1)[t]:
                        flat[t] = int(top_y[b, (i // 3) % bsy])
        mod = _model(zl, sdl, p)
        loss, rec = _run(mod, ids, labels, pm, tm, seed)
        if torch.isfinite(loss):
            loss.backward()
        gr = {k: pr.grad for k, pr in mod._model.named_parameters() if pr.grad is not None}
        ek = [k for k in gr if "item_emb" in k]
        wk = [k for k in gr if k.endswith("in_proj_weight")]
        out[f"{name}_params"] = np.array([n_b, bsx, bsy, int(mix)])
        out[f"{name}_seed"] = seed
        out[f"{name}_margin"] = m
        out[f"{name}_labels"] = labels.numpy()
        out[f"{name}_draw"] = rec["randn"][0].numpy()
        out[f"{name}_top_x"] = rec["topk"][0].numpy()
        out[f"{name}_top_y"] = rec["topk"][1].numpy()
        out[f"{name}_loss"] = loss.detach().numpy()
        d_model = int(zl["d"])
        out[f"{name}_gE"] = (gr[ek[0]].numpy().copy() if ek else np.zeros((n_items + 1, d_model), np.float32))
        out[f"{name}_gW"] = (gr[wk[0]].numpy().copy() if wk else np.zeros((3 * d_model, d_model), np.float32))
        print(name, "seed", seed, "margin", round(m, 4), "loss", float(loss))
    np.savez_compressed(os.path.join(OUT, "sce_losses.npz"), **out)
    print("wrote sce_losses")


if __name__ == "__main__":
    gen_sce_losses()
