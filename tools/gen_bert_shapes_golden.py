"""Golden vectors of BERT4Rec at hidden sizes that the kernels see padded, FROM THE REAL REFERENCE (run where the reference
source is installed; the tests only read the result).

    python tools/gen_bert_shapes_golden.py /path/to/reference

For every shape of tests/bert_shapes_golden.py SHAPES it runs oracle.gen_golden.gen_bert4rec (the reference's Bert4RecModel,
CE over the real and masked positions, one backward, eval logits) with the weights drawn by ``golden_weights`` instead of
the reference's own init, and writes tests/golden/bert4rec_<tag>.npz without the weights (the seed regenerates them) and
with every gradient packed by ``pack_grads`` (float16, large matrices as a subset of their rows).  It also writes tests/golden/bert4rec_bce_d300h4.npz: the legacy Bert4Rec(loss_type="BCE")
loss on the d300h4 weights and batch and the gradients tools/gen_bce_golden.py keeps for the tiny shapes."""
import os
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle", "shim"))
sys.path.insert(1, sys.argv[1] if len(sys.argv) > 1 else "/root/reference")
sys.path.insert(2, ROOT)
sys.path.insert(3, os.path.join(ROOT, "tests"))
warnings.filterwarnings("ignore")

import oracle.gen_golden as gg  # noqa: E402
from bert_shapes_golden import SHAPES, golden_weights, load, pack_grads  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def _meta(module, seed):
    names, shapes = [], []
    for k, p in module.named_parameters():
        names.append(k)
        shapes.append(list(p.shape) + [0] * (2 - p.dim()))
    return dict(param_names=np.array(names), param_shapes=np.array(shapes, dtype=np.int64), init_seed=np.int64(seed))


def gen_shape(tag):
    d, H, tied, n_items, nb, B, L, seed = SHAPES[tag]
    meta = {}

    def set_weights(model, g):   # replaces gen_golden's perturbation of the reference init
        meta.update(_meta(model, seed + 1000))
        w = golden_weights(list(meta["param_names"]), [s[s > 0] for s in meta["param_shapes"]], seed + 1000)
        with torch.no_grad():
            for k, p in model.named_parameters():
                p.copy_(w[k])

    orig, gg.randomise_small_params = gg.randomise_small_params, set_weights
    try:
        gg.gen_bert4rec(tag, B=B, L=L, d=d, H=H, n_items=n_items, n_blocks=nb, seed=seed, tying=tied)
    finally:
        gg.randomise_small_params = orig
    path = os.path.join(GOLDEN, f"bert4rec_{tag}.npz")
    z = dict(np.load(path))
    grads = {k[6:]: v for k, v in z.items() if k.startswith("grad::")}
    out = {k: v for k, v in z.items() if not k.startswith(("sd::", "grad::"))}
    out.update(meta)
    out.update(pack_grads(grads))
    np.savez_compressed(path, **out)
    print("packed", os.path.basename(path), os.path.getsize(path), "bytes")


def gen_bce(tag):
    from replay.models.nn.sequential.bert4rec.lightning import Bert4Rec

    z, sd, _ = load(os.path.join(GOLDEN, f"bert4rec_{tag}.npz"))
    n_items, d, H, L, nb, tying = (int(z[k]) for k in ("n_items", "d", "H", "L", "n_blocks", "tying"))
    m = Bert4Rec(gg.schema(n_items, d, 0), block_count=nb, head_count=H, hidden_size=d, max_seq_len=L, dropout_rate=0.0,
                 enable_embedding_tying=bool(tying), loss_type="BCE")
    m._model.load_state_dict(sd, strict=False)
    m.train()
    ids, pm, tok = (torch.from_numpy(z[k]) for k in ("ids", "pad_mask", "token_mask"))
    loss = m._compute_loss_bce({"item_id": ids}, torch.from_numpy(z["labels"]), pm, tok)
    loss.backward()
    # the gradients tools/gen_bce_golden.py keeps: item table, block 0's in_proj_weight, the head weight and its bias
    keep = ("item_embedder.cat_embeddings.item_id.weight", "transformer_blocks.0.attention.in_proj_weight", "_head.linear.weight",
            "_head.linear.bias", "_head.out_bias")
    grads = {k: p.grad.numpy().copy() for k, p in m._model.named_parameters() if k in keep}
    out = dict(source=np.array(f"bert4rec_{tag}.npz"), train_loss=loss.detach().numpy())
    out.update(pack_grads(grads))
    path = os.path.join(GOLDEN, f"bert4rec_bce_{tag}.npz")
    np.savez_compressed(path, **out)
    print("wrote", os.path.basename(path), "loss", float(loss), os.path.getsize(path), "bytes")


def main():
    for tag in SHAPES:
        if "bce" not in sys.argv[2:]:
            gen_shape(tag)
    gen_bce("d300h4")


if __name__ == "__main__":
    main()
