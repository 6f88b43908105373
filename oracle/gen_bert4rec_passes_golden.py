"""Generate the golden vectors of BERT4Rec's body options and catalog growth FROM THE REAL REFERENCE (run in the build
container only; the reference checkout is not on the GPU box).  TEST INFRASTRUCTURE.

    PYTHONPATH=oracle/shim:<reference checkout> python oracle/gen_bert4rec_passes_golden.py

Writes only the files below (the goldens of oracle/gen_golden.py are left alone: np.savez_compressed stamps the archive,
so rewriting them would change their bytes even where the arrays are the same):
- tests/golden/bert4rec_p2_d64h2.npz: 2 blocks x 2 passes, positional embedding, untied head, d 64, 2 heads;
- tests/golden/bert4rec_nopos_tied.npz: no positional embedding, tied head, 1 pass;
- tests/golden/bert4rec_p3_nopos_d96h2.npz: 1 block x 3 passes, no positional embedding, untied, d 96, 2 heads (48-wide
  heads in 64-wide feature slots);
- tests/golden/bert4rec_resize_shapes.npz: the state_dict shapes of the reference's Lightning ``Bert4Rec`` after each
  catalog-growth call, tied and untied.
Each model file holds the seeded batch, the train-mode hidden states, loss and gradients (dropout 0) and the eval logits
of ``predict``, as gen_golden.gen_bert4rec writes them, plus ``passes`` and ``positional``.  The weights are not stored:
oracle.bert4rec_passes.seeded_state_dict draws them from ``sd_seed`` in the order of ``sd_keys``, and
``golden_state_dict`` regenerates them and checks them against ``sd_checksum``.  This keeps each file under 0.8 MB.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from gen_golden import OUT, schema  # noqa: E402
from replay.models.nn.sequential.bert4rec.model import Bert4RecModel  # noqa: E402

sys.path.insert(0, os.path.dirname(HERE))
from oracle.bert4rec_passes import seeded_state_dict, state_dict_checksum  # noqa: E402


def gen_bert4rec_case(tag, B, L, d, H, n_items, n_blocks, seed, tying, passes, positional):
    """gen_golden.gen_bert4rec with the reference's num_passes_over_block and enable_positional_embedding."""
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    model = Bert4RecModel(schema(n_items, d, 0), max_len=L, hidden_size=d, num_blocks=n_blocks, num_heads=H,
                          num_passes_over_block=passes, dropout=0.0, enable_positional_embedding=positional,
                          enable_embedding_tying=tying)
    # the weights are drawn from a seed and not stored: the file keeps the seed, the key order, the shapes and a checksum
    keys = list(model.state_dict())
    shapes = [tuple(v.shape) for v in model.state_dict().values()]
    sd = seeded_state_dict(keys, shapes, seed)
    model.load_state_dict(sd)
    lens = torch.randint(2, L + 1, (B,), generator=g)
    lens[0] = L
    ids = torch.zeros(B, L, dtype=torch.int64)
    pmask = torch.zeros(B, L, dtype=torch.bool)
    for b in range(B):
        n = int(lens[b])
        ids[b, L - n:] = torch.randint(0, n_items, (n,), generator=g)
        pmask[b, L - n:] = True
    tok = (torch.rand(B, L, generator=g) > 0.3) & pmask
    tok[:, -1] = False
    labels = ids.clone()
    out = dict(sd_seed=seed, sd_keys=np.array(keys), sd_shapes=np.array(["x".join(map(str, t)) for t in shapes]),
               sd_checksum=state_dict_checksum(sd, keys))
    out.update(ids=ids.numpy(), pad_mask=pmask.numpy(), token_mask=tok.numpy(), labels=labels.numpy(), n_items=n_items, d=d,
               H=H, L=L, n_blocks=n_blocks, tying=int(tying), passes=passes, positional=int(positional))
    model.train()
    hidden = model.forward_step({"item_id": ids}, pmask, tok)
    logits = model.get_logits(hidden)
    masked = ~((~pmask) + tok)   # bert4rec/lightning.py:332-351
    loss = torch.nn.CrossEntropyLoss()(logits[masked], labels[masked])
    loss.backward()
    out["train_hidden"] = hidden.detach().numpy()
    out["train_loss"] = loss.detach().numpy()
    for k, p in model.named_parameters():
        out["grad::" + k] = (p.grad if p.grad is not None else torch.zeros_like(p)).numpy().copy()
    model.eval()
    with torch.no_grad():
        out["eval_logits"] = model.predict({"item_id": ids}, pmask, tok).numpy()
    np.savez_compressed(os.path.join(OUT, f"bert4rec_{tag}.npz"), **out)
    print("wrote bert4rec_" + tag, "loss", float(loss), "keys", len(keys))


def gen_resize_shapes():
    from replay.models.nn.sequential.bert4rec.lightning import Bert4Rec

    n_items, d = 40, 64
    out = {"n_items": n_items, "d": d}
    for tying in (False, True):
        for op, arg in (("by_size", 47), ("by_tensor", torch.rand(45, d)), ("append", torch.rand(3, d))):
            torch.manual_seed(3)
            m = Bert4Rec(schema(n_items, d, 0), block_count=2, head_count=2, hidden_size=d, max_seq_len=16,
                         dropout_rate=0.0, enable_embedding_tying=tying)
            getattr(m, {"by_size": "set_item_embeddings_by_size", "by_tensor": "set_item_embeddings_by_tensor",
                        "append": "append_item_embeddings"}[op])(arg)
            tag = f"{'tied' if tying else 'untied'}_{op}"
            for k, v in m.state_dict().items():
                out[f"{tag}::{k}"] = np.asarray(v.shape, dtype=np.int64)
            print(tag, {k: tuple(v.shape) for k, v in m.state_dict().items() if "item" in k or "_head" in k})
    np.savez_compressed(os.path.join(OUT, "bert4rec_resize_shapes.npz"), **out)
    print("wrote bert4rec_resize_shapes")


if __name__ == "__main__":
    gen_bert4rec_case("p2_d64h2", B=6, L=16, d=64, H=2, n_items=300, n_blocks=2, seed=31, tying=False, passes=2,
                      positional=True)
    gen_bert4rec_case("nopos_tied", B=6, L=16, d=64, H=1, n_items=300, n_blocks=2, seed=32, tying=True, passes=1,
                      positional=False)
    gen_bert4rec_case("p3_nopos_d96h2", B=6, L=16, d=96, H=2, n_items=300, n_blocks=1, seed=33, tying=False, passes=3,
                      positional=False)
    gen_resize_shapes()
