"""Generate the golden vectors of the sampled LogInCESampled / CESampledWeighted losses FROM THE REAL REFERENCE (run in the
build container only; the reference checkout is not on the GPU box).  TEST INFRASTRUCTURE.

    PYTHONPATH=oracle/shim:<reference checkout> python oracle/gen_sampled_ext_golden.py

Writes only tests/golden/sampled_ext_losses.npz (the goldens of oracle/gen_golden.py are left alone: np.savez_compressed
stamps the archive, so rewriting them would change their bytes even where the arrays are the same).  On the weights and
batch of sasrec_new_tiny, for each negative layout (shared [N], per sequence [B, N], per position [B, L, N]), the file
holds the reference's loss and the gradients of the item table and of block 0's ``in_proj_weight`` for
- ``login``: LogInCESampled() with its defaults;
- ``login_clamped``: LogInCESampled(log_epsilon=1e-3, clamp_border=4.37), whose clamp is active on some rows of every
  layout; the border lies at least 0.02 from every row's log(p + eps), so that bf16 logits clamp the same rows;
- ``weighted``: CESampledWeighted(feature_name="w") with seeded weights [B, L, 1] that include zeros and negative values;
plus the negatives (``neg_<layout>``), the weights and the ignore index.  Every layout holds negatives equal to the
ignore index and negatives equal to the row's positive.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from gen_golden import OUT, schema  # noqa: E402
from replay.nn.loss import CESampledWeighted, LogInCESampled  # noqa: E402
from replay.nn.sequential import SasRec  # noqa: E402

IGNORE = 5
N_NEG = 41


def negatives(labels, tm, n_items, g):
    B, L = labels.shape
    negs = {"shared": torch.randint(0, n_items, (N_NEG,), generator=g),
            "perseq": torch.randint(0, n_items, (B, N_NEG), generator=g),
            "perpos": torch.randint(0, n_items, (B, L, N_NEG), generator=g)}
    # collisions with the positive and entries equal to the ignore index in every layout
    negs["shared"][2] = labels[tm][1]
    negs["shared"][11] = IGNORE
    negs["perseq"][:, 3] = labels[:, -1]
    negs["perseq"][2, 6] = IGNORE
    negs["perpos"][:, :, 0] = labels.clamp(max=n_items - 1)
    negs["perpos"][:, :, 17] = labels.clamp(max=n_items - 1)
    negs["perpos"][1, -1, 8] = IGNORE
    return negs


def weights(B, L, g):
    w = torch.rand(B, L, 1, generator=g) * 2.0 - 0.5            # some negative weights
    w[torch.rand(B, L, 1, generator=g) < 0.15] = 0.0           # and some zero weights
    return w


def main():
    z = np.load(os.path.join(OUT, "sasrec_new_tiny.npz"))
    sd = {k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd::")}
    n_items, d, H, L, nb = int(z["n_items"]), int(z["d"]), int(z["H"]), int(z["L"]), int(z["n_blocks"])
    ids, pm = torch.from_numpy(z["ids"]), torch.from_numpy(z["pad_mask"])
    labels, tm = torch.from_numpy(z["labels"]), torch.from_numpy(z["target_mask"])
    B = ids.shape[0]
    g = torch.Generator().manual_seed(123)
    negs = negatives(labels, tm, n_items, g)
    w = weights(B, L, g)
    out = {"ignore_index": IGNORE, "weights": w.numpy()}
    for k, v in negs.items():
        out["neg_" + k] = v.numpy()
    cases = {"login": lambda: LogInCESampled(negative_labels_ignore_index=IGNORE),
             "login_clamped": lambda: LogInCESampled(log_epsilon=1e-3, clamp_border=4.37, negative_labels_ignore_index=IGNORE),
             "weighted": lambda: CESampledWeighted(feature_name="w", negative_labels_ignore_index=IGNORE)}
    for name, mk in cases.items():
        for shape, neg in negs.items():
            model = SasRec.from_params(schema(n_items, d, n_items), embedding_dim=d, num_heads=H, num_blocks=nb,
                                       max_sequence_length=L, dropout=0.0)
            model.load_state_dict(sd)
            model.loss = mk()
            model.loss.logits_callback = model.get_logits
            model.train()
            res = model(feature_tensors={"item_id": ids, "w": w}, padding_mask=pm, positive_labels=labels.unsqueeze(-1),
                        negative_labels=neg, target_padding_mask=tm.unsqueeze(-1).clone())
            res["loss"].backward()
            gr = {k: p.grad for k, p in model.named_parameters() if p.grad is not None}
            ek = [k for k in gr if "item_id" in k or "item_emb" in k]
            wk = [k for k in gr if k.endswith("in_proj_weight")]
            out[f"{name}_{shape}_loss"] = res["loss"].detach().numpy()
            out[f"{name}_{shape}_gE"] = gr[ek[0]].numpy().copy()
            out[f"{name}_{shape}_gW"] = gr[wk[0]].numpy().copy()
            print(name, shape, float(res["loss"]), ek[0], wk[0])
    np.savez_compressed(os.path.join(OUT, "sampled_ext_losses.npz"), **out)
    print("wrote sampled_ext_losses")


if __name__ == "__main__":
    main()
