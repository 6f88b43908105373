"""Generate the golden vectors of the multi-positive losses FROM THE REAL REFERENCE (run in the build container only; the
reference checkout is not on the GPU box).  TEST INFRASTRUCTURE.

    PYTHONPATH=oracle/shim:<reference checkout> python oracle/gen_multi_positive_golden.py

Writes only tests/golden/multi_positive_losses.npz.  On the weights and sequences of sasrec_new_tiny with P = 3 positives per
position (``labels`` / ``target_mask`` [B, L, 3]), the file holds the reference's loss and the gradients of the item table
and of block 0's ``in_proj_weight`` for BCE(), CESampled, BCESampled and CESampledWeighted(feature_name="w") with weights
[B, L, 3], each sampled loss at every negative layout (``neg_<layout>``: shared [N], per sequence [B, N], per position
[B, L, N]).  Slot 0 is the golden's own target; slots 1 and 2 hold other items, set on part of the live positions, so the
batch has padded slots inside live rows, live positions with one set slot, and a duplicated id within a row.  Every layout
holds negatives equal to a non-first positive, to a padded slot's value and to the ignore index.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from gen_golden import OUT, schema  # noqa: E402
from replay.nn.loss import BCE, BCESampled, CESampled, CESampledWeighted  # noqa: E402
from replay.nn.sequential import SasRec  # noqa: E402

IGNORE = 5
N_NEG = 37
P = 3


def targets(labels, tm, n_items, g):
    """[B, L, P] labels and mask from the golden's [B, L] targets."""
    B, L = labels.shape
    lab = torch.randint(0, n_items, (B, L, P), generator=g)
    lab[..., 0] = labels
    m = torch.zeros(B, L, P, dtype=torch.bool)
    m[..., 0] = tm
    m[..., 1] = tm & (torch.rand(B, L, generator=g) < 0.6)
    m[..., 2] = tm & (torch.rand(B, L, generator=g) < 0.5)
    live = tm.nonzero()
    b, l = live[0].tolist()
    m[b, l, 1:] = False                      # one set slot
    b, l = live[1].tolist()
    m[b, l, :] = True
    lab[b, l, 2] = lab[b, l, 0]              # a duplicated id, both slots set
    b, l = live[2].tolist()
    m[b, l, 1], m[b, l, 2] = True, False     # a padded slot after a set one
    return lab, m


def negatives(lab, m, n_items, g):
    B, L, _ = lab.shape
    live = m.any(-1).nonzero()
    b0, l0 = live[2].tolist()                # lab[b0, l0, 1] is set, lab[b0, l0, 2] is padded
    negs = {"shared": torch.randint(0, n_items, (N_NEG,), generator=g),
            "perseq": torch.randint(0, n_items, (B, N_NEG), generator=g),
            "perpos": torch.randint(0, n_items, (B, L, N_NEG), generator=g)}
    negs["shared"][1] = lab[b0, l0, 1]
    negs["shared"][4] = lab[b0, l0, 2]
    negs["shared"][9] = IGNORE
    negs["perseq"][:, 2] = lab[:, -1, 1]
    negs["perseq"][:, 3] = lab[:, -1, 2]
    negs["perseq"][b0, 5] = IGNORE
    negs["perpos"][:, :, 0] = lab[..., 1]
    negs["perpos"][:, :, 7] = lab[..., 2]
    negs["perpos"][b0, l0, 8] = IGNORE
    return negs


def main():
    z = np.load(os.path.join(OUT, "sasrec_new_tiny.npz"))
    sd = {k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd::")}
    n_items, d, H, L, nb = int(z["n_items"]), int(z["d"]), int(z["H"]), int(z["L"]), int(z["n_blocks"])
    ids, pm = torch.from_numpy(z["ids"]), torch.from_numpy(z["pad_mask"])
    g = torch.Generator().manual_seed(321)
    lab, m = targets(torch.from_numpy(z["labels"]), torch.from_numpy(z["target_mask"]), n_items, g)
    negs = negatives(lab, m, n_items, g)
    w = torch.rand(*lab.shape, generator=g) * 2.0 - 0.5
    out = {"ignore_index": IGNORE, "labels": lab.numpy(), "target_mask": m.numpy(), "weights": w.numpy()}
    for k, v in negs.items():
        out["neg_" + k] = v.numpy()
    cases = {"bce": (lambda: BCE(), ["none"]),
             "ce_sampled": (lambda: CESampled(negative_labels_ignore_index=IGNORE), list(negs)),
             "bce_sampled": (lambda: BCESampled(negative_labels_ignore_index=IGNORE), list(negs)),
             "ce_sampled_weighted": (lambda: CESampledWeighted(feature_name="w", negative_labels_ignore_index=IGNORE),
                                     list(negs))}
    for name, (mk, shapes) in cases.items():
        for shape in shapes:
            model = SasRec.from_params(schema(n_items, d, n_items), embedding_dim=d, num_heads=H, num_blocks=nb,
                                       max_sequence_length=L, dropout=0.0)
            model.load_state_dict(sd)
            model.loss = mk()
            model.loss.logits_callback = model.get_logits
            model.train()
            res = model(feature_tensors={"item_id": ids, "w": w}, padding_mask=pm, positive_labels=lab.clone(),
                        negative_labels=negs.get(shape), target_padding_mask=m.clone())
            res["loss"].backward()
            gr = {k: p.grad for k, p in model.named_parameters() if p.grad is not None}
            ek = [k for k in gr if "item_id" in k or "item_emb" in k]
            wk = [k for k in gr if k.endswith("in_proj_weight")]
            out[f"{name}_{shape}_loss"] = res["loss"].detach().numpy()
            out[f"{name}_{shape}_gE"] = gr[ek[0]].numpy().copy()
            out[f"{name}_{shape}_gW"] = gr[wk[0]].numpy().copy()
            print(name, shape, float(res["loss"]), ek[0], wk[0])
    np.savez_compressed(os.path.join(OUT, "multi_positive_losses.npz"), **out)
    print("wrote multi_positive_losses")


if __name__ == "__main__":
    main()
