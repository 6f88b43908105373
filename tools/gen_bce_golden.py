"""Golden vectors of the full-catalog BCE loss FROM THE REAL REFERENCE classes (run where the reference source is
installed; the GPU tests only read the result).

    python tools/gen_bce_golden.py /path/to/reference

Reads tests/golden/sasrec_new_tiny.npz, bert4rec_tiny.npz and bert4rec_tiny_tied.npz (weights and batches) and writes
tests/golden/full_bce_losses.npz:
  new_{loss,gE,gW}            replay.nn.loss.BCE through the new-path SasRec (replay/nn/loss/bce.py:10-95)
  bert_{untied,tied}_{loss,gE,gW,gHead,gBias}
                              legacy Bert4Rec(loss_type="BCE")._compute_loss_bce (bert4rec/lightning.py:273-305)
gE = item table, gW = in_proj_weight of block 0, gHead / gBias = the untied Linear head (gHead absent when tied, where the
head is the item table) and its bias or the tied head's out_bias."""
import os
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle", "shim"))
sys.path.insert(1, sys.argv[1] if len(sys.argv) > 1 else "/root/reference")
warnings.filterwarnings("ignore")

from replay.data import FeatureHint, FeatureSource, FeatureType  # noqa: E402
from replay.data.nn import TensorFeatureInfo, TensorFeatureSource, TensorSchema  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def schema(n_items, d, pad):
    return TensorSchema([TensorFeatureInfo(name="item_id", is_seq=True, cardinality=n_items, padding_value=pad, embedding_dim=d,
                                           feature_type=FeatureType.CATEGORICAL,
                                           feature_sources=[TensorFeatureSource(FeatureSource.INTERACTIONS, "item_id")],
                                           feature_hint=FeatureHint.ITEM_ID)])


def load(name):
    z = np.load(os.path.join(GOLDEN, name))
    return z, {k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd::")}


def gen_new_path(out):
    from replay.nn.loss import BCE
    from replay.nn.sequential import SasRec

    z, sd = load("sasrec_new_tiny.npz")
    n_items, d, H, L, nb = int(z["n_items"]), int(z["d"]), int(z["H"]), int(z["L"]), int(z["n_blocks"])
    model = SasRec.from_params(schema(n_items, d, n_items), embedding_dim=d, num_heads=H, num_blocks=nb, max_sequence_length=L,
                               dropout=0.0)
    model.load_state_dict(sd)
    model.loss = BCE()
    model.loss.logits_callback = model.get_logits
    model.train()
    ids, pm = torch.from_numpy(z["ids"]), torch.from_numpy(z["pad_mask"])
    labels, tm = torch.from_numpy(z["labels"]), torch.from_numpy(z["target_mask"])
    res = model(feature_tensors={"item_id": ids}, padding_mask=pm, positive_labels=labels.unsqueeze(-1), negative_labels=None,
                target_padding_mask=tm.unsqueeze(-1).clone())
    res["loss"].backward()
    gr = {k: p.grad for k, p in model.named_parameters() if p.grad is not None}
    out["new_loss"] = res["loss"].detach().numpy()
    out["new_gE"] = gr[[k for k in gr if "item_id" in k or "item_emb" in k][0]].numpy().copy()
    out["new_gW"] = gr[[k for k in gr if k.endswith("in_proj_weight")][0]].numpy().copy()
    print("new-path BCE", float(res["loss"]))


def gen_bert(out, tag):
    from replay.models.nn.sequential.bert4rec.lightning import Bert4Rec

    z, sd = load(f"bert4rec_{tag}.npz")
    n_items, d, H, L, nb, tying = (int(z[k]) for k in ("n_items", "d", "H", "L", "n_blocks", "tying"))
    m = Bert4Rec(schema(n_items, d, 0), block_count=nb, head_count=H, hidden_size=d, max_seq_len=L, dropout_rate=0.0,
                 enable_embedding_tying=bool(tying), loss_type="BCE")
    m._model.load_state_dict(sd)
    m.train()
    ids, pm, tok = (torch.from_numpy(z[k]) for k in ("ids", "pad_mask", "token_mask"))
    loss = m._compute_loss_bce({"item_id": ids}, torch.from_numpy(z["labels"]), pm, tok)
    loss.backward()
    gr = {k: p.grad for k, p in m._model.named_parameters() if p.grad is not None}
    name = "tied" if tying else "untied"
    out[f"bert_{name}_loss"] = loss.detach().numpy()
    out[f"bert_{name}_gE"] = gr["item_embedder.cat_embeddings.item_id.weight"].numpy().copy()
    out[f"bert_{name}_gW"] = gr["transformer_blocks.0.attention.in_proj_weight"].numpy().copy()
    if tying:
        out[f"bert_{name}_gBias"] = gr["_head.out_bias"].numpy().copy()
    else:
        out[f"bert_{name}_gHead"] = gr["_head.linear.weight"].numpy().copy()
        out[f"bert_{name}_gBias"] = gr["_head.linear.bias"].numpy().copy()
    print("bert4rec BCE", name, float(loss))


def main():
    torch.manual_seed(0)
    out = {}
    gen_new_path(out)
    gen_bert(out, "tiny")
    gen_bert(out, "tiny_tied")
    np.savez_compressed(os.path.join(GOLDEN, "full_bce_losses.npz"), **out)
    print("wrote full_bce_losses.npz")


if __name__ == "__main__":
    main()
