"""Generate the side-feature SASRec golden vectors FROM THE REAL REFERENCE (run in the build container only; the reference
checkout is not on the GPU box).  TEST INFRASTRUCTURE.

    python oracle/gen_side_features_golden.py

Writes tests/golden/sasrec_side_{d64h2_sum,d50h1_mean}.npz from ``replay.nn.sequential.SasRec.from_params`` on a schema
with the item id, two categoricals (one of cardinality 1), two categorical lists (K 3 and 5, with all-pad bags), numerical
features of tensor_dim 1 and 7 and an identity numerical (tensor_dim = d).  The reference takes one bag aggregation per
model, so the d 64 case sums its bags and the d 50 case (50-wide head in a 64-wide slot) averages them.  Inputs are
left-padded; numerical values at pad positions are non-zero and categorical pads hold the padding value.  Each file holds
the batch, the weights as a seed with a checksum (oracle.side_features.seeded_state_dict), the train loss and every
gradient (dropout 0) and the eval logits.  tests/test_side_features_cpu.py checks oracle/side_features.py against them;
tests/test_gpu_side_features.py the CUDA path.
"""
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "shim"))
sys.path.insert(1, "/root/reference")
sys.path.insert(2, HERE)
sys.path.insert(3, os.path.dirname(HERE))
warnings.filterwarnings("ignore")

from gen_golden import make_batch  # noqa: E402
from oracle.side_features import seeded_state_dict, state_dict_checksum  # noqa: E402
from replay.data import FeatureHint, FeatureSource, FeatureType  # noqa: E402
from replay.data.nn import TensorFeatureInfo, TensorFeatureSource, TensorSchema  # noqa: E402
from replay.nn.sequential import SasRec  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")


def specs(d):
    return [dict(name="genre", kind="cat", cardinality=12, padding_value=12, width=1),
            dict(name="flag", kind="cat", cardinality=1, padding_value=1, width=1),
            dict(name="tags", kind="bag", cardinality=20, padding_value=20, width=3),
            dict(name="cats", kind="bag", cardinality=15, padding_value=15, width=5),
            dict(name="price", kind="num", cardinality=0, padding_value=0, width=1),
            dict(name="stats", kind="num", cardinality=0, padding_value=0, width=7),
            dict(name="vec", kind="ident", cardinality=0, padding_value=0, width=d)]


def schema(n_items, d, fs):
    src = [TensorFeatureSource(FeatureSource.INTERACTIONS, "item_id")]
    out = [TensorFeatureInfo(name="item_id", is_seq=True, cardinality=n_items, padding_value=n_items, embedding_dim=d,
                             feature_type=FeatureType.CATEGORICAL, feature_sources=src, feature_hint=FeatureHint.ITEM_ID)]
    for f in fs:
        kind = {"cat": FeatureType.CATEGORICAL, "bag": FeatureType.CATEGORICAL_LIST, "num": FeatureType.NUMERICAL,
                "ident": FeatureType.NUMERICAL}[f["kind"]]
        extra = (dict(cardinality=f["cardinality"], padding_value=f["padding_value"]) if f["kind"] in ("cat", "bag")
                 else dict(tensor_dim=f["width"]))
        out.append(TensorFeatureInfo(name=f["name"], is_seq=True, embedding_dim=d, feature_type=kind,
                                     feature_sources=[TensorFeatureSource(FeatureSource.INTERACTIONS, f["name"])], **extra))
    return TensorSchema(out)


def side_batch(g, fs, pmask):
    """Side-feature tensors of a left-padded batch: categorical pads hold the padding value, numerical pads are non-zero."""
    B, L = pmask.shape
    out = {}
    for f in fs:
        if f["kind"] == "cat":
            v = torch.randint(0, f["cardinality"], (B, L), generator=g)
            v[torch.rand(B, L, generator=g) < 0.15] = f["padding_value"]   # padding ids inside real positions too
            out[f["name"]] = v.masked_fill(~pmask, f["padding_value"])
        elif f["kind"] == "bag":
            K = f["width"]
            v = torch.randint(0, f["cardinality"], (B, L, K), generator=g)
            v[torch.rand(B, L, K, generator=g) < 0.35] = f["padding_value"]
            v[torch.rand(B, L, generator=g) < 0.15] = f["padding_value"]  # all-pad bags at real positions
            out[f["name"]] = v.masked_fill(~pmask.unsqueeze(-1), f["padding_value"])
        else:
            shape = (B, L) if f["width"] == 1 else (B, L, f["width"])
            out[f["name"]] = torch.randn(shape, generator=g)
    return out


def gen(tag, B, L, d, H, n_items, n_blocks, seed, method):
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    fs = specs(d)
    model = SasRec.from_params(schema(n_items, d, fs), embedding_dim=d, num_heads=H, num_blocks=n_blocks,
                               max_sequence_length=L, dropout=0.0, categorical_list_feature_aggregation_method=method)
    keys = list(model.state_dict())
    shapes = [tuple(v.shape) for v in model.state_dict().values()]
    pads = {f"body.embedder.feature_embedders.{f['name']}.emb.weight": f["padding_value"] for f in fs if f["kind"] in ("cat", "bag")}
    pads["body.embedder.feature_embedders.item_id.emb.weight"] = n_items
    sd = seeded_state_dict(keys, shapes, seed, pads)
    model.load_state_dict(sd)
    ids, pmask, labels, tmask = make_batch(g, B, L, n_items, n_items)
    feats = side_batch(g, fs, pmask)
    ft = {"item_id": ids, **feats}
    out = dict(sd_seed=seed, sd_keys=np.array(keys), sd_shapes=np.array(["x".join(map(str, t)) for t in shapes]),
               sd_checksum=state_dict_checksum(sd, keys), pad_keys=np.array(list(pads)), pad_rows=np.array(list(pads.values())))
    out.update({f"f_{k}": np.array([f[k] for f in fs]) for k in ("name", "kind", "padding_value", "width")})
    out["f_card"] = np.array([f["cardinality"] for f in fs])
    out["f_pad"] = out.pop("f_padding_value")
    out.update(ids=ids.numpy(), pad_mask=pmask.numpy(), labels=labels.numpy(), target_mask=tmask.numpy(), n_items=n_items,
               d=d, H=H, L=L, n_blocks=n_blocks, method=method)
    out.update({"feat::" + k: v.numpy() for k, v in feats.items()})
    model.train()
    res = model(feature_tensors=ft, padding_mask=pmask, positive_labels=labels.unsqueeze(-1), negative_labels=None,
                target_padding_mask=tmask.unsqueeze(-1))
    res["loss"].backward()
    out["train_loss"] = res["loss"].detach().numpy()
    for k, p in model.named_parameters():
        out["grad::" + k] = (p.grad if p.grad is not None else torch.zeros_like(p)).numpy().copy()
    model.eval()
    with torch.no_grad():
        out["eval_logits"] = model(feature_tensors=ft, padding_mask=pmask)["logits"].numpy()
    path = os.path.join(OUT, f"sasrec_side_{tag}.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, "loss", float(res["loss"]), "bytes", os.path.getsize(path))


if __name__ == "__main__":
    gen("d64h2_sum", B=8, L=16, d=64, H=2, n_items=200, n_blocks=2, seed=41, method="sum")
    gen("d50h1_mean", B=8, L=16, d=50, H=1, n_items=200, n_blocks=2, seed=42, method="mean")
