"""Generate the ConcatAggregator SASRec golden vectors FROM THE REAL REFERENCE (run in the build container only; the reference
checkout is not on the GPU box).  TEST INFRASTRUCTURE.

    python oracle/gen_concat_features_golden.py

Writes tests/golden/sasrec_concat_{d64h2,d50h1_mean,item_only}.npz from ``replay.nn.sequential.SasRec(SasRecBody(...))`` with
``PositionAwareAggregator(ConcatAggregator(...))`` and ``SasRecTransformerLayer``:
- d64h2: d 64 / 2 heads, the item at 64, a categorical at 16, a sum bag at 32 (all-pad bags), a numerical of tensor_dim 3
  at 8 and an identity of width 5; the names put the item in the middle of the sorted order;
- d50h1_mean: d 50 / 1 head (a 50-wide head in a 64-wide slot), mean bags, the reference fixture's widths 11 / 12 / 13 / 14;
- item_only: the item alone, no projection.
Inputs are left-padded as in oracle/gen_side_features_golden.py.  Each file holds the batch, the feature specs with their
embedding widths, the weights as a seed with a checksum, the train loss and every gradient (dropout 0) and the eval
logits.  tests/test_concat_features_cpu.py checks oracle/concat_features.py against them; tests/test_gpu_concat_features.py
the CUDA path.
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
from gen_side_features_golden import side_batch  # noqa: E402
from oracle.side_features import seeded_state_dict, state_dict_checksum  # noqa: E402
from replay.data import FeatureHint, FeatureSource, FeatureType  # noqa: E402
from replay.data.nn import TensorFeatureInfo, TensorFeatureSource, TensorSchema  # noqa: E402
from replay.nn.agg import ConcatAggregator  # noqa: E402
from replay.nn.embedding import SequenceEmbedding  # noqa: E402
from replay.nn.loss import CE  # noqa: E402
from replay.nn.mask import DefaultAttentionMask  # noqa: E402
from replay.nn.sequential import PositionAwareAggregator, SasRec, SasRecBody  # noqa: E402
from replay.nn.sequential.sasrec.transformer import SasRecTransformerLayer  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")
ITEM = "item_id"


def spec(name, kind, dim, cardinality=0, width=1):
    return dict(name=name, kind=kind, cardinality=cardinality, padding_value=cardinality, width=width, dim=dim)


CASES = {
    "d64h2": dict(d=64, H=2, method="sum", seed=51,
                  fs=[spec("genre", "cat", 16, cardinality=12), spec("tags", "bag", 32, cardinality=20, width=4),
                      spec("price", "num", 8, width=3), spec("vec", "ident", 5, width=5)]),
    "d50h1_mean": dict(d=50, H=1, method="mean", seed=52,
                       fs=[spec("cat_list_feature", "bag", 11, cardinality=4, width=3), spec("num_feature", "num", 12),
                           spec("num_list_feature", "num", 13, width=6), spec("emb_list_feature", "ident", 14, width=14)]),
    "item_only": dict(d=64, H=2, method="sum", seed=53, fs=[]),
}


def schema(n_items, d, fs):
    src = [TensorFeatureSource(FeatureSource.INTERACTIONS, ITEM)]
    out = [TensorFeatureInfo(name=ITEM, is_seq=True, cardinality=n_items, padding_value=n_items, embedding_dim=d,
                             feature_type=FeatureType.CATEGORICAL, feature_sources=src, feature_hint=FeatureHint.ITEM_ID)]
    for f in fs:
        kind = {"cat": FeatureType.CATEGORICAL, "bag": FeatureType.CATEGORICAL_LIST, "num": FeatureType.NUMERICAL,
                "ident": FeatureType.NUMERICAL}[f["kind"]]
        extra = (dict(cardinality=f["cardinality"], padding_value=f["padding_value"]) if f["kind"] in ("cat", "bag")
                 else dict(tensor_dim=f["width"]))
        out.append(TensorFeatureInfo(name=f["name"], is_seq=True, embedding_dim=f["dim"], feature_type=kind,
                                     feature_sources=[TensorFeatureSource(FeatureSource.INTERACTIONS, f["name"])], **extra))
    return TensorSchema(out)


def model_of(sch, d, H, L, n_blocks, method, n_items):
    body = SasRecBody(
        embedder=SequenceEmbedding(sch, categorical_list_feature_aggregation_method=method),
        embedding_aggregator=PositionAwareAggregator(
            ConcatAggregator(input_embedding_dims=[x.embedding_dim for x in sch.values()], output_embedding_dim=d),
            max_sequence_length=L, dropout=0.0),
        attn_mask_builder=DefaultAttentionMask(ITEM, H),
        encoder=SasRecTransformerLayer(embedding_dim=d, num_heads=H, num_blocks=n_blocks, dropout=0.0, activation="relu"),
        output_normalization=torch.nn.LayerNorm(d))
    return SasRec(body=body, loss=CE(ignore_index=n_items))


def gen(tag, B=8, L=16, n_items=200, n_blocks=2):
    c = CASES[tag]
    d, H, method, seed, fs = c["d"], c["H"], c["method"], c["seed"], c["fs"]
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    model = model_of(schema(n_items, d, fs), d, H, L, n_blocks, method, n_items)
    keys = list(model.state_dict())
    shapes = [tuple(v.shape) for v in model.state_dict().values()]
    pads = {f"body.embedder.feature_embedders.{f['name']}.emb.weight": f["padding_value"] for f in fs if f["kind"] in ("cat", "bag")}
    pads[f"body.embedder.feature_embedders.{ITEM}.emb.weight"] = n_items
    sd = seeded_state_dict(keys, shapes, seed, pads)
    model.load_state_dict(sd)
    ids, pmask, labels, tmask = make_batch(g, B, L, n_items, n_items)
    feats = side_batch(g, fs, pmask)
    ft = {ITEM: ids, **feats}
    out = dict(sd_seed=seed, sd_keys=np.array(keys), sd_shapes=np.array(["x".join(map(str, t)) for t in shapes]),
               sd_checksum=state_dict_checksum(sd, keys), pad_keys=np.array(list(pads)), pad_rows=np.array(list(pads.values())))
    for k in ("name", "kind", "cardinality", "padding_value", "width", "dim"):
        out[f"f_{k}"] = np.array([f[k] for f in fs], dtype=str if k in ("name", "kind") else np.int64)
    out["f_card"] = out.pop("f_cardinality")
    out["f_pad"] = out.pop("f_padding_value")
    out.update(ids=ids.numpy(), pad_mask=pmask.numpy(), labels=labels.numpy(), target_mask=tmask.numpy(), n_items=n_items,
               d=d, H=H, L=L, n_blocks=n_blocks, method=method, item_name=ITEM)
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
    path = os.path.join(OUT, f"sasrec_concat_{tag}.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, "loss", float(res["loss"]), "bytes", os.path.getsize(path))


if __name__ == "__main__":
    for tag in CASES:
        gen(tag)
