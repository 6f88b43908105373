"""Generate the golden vectors of the legacy BERT4Rec with side features FROM THE REAL REFERENCE (run in the build
container only; the reference checkout is not on the GPU box).  TEST INFRASTRUCTURE.

    python oracle/gen_bert4rec_side_features_golden.py

Writes tests/golden/bert4rec_side_{d64h2,d300h4,d96h2_tied_bce}.npz from the reference's Lightning ``Bert4Rec`` on a schema
whose item id is followed by categorical features (one of cardinality 1) and NUMERICAL / NUMERICAL_LIST features of
tensor_dim d, all summed into the item embedding (BertEmbedding, bert4rec/model.py:173-296):
- d64h2: d 64, 2 heads, untied head, positional embedding, CE, two categoricals and two numericals;
- d300h4: d 300, 4 heads (75-wide heads in 128-wide feature slots), untied, CE, one categorical and a numerical of width 300,
  and no transformer block (the embedding feeds the head directly), which keeps the file small;
- d96h2_tied_bce: d 96, 2 heads, tied head, no positional embedding, 2 passes per block, BCE.
The batch is left-padded, its token masks come from the reference's uniform masker, categorical ids include the padding
value at real positions and numerical values are non-zero at pads.  Each file holds that batch, the weights as a seed with
a checksum (oracle.bert4rec_passes.seeded_state_dict), the train loss and every gradient (dropout 0), and the eval logits of
``predict`` on the batch shifted as the prediction dataset shifts it (dataset.py:322-345).
tests/test_bert4rec_side_features_cpu.py checks oracle/bert4rec_side_features.py against them; the GPU tests the CUDA path.
"""
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "shim"))
sys.path.insert(1, "/root/reference")
sys.path.insert(2, os.path.dirname(HERE))
warnings.filterwarnings("ignore")

from oracle.bert4rec_passes import seeded_state_dict, state_dict_checksum  # noqa: E402
from replay.data import FeatureHint, FeatureSource, FeatureType  # noqa: E402
from replay.data.nn import TensorFeatureInfo, TensorFeatureSource, TensorSchema  # noqa: E402
from replay.models.nn.sequential.bert4rec.dataset import Bert4RecUniformMasker  # noqa: E402
from replay.models.nn.sequential.bert4rec.lightning import Bert4Rec  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")
_TYPES = {"cat": FeatureType.CATEGORICAL, "num": FeatureType.NUMERICAL, "num_list": FeatureType.NUMERICAL_LIST}


def schema(n_items, d, fs):
    out = [TensorFeatureInfo(name="item_id", is_seq=True, cardinality=n_items, padding_value=0, embedding_dim=d,
                             feature_type=FeatureType.CATEGORICAL, feature_hint=FeatureHint.ITEM_ID,
                             feature_sources=[TensorFeatureSource(FeatureSource.INTERACTIONS, "item_id")])]
    for f in fs:
        extra = (dict(cardinality=f["cardinality"], padding_value=f["padding_value"], embedding_dim=d) if f["kind"] == "cat"
                 else dict(tensor_dim=d))
        out.append(TensorFeatureInfo(name=f["name"], is_seq=True, feature_type=_TYPES[f["kind"]],
                                     feature_sources=[TensorFeatureSource(FeatureSource.INTERACTIONS, f["name"])], **extra))
    return TensorSchema(out)


def batch(g, B, L, n_items, d, fs, mask_prob=0.3):
    lens = torch.randint(2, L + 1, (B,), generator=g)
    lens[0] = L
    pm = torch.arange(L)[None, :] >= (L - lens)[:, None]
    ids = torch.where(pm, torch.randint(0, n_items, (B, L), generator=g), torch.zeros(B, L, dtype=torch.int64))
    masker = Bert4RecUniformMasker(mask_prob, generator=g)
    tok = torch.stack([masker.mask(pm[b]) for b in range(B)])
    feats = {}
    for f in fs:
        if f["kind"] == "cat":
            v = torch.randint(0, f["cardinality"], (B, L), generator=g)
            v[torch.rand(B, L, generator=g) < 0.2] = f["padding_value"]   # the padding value at real positions: a real row
            feats[f["name"]] = v.masked_fill(~pm, f["padding_value"])
        else:
            feats[f["name"]] = torch.randn(B, L, d, generator=g)           # non-zero at pads too
    return ids, pm, tok, feats


def shifted(sch, ft, pm):
    """_shift_features (dataset.py:322-345) row by row: every feature rolled left, the last position its padding value,
    token mask = the rolled padding mask, padding mask the same with the last position real."""
    out = {}
    for name, info in sch.items():
        v = torch.roll(ft[name], -1, dims=1)
        v[:, -1] = info.padding_value
        out[name] = v
    tok = torch.roll(pm, -1, dims=1)
    tok[:, -1] = False
    pm2 = tok.clone()
    pm2[:, -1] = True
    return out, pm2, tok


def gen(tag, B, L, d, H, n_items, n_blocks, seed, fs, tying=False, positional=True, passes=1, loss="CE"):
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    sch = schema(n_items, d, fs)
    mod = Bert4Rec(sch, block_count=n_blocks, head_count=H, hidden_size=d, max_seq_len=L, dropout_rate=0.0,
                   pass_per_transformer_block_count=passes, enable_positional_embedding=positional,
                   enable_embedding_tying=tying, loss_type=loss)
    model = mod._model
    keys = list(model.state_dict())
    shapes = [tuple(v.shape) for v in model.state_dict().values()]
    sd = seeded_state_dict(keys, shapes, seed)
    model.load_state_dict(sd)
    ids, pm, tok, feats = batch(g, B, L, n_items, d, fs)
    ft = {"item_id": ids, **feats}
    out = dict(sd_seed=seed, sd_keys=np.array(keys), sd_shapes=np.array(["x".join(map(str, t)) for t in shapes]),
               sd_checksum=state_dict_checksum(sd, keys))
    out.update(f_name=np.array([f["name"] for f in fs]), f_kind=np.array([f["kind"] for f in fs]),
               f_card=np.array([f.get("cardinality", 0) for f in fs]), f_pad=np.array([f.get("padding_value", 0) for f in fs]))
    out.update(ids=ids.numpy(), pad_mask=pm.numpy(), token_mask=tok.numpy(), labels=ids.numpy(), n_items=n_items, d=d, H=H,
               L=L, n_blocks=n_blocks, tying=int(tying), passes=passes, positional=int(positional), loss=loss)
    out.update({"feat::" + k: v.numpy() for k, v in feats.items()})
    mod.train()
    fn = mod._compute_loss_ce if loss == "CE" else mod._compute_loss_bce
    res = fn(ft, ids, pm, tok)
    res.backward()
    out["train_loss"] = res.detach().numpy()
    for k, p in model.named_parameters():
        out["grad::" + k] = (p.grad if p.grad is not None else torch.zeros_like(p)).numpy().copy()
    model.eval()
    pft, ppm, ptok = shifted(sch, ft, pm)
    with torch.no_grad():
        out["eval_logits"] = model.predict(pft, ppm, ptok).numpy()
    out.update(p_pad_mask=ppm.numpy(), p_token_mask=ptok.numpy())
    out.update({"pfeat::" + k: v.numpy() for k, v in pft.items()})
    path = os.path.join(OUT, f"bert4rec_side_{tag}.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, "loss", float(res), "bytes", os.path.getsize(path))


if __name__ == "__main__":
    gen("d64h2", B=6, L=16, d=64, H=2, n_items=300, n_blocks=2, seed=51,
        fs=[dict(name="genre", kind="cat", cardinality=7, padding_value=3), dict(name="flag", kind="cat", cardinality=1,
            padding_value=0), dict(name="vec", kind="num"), dict(name="vl", kind="num_list")])
    gen("d300h4", B=6, L=16, d=300, H=4, n_items=100, n_blocks=0, seed=52,
        fs=[dict(name="genre", kind="cat", cardinality=11, padding_value=0), dict(name="vec", kind="num")])
    gen("d96h2_tied_bce", B=6, L=16, d=96, H=2, n_items=250, n_blocks=1, seed=53, tying=True, positional=False, passes=2,
        loss="BCE", fs=[dict(name="genre", kind="cat", cardinality=5, padding_value=4), dict(name="vec", kind="num")])
