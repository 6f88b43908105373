"""Generate the DiffTransformer golden vectors FROM THE REAL REFERENCE (run in the build container only).  TEST INFRASTRUCTURE.

    python oracle/gen_diff_golden.py

Writes tests/golden/sasrec_diff_*.npz: seeded inputs, the reference model's weights as a seed (oracle.diff.seeded_state_dict)
with the reference's key list and a checksum of every tensor, hidden states of every position (train mode, dropout 0), the
CE loss, every gradient (bf16) and the eval logits of the last position.  Weights as a seed and bf16 gradients keep each
file well under a megabyte.
tests/test_diff_cpu.py checks oracle/diff.py against them; tests/test_gpu_diff_sasrec.py checks the CUDA path.
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

from gen_golden import make_batch, schema  # noqa: E402
from oracle.diff import checksum, seeded_state_dict, to_bf16_bits  # noqa: E402
from replay.nn.agg import SumAggregator  # noqa: E402
from replay.nn.embedding import SequenceEmbedding  # noqa: E402
from replay.nn.loss import CE  # noqa: E402
from replay.nn.mask import DefaultAttentionMask  # noqa: E402
from replay.nn.sequential import DiffTransformerLayer, PositionAwareAggregator, SasRec, SasRecBody  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")


def build(n_items, d, H, L, n_blocks, norm):
    sch = schema(n_items, d, n_items)
    body = SasRecBody(
        embedder=SequenceEmbedding(schema=sch, excluded_features=[sch.query_id_feature_name, sch.timestamp_feature_name]),
        embedding_aggregator=PositionAwareAggregator(SumAggregator(embedding_dim=d), max_sequence_length=L, dropout=0.0),
        attn_mask_builder=DefaultAttentionMask(reference_feature_name="item_id", num_heads=H),
        encoder=DiffTransformerLayer(embedding_dim=d, num_heads=H, num_blocks=n_blocks),
        output_normalization=torch.nn.LayerNorm(d) if norm == "layernorm" else torch.nn.RMSNorm(d),
    )
    return SasRec(body=body, loss=CE(ignore_index=n_items))


def gen(tag, B, L, d, H, n_items, n_blocks, norm, seed):
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    model = build(n_items, d, H, L, n_blocks, norm)
    model.load_state_dict(seeded_state_dict(n_items, d, H, L, n_blocks, norm, seed), strict=True)
    ids, pmask, labels, tmask = make_batch(g, B, L, n_items, n_items)
    keys = list(model.state_dict())
    out = dict(sd_keys=np.array(keys), sd_sums=np.array([checksum(model.state_dict()[k]) for k in keys]), seed=seed)
    out.update(ids=ids.numpy(), pad_mask=pmask.numpy(), labels=labels.numpy(), target_mask=tmask.numpy(), n_items=n_items,
               d=d, H=H, L=L, n_blocks=n_blocks, norm=norm)
    model.train()
    res = model(feature_tensors={"item_id": ids}, padding_mask=pmask, positive_labels=labels.unsqueeze(-1),
                negative_labels=None, target_padding_mask=tmask.unsqueeze(-1))
    res["loss"].backward()
    hidden = model.body(feature_tensors={"item_id": ids}, padding_mask=pmask)
    out["train_hidden"] = hidden.detach().numpy()
    out["train_loss"] = res["loss"].detach().numpy()
    for k, p in model.named_parameters():
        out["grad::" + k] = to_bf16_bits(p.grad if p.grad is not None else torch.zeros_like(p))
    model.eval()
    with torch.no_grad():
        out["eval_logits"] = model(feature_tensors={"item_id": ids}, padding_mask=pmask)["logits"].numpy()
    np.savez_compressed(os.path.join(OUT, f"sasrec_diff_{tag}.npz"), **out)
    print("wrote sasrec_diff_" + tag, "loss", float(res["loss"]))


if __name__ == "__main__":
    gen("tiny", B=4, L=8, d=64, H=2, n_items=50, n_blocks=2, norm="layernorm", seed=11)
    gen("tiny_rms", B=4, L=8, d=64, H=2, n_items=50, n_blocks=2, norm="rmsnorm", seed=12)
    gen("d128h2", B=8, L=50, d=128, H=2, n_items=200, n_blocks=1, norm="layernorm", seed=13)
