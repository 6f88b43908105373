"""The padded parameter layout without a GPU: every parameter's true shape (BaseConfig.true_shapes, from the pad kind of each
axis) equals the reference model's shape, for SASRec (new and legacy) and BERT4Rec - also where a non-feature axis (the
item table's rows, the positional table's rows) happens to equal a multiple of the padded width."""
import os

import numpy as np
import pytest

from bert_shapes_golden import SHAPES

# (d, H) -> padded width dp: 192 / 4 -> 256, 50 / 1 -> 64, 300 / 4 -> 512, 64 / 2 -> 128 (every one has padded slots)
DH = [(192, 4, 256), (50, 1, 64), (300, 4, 512), (64, 2, 128)]


def _sasrec_ref_shapes(n_items, d, max_len, n_blocks):
    """the reference SASRec's parameters (oracle.sasrec.random_params mirrors its state_dict), conv weights squeezed"""
    from oracle.sasrec import random_params

    P = random_params(n_items, d, max_len, n_blocks)
    out = {k: tuple(P[k].shape) for k in ("item_emb", "pos_emb", "lnf_w", "lnf_b")}
    for i, blk in enumerate(P["blocks"]):
        out.update({f"b{i}.{k}": tuple(v.shape) for k, v in blk.items()})
    return out


def _bert_ref_shapes(n_items, d, max_len, n_blocks, tying):
    """bert4rec/model.py: item table [|I|, d], one <MASK> row, positions, pre-LN blocks with a Linear(d, 4d) FFN, the head"""
    out = {"item_emb": (n_items, d), "mask_emb": (1, d), "pos_emb": (max_len, d), "head_b": (n_items,)}
    blk = {"ln1_w": (d,), "ln1_b": (d,), "in_w": (3 * d, d), "in_b": (3 * d,), "out_w": (d, d), "out_b": (d,), "ln2_w": (d,),
           "ln2_b": (d,), "w1": (4 * d, d), "b1": (4 * d,), "w2": (d, 4 * d), "b2": (d,)}
    for i in range(n_blocks):
        out.update({f"b{i}.{k}": v for k, v in blk.items()})
    if not tying:
        out["head_w"] = (n_items, d)
    return out


@pytest.mark.parametrize("k", [1, 2, 3])
@pytest.mark.parametrize("d,H,dp", DH)
@pytest.mark.parametrize("variant", ["new", "legacy"])
def test_sasrec_true_shapes_match_reference(variant, d, H, dp, k):
    """max_len and the item table's rows (n_items + 1) equal k * dp"""
    from replay_b200.engine import EncoderConfig

    cfg = EncoderConfig(n_items=k * dp - 1, d=d, n_heads=H, n_blocks=2, max_len=k * dp, variant=variant)
    assert cfg.dp == dp
    assert cfg.true_shapes() == _sasrec_ref_shapes(cfg.n_items, d, cfg.max_len, 2)
    padded = {name: shp for name, shp, _ in cfg.param_layout()}
    assert padded["item_emb"] == (k * dp, dp) and padded["pos_emb"] == (k * dp, dp) and padded["b0.in_w"] == (3 * dp, dp)


@pytest.mark.parametrize("tying", [False, True])
@pytest.mark.parametrize("k", [1, 2, 3])
@pytest.mark.parametrize("d,H,dp", DH)
def test_bert_true_shapes_match_reference(d, H, dp, k, tying):
    """max_len and the item table's rows (n_items) equal k * dp"""
    from replay_b200.engine_bert import BertConfig

    cfg = BertConfig(n_items=k * dp, d=d, n_heads=H, n_blocks=2, max_len=k * dp, tying=tying)
    assert cfg.dp == dp
    assert cfg.true_shapes() == _bert_ref_shapes(cfg.n_items, d, cfg.max_len, 2, tying)


@pytest.mark.parametrize("tag", ["sasrec_new_d192h4", "sasrec_new_d64h2", "sasrec_legacy_d50h1", "sasrec_new_tiny",
                                 "sasrec_legacy_tiny"])
def test_sasrec_true_shapes_match_reference_state_dict(golden_dir, tag):
    """against the shapes of the real reference's state_dict stored in the goldens"""
    from replay_b200.core import reference_key_map
    from replay_b200.engine import EncoderConfig

    z = np.load(os.path.join(golden_dir, f"{tag}.npz"))
    variant = "legacy" if "legacy" in tag else "new"
    cfg = EncoderConfig(n_items=int(z["n_items"]), d=int(z["d"]), n_heads=int(z["H"]), n_blocks=int(z["n_blocks"]),
                        max_len=int(z["L"]), variant=variant)
    keymap = reference_key_map(variant, cfg.n_blocks)
    ref = {k: tuple(z["sd::" + rk].shape) for k, rk in keymap.items()}
    ref = {k: s[:2] if k.endswith((".w1", ".w2")) else s for k, s in ref.items()}   # Conv1d weights [d, d, 1]
    assert cfg.true_shapes() == ref


@pytest.mark.parametrize("tag", list(SHAPES))
def test_bert_true_shapes_match_reference_state_dict(golden_dir, tag):
    """against the shapes of the real reference's state_dict stored in the goldens (padded hidden sizes included)"""
    from replay_b200.engine_bert import BertConfig
    from replay_b200.models.nn.sequential.bert4rec import bert_key_map

    z = np.load(os.path.join(golden_dir, f"bert4rec_{tag}.npz"))
    ref = {str(n): tuple(int(v) for v in s[s > 0]) for n, s in zip(z["param_names"], z["param_shapes"])}
    cfg = BertConfig(n_items=int(z["n_items"]), d=int(z["d"]), n_heads=int(z["H"]), n_blocks=int(z["n_blocks"]),
                     max_len=int(z["L"]), tying=bool(int(z["tying"])))
    keymap = bert_key_map(cfg.n_blocks, cfg.tying)
    assert {keymap[k]: s for k, s in cfg.true_shapes().items()} == {k: ref[k] for k in keymap.values()}
