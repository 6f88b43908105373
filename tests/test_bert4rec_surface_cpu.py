"""BERT4Rec's repeated block passes, the model without positional embedding and the catalog-growth surface, on the CPU:
the oracle against the reference's goldens (tests/golden/bert4rec_{p2_d64h2, nopos_tied, p3_nopos_d96h2}.npz, written by
oracle/gen_bert4rec_passes_golden.py), the mirror's checkpoint keys, and the constructor and resize argument errors."""
import os

import numpy as np
import pytest
import torch

CASES = ["bert4rec_p2_d64h2.npz", "bert4rec_nopos_tied.npz", "bert4rec_p3_nopos_d96h2.npz"]


def _load(golden_dir, name):
    from oracle import bert4rec_passes as op

    z = np.load(os.path.join(golden_dir, name))
    return z, op.golden_state_dict(z)


def _schema(n_items, d):
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    return TensorSchema(TensorFeatureInfo("item_id", n_items, 0, d))


@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_reference(golden_dir, name):
    from oracle import bert4rec_passes as op

    z, sd = _load(golden_dir, name)
    P = op.params_from_state_dict(sd)
    assert ("pos_emb" in P) == bool(int(z["positional"]))
    H, p = int(z["H"]), int(z["passes"])
    ids, pm, tok, labels = (torch.from_numpy(z[k]) for k in ("ids", "pad_mask", "token_mask", "labels"))
    Pd = {k: ([{a: b.double() for a, b in blk.items()} for blk in v] if k == "blocks" else v.double()) for k, v in P.items()}
    h = op.body(Pd, ids, pm, tok, H, p)
    torch.testing.assert_close(h.float(), torch.from_numpy(z["train_hidden"]), atol=2e-5, rtol=2e-5)
    # the passes matter: one pass gives other hidden states
    if p > 1:
        assert (op.body(Pd, ids, pm, tok, H, 1).float() - h.float()).abs().max() > 1e-2
    # loss and every gradient through autograd
    Pg = {k: ([{a: b.clone().requires_grad_(True) for a, b in blk.items()} for blk in v] if k == "blocks"
              else v.clone().requires_grad_(True)) for k, v in Pd.items()}
    loss = op.train_loss(Pg, ids, pm, tok, labels, H, p)
    assert abs(float(loss.detach()) - float(z["train_loss"])) < 1e-5 * float(z["train_loss"])
    loss.backward()
    Gref = op.params_from_state_dict({k[6:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("grad::")})
    for k, v in Pg.items():
        if k == "blocks":
            for i, blk in enumerate(v):
                for a, b in blk.items():
                    torch.testing.assert_close(b.grad.float(), Gref["blocks"][i][a], atol=1e-6, rtol=1e-4, msg=f"b{i}.{a}")
        else:
            torch.testing.assert_close(v.grad.float(), Gref[k], atol=1e-6, rtol=1e-4, msg=k)
    # eval logits of predict: the last position through the biased head
    with torch.no_grad():
        lg = op.logits(Pd, op.body(Pd, ids, pm, tok, H, p)[:, -1])
    torch.testing.assert_close(lg.float(), torch.from_numpy(z["eval_logits"]), atol=5e-5, rtol=5e-5)


@pytest.mark.parametrize("name", CASES)
def test_mirror_keys_equal_reference(golden_dir, name):
    from replay_b200.models.nn.sequential import Bert4Rec
    from replay_b200.models.nn.sequential.bert4rec import bert_key_map

    z, sd = _load(golden_dir, name)
    nb, tying, pos = int(z["n_blocks"]), bool(int(z["tying"])), bool(int(z["positional"]))
    aliases = {k for k in sd if k.startswith("_head._item_embedder.")}
    assert set(bert_key_map(nb, tying, "item_id", pos).values()) == set(sd) - aliases
    m = Bert4Rec(_schema(int(z["n_items"]), int(z["d"])), block_count=nb, head_count=int(z["H"]), hidden_size=int(z["d"]),
                 max_seq_len=int(z["L"]), dropout_rate=0.0, pass_per_transformer_block_count=int(z["passes"]),
                 enable_positional_embedding=pos, enable_embedding_tying=tying, device="cpu")
    m.load_state_dict({"_model." + k: v for k, v in sd.items()})   # strict: every key the mirror expects is present
    assert set(m.state_dict()) == {"_model." + k for k in sd}


@pytest.mark.parametrize("passes", [0, 1, 2, 5])
@pytest.mark.parametrize("positional", [True, False])
def test_constructor_accepts_options(passes, positional):
    from replay_b200.models.nn.sequential import Bert4Rec

    m = Bert4Rec(_schema(50, 64), block_count=2, head_count=2, hidden_size=64, max_seq_len=16,
                 pass_per_transformer_block_count=passes, enable_positional_embedding=positional, device="cpu")
    cfg = m._model.core.cfg
    assert (cfg.passes, cfg.positional, cfg.n_apps) == (passes, positional, 2 * passes)
    names = [n for n, _, _ in cfg.param_layout()]
    assert ("pos_emb" in names) == positional
    assert sum(n.endswith(".in_w") for n in names) == 2   # weights per block, whatever the passes


@pytest.mark.parametrize("passes", [-1, -3, 1.5])
def test_negative_passes_raise(passes):
    from replay_b200.models.nn.sequential import Bert4Rec

    with pytest.raises(ValueError):
        Bert4Rec(_schema(50, 64), block_count=2, head_count=2, hidden_size=64, max_seq_len=16,
                 pass_per_transformer_block_count=passes, device="cpu")


def test_resize_argument_errors():
    """test_bert4rec_fine_tuning_errors' cases, scaled to this model (4 items there, 40 here; hidden 64)."""
    from replay_b200.models.nn.sequential import Bert4Rec

    m = Bert4Rec(_schema(40, 64), block_count=2, head_count=2, hidden_size=64, max_seq_len=16, device="cpu")
    with pytest.raises(ValueError, match="greater then already fitted"):
        m.set_item_embeddings_by_size(3)
    with pytest.raises(ValueError, match="greater then already fitted"):
        m.set_item_embeddings_by_size(40)
    with pytest.raises(ValueError, match="shape"):
        m.set_item_embeddings_by_tensor(torch.rand(1, 1, 1))
    with pytest.raises(ValueError, match="less then already fitted"):
        m.set_item_embeddings_by_tensor(torch.rand(39, 64))
    with pytest.raises(ValueError, match="second dimension"):
        m.set_item_embeddings_by_tensor(torch.rand(40, 1))
    with pytest.raises(ValueError, match="shape"):
        m.append_item_embeddings(torch.rand(1, 1, 1))
    with pytest.raises(ValueError, match="second dimension"):
        m.append_item_embeddings(torch.rand(1, 1))
    assert m._vocab_size == 40 and m._schema.item_id_features.item().cardinality == 40


def test_optimizer_factory_property():
    from replay_b200.models.nn.sequential import Bert4Rec

    class Factory:
        learning_rate, betas = 3e-4, (0.8, 0.9)

        def create(self, params):
            return torch.optim.Adam(params, lr=self.learning_rate, betas=self.betas)

    m = Bert4Rec(_schema(40, 64), block_count=1, head_count=1, hidden_size=64, max_seq_len=8, device="cpu")
    assert m.optimizer_factory is None
    f = Factory()
    m.optimizer_factory = f
    assert m.optimizer_factory is f and m._lr == 3e-4 and m._model.core.adam_betas == (0.8, 0.9)
    with pytest.raises(ValueError, match="OptimizerFactory"):
        m.optimizer_factory = object()
