"""SASRec where a non-feature axis of a parameter equals a multiple of the padded width: the engine builds, a state_dict
survives a round trip exactly, and one training step runs.  The true shape of every axis comes from its pad kind, not from
its size."""
import pytest
import torch


# (item count, embedding_dim, heads, max_sequence_length): pos_emb [256, 256] at dp 256 (head_dim 48 in 64-wide slots);
# item_emb [64, 64] at dp 64 (hidden 50 in one 64-wide slot)
CASES = [(300, 192, 4, 256), (63, 50, 1, 50)]


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("n_items,d,H,max_len", CASES, ids=["d192h4_L256", "d50h1_I63"])
def test_padded_layout_round_trip_and_step(cuda, n_items, d, H, max_len):
    from replay_b200.nn.sequential import SasRec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema
    from replay_b200.synthetic import make_sequences

    schema = TensorSchema(TensorFeatureInfo("item_id", n_items, n_items, d))
    m = SasRec.from_params(schema, embedding_dim=d, num_heads=H, max_sequence_length=max_len, dropout=0.0, device=cuda, seed=3)
    eng = m.core.engine
    assert eng.cfg.hd_valid != 0
    for name in eng.layout:
        assert tuple(eng.export_named(name).shape) == eng.true_shape(name), name
    sd = m.state_dict()
    assert sd["body.embedder.feature_embedders.item_id.emb.weight"].shape == (n_items + 1, d)
    assert sd["body.embedding_aggregator.pe.weight"].shape == (max_len, d)

    m2 = SasRec.from_params(schema, embedding_dim=d, num_heads=H, max_sequence_length=max_len, dropout=0.0, device=cuda, seed=4)
    m2.load_state_dict(sd)
    sd2 = m2.state_dict()
    assert sd2.keys() == sd.keys()
    for k in sd:
        assert torch.equal(sd2[k], sd[k]), k
    m2.core.engine.refresh_shadow()
    assert torch.equal(m2.core.engine.p32, eng.p32)   # padded entries are zero in both

    ids, pm, lab, tm = (t.to(cuda) for t in make_sequences(2, n_items, max_len, seed=5))
    before = eng.p32.clone()
    loss = m.core.fused_step(ids, pm, lab, tm, all_reduce=None, lr=1e-3)
    torch.cuda.synchronize()
    assert torch.isfinite(loss).all()
    assert not torch.equal(eng.p32, before)
    pad = torch.ones(eng.cfg.dp, dtype=torch.bool, device=cuda)
    pad[eng.cfg.feat_index(cuda)] = False
    assert not eng.params["pos_emb"][:, pad].any() and not eng.params["item_emb"][:, pad].any()
