"""SasRec with the DiffTransformer encoder without a GPU: the fp64 oracle reproduces the reference's golden vectors, the
reference-style constructors map onto the right engine configuration (or raise), the state_dict keys are the reference's,
and the new C entry points refuse bad arguments before any CUDA call."""
import ctypes
import os

import pytest
import torch

from replay_b200.schema import TensorFeatureInfo, TensorSchema

GOLDENS = ["sasrec_diff_tiny.npz", "sasrec_diff_tiny_rms.npz", "sasrec_diff_d128h2.npz"]
EINVAL, ESHAPE = -1, -2


def _load(golden_dir, name):
    from oracle import diff as od

    return od.load_golden(os.path.join(golden_dir, name))


@pytest.mark.parametrize("name", GOLDENS)
def test_oracle_reproduces_reference(golden_dir, name):
    from oracle import diff as od

    z, sd, grads = _load(golden_dir, name)
    sd64 = {k: v.double() for k, v in sd.items()}
    ids, pm = torch.from_numpy(z["ids"]), torch.from_numpy(z["pad_mask"])
    labels, tm = torch.from_numpy(z["labels"]), torch.from_numpy(z["target_mask"])
    H = int(z["H"])
    h = od.diff_body(sd64, ids, pm, H)
    torch.testing.assert_close(h, torch.from_numpy(z["train_hidden"]).double(), rtol=1e-4, atol=1e-4)
    loss, G = od.loss_and_grads(sd64, ids, pm, labels, tm, H)
    assert abs(float(loss) - float(z["train_loss"])) < 1e-5 * abs(float(z["train_loss"]))
    assert set(grads) == set(G)
    for k, ref in grads.items():   # stored as bf16: half an ulp is 2^-9 of the value
        ref = ref.double()
        torch.testing.assert_close(G[k], ref, rtol=4e-3, atol=1e-5 * max(1.0, float(ref.abs().max())))
    n_items = int(z["n_items"])
    table = sd64["body.embedder.feature_embedders.item_id.emb.weight"][:n_items]
    torch.testing.assert_close(h[:, -1] @ table.T, torch.from_numpy(z["eval_logits"]).double(), rtol=1e-4, atol=1e-4)


def _schema(n_items=100, d=64):
    return TensorSchema(TensorFeatureInfo("item_id", n_items, n_items, d))


def _body(enc, norm, d=64, H=2, L=50, dropout=0.0, mask_name="item_id", mask_heads=None, agg_d=None):
    from replay_b200.nn.agg import SumAggregator
    from replay_b200.nn.embedding import SequenceEmbedding
    from replay_b200.nn.mask import DefaultAttentionMask
    from replay_b200.nn.sequential import PositionAwareAggregator, SasRecBody

    return SasRecBody(embedder=SequenceEmbedding(_schema(d=d)),
                      embedding_aggregator=PositionAwareAggregator(SumAggregator(agg_d or d), max_sequence_length=L, dropout=dropout),
                      attn_mask_builder=DefaultAttentionMask(mask_name, mask_heads or H), encoder=enc, output_normalization=norm)


@pytest.mark.parametrize("d,H,L,norm", [(64, 2, 50, "ln"), (128, 2, 200, "rms"), (192, 4, 100, "ln"), (256, 4, 256, "rms"),
                                        (64, 1, 1, "ln"), (48, 1, 20, "rms")])
def test_diff_body_builds_config(d, H, L, norm):
    from replay_b200.engine_diff import RMS_EPS, DiffConfig
    from replay_b200.nn.sequential import DiffTransformerLayer, SasRec

    nrm = torch.nn.LayerNorm(d, eps=1e-6) if norm == "ln" else torch.nn.RMSNorm(d)
    m = SasRec(_body(DiffTransformerLayer(d, H, 2), nrm, d, H, L, dropout=0.1), device="cpu")
    cfg = m.core.cfg
    assert isinstance(cfg, DiffConfig)
    assert (cfg.n_items, cfg.d, cfg.n_heads, cfg.n_blocks, cfg.max_len, cfg.dropout) == (100, d, H, 2, L, 0.1)
    assert cfg.out_norm == ("layernorm" if norm == "ln" else "rmsnorm")
    assert cfg.lnf_eps == (1e-6 if norm == "ln" else RMS_EPS)
    assert cfg.v_slot == (64 if d // H <= 32 else 128)


@pytest.mark.parametrize("d,H,L", [(256, 2, 50), (128, 1, 50), (512, 8, 50), (320, 5, 50), (64, 2, 257), (64, 3, 50)])
def test_diff_body_rejects_unsupported_shapes(d, H, L):
    from replay_b200.nn.sequential import DiffTransformerLayer, SasRec

    with pytest.raises(ValueError):
        SasRec(_body(DiffTransformerLayer(d, H, 1), torch.nn.LayerNorm(d), d, H, L), device="cpu")


def test_body_rejects_mismatched_parts():
    from replay_b200.nn.sequential import DiffTransformerLayer, SasRec, SasRecTransformerLayer

    bad = [_body(DiffTransformerLayer(64, 2, 1), torch.nn.LayerNorm(32)),
           _body(DiffTransformerLayer(64, 2, 1), torch.nn.BatchNorm1d(64)),
           _body(DiffTransformerLayer(64, 2, 1), torch.nn.LayerNorm(64), mask_name="other"),
           _body(DiffTransformerLayer(64, 2, 1), torch.nn.LayerNorm(64), mask_heads=4),
           _body(DiffTransformerLayer(64, 2, 1), torch.nn.LayerNorm(64), agg_d=32),
           _body(SasRecTransformerLayer(64, 2, 1, 0.0, activation="gelu"), torch.nn.LayerNorm(64)),
           _body(SasRecTransformerLayer(64, 2, 1, 0.0, activation="relu"), torch.nn.RMSNorm(64)),
           _body(SasRecTransformerLayer(64, 2, 1, 0.2, activation="relu"), torch.nn.LayerNorm(64), dropout=0.1)]
    for body in bad:
        with pytest.raises(ValueError):
            SasRec(body, device="cpu")


@pytest.mark.parametrize("d,H,L,n_blocks", [(64, 2, 50, 2), (192, 4, 100, 1), (50, 1, 30, 3)])
def test_transformer_body_equals_from_params(d, H, L, n_blocks):
    from replay_b200.nn.sequential import SasRec, SasRecTransformerLayer

    a = SasRec(_body(SasRecTransformerLayer(d, H, n_blocks, 0.2, activation="relu"), torch.nn.LayerNorm(d), d, H, L, dropout=0.2),
               device="cpu")
    b = SasRec.from_params(_schema(d=d), embedding_dim=d, num_heads=H, num_blocks=n_blocks, max_sequence_length=L, dropout=0.2,
                           device="cpu")
    assert a.core.cfg == b.core.cfg
    assert type(a.core) is type(b.core)
    assert a.core._keymap == b.core._keymap


@pytest.mark.parametrize("name", GOLDENS)
def test_state_dict_keys_equal_reference(golden_dir, name):
    from replay_b200.nn.sequential import DiffTransformerLayer, SasRec

    z, sd, _ = _load(golden_dir, name)
    d, H, L, n_blocks = int(z["d"]), int(z["H"]), int(z["L"]), int(z["n_blocks"])
    norm = torch.nn.LayerNorm(d) if str(z["norm"]) == "layernorm" else torch.nn.RMSNorm(d)
    sch = TensorSchema(TensorFeatureInfo("item_id", int(z["n_items"]), int(z["n_items"]), d))
    from replay_b200.nn.agg import SumAggregator
    from replay_b200.nn.embedding import SequenceEmbedding
    from replay_b200.nn.mask import DefaultAttentionMask
    from replay_b200.nn.sequential import PositionAwareAggregator, SasRecBody

    body = SasRecBody(SequenceEmbedding(sch), PositionAwareAggregator(SumAggregator(d), L, 0.0), DefaultAttentionMask("item_id", H),
                      DiffTransformerLayer(d, H, n_blocks), norm)
    m = SasRec(body, device="cpu")
    m.load_state_dict(sd)
    assert set(m.state_dict()) == {str(k) for k in z["sd_keys"]}
    # true shapes of the engine layout equal the reference's tensors
    shapes = m.core.cfg.true_shapes()
    for k, rk in m.core._keymap.items():
        assert tuple(sd[rk].shape) == shapes[k], (k, rk)
    bad = dict(sd)
    bad["body.encoder.layers.0.attn.scaling"] = torch.tensor(0.5)
    with pytest.raises(ValueError):
        m.load_state_dict(bad)


def _lam():
    from replay_b200._lib import DiffLambda

    lam = DiffLambda()
    lam.q1 = lam.k1 = lam.q2 = lam.k2 = 1 << 20
    lam.head_dim, lam.lambda_init = 32, 0.2
    return lam


def _attn_desc(**kw):
    from replay_b200._lib import DiffAttnDesc

    a = DiffAttnDesc()
    fake = 1 << 20   # never dereferenced: the argument checks come first
    a.qk = a.v = a.pad_mask = a.out = a.rms_scale = fake
    a.ld_qk, a.ldv, a.ldo, a.k_c0, a.v_c0 = 320, 320, 64, 128, 256
    a.B, a.H, a.L, a.head_dim, a.v_slot = 2, 1, 50, 32, 64
    a.lam = _lam()
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("kw,rc", [(dict(qk=None), EINVAL), (dict(pad_mask=None), EINVAL), (dict(rms_scale=None), EINVAL),
                                   (dict(L=257), ESHAPE), (dict(L=0), ESHAPE), (dict(v_slot=96), ESHAPE),
                                   (dict(head_dim=48), ESHAPE), (dict(e1_save=1 << 20), EINVAL), (dict(B=0), ESHAPE)])
def test_diff_attn_fwd_rejects_bad_arguments(kw, rc):
    from replay_b200._lib import lib

    assert lib().rp_diff_attn_fwd(ctypes.byref(_attn_desc(**kw)), None) == rc


def test_diff_entry_points_reject_bad_arguments():
    from replay_b200._lib import lib

    L, f, lam = lib(), 1 << 20, _lam()
    assert L.rp_diff_attn_softmax_bwd(f, f, f, f, f, f, f, f, None, 4, 2, 50, 0.1, ctypes.byref(lam), f, f, f, f, 1e-5, 128, 64, None) == EINVAL
    assert L.rp_diff_attn_softmax_bwd(f, f, f, f, f, f, f, f, f, 3, 2, 50, 0.1, ctypes.byref(lam), f, f, f, f, 1e-5, 128, 64, None) == ESHAPE
    assert L.rp_diff_attn_softmax_bwd(f, f, f, f, f, f, f, f, f, 4, 2, 300, 0.1, ctypes.byref(lam), f, f, f, f, 1e-5, 128, 64, None) == ESHAPE
    big = _lam()
    big.head_dim = 65
    assert L.rp_diff_attn_softmax_bwd(f, f, f, f, f, f, f, f, f, 4, 2, 50, 0.1, ctypes.byref(big), f, f, f, f, 1e-5, 128, 64, None) == EINVAL
    assert L.rp_diff_attn_softmax_bwd(f, f, f, f, f, f, f, f, f, 4, 2, 50, 0.1, ctypes.byref(lam), None, f, f, f, 1e-5, 128, 64, None) == EINVAL
    assert L.rp_diff_attn_softmax_bwd(f, f, f, f, f, f, f, f, f, 4, 2, 50, 0.1, ctypes.byref(lam), f, f, f, f, 1e-5, 128, 96, None) == ESHAPE
    assert L.rp_diff_lambda_bwd(f, 2, 2, 50, ctypes.byref(lam), f, f, None, f, None) == EINVAL
    assert L.rp_diff_lambda_bwd(f, 2, 2, 257, ctypes.byref(lam), f, f, f, f, None) == ESHAPE
    assert L.rp_rmsnorm_fwd(None, f, 1e-5, 1.0, 10, 64, 64, 64, None, None, f, None) == EINVAL
    for d, group, n_true in ((96, 96, 96), (128, 256, 128), (192, 128, 128), (64, 64, 65), (64, 64, 0), (1024, 256, 256)):
        assert L.rp_rmsnorm_fwd(f, f, 1e-5, 1.0, 10, d, group, n_true, None, None, f, None) == ESHAPE
        assert L.rp_rmsnorm_bwd(f, f, f, 1e-5, 1.0, 10, d, group, n_true, None, None, f, f, f, 1 << 30, None) == ESHAPE
    assert L.rp_rmsnorm_bwd_workspace(96) == 0
    ws = L.rp_rmsnorm_bwd_workspace(128)
    assert ws > 0
    assert L.rp_rmsnorm_bwd(f, f, f, 1e-5, 1.0, 10, 128, 128, 128, None, None, f, f, f, ws - 4, None) == -5
    assert L.rp_rmsnorm_bwd(f, f, f, 1e-5, 1.0, 10, 128, 128, 128, None, None, f, None, f, ws, None) == EINVAL
    assert L.rp_swiglu_fwd(None, 10, 64, f, None) == EINVAL
    assert L.rp_swiglu_fwd(f, 10, 0, f, None) == ESHAPE
    assert L.rp_swiglu_bwd(f, None, 10, 64, f, None) == EINVAL
    assert L.rp_swiglu_bwd(f, f, -1, 64, f, None) == ESHAPE
