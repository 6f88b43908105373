"""TiSASRec without a GPU: the float64 restatement (oracle/tisasrec.py) reproduces the reference's goldens, the interval
matrix clips and floors as the reference does in every timestamp dtype, the state_dict has the reference's keys and
shapes, and the configurations outside the kernels' limits raise at construction."""
import glob
import os

import numpy as np
import pytest
import torch

import oracle.tisasrec as oti

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sasrec_ti_*.npz")))


def test_goldens_exist():
    assert {os.path.basename(p) for p in GOLDEN} == {"sasrec_ti_tiny.npz", "sasrec_ti_d64h2.npz", "sasrec_ti_fp32_times.npz"}


@pytest.mark.parametrize("path", GOLDEN, ids=os.path.basename)
def test_oracle_reproduces_golden(path):
    z = np.load(path)
    sd = {k[4:]: torch.from_numpy(z[k]).double() for k in z.files if k.startswith("sd::")}
    P = oti.params_from_state_dict(sd)
    ids, pad, times, labels, tmask = (torch.from_numpy(z[k]) for k in ("ids", "pad", "times", "labels", "tmask"))
    H, span = int(z["n_heads"]), int(z["time_span"])
    hid = oti.body(P, ids, pad, times, H, span)
    assert torch.allclose(hid.float(), torch.from_numpy(z["hidden"]), atol=1e-5)
    loss, G = oti.loss_and_grads(P, ids, pad, times, labels, tmask, H, span)
    assert abs(float(loss) - float(z["loss"])) < 1e-6 * abs(float(z["loss"]))
    ref_G = oti.params_from_state_dict({k[6:]: torch.from_numpy(z[k]).double() for k in z.files if k.startswith("grad::")})
    for k in ("item_emb", "pos_k", "pos_v", "time_k", "time_v", "lnf_w", "lnf_b"):
        assert torch.allclose(G[k], ref_G[k], atol=1e-6), k
    for b, rb in zip(G["blocks"], ref_G["blocks"]):
        for k in b:
            assert torch.allclose(b[k], rb[k], atol=1e-6), k


def test_golden_intervals_clip_and_tie():
    z = np.load([p for p in GOLDEN if p.endswith("tiny.npz")][0])
    r = oti.time_matrix(torch.from_numpy(z["times"]), int(z["time_span"]))
    assert int(r.max()) == 8 and bool((r == 0).any())
    live = torch.from_numpy(z["pad"])
    offdiag = (r == 0) & ~torch.eye(r.shape[1], dtype=torch.bool) & live[:, :, None] & live[:, None, :]
    assert bool(offdiag.any()), "no tie between two live positions"


@pytest.mark.parametrize("dtype", [torch.int64, torch.float32, torch.float64])
def test_time_matrix_clips_and_floors(dtype):
    t = torch.tensor([[0.0, 0.4, 1.6, 2.5, 300.0, 1.7e9, 1.7e9 + 100.7]]).to(dtype)
    r = oti.time_matrix(t, 256)
    assert r.dtype == torch.int64
    assert int(r[0, 0, 1]) == 0 and int(r[0, 0, 4]) == 256 and int(r[0, 2, 3]) == (0 if dtype.is_floating_point else 1)
    d = (t[0, 6] - t[0, 5]).abs()
    assert int(r[0, 5, 6]) == int(torch.floor(d)) if dtype.is_floating_point else int(d)
    if dtype == torch.float32:   # the difference is taken in float32: 1.7e9 + 100.7 rounds to a multiple of 128
        assert int(r[0, 5, 6]) == 128
    assert bool((r == r.transpose(1, 2)).all())


def _schema(ts=True):
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    return TensorSchema(TensorFeatureInfo("item_id", 100, 100, 50), timestamp_feature_name="timestamp" if ts else None)


def test_state_dict_keys_and_shapes_match_reference():
    from replay_b200.engine_tisasrec import TiConfig, ti_reference_key_map

    cfg = TiConfig(n_items=10, d=50, n_heads=1, n_blocks=2, max_len=12, time_span=8)
    km, shapes = ti_reference_key_map(2), cfg.true_shapes()
    got = {km[k]: shapes[k] for k in shapes}
    d, e = 50, "item_embedder."
    want = {e + "item_emb.weight": (11, d), e + "abs_pos_k_emb.pe.weight": (12, d), e + "abs_pos_v_emb.pe.weight": (12, d),
            e + "time_matrix_k_emb.weight": (9, d), e + "time_matrix_v_emb.weight": (9, d),
            "output_normalization.last_layernorm.weight": (d,), "output_normalization.last_layernorm.bias": (d,)}
    for i in range(2):
        s = f"sasrec_layers."
        for m in ("query_w", "key_w", "value_w"):
            want.update({f"{s}attention_layers.{i}.{m}.weight": (d, d), f"{s}attention_layers.{i}.{m}.bias": (d,)})
        for m in ("attention_layernorms", "forward_layernorms"):
            want.update({f"{s}{m}.{i}.weight": (d,), f"{s}{m}.{i}.bias": (d,)})
        for c in ("conv1", "conv2"):   # Conv1d(d, d, 1): the state_dict adds the trailing 1 (SasRecCore._to_ref)
            want.update({f"{s}forward_layers.{i}.{c}.weight": (d, d), f"{s}forward_layers.{i}.{c}.bias": (d,)})
    assert got == want


@pytest.mark.parametrize("kw,what", [
    (dict(hidden_size=130, num_heads=2), "head width"),
    (dict(hidden_size=320, num_heads=5), "padded columns"),
    (dict(max_len=257), "max_seq_len"),
    (dict(time_span=0), "time_span"),
    (dict(time_span=321), "time_span"),
])
def test_limits_raise_value_error(kw, what):
    from replay_b200.models.nn.sequential.sasrec import SasRecModel

    with pytest.raises(ValueError, match=what):
        SasRecModel(_schema(), ti_modification=True, device="cpu", **kw)


@pytest.mark.parametrize("kw", [dict(), dict(hidden_size=128, num_heads=2), dict(time_span=320)])
def test_reference_defaults_and_config2_fit(kw):
    from replay_b200.models.nn.sequential.sasrec import SasRecModel

    m = SasRecModel(_schema(), ti_modification=True, device="cpu", **kw)
    assert m.core.cfg.time_span == kw.get("time_span", 256)


def test_schema_without_timestamp_raises_assertion():
    from replay_b200.models.nn.sequential import SasRec
    from replay_b200.models.nn.sequential.sasrec import SasRecModel

    with pytest.raises(AssertionError):
        SasRecModel(_schema(ts=False), ti_modification=True, device="cpu")
    with pytest.raises(AssertionError):
        SasRec(_schema(ts=False), ti_modification=True, device="cpu")
