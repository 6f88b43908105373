"""The legacy SasRec with ti_modification=True on the GPU: the training step against the float64 restatement
(oracle/tisasrec.py) and the goldens of the reference (tests/golden/sasrec_ti_*.npz), dead padded rows, predict, the
Lightning module's three training paths, checkpoints with the reference's keys, catalog growth, the sampled and SCE
losses, and the memory of a config-2 step."""
import glob
import os

import numpy as np
import pytest
import torch

import oracle.tisasrec as oti

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda")


def _schema(n_items, d):
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    return TensorSchema(TensorFeatureInfo("item_id", n_items, n_items, d), timestamp_feature_name="timestamp")


def _batch(B, L, n_items, g, ts_dtype=torch.int64, span=256):
    """Left-padded windows with ties, zero gaps and gaps beyond the span; pads carry timestamp 0."""
    lens = torch.randint(1, L + 2, (B,), generator=g)
    lens[0], lens[1] = L + 1, 2
    full = torch.full((B, L + 1), n_items, dtype=torch.int64)
    msk = torch.zeros(B, L + 1, dtype=torch.bool)
    ts = torch.zeros(B, L + 1, dtype=torch.float64)
    for b in range(B):
        n = int(lens[b])
        full[b, L + 1 - n:] = torch.randint(0, n_items, (n,), generator=g)
        msk[b, L + 1 - n:] = True
        steps = torch.randint(0, 3, (n,), generator=g).double() * torch.rand(n, generator=g, dtype=torch.float64) * span * 0.7
        ts[b, L + 1 - n:] = 1.0e6 + steps.cumsum(0)
    ts = ts.to(ts_dtype) if ts_dtype.is_floating_point else ts.floor().to(ts_dtype)
    return full[:, :-1], msk[:, :-1], ts[:, :-1], full[:, 1:], msk[:, 1:]


def _engine(dev, P, n_items, d, H, L, span, B, drop=0.0):
    from replay_b200.engine_tisasrec import TiConfig, TiSasRecEngine

    cfg = TiConfig(n_items=n_items, d=d, n_heads=H, n_blocks=len(P["blocks"]), max_len=L, dropout=drop, time_span=span)
    eng = TiSasRecEngine(cfg, B, L, dev, seed=7)
    eng.load_canonical(P)
    return eng


def _step(eng, ids, pm, ts, lab, tm):
    dev = eng.dev
    eng.set_batch(ids.to(dev), pm.to(dev), lab.to(dev), tm.to(dev))
    eng.set_times(ts.to(dev))
    eng.tick_rng()
    loss = eng.forward_train()
    eng.g32.zero_()
    eng.backward()
    torch.cuda.synchronize()
    return float(loss[0]), eng.export_canonical(eng.grads)


def _compare(loss, G, ref_loss, ref_G):
    assert abs(loss - ref_loss) <= 5e-3 * abs(ref_loss), (loss, ref_loss)
    flat = lambda P: torch.cat([P[k].double().flatten() for k in sorted(P) if k != "blocks"]  # noqa: E731
                               + [b[k].double().flatten() for b in P["blocks"] for k in sorted(b)])
    for name in ("item_emb", "pos_k", "pos_v", "time_k", "time_v"):
        g, r = G[name].double(), ref_G[name].double()
        assert torch.nn.functional.cosine_similarity(g.flatten(), r.flatten(), dim=0) > 0.995, name
        assert abs(float(g.norm() / r.norm()) - 1) < 0.03, name
    g, r = flat(G), flat(ref_G)
    assert torch.nn.functional.cosine_similarity(g, r, dim=0) > 0.995
    assert abs(float(g.norm() / r.norm()) - 1) < 0.03


CASES = [  # (n_items, d, H, L, span, timestamp dtype)
    (60, 50, 1, 12, 8, torch.int64),
    (300, 64, 2, 50, 256, torch.int64),
    (200, 64, 2, 40, 64, torch.float32),
    (150, 64, 2, 33, 32, torch.float64),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=["d50h1_span8", "d64h2_span256", "fp32_times", "fp64_times"])
def test_train_step_matches_fp64_oracle(cuda, case):
    n_items, d, H, L, span, ts_dtype = case
    g = torch.Generator().manual_seed(11)
    P = oti.random_params(n_items, d, L, 2, span, seed=3)
    ids, pm, ts, lab, tm = _batch(6, L, n_items, g, ts_dtype, span)
    eng = _engine(cuda, P, n_items, d, H, L, span, 6)
    loss, G = _step(eng, ids, pm, ts, lab, tm)
    ref_loss, ref_G = oti.loss_and_grads(oti.params_to(P, torch.float64), ids, pm, ts, lab, tm, H, span)
    _compare(loss, G, float(ref_loss), ref_G)


@pytest.mark.gpu
@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(GOLDEN, "sasrec_ti_*.npz"))), ids=os.path.basename)
def test_train_step_matches_reference_golden(cuda, path):
    z = np.load(path)
    sd = {k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd::")}
    P = oti.params_from_state_dict(sd)
    n_items, d = P["item_emb"].shape[0] - 1, P["item_emb"].shape[1]
    H, span, L = int(z["n_heads"]), int(z["time_span"]), P["pos_k"].shape[0]
    batch = [torch.from_numpy(z[k]) for k in ("ids", "pad", "times", "labels", "tmask")]
    eng = _engine(cuda, P, n_items, d, H, L, span, batch[0].shape[0])
    loss, G = _step(eng, *batch)
    ref_G = oti.params_from_state_dict({k[6:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("grad::")})
    _compare(loss, G, float(z["loss"]), ref_G)
    eng.set_batch(batch[0].to(cuda), batch[1].to(cuda))
    eng.set_times(batch[2].to(cuda))
    hid = eng.unpad_features(eng.forward_hidden_all()).float().cpu().view(*batch[0].shape, d)
    ref_h = torch.from_numpy(z["hidden"])
    assert float((hid - ref_h).norm() / ref_h.norm()) < 2e-2


@pytest.mark.gpu
@pytest.mark.parametrize("drop", [0.0, 0.2])
def test_padded_rows_are_exactly_zero(cuda, drop):
    g = torch.Generator().manual_seed(5)
    P = oti.random_params(100, 64, 32, 2, 16, seed=1)
    ids, pm, ts, lab, tm = _batch(8, 32, 100, g, span=16)
    eng = _engine(cuda, P, 100, 64, 2, 32, 16, 8, drop)
    _step(eng, ids, pm, ts, lab, tm)
    pad = ~pm.reshape(-1).to(cuda)
    for x in eng.x[1:]:
        assert torch.equal(x[pad], torch.zeros_like(x[pad]))
    assert bool(torch.isfinite(eng.g32).all())


def _module(dev, n_items=500, d=64, H=2, L=32, span=64, **kw):
    from replay_b200.models.nn.sequential import SasRec

    torch.manual_seed(0)
    return SasRec(_schema(n_items, d), block_count=2, head_count=H, hidden_size=d, max_seq_len=L, dropout_rate=kw.pop("drop", 0.0),
                  ti_modification=True, time_span=span, device=dev, **kw)


def _lbatch(dev, B, L, n_items, seed=0):
    g = torch.Generator().manual_seed(seed)
    ids, pm, ts, lab, tm = _batch(B, L, n_items, g, span=64)
    return {"feature_tensor": {"item_id": ids.to(dev), "timestamp": ts.to(dev)}, "padding_mask": pm.to(dev),
            "positive_labels": lab.to(dev), "target_padding_mask": tm.to(dev)}


@pytest.mark.gpu
def test_predict_topk_agrees_with_logits(cuda):
    m = _module(cuda)
    b = _lbatch(cuda, 64, 32, 500, seed=2)
    b["feature_tensor"] = {k: v[:, 4:] for k, v in b["feature_tensor"].items()}   # short batch: left-padded to max_len
    b["padding_mask"] = b["padding_mask"][:, 4:]
    seen = b["feature_tensor"]["item_id"]
    ids, scores = m.predict_topk(b, 10, seen_ids=seen)
    logits = m.predict(b).float()
    rows, cols = (seen < 500).nonzero(as_tuple=True)
    logits[rows, seen[rows, cols]] = float("-inf")
    # near-ties: every returned item scores within bf16 rounding of the k-th best of the materialised fp32 logits
    kth = logits.topk(10, dim=1).values[:, -1:]
    got = logits.gather(1, ids)
    assert bool((got >= kth - 2e-2 * kth.abs().clamp_min(1)).all())
    assert float((scores.float() - got).abs().max()) < 5e-2


@pytest.mark.gpu
def test_lightning_training_paths_agree(cuda):
    from replay_b200.core import SasRecCore

    b = _lbatch(cuda, 16, 32, 500, seed=4)
    losses = []
    for fused, graph in ((True, True), (True, False), (False, False)):
        old = SasRecCore.use_cuda_graph
        SasRecCore.use_cuda_graph = graph
        try:
            m = _module(cuda, fused_optimizer=fused)
            losses.append(float(m.training_step(b)))
        finally:
            SasRecCore.use_cuda_graph = old
    assert abs(losses[0] - losses[1]) < 1e-4 * abs(losses[0]) and abs(losses[0] - losses[2]) < 1e-4 * abs(losses[0]), losses
    m = _module(cuda)   # a few graph-replayed steps train
    first = float(m.training_step(b))
    for _ in range(20):
        last = float(m.training_step(b))
    assert last < first


@pytest.mark.gpu
def test_timestamp_dtype_change_rebuilds_the_captured_step(cuda):
    """Graph-replayed steps on int64 timestamps, then the same values as float64: the captured launches carry the
    timestamps' dtype, so the core must drop them.  The float64 step's loss equals an eager step's on the same state."""
    from replay_b200.core import SasRecCore

    b = _lbatch(cuda, 16, 32, 500, seed=12)
    b["feature_tensor"]["timestamp"] = b["feature_tensor"]["timestamp"].floor().to(torch.int64)
    b64 = dict(b, feature_tensor=dict(b["feature_tensor"], timestamp=b["feature_tensor"]["timestamp"].double()))
    graph, eager = _module(cuda), _module(cuda)
    old = SasRecCore.use_cuda_graph
    try:
        SasRecCore.use_cuda_graph = True
        for _ in range(3):
            graph.training_step(b)
        eager.load_state_dict(graph.state_dict())
        got = float(graph.training_step(b64))
        SasRecCore.use_cuda_graph = False
        want = float(eager.training_step(b64))
    finally:
        SasRecCore.use_cuda_graph = old
    assert graph._model.core.engine.times_dtype == 2
    assert abs(got - want) <= 1e-4 * abs(want), (got, want)


@pytest.mark.gpu
def test_checkpoint_round_trip_and_catalog_growth(cuda):
    m = _module(cuda)
    b = _lbatch(cuda, 8, 32, 500, seed=6)
    m.training_step(b)
    sd = m.state_dict()
    m2 = _module(cuda)
    m2.load_state_dict(sd)
    assert torch.allclose(m.predict(b), m2.predict(b))
    before = m.get_all_embeddings()
    assert set(before) == {"item_embedding", "abs_pos_k_emb", "abs_pos_v_emb", "time_matrix_k_emb", "time_matrix_v_emb"}
    m.set_item_embeddings_by_size(520)
    after = m.get_all_embeddings()
    assert after["item_embedding"].shape[0] == 520
    for k in ("abs_pos_k_emb", "abs_pos_v_emb", "time_matrix_k_emb", "time_matrix_v_emb"):
        assert torch.equal(before[k], after[k]), k
    assert torch.isfinite(m.training_step(b))


@pytest.mark.gpu
@pytest.mark.parametrize("loss", ["CE_sampled", "BCE_sampled", "SCE"])
def test_sampled_and_sce_losses_train(cuda, loss):
    from replay_b200.models.nn.loss import SCEParams

    if loss == "SCE":
        kw = dict(loss_type="SCE", sce_params=SCEParams(n_buckets=4, bucket_size_x=16, bucket_size_y=16))
    else:
        kw = dict(loss_type=loss.split("_")[0], loss_sample_count=20)
    m = _module(cuda, **kw)
    b = _lbatch(cuda, 16, 32, 500, seed=8)
    losses = [float(m.training_step(b)) for _ in range(5)]
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses


@pytest.mark.gpu
def test_config2_step_memory_has_no_b_l2_d_term(cuda):
    """B 256, L 200, d 128, 2 heads, dropout 0.2: the step trains, and its peak memory stays below a bound with B*H*L^2
    (probabilities) and B*L*d (activations) terms only - the reference's [B, L, L, d] time tensors would be 1.3 GB each."""
    B, L, d, H, n_items, span = 256, 200, 128, 2, 50_000, 256
    m = _module(cuda, n_items=n_items, d=d, H=H, L=L, span=span, drop=0.2)
    b = _lbatch(cuda, B, L, n_items, seed=9)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(cuda)
    base = torch.cuda.memory_allocated(cuda)
    losses = [float(m.training_step(b)) for _ in range(3)]
    peak = torch.cuda.max_memory_allocated(cuda) - base
    Lp, T, n_blocks = 256, B * L, 2
    probs = B * H * Lp * Lp * (4 + 2 + 2 + 2 * n_blocks)          # S fp32, Ad, dS bf16, A per block
    acts = T * d * 2 * (8 * n_blocks + 16) + T * 64               # bf16 activations / scratch, row statistics
    head = T * n_items * 0 + 64 * n_items * d * 4 + (1 << 28)     # CE head workspace and slack
    bound = probs + acts + head
    assert all(np.isfinite(losses))
    assert peak < bound, (peak / 2**20, bound / 2**20)
    assert peak < B * L * L * d * 4, "a [B, L, L, d] fp32 tensor would not fit this budget"
