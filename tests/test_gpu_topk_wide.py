"""Fused top-K for 32 < K <= 1024 (score_topk_wide_kernel + topk_wide_merge_kernel) against the fp64 oracle on the same bf16
inputs, at tile, split and K-th-place ties, with fewer than K unmasked items, on adversarial item orders, at the config-4
predict shape, and through the modules and callbacks that pick it up via ops.MAX_FUSED_K."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from replay_b200 import ops as _ops

    return _ops


def _oracle(hq, table, seen, K, bias=None, candidates=None):
    """oracle.sasrec.score_topk in fp64; a bias enters as one more feature column (hq . 1 + bias)."""
    from oracle import sasrec as osr

    hq, table = hq.double(), table.double()
    if bias is not None:
        hq = torch.cat([hq, torch.ones(hq.shape[0], 1, dtype=torch.float64)], 1)
        table = torch.cat([table, bias[:table.shape[0], None].double()], 1)
    return osr.score_topk(hq, table, seen, K, candidates=candidates, acc_dtype=torch.float64), hq, table


def _check(ids, sc, ref, hq64, tb64, columns=True):
    """_topk_case's adjudication: scores within fp32 noise; an index swap only between scores closer than fp32 accumulation
    noise and never inside an exact tie.  ids are item ids, i.e. rows of tb64 (the full, bias-augmented table)."""
    (ids_ref, sc_ref) = ref
    ids, sc = ids.cpu(), sc.cpu()
    torch.testing.assert_close(sc.double(), sc_ref, rtol=1e-4, atol=1e-4)
    assert ((sc[:, :-1] > sc[:, 1:]) | (sc[:, :-1] == sc[:, 1:])).all()
    mism = ids != ids_ref
    if mism.any():
        full = hq64 @ tb64.T
        gap = (torch.gather(full, 1, ids.clamp_min(0)) - torch.gather(full, 1, ids_ref.clamp_min(0))).abs()
        assert (gap[mism] < 1e-5).all(), f"{int(mism.sum())} index mismatches"
        assert mism.float().mean() < 1e-3
        # two rows can tie exactly in fp64 yet round to different fp32 sums; the kernel orders by its own scores, and
        # bit-equal kernel scores by ascending column (bit-equal table rows are checked exactly in the tie test)
        if columns:
            same = sc[:, :-1] == sc[:, 1:]
            assert (ids[:, :-1][same] < ids[:, 1:][same]).all()


def _case(ops, B, I, d, K, S, seed, bias=False, cands=False):
    g = torch.Generator().manual_seed(seed)
    hq = (torch.randn(B, d, generator=g) * 0.5).to(torch.bfloat16)
    table = (torch.randn(I, d, generator=g) * 0.5).to(torch.bfloat16)
    b = torch.randn(I, generator=g) * 2.0 if bias else None
    seen = None
    if S:
        seen = torch.randint(-3, I + 5, (B, S), generator=g)  # ids outside [0, I) are padding
        seen[0, :] = I                                       # a user with nothing seen
        if B > 1:
            seen[1, : S // 2] = seen[1, 0]                   # duplicates
    c = torch.randperm(I, generator=g)[: max(K, I * 3 // 4)] if cands else None
    ref, hq64, tb64 = _oracle(hq, table, seen, K, b, c)
    # the kernel scores the gathered rows; its bias is per scored column, padded to a multiple of 128
    tb_k = table if c is None else table[c]
    b_k = None
    if b is not None:
        b_k = torch.zeros((tb_k.shape[0] + 127) // 128 * 128)
        b_k[:tb_k.shape[0]] = b if c is None else b[c]
    inv = None
    if c is not None:
        inv = torch.full((I,), -1, dtype=torch.int32)
        inv[c] = torch.arange(c.numel(), dtype=torch.int32)
    seen_sorted = ops.seen_prepare(seen.cuda(), I, None if inv is None else inv.cuda()) if seen is not None else None
    ids, sc = ops.score_topk(hq.cuda(), tb_k.contiguous().cuda(), K, seen_sorted, None if c is None else c.cuda(),
                             bias=None if b_k is None else b_k.cuda())
    _check(ids, sc, ref, hq64, tb64, columns=c is None)
    return ids, sc


@pytest.mark.parametrize("B,I,d,K,S,bias,cands", [
    (1, 33, 64, 33, 0, False, False),           # n_items = K
    (127, 65, 128, 64, 0, True, False),         # n_items = K + 1
    (128, 5000, 256, 100, 200, False, False),
    (129, 5000, 512, 128, 64, True, False),
    (4096, 5000, 128, 100, 200, False, False),
    (129, 50_000, 64, 257, 200, True, False),
    (127, 1001, 256, 1000, 16, False, False),
    (128, 5003, 512, 1000, 100, False, True),   # candidates, seen mapped through inv_map
    (129, 1025, 64, 1024, 0, True, False),
    (1, 50_000, 128, 1024, 200, False, False),
    (4096, 5000, 64, 1024, 50, False, False),
    (130, 50_000, 512, 33, 200, False, True),
    (200, 5000, 128, 257, 0, True, True),       # candidates + bias
])
def test_wide_topk_matches_oracle(ops, B, I, d, K, S, bias, cands):
    _case(ops, B, I, d, K, S, seed=B + I + K + d, bias=bias, cands=cands)


def _wide_splits(B, I, K):
    """item-split boundaries of the wide kernel (rp_score_topk.cu wide_splits)"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    C = 128
    while C < 2 * K or C < K + 64:
        C *= 2
    n_tiles, ut = (I + 127) // 128, (B + 127) // 128
    p = min(max(1, sms // ut), n_tiles, 64, 65536 // C)
    return [(n_tiles * s // p) * 128 for s in range(1, p)]


@pytest.mark.parametrize("K", [100, 1000])
def test_wide_topk_ties_at_every_boundary(ops, K):
    """Bit-equal table rows straddle the 32-column part, 64-column half, 128-column tile and item-split boundaries; the K-th
    place falls inside the second tie group.  The result is (score desc, column asc), exactly the oracle's."""
    B, I, d = 130, 50_000, 128
    g = torch.Generator().manual_seed(K)
    u = torch.nn.functional.normalize(torch.randn(d, generator=g), dim=0)
    hq = (u[None, :] * 1.5 + torch.randn(B, d, generator=g) * 0.05).to(torch.bfloat16)
    table = (torch.randn(I, d, generator=g) * 0.05).to(torch.bfloat16)
    cuts = _wide_splits(B, I, K)
    assert len(cuts) >= 2
    edges = [31, 32, 63, 64, 127, 128, 255, 256] + [c + o for c in (cuts[0], cuts[len(cuts) // 2], cuts[-1]) for o in (-1, 0)]
    n_a, n_b = K * 6 // 10, K * 8 // 10     # group A fully in, group B's K - n_a smallest columns in
    rest = torch.randperm(I, generator=g)
    rest = rest[~torch.isin(rest, torch.tensor(edges))]
    ga = sorted(edges[: len(edges) // 2] + rest[: n_a - len(edges) // 2].tolist())
    gb = sorted(edges[len(edges) // 2:] + rest[n_a: n_a + n_b - (len(edges) - len(edges) // 2)].tolist())
    for c, pos in ((3.0, ga), (2.8, gb)):
        table[torch.tensor(pos)] = (u * c + torch.randn(d, generator=g) * 0.01).to(torch.bfloat16)
    seen = torch.randint(0, I + 50, (B, 50), generator=g)
    seen[0] = I                                               # user 0: nothing seen
    seen[5, :4] = torch.tensor([ga[0], ga[-1], gb[0], gb[3]])  # user 5: tie rows seen
    ids, sc = ops.score_topk(hq.cuda(), table.cuda(), K, ops.seen_prepare(seen.cuda(), I))
    ids, sc = ids.cpu(), sc.cpu()
    (ids_ref, sc_ref), hq64, tb64 = _oracle(hq, table, seen, K)
    for user in (0, 1, 5, 127, 128, 129):
        assert torch.equal(ids[user], ids_ref[user]), user
    want0 = ga + gb[: K - n_a]
    assert ids[0].tolist() == want0
    assert (sc[0, :n_a] == sc[0, 0]).all() and (sc[0, n_a:] == sc[0, n_a]).all() and sc[0, 0] > sc[0, n_a]
    _check(ids, sc, (ids_ref, sc_ref), hq64, tb64)


@pytest.mark.parametrize("K,d", [(100, 128), (1000, 512)])
def test_wide_topk_fewer_than_k_unseen(ops, K, d):
    """n_items = K + 5 with 20 distinct seen items: the last 15 slots hold the seen columns in ascending order, score -inf."""
    B, I = 3, K + 5
    g = torch.Generator().manual_seed(K)
    hq = torch.randn(B, d, generator=g).to(torch.bfloat16)
    table = torch.randn(I, d, generator=g).to(torch.bfloat16)
    seen = torch.stack([torch.randperm(I, generator=g)[:20] for _ in range(B)])
    seen = torch.cat([seen, seen[:, :5], torch.full((B, 3), I + 7)], 1)  # duplicates and padding
    ids, sc = ops.score_topk(hq.cuda(), table.cuda(), K, ops.seen_prepare(seen.cuda(), I))
    ids, sc = ids.cpu(), sc.cpu()
    (ids_ref, sc_ref), _, _ = _oracle(hq, table, seen, K)
    assert torch.equal(ids, ids_ref)
    assert torch.isinf(sc[:, K - 15:]).all() and torch.isfinite(sc[:, : K - 15]).all()
    for b in range(B):
        assert ids[b, K - 15:].tolist() == sorted(set(seen[b].tolist()) - {I + 7})[:15]


def _ordered_table(I, d, descending):
    """hq = (1, 2^-8, 2^-16, 0, ...) and rows = base-256 digits of the column: every score is exact in bf16 x fp32 and
    strictly increasing (or decreasing) with the column."""
    j = torch.arange(I)
    v = (I - j) if descending else (j + 1)
    table = torch.zeros(I, d)
    table[:, 0], table[:, 1], table[:, 2] = (v // 65536).float(), ((v // 256) % 256).float(), (v % 256).float()
    return table.to(torch.bfloat16)


@pytest.mark.parametrize("descending", [False, True])
@pytest.mark.parametrize("K", [100, 1024])
def test_wide_topk_adversarial_item_orders(ops, K, descending):
    """Ascending scores admit every item (compaction as often as it can run); descending ones admit only the first tiles."""
    B, I, d = 256, 50_000, 128
    hq = torch.zeros(B, d)
    hq[:, 0], hq[:, 1], hq[:, 2] = 1.0, 2.0 ** -8, 2.0 ** -16
    hq = hq.to(torch.bfloat16)
    table = _ordered_table(I, d, descending)
    g = torch.Generator().manual_seed(1)
    seen = torch.randint(0, I + 10, (B, 200), generator=g)
    hi = torch.arange(I - 2 * K, I) if not descending else torch.arange(0, 2 * K)
    seen[:, :50] = hi[torch.randint(0, hi.numel(), (B, 50), generator=g)]  # seen items among the winners
    ids, sc = ops.score_topk(hq.cuda(), table.cuda(), K, ops.seen_prepare(seen.cuda(), I))
    (ids_ref, sc_ref), _, _ = _oracle(hq, table, seen, K)
    assert torch.equal(ids.cpu(), ids_ref)
    assert torch.equal(sc.cpu().double(), sc_ref)


def test_wide_topk_exact_zero_tie_across_splits(ops):
    """The K-th place is an exact-zero tie.  The later item splits hold only zeros (and the positives), so they publish a
    shared K-th best of exactly 0 within their first tiles.  Split 0 holds -1 scores and meets its zeros only in its last
    tile, long after that.  Its zeros have the smallest columns, so they win the tie and must still be admitted."""
    B, I, d, K = 4096, 200_000, 64, 100
    cuts = _wide_splits(B, I, K)
    assert len(cuts) >= 2 and cuts[0] >= 1024
    z0 = cuts[0] - 128                                       # split 0's last tile: its first zero column
    n_pos = K - 5
    pos = torch.arange(n_pos) * 7 + cuts[-1] + 1000          # positives inside the last split
    col0 = torch.zeros(I)
    col0[:z0] = -1.0
    col0[pos] = 1.0 + torch.arange(n_pos, dtype=torch.float32) / 128   # distinct, exact in bf16
    table = torch.zeros(I, d)
    table[:, 0] = col0
    hq = torch.zeros(B, d)
    hq[:, 0] = 1.0
    ids, sc = ops.score_topk(hq.to(torch.bfloat16).cuda(), table.to(torch.bfloat16).cuda(), K)
    want = pos.flip(0).tolist() + list(range(z0, z0 + 5))
    want_sc = (1.0 + torch.arange(n_pos, dtype=torch.float32) / 128).flip(0).tolist() + [0.0] * 5
    assert (ids.cpu() == torch.tensor(want)).all(), ids[0].tolist()
    assert (sc.cpu() == torch.tensor(want_sc)).all()


# ----------------------------------------------------------------------------------------------------------------------
# config 4: 4096 users x 500 000 items, d = 128, S = 200 (construction of test_gpu_fullshape._c4_case)
# ----------------------------------------------------------------------------------------------------------------------
def _c4_case(seed=7, B=4096, I=500_000, d=128, S=200):
    g = torch.Generator().manual_seed(seed)
    u = torch.nn.functional.normalize(torch.randn(d, generator=g), dim=0)
    hq = (u[None, :] * 1.5 + torch.randn(B, d, generator=g) * 0.3).to(torch.bfloat16)
    table = (torch.randn(I, d, generator=g) * 0.05).to(torch.bfloat16)
    n_tiles, p = (I + 127) // 128, max(1, 148 // ((B + 127) // 128))
    cuts = [(n_tiles * s // p) * 128 for s in range(1, p)]
    groups = [
        (3.0, [31, 32, 127, 128]),
        (2.8, [cuts[0] - 1, cuts[0], cuts[-1] - 1, cuts[-1]]),
        (2.6, [63, 64, cuts[len(cuts) // 2] - 1, cuts[len(cuts) // 2], I - 2, I - 1]),
    ]
    for c, pos in groups:
        v = (u * c + torch.randn(d, generator=g) * 0.02).to(torch.bfloat16)
        table[torch.tensor(pos)] = v
    seen = torch.randint(0, I + 50, (B, S), generator=g)
    seen[5, :4] = torch.tensor([31, 128, cuts[0], 63])
    return hq, table, seen


@pytest.mark.parametrize("K", [100, 1024])
def test_c4_wide_topk(ops, K):
    hq, table, seen = _c4_case()
    B, I = hq.shape[0], table.shape[0]
    hq_d, tb_d, seen_d = hq.cuda(), table.cuda(), seen.cuda()
    seen_sorted = ops.seen_prepare(seen_d, I)
    ids0, sc0 = ops.score_topk(hq_d, tb_d, K, seen_sorted)
    # every user against chunked fp64 torch on the GPU: the scores, and the returned ids carry them and were not seen
    tb64 = tb_d.double()
    for lo in range(0, B, 256):
        s64 = hq_d[lo:lo + 256].double() @ tb64.T
        sd = seen_d[lo:lo + 256]
        ok = (sd >= 0) & (sd < I)
        rows = torch.arange(s64.shape[0], device=sd.device)[:, None].expand_as(sd)
        s64[rows[ok], sd[ok]] = float("-inf")
        ref = torch.topk(s64, K, dim=1)
        torch.testing.assert_close(sc0[lo:lo + 256].double(), ref.values, rtol=1e-4, atol=1e-4)
        torch.testing.assert_close(torch.gather(s64, 1, ids0[lo:lo + 256]), ref.values, rtol=1e-4, atol=1e-4)
        assert (torch.sort(ids0[lo:lo + 256], 1).values[:, 1:] != torch.sort(ids0[lo:lo + 256], 1).values[:, :-1]).all()
    assert (sc0[:, :-1] >= sc0[:, 1:]).all()
    if K == 100:  # same total order as the K = 32 kernel: its output is our prefix, bit for bit
        ids32, sc32 = ops.score_topk(hq_d, tb_d, 32, seen_sorted)
        assert torch.equal(ids0[:, :32], ids32) and torch.equal(sc0[:, :32], sc32)
    for _ in range(10):
        ids, sc = ops.score_topk(hq_d, tb_d, K, seen_sorted)
        assert torch.equal(ids, ids0) and torch.equal(sc, sc0)
    for users in (512, 32768):
        rep = (users + B - 1) // B
        hq_u = hq_d.repeat(rep, 1)[:users].contiguous()
        ids_u, sc_u = ops.score_topk(hq_u, tb_d, K, ops.seen_prepare(seen_d.repeat(rep, 1)[:users].contiguous(), I))
        n = min(users, B)
        assert torch.equal(ids_u[:n], ids0[:n]) and torch.equal(sc_u[:n], sc0[:n])
        if users > B:
            assert torch.equal(ids_u[B:2 * B], ids0) and torch.equal(sc_u[B:2 * B], sc0)
        del hq_u, ids_u, sc_u


# ----------------------------------------------------------------------------------------------------------------------
# public surfaces
# ----------------------------------------------------------------------------------------------------------------------
class _Seqs:
    """The ``sequential`` that RemoveSeenItems reads: each query's stored item ids."""

    def __init__(self, ids, n_items):
        from replay_b200.schema import TensorFeatureInfo, TensorSchema

        self.schema = TensorSchema(TensorFeatureInfo("item_id", n_items, 0, 8))
        self._ids = ids.cpu()

    def get_sequence_by_query_id(self, query_ids, feature):
        return [self._ids[int(q)][self._ids[int(q)] < self.schema.item_id_features.item().cardinality].numpy()
                for q in query_ids]


def _tutorial_bert4rec(B=96):
    """Bert4Rec(hidden 300, 4 heads, L = 100, 3 700 items) and a prediction batch as its dataset builds it: shifted, with
    ``pad_mask`` / ``token_mask`` (no ``padding_mask``), plus the RemoveSeenItems that reads each user's history."""
    from replay_b200.models.nn.sequential import Bert4Rec, RemoveSeenItems
    from replay_b200.models.nn.sequential.bert4rec import shift_features
    from replay_b200.schema import TensorFeatureInfo, TensorSchema
    from replay_b200.synthetic import make_sequences

    n_items, d, H, L = 3700, 300, 4, 100
    m = Bert4Rec(TensorSchema(TensorFeatureInfo("item_id", n_items, 0, d)), block_count=2, head_count=H, hidden_size=d,
                 max_seq_len=L, dropout_rate=0.0)
    ids, pm, _, _ = make_sequences(B, n_items, L, seed=3, pad_value=0)
    ids, pm = ids.cuda(), pm.cuda()
    sids, spm, stm = shift_features(ids, pm, pm, 0)
    batch = {"query_id": torch.arange(B).cuda()[:, None], "inputs": {"item_id": sids}, "pad_mask": spm, "token_mask": stm}
    return m, batch, RemoveSeenItems(_Seqs(ids.masked_fill(~pm, n_items), n_items))


def _count_fused_calls(m):
    calls = []
    orig = m.predict_topk
    m.predict_topk = lambda *a, **k: (calls.append(a[1]), orig(*a, **k))[1]
    return calls


@pytest.mark.parametrize("top_k", [10, 100])
def test_legacy_bert4rec_tutorial_prediction_callback(ops, top_k):
    """PandasPredictionCallback(top_k, RemoveSeenItems) on the tutorial-shaped Bert4Rec runs fused (its batches carry
    ``pad_mask``, so this also covers K <= 32) and equals the module's own dense scores -> RemoveSeenItems -> torch.topk."""
    from replay_b200.models.nn.sequential import PandasPredictionCallback

    m, batch, post = _tutorial_bert4rec()
    B = batch["query_id"].shape[0]
    cb = PandasPredictionCallback(top_k=top_k, query_column="user", item_column="item", postprocessors=[post])
    cb.on_predict_epoch_start(None, m)
    calls = _count_fused_calls(m)
    cb.on_predict_batch_end(None, m, None, batch, 0)   # the fused path never reads the dense outputs
    assert calls == [top_k]
    df = cb.get_result()
    got_ids = torch.tensor(df["item"].to_numpy()).view(B, top_k)
    got_sc = torch.tensor(df["rating"].to_numpy()).view(B, top_k)
    dense = m.predict_step(batch, 0)
    _, filt = post.on_prediction(batch["query_id"], dense)
    ref = torch.topk(filt, top_k, dim=1)
    torch.testing.assert_close(got_sc, ref.values.cpu(), rtol=0, atol=1e-4)
    mism = got_ids != ref.indices.cpu()
    if mism.any():  # only swaps between (near-)tied scores
        gap = (torch.gather(filt.cpu(), 1, got_ids) - torch.gather(filt.cpu(), 1, ref.indices.cpu())).abs()
        assert (gap[mism] <= 1e-4).all()


def test_legacy_validation_metrics_ks_up_to_100_fused_on_bert4rec(ops):
    """ValidationMetricsCallback(ks=[1, 10, 20, 100], RemoveSeenItems) on Bert4Rec: fused top-100, metrics equal to the
    dense scores -> RemoveSeenItems -> torch.topk path."""
    from replay_b200.models.nn.sequential import ValidationMetricsCallback

    m, batch, post = _tutorial_bert4rec()
    g = torch.Generator().manual_seed(4)
    batch["ground_truth"] = torch.randint(0, 3700, (batch["query_id"].shape[0], 3), generator=g).cuda()
    mk = lambda: ValidationMetricsCallback(metrics=("recall", "ndcg", "map", "mrr", "precision"), ks=[1, 10, 20, 100],  # noqa: E731
                                           postprocessors=[post])
    fused, dense = mk(), mk()
    fused.on_validation_epoch_start(None, m)
    calls = _count_fused_calls(m)
    fused.on_validation_batch_end(None, m, None, batch, 0)
    assert calls == [100]

    class _NoFusedHead:                                # same scores, no predict_topk: the dense path
        pass

    dense.on_validation_epoch_start(None, _NoFusedHead())
    dense.on_validation_batch_end(None, _NoFusedHead(), m.predict_step(batch, 0), batch, 0)
    mf, md = fused.on_validation_epoch_end(None, _NoFusedHead()), dense.on_validation_epoch_end(None, _NoFusedHead())
    assert set(mf) == set(md) and any(k.endswith("@100") for k in mf)
    for k in mf:
        assert abs(mf[k] - md[k]) < 1e-6, (k, mf[k], md[k])


def test_legacy_sasrec_predict_topk_100_cuda_graph(ops):
    """Legacy SasRec.predict_topk at K = 100 through the CUDA-graph path: three eager calls, then capture; replay == eager."""
    from replay_b200.models.nn.sequential import SasRec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema
    from replay_b200.synthetic import make_sequences

    n_items, d, L, B = 20_000, 64, 50, 256
    m = SasRec(TensorSchema(TensorFeatureInfo("item_id", n_items, 0, d)), block_count=2, head_count=1, hidden_size=d,
               max_seq_len=L, dropout_rate=0.0)
    m.eval()
    ids, pm, _, _ = make_sequences(B, n_items, L, seed=4)
    batch = {"feature_tensor": {"item_id": ids.cuda()}, "padding_mask": pm.bool().cuda()}
    seen = ids.cuda()
    core = m._model.core
    assert core.use_cuda_graph
    outs = [m.predict_topk(dict(batch), 100, seen_ids=seen) for _ in range(5)]
    key = [k for k in core._predict_graphs if k[2] == 100]
    assert key and "graph" in core._predict_graphs[key[0]]
    for ids_, sc_ in outs[1:]:
        assert torch.equal(ids_, outs[0][0]) and torch.equal(sc_, outs[0][1])
    dense = m.predict(dict(batch)).float()
    col = torch.where((seen >= 0) & (seen < n_items), seen, torch.full_like(seen, n_items))
    masked = torch.zeros(B, n_items + 1, dtype=torch.bool, device=seen.device).scatter_(1, col, True)[:, :n_items]
    torch.testing.assert_close(outs[0][1], torch.topk(dense.masked_fill(masked, float("-inf")), 100, dim=1).values,
                               rtol=0, atol=1e-3)


def _new_path(n_items=4000, d=64, L=32, B=200):
    from replay_b200.nn.lightning import LightningModule
    from replay_b200.nn.sequential import SasRec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema
    from replay_b200.synthetic import make_sequences

    model = SasRec.from_params(TensorSchema(TensorFeatureInfo("item_id", n_items, n_items, d)), embedding_dim=d,
                               num_heads=1, num_blocks=2, max_sequence_length=L, dropout=0.0, seed=5)
    model.eval()
    lm = LightningModule(model)
    ids, pm, _, _ = (t.cuda() for t in make_sequences(B, n_items, L, seed=6))
    g = torch.Generator().manual_seed(2)
    gt = torch.randint(0, n_items, (B, 3), generator=g).cuda()
    batch = {"query_id": torch.arange(B).cuda(), "feature_tensors": {"item_id": ids}, "padding_mask": pm, "seen_ids": ids,
             "ground_truth": gt}
    return lm, batch, n_items


def test_top_items_callback_top100_fused_equals_logits_path(ops):
    from replay_b200.nn.lightning import SeenItemsFilter, TorchTopItemsCallback

    lm, batch, n_items = _new_path()
    filt = SeenItemsFilter(item_count=n_items, seen_items_column="seen_ids")
    cb = TorchTopItemsCallback(top_k=100, query_column="query_id", item_column="item_id", postprocessors=[filt])
    cb.on_predict_epoch_start(None, lm)
    out = lm.predict_step(batch, 0)
    cb.on_predict_batch_end(None, lm, out, batch, 0)
    assert not out.materialised                       # fused: the logits were never built
    _, items, scores = cb.get_result()
    logits = filt.on_prediction(batch, out["logits"])
    ref = torch.topk(logits, 100, dim=1)
    torch.testing.assert_close(scores, ref.values.cpu(), rtol=0, atol=1e-3)
    mism = items != ref.indices.cpu()
    if mism.any():
        lc = logits.cpu()
        assert ((torch.gather(lc, 1, items) - torch.gather(lc, 1, ref.indices.cpu())).abs()[mism] <= 1e-3).all()


def test_compute_metrics_callback_ks_up_to_100_fused_equals_materialised(ops):
    from replay_b200.nn.lightning import ComputeMetricsCallback, SeenItemsFilter

    lm, batch, n_items = _new_path()
    ks = [1, 10, 20, 100]
    mk = lambda: ComputeMetricsCallback(metrics=("recall", "ndcg", "map", "mrr", "precision"), ks=ks,  # noqa: E731
                                        postprocessors=[SeenItemsFilter(item_count=n_items, seen_items_column="seen_ids")])
    fused, dense = mk(), mk()
    fused.on_validation_epoch_start(None, lm)
    out = lm.predict_step(batch, 0)
    fused.on_validation_batch_end(None, lm, out, batch, 0)
    assert not out.materialised

    class _NoEngine:                                   # same logits, no engine: the materialised path
        candidates_to_score = None
        model = None

    dense.on_validation_epoch_start(None, _NoEngine())
    dense.on_validation_batch_end(None, _NoEngine(), {"logits": out["logits"]}, batch, 0)
    mf, md = fused.on_validation_epoch_end(None, lm), dense.on_validation_epoch_end(None, _NoEngine())
    assert set(mf) == set(md) and any(k.endswith("@100") for k in mf)
    for k in mf:
        assert abs(mf[k] - md[k]) < 1e-6, (k, mf[k], md[k])
