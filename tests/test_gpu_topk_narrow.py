"""Fused top-K for K <= 32 (score_topk_kernel + topk_merge_kernel, the register path) and the seen-list sort
(seen_prepare_kernel) against the fp64 oracle on the same bf16 inputs: at the K edges of the register templates (KMAX 10, 16,
32), every d and its ring depth, ragged catalogs smaller than one tile, the BERT4Rec bias, candidates, ties at the column-part,
half, tile, item-split and ragged-tile boundaries, an exact-zero tie at the K-th place across item splits, fewer than K unseen
items, adversarial item orders, seen items at the split cuts, and seen lists longer than one block can sort."""
import numpy as np
import pytest
import torch

import topk_reference as tr

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from replay_b200 import ops as _ops

    return _ops


def _repeat_equal(fn, ids0, sc0, n=10):
    """the result is bit-identical from run to run, whatever order the CTAs publish their thresholds in"""
    for _ in range(n):
        ids, sc = fn()
        assert torch.equal(ids, ids0) and torch.equal(sc, sc0)


# ----------------------------------------------------------------------------------------------------------------------
# shape grid: K at the template edges, d at every ring depth, B and I at the tile edges
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,I,d,K,S,bias,cands", [
    (1, 1, 64, 1, 0, False, False),             # n_items = K = 1
    (127, 2, 128, 1, 4, True, False),           # n_items = K + 1, most users have seen everything
    (4096, 5003, 128, 1, 64, True, False),
    (128, 10, 256, 10, 8, False, False),        # n_items = K
    (129, 11, 512, 10, 0, True, False),         # n_items = K + 1
    (1, 127, 256, 10, 16, False, False),
    (129, 5003, 128, 10, 5000, False, False),   # a seen list longer than seen_prepare_kernel sorts
    (4096, 127, 64, 11, 16, False, True),
    (129, 128, 64, 11, 16, True, True),
    (1, 128, 128, 16, 32, True, False),
    (128, 17, 64, 16, 0, False, False),         # n_items = K + 1
    (4096, 129, 256, 16, 8, False, False),
    (127, 50_000, 512, 16, 200, False, False),
    (127, 129, 256, 17, 32, False, False),
    (128, 5003, 64, 17, 50, False, False),
    (1, 50_000, 256, 17, 50, False, True),
    (128, 32, 512, 32, 0, True, False),         # n_items = K
    (127, 33, 128, 32, 20, False, True),        # 33 items, K = 32 candidates
    (129, 5003, 512, 32, 100, True, True),      # bias + candidates
    (4096, 5003, 64, 32, 200, False, False),
    (130, 50_000, 128, 10, 200, True, False),
    (128, 50_000, 64, 32, 4500, True, True),    # long seen list through inv_map, bias + candidates
])
def test_narrow_topk_matches_oracle(ops, B, I, d, K, S, bias, cands):
    tr.run_case(ops, B, I, d, K, S, seed=B + I + K + d, bias=bias, cands=cands)


# ----------------------------------------------------------------------------------------------------------------------
# ties at every boundary
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [64, 256])
@pytest.mark.parametrize("K", [1, 10, 16, 32])
def test_narrow_topk_ties_at_every_boundary(ops, K, d):
    """Two groups of bit-equal table rows.  Group A holds the K // 2 lowest 32-column-part / 64-column-half / 128-column-tile
    edges; group B the other such edges, both sides of three item-split cuts, both sides of the ragged last tile and I - 1,
    and columns past the last cut.  The K-th place falls inside group B, whose smallest columns win: for user 0 a low edge,
    for user 1 (who has seen every low edge) the split cuts, for user 2 (who has seen the first cut pair and I - 1) the
    next ones, for user 4 (who has seen all but group B's last K + 2 rows) the last column before the ragged tile.  Every
    user's ids equal the oracle's exactly."""
    B, I = 130, 50_000
    cuts = tr.narrow_cuts(B, I, tr.sm_count())
    assert len(cuts) >= 3
    ragged = I // 128 * 128                                   # first column of the ragged last tile
    low = [31, 32, 63, 64, 127, 128, 255, 256]
    hi = [c + o for c in (cuts[0], cuts[len(cuts) // 2], cuts[-1]) for o in (-1, 0)] + [ragged - 1, ragged, I - 1]
    g = torch.Generator().manual_seed(K * 1000 + d)
    u = torch.nn.functional.normalize(torch.randn(d, generator=g), dim=0)
    hq = (u[None, :] * 1.5 + torch.randn(B, d, generator=g) * 0.05).to(torch.bfloat16)
    table = (torch.randn(I, d, generator=g) * 0.05).to(torch.bfloat16)
    n_a = K // 2
    free = torch.arange(cuts[-1] + 1, ragged - 1)
    free = free[torch.randperm(free.numel(), generator=g)].tolist()
    ga = sorted(low[:n_a] + free[: max(0, n_a - 8)])
    gb = sorted(low[n_a:] + hi + free[max(0, n_a - 8): max(0, n_a - 8) + K + 4])
    for c, pos in ((3.0, ga), (2.8, gb)):
        if pos:
            table[torch.tensor(pos)] = (u * c + torch.randn(d, generator=g) * 0.01).to(torch.bfloat16)
    seen = torch.randint(0, I + 50, (B, 50), generator=g)
    seen[0] = I                                               # user 0: nothing seen
    seen[1] = I
    seen[1, :8] = torch.tensor(low)                           # user 1: every low edge
    seen[2] = I
    seen[2, :3] = torch.tensor([hi[0], hi[1], I - 1])         # user 2: the first cut pair and the last item
    seen[4] = I
    seen4 = ga + gb[: len(gb) - (K + 2)]
    seen[4, :len(seen4)] = torch.tensor(seen4)
    assert gb[-3:] == [ragged - 1, ragged, I - 1]
    seen[5, :3] = torch.tensor([gb[0], gb[3], (ga or gb)[-1]])
    hq_d, tb_d, ss = hq.cuda(), table.cuda(), ops.seen_prepare(seen.cuda(), I)
    ids0, sc0 = ops.score_topk(hq_d, tb_d, K, ss)
    ids, sc = ids0.cpu(), sc0.cpu()
    (ids_ref, sc_ref), hq64, tb64 = tr.oracle(hq, table, seen, K)
    assert torch.equal(ids, ids_ref)
    tr.check(ids, sc, (ids_ref, sc_ref), hq64, tb64)
    assert ids[0].tolist() == (ga + gb)[:K]
    want1 = [c for c in ga + gb if c not in low][:K]
    assert ids[1].tolist() == want1
    assert ids[2].tolist() == [c for c in ga + gb if c not in (hi[0], hi[1], I - 1)][:K]
    assert ids[4].tolist() == gb[len(gb) - (K + 2):][:K] and ids[4, K - 1] == ragged - 1
    in_a = torch.isin(ids[0], torch.tensor(ga or [-1]))
    assert (sc[0][in_a] == sc[0, 0]).all() and (sc[0][~in_a] == sc[0, K - 1]).all()
    _repeat_equal(lambda: ops.score_topk(hq_d, tb_d, K, ss), ids0, sc0)


# ----------------------------------------------------------------------------------------------------------------------
# exact-zero tie at the K-th place across item splits
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("signed_zeros", [False, True])
@pytest.mark.parametrize("K", [10, 32])
def test_narrow_topk_exact_zero_tie_across_splits(ops, K, signed_zeros):
    """The K-th place is an exact-zero tie.  The later item splits hold only zeros (and K - 5 positives), so they publish a
    shared K-th best of exactly 0 within their first tiles.  Split 0 holds -1 scores and meets its zeros only in its last
    tile, long after that.  Its zeros have the smallest columns, so they win the tie and must still be admitted.  With
    signed_zeros, hq = (1, -0, -0, ...) and the zero rows alternate +0 / -0 in feature 0, so the zero scores alternate
    +0 / -0 as well; -0 == +0, so the order is by column alone."""
    B, I, d = 4096, 200_000, 64
    cuts = tr.narrow_cuts(B, I, tr.sm_count())
    assert len(cuts) >= 2 and cuts[0] >= 1024
    z0 = cuts[0] - 128                                       # split 0's last tile: its first zero column
    n_pos = K - 5
    pos = torch.arange(n_pos) * 7 + cuts[-1] + 1000          # positives inside the last split
    col0 = torch.zeros(I)
    if signed_zeros:
        col0[1::2] = -0.0
    col0[:z0] = -1.0
    col0[pos] = 1.0 + torch.arange(n_pos, dtype=torch.float32) / 128   # distinct, exact in bf16
    table = torch.zeros(I, d)
    table[:, 0] = col0
    hq = torch.full((B, d), -0.0 if signed_zeros else 0.0)
    hq[:, 0] = 1.0
    hq_d, tb_d = hq.to(torch.bfloat16).cuda(), table.to(torch.bfloat16).cuda()
    assert bool(torch.signbit(tb_d[z0 + 1, 0])) == signed_zeros and bool(torch.signbit(hq_d[0, 1])) == signed_zeros
    ids0, sc0 = ops.score_topk(hq_d, tb_d, K)
    want = pos.flip(0).tolist() + list(range(z0, z0 + 5))
    want_sc = (1.0 + torch.arange(n_pos, dtype=torch.float32) / 128).flip(0).tolist() + [0.0] * 5
    assert (ids0.cpu() == torch.tensor(want)).all(), ids0[0].tolist()
    assert (sc0.cpu() == torch.tensor(want_sc)).all()
    _repeat_equal(lambda: ops.score_topk(hq_d, tb_d, K), ids0, sc0)


# ----------------------------------------------------------------------------------------------------------------------
# fewer than K unseen items: the merge kernel's -inf fill
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cands", [False, True])
@pytest.mark.parametrize("K,d", [(16, 64), (17, 256), (32, 512)])
def test_narrow_topk_fewer_than_k_unseen(ops, K, d, cands):
    """n_items = K + 5 scored columns; users 0-2 have seen 20 distinct of them (plus duplicates, padding and, with
    candidates, items that are not candidates): the last 15 slots hold the seen columns in ascending order, score -inf.
    User 3 has seen every item: all K slots are -inf, columns 0 .. K-1."""
    B, n = 4, K + 5
    g = torch.Generator().manual_seed(K + d)
    N = 3 * n if cands else n                                 # catalog size
    c = torch.randperm(N, generator=g)[:n] if cands else torch.arange(n)
    hq = torch.randn(B, d, generator=g).to(torch.bfloat16)
    table = torch.randn(N, d, generator=g).to(torch.bfloat16)
    others = torch.tensor(sorted(set(range(N)) - set(c.tolist())) or [N + 1])
    S = N + 12
    seen = torch.full((B, S), -1, dtype=torch.int64)
    for b in range(3):
        s = c[torch.randperm(n, generator=g)[:20]]
        row = torch.cat([s, s[:5], torch.full((3,), N + 7), others[:4]])
        seen[b, :row.numel()] = row[torch.randperm(row.numel(), generator=g)]
    seen[3, :n] = c[torch.randperm(n, generator=g)]
    inv = None
    if cands:
        inv = torch.full((N,), -1, dtype=torch.int32)
        inv[c] = torch.arange(n, dtype=torch.int32)
    ss = ops.seen_prepare(seen.cuda(), N, None if inv is None else inv.cuda())
    ids, sc = ops.score_topk(hq.cuda(), table[c].contiguous().cuda(), K, ss, c.cuda() if cands else None)
    ids, sc = ids.cpu(), sc.cpu()
    (ids_ref, sc_ref), _, _ = tr.oracle(hq, table, seen, K, candidates=c if cands else None)
    assert torch.equal(ids, ids_ref)
    assert torch.equal(sc[:3, K - 15:], torch.full((3, 15), float("-inf")))
    assert torch.isfinite(sc[:3, : K - 15]).all()
    torch.testing.assert_close(sc[:3, : K - 15].double(), sc_ref[:3, : K - 15], rtol=1e-4, atol=1e-4)
    pos_of = {int(x): i for i, x in enumerate(c.tolist())}
    for b in range(3):
        seen_cols = sorted({pos_of[int(x)] for x in seen[b].tolist() if int(x) in pos_of})
        assert ids[b, K - 15:].tolist() == c[torch.tensor(seen_cols[:15])].tolist()
    assert ids[3].tolist() == c[:K].tolist() and torch.isinf(sc[3]).all()


# ----------------------------------------------------------------------------------------------------------------------
# adversarial item orders
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("descending", [False, True])
@pytest.mark.parametrize("K", [10, 32])
def test_narrow_topk_adversarial_item_orders(ops, K, descending):
    """Ascending scores improve every list on every tile (the slow path and the threshold publish run as often as they
    can); descending ones fill the lists in the first tiles of split 0 and reject everything after.  Exact scores: ids
    and scores equal the oracle bit for bit."""
    B, I, d = 256, 50_000, 128
    hq = tr.ordered_hq(B, d)
    table = tr.ordered_table(I, d, descending)
    g = torch.Generator().manual_seed(K)
    seen = torch.randint(0, I + 10, (B, 200), generator=g)
    hi = torch.arange(I - 2 * K, I) if not descending else torch.arange(0, 2 * K)
    seen[:, :K] = hi[torch.randint(0, hi.numel(), (B, K), generator=g)]  # seen items among the winners
    ids, sc = ops.score_topk(hq.cuda(), table.cuda(), K, ops.seen_prepare(seen.cuda(), I))
    (ids_ref, sc_ref), _, _ = tr.oracle(hq, table, seen, K)
    assert torch.equal(ids.cpu(), ids_ref)
    assert torch.equal(sc.cpu().double(), sc_ref)


# ----------------------------------------------------------------------------------------------------------------------
# seen filter
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("with_inv", [False, True])
@pytest.mark.parametrize("S", [1, 63, 64, 65, 255, 256, 257, 1024, 1025, 4096, 4097, 20_000])
def test_seen_prepare_matches_reference(ops, S, with_inv):
    """ops.seen_prepare at each kernel template's edges and past the largest (S > 4096, a device-side sort): ids outside
    [0, item_count) and, with inv_map, items that are not candidates become INT32_MAX; the rest sorted ascending."""
    B, n_items = 7, 30_000
    g = torch.Generator().manual_seed(S)
    seen = torch.randint(-5, n_items + 5, (B, S), generator=g)
    seen[0] = -1                                              # nothing seen
    seen[1, : (S + 1) // 2] = seen[1, 0]                      # duplicates
    seen[2, :: 3] = n_items                                   # padding at ids >= item_count
    inv = None
    if with_inv:
        c = torch.randperm(n_items, generator=g)[: n_items // 2]
        inv = torch.full((n_items,), -1, dtype=torch.int32)
        inv[c] = torch.arange(c.numel(), dtype=torch.int32)
    out = ops.seen_prepare(seen.cuda(), n_items, None if inv is None else inv.cuda())
    assert out.dtype == torch.int32 and out.shape == (B, S) and out.is_cuda
    assert torch.equal(out.cpu(), tr.seen_prepare_reference(seen, n_items, inv))


@pytest.mark.parametrize("K", [10, 32])
def test_narrow_topk_seen_at_split_cuts(ops, K):
    """The best items sit both sides of item-split cuts, in both 32-column parts of a half and at I - 1, with distinct
    scores.  User 1 has seen all of them, users 2 and 3 every other one: the seen cursor's lower_bound at each split's first
    column and its advance across parts must drop exactly these."""
    B, I, d = 130, 50_000, 128
    cuts = tr.narrow_cuts(B, I, tr.sm_count())
    assert len(cuts) >= 3
    c1 = cuts[1]
    top = [cuts[0] - 1, cuts[0], cuts[-1] - 1, cuts[-1], I - 1] + [c1 + o for o in (31, 32, 63, 64, 95, 96)]
    g = torch.Generator().manual_seed(K)
    u = torch.nn.functional.normalize(torch.randn(d, generator=g), dim=0)
    hq = (u[None, :] * 1.5 + torch.randn(B, d, generator=g) * 0.05).to(torch.bfloat16)
    table = (torch.randn(I, d, generator=g) * 0.05).to(torch.bfloat16)
    for i, p in enumerate(top):
        table[p] = (u * (3.0 - 0.1 * i)).to(torch.bfloat16)  # descending in list order, well apart
    seen = torch.randint(-2, I + 50, (B, 64), generator=g)
    seen[0] = -1
    seen[1] = -1
    seen[1, : len(top)] = torch.tensor(top)
    seen[2] = -1
    seen[2, : len(top[::2])] = torch.tensor(top[::2])
    seen[3] = -1
    seen[3, : len(top[1::2])] = torch.tensor(top[1::2])
    ids, sc = ops.score_topk(hq.cuda(), table.cuda(), K, ops.seen_prepare(seen.cuda(), I))
    ids, sc = ids.cpu(), sc.cpu()
    ref, hq64, tb64 = tr.oracle(hq, table, seen, K)
    tr.check(ids, sc, ref, hq64, tb64)
    for user, want in ((0, top), (2, top[1::2]), (3, top[::2])):
        n = min(K, len(want))
        assert ids[user, :n].tolist() == want[:n], user
    assert not torch.isin(ids[1], torch.tensor(top)).any()


class _Histories:
    """The ``sequential`` that RemoveSeenItems reads: each query's whole stored history."""

    def __init__(self, histories, n_items):
        from replay_b200.schema import TensorFeatureInfo, TensorSchema

        self.schema = TensorSchema(TensorFeatureInfo("item_id", n_items, 0, 8))
        self._h = histories

    def get_sequence_by_query_id(self, query_ids, feature):
        return [self._h[int(q)] for q in query_ids]


def test_legacy_prediction_callback_history_longer_than_4096(ops):
    """TorchPredictionCallback + RemoveSeenItems on the legacy SasRec, one user with a 6 000-item history: the batch's seen
    matrix is padded to it.  The fused path equals the module's dense scores -> RemoveSeenItems -> torch.topk, through
    two eager calls, the CUDA-graph capture and a replay."""
    from replay_b200.models.nn.sequential import RemoveSeenItems, SasRec, TorchPredictionCallback
    from replay_b200.schema import TensorFeatureInfo, TensorSchema
    from replay_b200.synthetic import make_sequences

    n_items, d, L, B, K = 20_000, 64, 50, 64, 10
    m = SasRec(TensorSchema(TensorFeatureInfo("item_id", n_items, 0, d)), block_count=2, head_count=1, hidden_size=d,
               max_seq_len=L, dropout_rate=0.0)
    m.eval()
    ids, pm, _, _ = make_sequences(B, n_items, L, seed=4)
    rng = np.random.default_rng(5)
    hist = [rng.integers(0, n_items, 30) for _ in range(B)]
    hist[3] = rng.integers(0, n_items, 6000)
    post = RemoveSeenItems(_Histories(hist, n_items))
    batch = {"query_id": torch.arange(B).cuda()[:, None], "feature_tensor": {"item_id": ids.cuda()},
             "padding_mask": pm.bool().cuda()}
    cb = TorchPredictionCallback(top_k=K, query_column="query_id", item_column="item_id", postprocessors=[post])
    cb.on_predict_epoch_start(None, m)
    for _ in range(4):
        cb.on_predict_batch_end(None, m, None, batch, 0)  # the fused path never reads the dense outputs
    graphs = m._model.core._predict_graphs
    assert any(k[3] == (B, 6000) and "graph" in st for k, st in graphs.items())
    _, got_ids, got_sc = cb.get_result()
    got_ids, got_sc = got_ids.view(4, B, K), got_sc.view(4, B, K)
    for r in range(1, 4):
        assert torch.equal(got_ids[r], got_ids[0]) and torch.equal(got_sc[r], got_sc[0])
    got_ids, got_sc = got_ids[0], got_sc[0]
    assert not np.isin(got_ids[3].numpy(), hist[3]).any()
    dense = m.predict_step(batch, 0)
    _, filt = post.on_prediction(batch["query_id"], dense)
    ref = torch.topk(filt, K, dim=1)
    torch.testing.assert_close(got_sc, ref.values.cpu(), rtol=0, atol=1e-3)
    mism = got_ids != ref.indices.cpu()
    if mism.any():  # only swaps between (near-)tied scores
        fc = filt.cpu()
        assert ((torch.gather(fc, 1, got_ids) - torch.gather(fc, 1, ref.indices.cpu())).abs()[mism] <= 1e-3).all()
