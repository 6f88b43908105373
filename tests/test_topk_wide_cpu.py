"""Wide fused top-K (32 < K <= 1024) without a GPU: the C ABI's shape errors and workspace sizes, and the legacy prediction
callback's choice between the fused head and dense scores."""
import ctypes

import torch

ESHAPE = -2


def _sms():
    # rp_score_topk sizes its item splits by the SM count; without a device it assumes an H100 SXM (132 SMs)
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


def test_score_topk_shape_errors_for_wide_k_without_a_gpu():
    from replay_b200._lib import lib

    L = lib()
    bufs = [ctypes.create_string_buffer(64) for _ in range(5)]
    hq, table, out_ids, out_scores, ws = (ctypes.cast(b, ctypes.c_void_p) for b in bufs)
    call = lambda n_users, n_items, K: L.rp_score_topk(hq, table, None, None, 0, n_users, n_items, 128, K, None,  # noqa: E731
                                                       out_ids, out_scores, ws, 1 << 40, None)
    assert call(4, 5000, 1025) == ESHAPE      # above the widest kernel
    assert call(4, 5000, 1 << 20) == ESHAPE
    assert call(4, 99, 100) == ESHAPE         # more slots than items
    assert call(4, 32, 33) == ESHAPE
    assert call(4, 5000, 0) == ESHAPE


def test_score_topk_workspace_sizes():
    from replay_b200._lib import lib

    L = lib()
    sms = _sms()
    for users, items, K in [(1, 100, 1), (130, 5000, 10), (4096, 500_000, 10), (4096, 500_000, 32), (32768, 500_000, 17)]:
        ut, it = (users + 127) // 128, (items + 127) // 128
        p = min(max(1, sms // ut), it, 64)
        assert L.rp_score_topk_workspace(users, items, 128, K) == users * p * 2 * K * 8 + users * 4 + 256
    # wide K: monotone in K and in users, and at least one C >= K + 64 buffer per user
    for items in (1100, 50_000, 500_000):
        ks = [33, 64, 100, 128, 257, 1000, 1024]
        for users in (1, 129, 4096, 32768):
            w = [L.rp_score_topk_workspace(users, items, 128, k) for k in ks]
            assert all(a <= b for a, b in zip(w, w[1:])), (users, items, w)
            assert all(x >= users * (k + 64) * 8 for x, k in zip(w, ks))
        for k in ks:
            w = [L.rp_score_topk_workspace(u, items, 128, k) for u in (1, 127, 128, 129, 512, 1000, 1024, 4096, 32768)]
            assert all(a <= b for a, b in zip(w, w[1:])), (k, items, w)
            assert w[-1] > w[0]
    # the per-user buffers stay bounded however few users share the GPU
    assert L.rp_score_topk_workspace(1, 500_000, 128, 1024) <= 65536 * 8 + 1024


class _LegacyStub:
    """A legacy module with the fused head: records the K it was asked for."""
    candidates_to_score = None

    def __init__(self):
        self.calls = []

    def predict_topk(self, batch, k, seen_ids=None, candidates_to_score=None):
        self.calls.append(k)
        B = batch["query_id"].shape[0]
        return torch.zeros(B, k, dtype=torch.long), torch.zeros(B, k)


def test_legacy_prediction_callback_routes_on_max_fused_k():
    from replay_b200.models.nn.sequential import TorchPredictionCallback
    from replay_b200.ops import MAX_FUSED_K

    assert MAX_FUSED_K == 1024
    n_items, B = MAX_FUSED_K + 10, 3
    scores = torch.randn(B, n_items)
    batch = {"query_id": torch.arange(B)[:, None], "padding_mask": torch.ones(B, 4, dtype=torch.bool)}
    for k in (1, 32, 33, 100, MAX_FUSED_K):
        pl = _LegacyStub()
        cb = TorchPredictionCallback(top_k=k, query_column="query_id", item_column="item_id")
        cb.on_predict_epoch_start(None, pl)
        cb.on_predict_batch_end(None, pl, scores, batch, 0)
        assert pl.calls == [k]
        assert cb.get_result()[1].shape == (B, k)
    # above the fused limit: dense scores and torch.topk, the module's fused head is not asked
    pl = _LegacyStub()
    cb = TorchPredictionCallback(top_k=MAX_FUSED_K + 1, query_column="query_id", item_column="item_id")
    cb.on_predict_epoch_start(None, pl)
    cb.on_predict_batch_end(None, pl, scores, batch, 0)
    assert pl.calls == []
    _, ids, sc = cb.get_result()
    ref = torch.topk(scores, MAX_FUSED_K + 1, dim=1)
    assert torch.equal(ids, ref.indices) and torch.equal(sc, ref.values)
