"""Register-path fused top-K (K <= 32) and the seen-list sort without a GPU: rp_seen_prepare's length limit through the C
ABI, and the workspace the register path sizes from its item-split count (which the GPU tests' split cuts restate)."""
import ctypes

import torch

import topk_reference as tr

ESHAPE = -2


def _sms():
    # rp_score_topk sizes its item splits by the SM count; without a device it assumes an H100 SXM (132 SMs)
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


def test_seen_prepare_rejects_lists_longer_than_one_block_sorts():
    from replay_b200._lib import lib
    from replay_b200.ops import SEEN_PREPARE_MAX_S

    L = lib()
    seen, out = ctypes.create_string_buffer(64), ctypes.create_string_buffer(64)
    call = lambda n_users, S: L.rp_seen_prepare(seen, n_users, S, 1000, None, out, None)  # noqa: E731
    assert SEEN_PREPARE_MAX_S == 4096
    assert call(1, SEEN_PREPARE_MAX_S + 1) == ESHAPE
    assert call(3, 20_000) == ESHAPE
    assert call(1, 0) == ESHAPE
    assert call(0, 16) == ESHAPE


def test_register_path_workspace_follows_its_split_count():
    """K <= 32: per (user, item split, 32-column part) K fp32 scores and K int32 columns, then one shared threshold per user.
    The split count is the one tr.narrow_splits restates for the tie and cut tests."""
    from replay_b200._lib import lib

    L = lib()
    sms = _sms()
    for K in (1, 10, 11, 16, 17, 32):
        for users in (1, 127, 128, 129, 130, 4096, 32768):
            for items in (1, 127, 128, 129, 5003, 50_000, 200_000, 500_000):
                if K > items:
                    continue
                p = tr.narrow_splits(users, items, sms)
                want = users * p * 2 * K * 8 + users * 4 + 256
                assert L.rp_score_topk_workspace(users, items, 128, K) == want, (K, users, items)
    # the shapes the GPU tests cut at: several splits, the first cut past the first tile
    assert tr.narrow_splits(130, 50_000, sms) >= 4 and tr.narrow_cuts(130, 50_000, sms)[0] >= 256
    assert tr.narrow_splits(4096, 200_000, sms) >= 3 and tr.narrow_cuts(4096, 200_000, sms)[0] >= 1024
