"""float64 restatement of the fused predict head (rp_score_topk: scores -> seen filter -> top-K) and the item-split cuts of
its two kernels, shared by the register-path (K <= 32) and wide (32 < K <= 1024) GPU tests.

The reference is oracle.sasrec.score_topk on the kernel's own bf16 inputs, accumulated in fp64, ordered by (score desc,
scored column asc).  A bias enters as one more feature column (hq . 1 + bias)."""
import torch

INT32_MAX = 2 ** 31 - 1


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def oracle(hq, table, seen, K, bias=None, candidates=None):
    """Returns ((ids, scores) in fp64, hq64, table64): the bias-augmented fp64 operands adjudicate index swaps."""
    from oracle import sasrec as osr

    hq, table = hq.double(), table.double()
    if bias is not None:
        hq = torch.cat([hq, torch.ones(hq.shape[0], 1, dtype=torch.float64)], 1)
        table = torch.cat([table, bias[:table.shape[0], None].double()], 1)
    return osr.score_topk(hq, table, seen, K, candidates=candidates, acc_dtype=torch.float64), hq, table


def check(ids, sc, ref, hq64, tb64, columns=True):
    """Scores within fp32 noise; an index swap only between scores closer than fp32 accumulation noise and never inside an
    exact tie.  ids are item ids, i.e. rows of tb64 (the full, bias-augmented table)."""
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
        # bit-equal kernel scores by ascending column (bit-equal table rows are checked exactly in the tie tests)
        if columns:
            same = sc[:, :-1] == sc[:, 1:]
            assert (ids[:, :-1][same] < ids[:, 1:][same]).all()


# the bias the kernel reads past the scored columns (it is padded to a multiple of 128): large, so that an out-of-catalog
# column that leaked into a result would show up at its head
BIAS_PAD = 1.0e4


def run_case(ops, B, I, d, K, S, seed, bias=False, cands=False):
    """Random bf16 case through ops.seen_prepare + ops.score_topk, checked against the oracle.  Seen ids include negative
    ids, ids >= I, duplicates (user 1) and a user with nothing seen (user 0)."""
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
    ref, hq64, tb64 = oracle(hq, table, seen, K, b, c)
    # the kernel scores the gathered rows; its bias is per scored column, padded to a multiple of 128
    tb_k = table if c is None else table[c]
    b_k = None
    if b is not None:
        b_k = torch.full(((tb_k.shape[0] + 127) // 128 * 128,), BIAS_PAD)
        b_k[:tb_k.shape[0]] = b if c is None else b[c]
    inv = None
    if c is not None:
        inv = torch.full((I,), -1, dtype=torch.int32)
        inv[c] = torch.arange(c.numel(), dtype=torch.int32)
    seen_sorted = ops.seen_prepare(seen.cuda(), I, None if inv is None else inv.cuda()) if seen is not None else None
    ids, sc = ops.score_topk(hq.cuda(), tb_k.contiguous().cuda(), K, seen_sorted, None if c is None else c.cuda(),
                             bias=None if b_k is None else b_k.cuda())
    check(ids, sc, ref, hq64, tb64, columns=c is None)
    return ids, sc


def ordered_table(I, d, descending):
    """hq = (1, 2^-8, 2^-16, 0, ...) and rows = base-256 digits of the column: every score is exact in bf16 x fp32 and
    strictly increasing (or decreasing) with the column."""
    j = torch.arange(I)
    v = (I - j) if descending else (j + 1)
    table = torch.zeros(I, d)
    table[:, 0], table[:, 1], table[:, 2] = (v // 65536).float(), ((v // 256) % 256).float(), (v % 256).float()
    return table.to(torch.bfloat16)


def ordered_hq(B, d):
    hq = torch.zeros(B, d)
    hq[:, 0], hq[:, 1], hq[:, 2] = 1.0, 2.0 ** -8, 2.0 ** -16
    return hq.to(torch.bfloat16)


def narrow_splits(B, I, sms):
    """item splits of the register path (rp_score_topk.cu choose_splits): one CTA per (128 users, item split)"""
    n_tiles, ut = (I + 127) // 128, (B + 127) // 128
    return min(max(1, sms // ut), n_tiles, 64)


def narrow_cuts(B, I, sms):
    """first column of each item split after the first"""
    n_tiles, p = (I + 127) // 128, narrow_splits(B, I, sms)
    return [(n_tiles * s // p) * 128 for s in range(1, p)]


def wide_cuts(B, I, K, sms):
    """item-split boundaries of the wide kernel (rp_score_topk.cu wide_splits): the narrow split count, capped so that one
    user's candidate buffers of C keys hold at most 65 536 keys"""
    C = 128
    while C < 2 * K or C < K + 64:
        C *= 2
    n_tiles = (I + 127) // 128
    p = min(narrow_splits(B, I, sms), 65536 // C)
    return [(n_tiles * s // p) * 128 for s in range(1, p)]


def seen_prepare_reference(seen, item_count, inv_map=None):
    """rp_seen_prepare's contract on the CPU: ids outside [0, item_count) (or, with inv_map, not candidates) become
    INT32_MAX; the rest are item ids (or candidate positions); each row sorted ascending, int32."""
    seen = seen.cpu().long()
    pad = (seen < 0) | (seen >= item_count)
    v = seen.masked_fill(pad, 0)
    if inv_map is not None:
        v = inv_map.cpu().long()[v]
        pad = pad | (v < 0)
    v = v.masked_fill(pad, INT32_MAX)
    return torch.sort(v, dim=1).values.to(torch.int32)
