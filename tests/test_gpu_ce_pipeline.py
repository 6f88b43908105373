"""GPU tests of the column-tile loop of the full-catalog CE head (ce_bwd_kernel in csrc/rp_ce_head.cu): thread 0 refills a
ring of NSTAGE column tiles of TN columns while the fused pass splits the catalog on a 64-column grid, so the edge cases are
the number of column tiles a CTA loops over (against the ring depth), ragged last tiles and splits that end inside a tile,
every hidden size with and without bias, the fused pass behind the two-pass forward, an empty batch, and run-to-run
determinism.  TILE and _pick_splits restate dispatch_ce_bwd and pick_splits; test_ce_tile_table.py checks them against
the source so the cases keep hitting the tile counts they are named for."""
import pytest
import torch

pytestmark = pytest.mark.gpu

GRID = 64                                      # column grid of the fused pass's splits (kTN)
TILE = {64: (128, 8), 128: (128, 4), 256: (64, 4)}   # ce_bwd_kernel's (column tile TN, ring depth NSTAGE) per d (dispatch_ce_bwd)
NSTAGE = {d: ns for d, (_, ns) in TILE.items()}


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from replay_b200 import ops as _ops

    return _ops


def _cdiv(a, b):
    return (a + b - 1) // b


def _pick_splits(n_row_tiles, n_col_tiles, sms, max_splits=8):
    """pick_splits of rp_ce_head.cu: the column split count of the fused pass"""
    best, best_eff = 1, 0.0
    for p in range(1, min(max_splits, n_col_tiles) + 1):
        ctas = n_row_tiles * p
        eff = ctas / (_cdiv(ctas, sms) * sms)
        if eff > best_eff + 0.02:
            best, best_eff = p, eff
    return best


def _fused_tiles(capacity, hint, n_items, d, sms):
    """(split count, set of column-tile counts per CTA) of the fused pass (MODE 2)"""
    hint_tiles = _cdiv(hint, 128) if 0 < hint <= capacity else _cdiv(capacity, 128)
    P = _pick_splits(hint_tiles, _cdiv(n_items, 128), sms)
    n_grid, tn = _cdiv(n_items, GRID), TILE[d][0]
    spans = [min(n_items, n_grid * (s + 1) // P * GRID) - n_grid * s // P * GRID for s in range(P)]
    return P, {_cdiv(c, tn) for c in spans}


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _layout(n_ct, d, split):
    """(capacity, n_valid, n_items, hint) whose CTAs loop over n_ct column tiles, last tiles ragged.
    split "P1": the fused pass with one split (row tiles fill the GPU), "Pn": the fused pass split over several CTAs per row
    tile, "twopass": the two-pass forward and the separate dH pass (MODE 0).  The dE pass (MODE 1) loops over
    ceil(n_valid / TN) token tiles: n_ct of them, except in "Pn" (one row tile of tokens)."""
    sms, tn = _sms(), TILE[d][0]
    if split == "Pn":
        n_valid = min(tn * n_ct - 5, 123)
        for n_items in range(GRID + 1, tn * 16 * (n_ct + 2)):
            if n_items % tn == 0:
                continue
            P, counts = _fused_tiles(128, n_valid, n_items, d, sms)
            if P > 1 and n_ct in counts:
                return 128, n_valid, n_items, n_valid
        raise AssertionError(f"no catalog size splits into CTAs of {n_ct} column tiles on {sms} SMs")
    n_valid, n_items = tn * n_ct - 5, tn * n_ct - 17
    if split == "twopass":
        return _cdiv(n_valid, 128) * 128, n_valid, n_items, n_valid
    capacity = sms * 128   # as many row tiles as SMs: one split is the best balance
    P, counts = _fused_tiles(capacity, capacity, n_items, d, sms)
    assert P == 1 and counts == {n_ct}
    return capacity, n_valid, n_items, capacity


def _case(ops, T, n_valid, I, d, *, fused, bias, hint, scale_h=0.5, scale_e=0.3, seed=0, oracle=True):
    """one forward + backward of the head; returns the device outputs and the fp64 oracle on the same bf16 inputs"""
    g = torch.Generator().manual_seed(seed + 7 * T + I + d)
    hc = (torch.randn(T, d, generator=g) * scale_h).to(torch.bfloat16)
    hc[n_valid:] = 0
    table = (torch.randn(I, d, generator=g) * scale_e).to(torch.bfloat16)
    b = (torch.randn(I, generator=g) * 0.5).float() if bias else None
    labels = torch.randint(0, I, (T,), generator=g, dtype=torch.int64)
    ref = None
    if oracle and n_valid > 0:
        h64, e64 = hc[:n_valid].double().requires_grad_(True), table.double().requires_grad_(True)
        b64 = b.double().requires_grad_(True) if bias else None
        logits = h64 @ e64.T + (b64 if bias else 0.0)
        loss = (torch.logsumexp(logits, -1) - logits.gather(1, labels[:n_valid, None])[:, 0]).mean()
        loss.backward()
        ref = dict(loss=loss.item(), d_hc=h64.grad, d_table=e64.grad, d_bias=b64.grad if bias else None)

    st = ops.CEHeadState(T, I, d, "cuda")
    nv = torch.tensor([n_valid], dtype=torch.int32, device="cuda")
    hc_c, tab_c, lab_c = hc.cuda(), table.cuda(), labels.int().cuda()
    b_c = b.cuda() if bias else None
    d_hc = torch.zeros(T, d, device="cuda", dtype=torch.bfloat16)
    d_tab = torch.full((I + 1, d), 7.0, device="cuda")   # rows < I are overwritten, the pad row stays
    d_b = torch.full((I + 1,), 7.0, device="cuda") if bias else None
    out = ops.ce_head_fwd(st, hc_c, tab_c, lab_c, nv, bias=b_c, d_hc=d_hc if fused else None, n_valid_hint=hint)
    loss = out.clone()
    fused_taken = ops.ce_head_fused_taken(st) if fused else None
    ops.ce_head_bwd(st, hc_c, tab_c, lab_c, nv, d_hc, d_tab, bias=b_c, d_bias=d_b)
    torch.cuda.synchronize()
    got = dict(loss=loss.cpu(), d_hc=d_hc.cpu(), d_table=d_tab.cpu(), d_bias=d_b.cpu() if bias else None,
               fused_taken=fused_taken)
    return got, ref


def _check(got, ref, n_valid, I, bias, loss_rtol):
    assert abs(got["loss"][0].item() - ref["loss"]) < loss_rtol * max(1.0, abs(ref["loss"])), (got["loss"][0].item(), ref["loss"])

    def rel(a, b):
        return ((a.double() - b).norm() / b.norm()).item()

    # the softmax reaches the gradient GEMMs in bf16: norm-relative tolerances
    assert rel(got["d_hc"][:n_valid], ref["d_hc"]) < 1e-2
    assert rel(got["d_table"][:I], ref["d_table"]) < 1e-2
    assert (got["d_table"][I] == 7.0).all()
    assert (got["d_hc"][n_valid:] == 0).all()
    if bias:
        assert rel(got["d_bias"][:I], ref["d_bias"]) < 1e-2
        assert got["d_bias"][I].item() == 7.0


_TILE_CASES = [(d, n) for d in (64, 128, 256) for n in sorted({1, 2, 3, NSTAGE[d] - 1, NSTAGE[d], NSTAGE[d] + 1})]


@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("split", ["P1", "Pn", "twopass"])
@pytest.mark.parametrize("d,n_ct", _TILE_CASES)
def test_ce_head_column_tiles_per_cta(ops, d, n_ct, split, bias):
    """1, 2, 3, NSTAGE - 1, NSTAGE and NSTAGE + 1 column tiles per CTA in every pass of the head, ragged last tiles"""
    T, n_valid, I, hint = _layout(n_ct, d, split)
    got, ref = _case(ops, T, n_valid, I, d, fused=split != "twopass", bias=bias, hint=hint)
    if split != "twopass":
        assert got["fused_taken"], "the logit bound should hold at these input scales"
    _check(got, ref, n_valid, I, bias, 2e-4)


@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("split", ["P1", "Pn"])
@pytest.mark.parametrize("d", [64, 128, 256])
def test_ce_head_fused_pass_behind_two_pass_forward(ops, d, split, bias):
    """logits too large for the fixed reference maximum: the fused kernel runs as the gradient pass with exponent offsets
    -lse from the two-pass forward"""
    T, n_valid, I, hint = _layout(NSTAGE[d] + 1, d, split)
    got, ref = _case(ops, T, n_valid, I, d, fused=True, bias=bias, hint=hint, scale_h=2.0, scale_e=1.0)
    assert not got["fused_taken"], "the logit bound should fail at these input scales"
    _check(got, ref, n_valid, I, bias, 1e-3)


@pytest.mark.parametrize("fused", [False, True])
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("d", [64, 128, 256])
def test_ce_head_without_valid_targets(ops, d, bias, fused):
    """T_v = 0: the dE pass has no token tiles; d_table (and d_bias) come out zero, pad rows untouched"""
    T, I = 256, 1000
    got, _ = _case(ops, T, 0, I, d, fused=fused, bias=bias, hint=0)
    assert (got["d_table"][:I] == 0).all()
    assert (got["d_table"][I] == 7.0).all()
    assert (got["d_hc"] == 0).all()
    assert torch.isfinite(got["loss"]).all()
    if bias:
        assert (got["d_bias"][:I] == 0).all()
        assert got["d_bias"][I].item() == 7.0


@pytest.mark.parametrize("d,T,n_valid,I,hint", [(64, 4096, 4000, 20001, 4000), (128, 4096, 4000, 50000, 4000),
                                                (128, 132 * 128, 3000, 5003, 132 * 128), (256, 2048, 1900, 9999, 1900)])
def test_ce_head_is_deterministic(ops, d, T, n_valid, I, hint):
    """two identical calls: bitwise-equal d_hc and loss (d_table is not compared: the label scatter adds with fp32 atomics)"""
    a, _ = _case(ops, T, n_valid, I, d, fused=True, bias=False, hint=hint, oracle=False)
    b, _ = _case(ops, T, n_valid, I, d, fused=True, bias=False, hint=hint, oracle=False)
    assert torch.equal(a["loss"], b["loss"])
    assert torch.equal(a["d_hc"], b["d_hc"])
