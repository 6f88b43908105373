"""GPU tests of the CE head's dE pass (ce_bwd_kernel MODE 1 in csrc/rp_ce_head.cu) against an fp64 reference.  The pass walks
the valid tokens in column tiles of TN and reads each tile's exponent offsets (cvec, -inf past T_v up to the next multiple of
128) from a shared-memory slot that the tile ring fills together with the tile, so the cases are the token counts around the
tile and buffer edges (T_v below one tile, not a multiple of 128, up to the end of a capacity that is not one either), fewer
and more token tiles than ring stages, offsets written by the two-pass forward (-lse, the bound failed) and by the un-fused
forward, and bitwise repeatability.  d_table is held to the per-element bounds of tests/ce_reference.py."""
import pytest
import torch

import ce_reference as cr
from ce_reference import TILE

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from replay_b200 import ops as _ops

    return _ops


def _run(ops, T, n_valid, I, d, *, fused=True, scale_h=0.5, scale_e=0.3, seed=0, distinct_labels=False):
    """forward + backward of the head; d_table [I, d] from the device and the fp64 reference on the same bf16 inputs"""
    g = torch.Generator().manual_seed(seed + 31 * T + 7 * n_valid + I + d)
    hc = (torch.randn(T, d, generator=g) * scale_h).to(torch.bfloat16)
    hc[n_valid:] = 0
    table = (torch.randn(I, d, generator=g) * scale_e).to(torch.bfloat16)
    if distinct_labels:   # every item row takes at most one one-hot correction: the fp32 atomics add in a fixed order
        labels = torch.randperm(I, generator=g)[:T].to(torch.int64)
    else:
        labels = torch.randint(0, I, (T,), generator=g, dtype=torch.int64)
    ref = cr.reference(hc, table, None, labels, n_valid)
    st = ops.CEHeadState(T, I, d, "cuda")
    nv = torch.tensor([n_valid], dtype=torch.int32, device="cuda")
    hc_c, tab_c, lab_c = hc.cuda(), table.cuda(), labels.int().cuda()
    d_hc = torch.zeros(T, d, device="cuda", dtype=torch.bfloat16)
    d_tab = torch.full((I, d), 7.0, device="cuda")
    ops.ce_head_fwd(st, hc_c, tab_c, lab_c, nv, d_hc=d_hc if fused else None, n_valid_hint=n_valid)
    taken = ops.ce_head_fused_taken(st) if fused else None
    ops.ce_head_bwd(st, hc_c, tab_c, lab_c, nv, d_hc, d_tab)
    torch.cuda.synchronize()
    return d_tab.cpu(), ref, taken


def _check(got, ref):
    assert cr.worst(got, ref["d_W"], ref["bound_W"]) <= 1.0


def _tokens(d, n_tiles, tail):
    """a token count that the dE pass covers with n_tiles column tiles, the last one holding `tail` tokens"""
    return (n_tiles - 1) * TILE[d][0] + tail


def _cap(n_valid):
    return (n_valid + 127) // 128 * 128 + 128


_D = [64, 128, 256]


@pytest.mark.parametrize("d", _D)
@pytest.mark.parametrize("n_valid", [1, 37, 127])
def test_de_pass_fewer_tokens_than_one_tile(ops, d, n_valid):
    """T_v < 128: one (at d = 256, at most two) token tiles, the slot mostly -inf"""
    got, ref, taken = _run(ops, 128, n_valid, 1031, d)
    assert taken
    _check(got, ref)


@pytest.mark.parametrize("d", _D)
@pytest.mark.parametrize("where", ["fewer", "equal", "more"])
def test_de_pass_token_tiles_against_ring_depth(ops, d, where):
    """fewer token tiles than ring stages, exactly as many, and more (the slots are refilled), last tile ragged"""
    tn, ns = TILE[d]
    n_tiles = {"fewer": max(1, ns - 2), "equal": ns, "more": 2 * ns + 1}[where]
    n_valid = _tokens(d, n_tiles, tn - 19)
    got, ref, taken = _run(ops, _cap(n_valid), n_valid, 2003, d)
    assert taken
    _check(got, ref)


@pytest.mark.parametrize("d", _D)
def test_de_pass_up_to_a_capacity_off_the_tile_grid(ops, d):
    """capacity 300 (cvec holds 384 entries) and T_v = 298: the last tile's offsets run past the capacity into the -inf pad"""
    got, ref, taken = _run(ops, 300, 298, 1500, d)
    assert taken
    _check(got, ref)


@pytest.mark.parametrize("d", _D)
def test_de_pass_offsets_from_two_pass_forward(ops, d):
    """logits too large for the fused pass's bound: the offsets come from the two-pass forward (-lse per token)"""
    tn, ns = TILE[d]
    n_valid = _tokens(d, ns + 1, 77)
    got, ref, taken = _run(ops, _cap(n_valid), n_valid, 3001, d, scale_h=2.0, scale_e=1.0)
    assert not taken, "the logit bound should fail at these input scales"
    _check(got, ref)


@pytest.mark.parametrize("d", _D)
def test_de_pass_offsets_from_unfused_forward(ops, d):
    """forward without d_hc: the two-pass forward writes the offsets, the backward runs the token pass and then dE"""
    tn, ns = TILE[d]
    n_valid = _tokens(d, ns + 2, 5)
    got, ref, _ = _run(ops, _cap(n_valid), n_valid, 3001, d, fused=False)
    _check(got, ref)


@pytest.mark.parametrize("d", _D)
def test_de_pass_is_bitwise_repeatable(ops, d):
    """two identical calls give the same d_table bit for bit (distinct labels keep the one-hot atomics order-free)"""
    tn, ns = TILE[d]
    n_valid = _tokens(d, 2 * ns + 3, 50)
    a, ref, _ = _run(ops, _cap(n_valid), n_valid, 4099, d, distinct_labels=True)
    b, _, _ = _run(ops, _cap(n_valid), n_valid, 4099, d, distinct_labels=True)
    assert torch.equal(a, b)
    _check(a, ref)
