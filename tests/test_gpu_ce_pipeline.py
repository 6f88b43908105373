"""GPU tests of the column-tile loop of the full-catalog CE head (ce_bwd_kernel in csrc/rp_ce_head.cu): thread 0 refills a
ring of NSTAGE column tiles of TN columns while the fused pass splits the catalog on a 64-column grid, so the edge cases are
the number of column tiles a CTA loops over (against the ring depth), ragged last tiles and splits that end inside a tile,
every hidden size with and without bias, the fused pass behind the two-pass forward, an empty batch, and run-to-run
determinism.  Shapes come from the dispatch restatement in tests/ce_reference.py (test_ce_tile_table.py checks it against
the source), so the cases keep hitting the tile counts they are named for; results are held to that module's per-element
bounds."""
import pytest
import torch

import ce_reference as cr
from ce_reference import NSTAGE

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from replay_b200 import ops as _ops

    return _ops


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _layout(n_ct, d, split):
    return cr.layout(n_ct, d, split, _sms())


def _case(ops, T, n_valid, I, d, *, fused, bias, hint, scale_h=0.5, scale_e=0.3, seed=0, oracle=True):
    """one forward + backward of the head; returns the device outputs and the fp64 oracle on the same bf16 inputs"""
    g = torch.Generator().manual_seed(seed + 7 * T + I + d)
    hc = (torch.randn(T, d, generator=g) * scale_h).to(torch.bfloat16)
    hc[n_valid:] = 0
    table = (torch.randn(I, d, generator=g) * scale_e).to(torch.bfloat16)
    b = (torch.randn(I, generator=g) * 0.5).float() if bias else None
    labels = torch.randint(0, I, (T,), generator=g, dtype=torch.int64)
    ref = cr.reference(hc, table, b, labels, n_valid) if oracle else None
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


def _check(got, ref, n_valid, I, bias):
    loss = got["loss"][0].item()
    assert abs(loss - float(ref["loss"])) <= float(ref["bound_loss"]), (loss, float(ref["loss"]))
    assert cr.worst(got["d_hc"][:n_valid], ref["d_h"], ref["bound_h"]) <= 1.0
    assert cr.worst(got["d_table"][:I], ref["d_W"], ref["bound_W"]) <= 1.0
    assert (got["d_table"][I] == 7.0).all()
    assert (got["d_hc"][n_valid:] == 0).all()
    if bias:
        assert cr.worst(got["d_bias"][:I], ref["d_b"], ref["bound_b"]) <= 1.0
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
    _check(got, ref, n_valid, I, bias)


@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("split", ["P1", "Pn"])
@pytest.mark.parametrize("d", [64, 128, 256])
def test_ce_head_fused_pass_behind_two_pass_forward(ops, d, split, bias):
    """logits too large for the fixed reference maximum: the fused kernel runs as the gradient pass with exponent offsets
    -lse from the two-pass forward"""
    T, n_valid, I, hint = _layout(NSTAGE[d] + 1, d, split)
    got, ref = _case(ops, T, n_valid, I, d, fused=True, bias=bias, hint=hint, scale_h=2.0, scale_e=1.0)
    assert not got["fused_taken"], "the logit bound should fail at these input scales"
    _check(got, ref, n_valid, I, bias)


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
