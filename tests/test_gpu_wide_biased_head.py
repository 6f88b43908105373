"""GPU tests of the biased full-catalog CE and BCE heads at d = 512 against float64 on the same bf16 inputs.  This is BERT4Rec's
head at hidden 512, or at any shape that pads to 512 columns such as 300 / 4.  The backward materialises the softmax / sigmoid
G of a token chunk in bf16 with the bias inside the exponent / sigmoid.  d_bias is the fixed-order column sums of every
chunk.

Bounds as in tests/bce_reference.py and tests/ce_reference.py.  G is a bf16 operand (relative 2^-8 with margin) and d_bias
sums the same bf16 G.
Rows past n_valid hold finite garbage, as stale rows do in the engine.  Column n_items of d_table / d_bias is a sentinel that
must stay untouched."""
import pytest
import torch

from bce_reference import reference as bce_reference, worst
from ce_reference import reference as ce_reference

pytestmark = pytest.mark.gpu

D = 512
CAP = 384
SENTINEL = 3.0


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from replay_b200 import ops as _ops

    return _ops


def _inputs(n_valid, I, seed=0):
    g = torch.Generator().manual_seed(seed + 7 * I + n_valid)
    h = torch.randn(CAP, D, generator=g) * 0.05
    h[n_valid:] = torch.randn(CAP - n_valid, D, generator=g) * 0.5 + 0.2   # stale rows: finite, non-zero
    W = torch.randn(I, D, generator=g) * 0.1
    labels = torch.randint(0, I, (CAP,), generator=g, dtype=torch.int32)
    b = torch.zeros((I + 127) // 128 * 128)
    b[:I] = torch.randn(I, generator=g) * 1.0
    b[I:] = 7.0   # padding entries are never read as a live item's bias
    dev = torch.device("cuda")
    return (h.to(dev, torch.bfloat16), W.to(dev, torch.bfloat16), b.to(dev), labels.to(dev),
            torch.tensor([n_valid], dtype=torch.int32, device=dev))


def _run(ops, kind, h, W, b, labels, nv):
    I = W.shape[0]
    st = ops.CEHeadState(CAP, I, D, h.device)
    d_hc = torch.full((CAP, D), SENTINEL, device=h.device, dtype=torch.bfloat16)
    d_W = torch.full((I + 1, D), 9.0, device=h.device)
    d_b = torch.full((I + 1,), 9.0, device=h.device)
    fwd, bwd = (ops.ce_head_fwd, ops.ce_head_bwd) if kind == "ce" else (ops.bce_head_fwd, ops.bce_head_bwd)
    loss = fwd(st, h, W, labels, nv, bias=b, d_hc=d_hc).clone()   # d_hc as the engine passes it (no fused pass at 512)
    bwd(st, h, W, labels, nv, d_hc, d_W, bias=b, d_bias=d_b)
    torch.cuda.synchronize()
    return loss, d_hc, d_W, d_b


@pytest.mark.parametrize("chunks", ["one", "several"])
@pytest.mark.parametrize("n_valid", [0, 1, 127, 128, 129, CAP])
@pytest.mark.parametrize("n_items", [1, 129, 30000])
@pytest.mark.parametrize("kind", ["ce", "bce"])
def test_biased_wide_head_matches_fp64(ops, kind, n_items, n_valid, chunks, monkeypatch):
    """Loss, d_hc, d_table and d_bias; one G chunk for the whole capacity, or 128-row chunks (three here, the later ones
    past n_valid for small n_valid).  30 000 items leave a ragged last column tile (30 000 = 234 x 128 + 48)."""
    if chunks == "several":
        monkeypatch.setenv("RP_CE_WIDE_G_BYTES", "1")   # the smallest budget: 128-row chunks
    h, W, b, labels, nv = _inputs(n_valid, n_items)
    loss, d_hc, d_W, d_b = _run(ops, kind, h, W, b, labels, nv)
    ref = (ce_reference if kind == "ce" else bce_reference)(h, W, b[:n_items], labels, n_valid)
    assert abs(float(loss[0]) - float(ref["loss"])) <= float(ref["bound_loss"]), (float(loss[0]), float(ref["loss"]))
    assert worst(d_hc[:n_valid], ref["d_h"], ref["bound_h"]) <= 1.0
    assert (d_hc[n_valid:] == SENTINEL).all(), "d_hc rows past n_valid were written"
    assert worst(d_W[:n_items], ref["d_W"], ref["bound_W"]) <= 1.0
    assert worst(d_b[:n_items], ref["d_b"], ref["bound_b"]) <= 1.0
    assert (d_W[n_items] == 9.0).all() and float(d_b[n_items]) == 9.0, "column n_items was written"
    if n_valid == 0:
        assert not d_b[:n_items].any() and not d_W[:n_items].any()
    # d_bias: fixed-order column sums and a one-hot part of equal terms -> bitwise identical on a rerun
    _, d_hc2, _, d_b2 = _run(ops, kind, h, W, b, labels, nv)
    assert torch.equal(d_b2, d_b) and torch.equal(d_hc2, d_hc)


@pytest.mark.parametrize("kind", ["ce", "bce"])
def test_bias_moves_the_wide_head(ops, kind):
    """The bias enters the exponent / sigmoid of the G GEMM: with a large bias on one item, that item's d_bias and d_table row
    follow the float64 reference, and differ from the head run without the bias."""
    h, W, b, labels, nv = _inputs(200, 5000)
    b[17] = 6.0
    loss, _, d_W, d_b = _run(ops, kind, h, W, b, labels, nv)
    ref = (ce_reference if kind == "ce" else bce_reference)(h, W, b[:5000], labels, 200)
    assert worst(d_b[:5000], ref["d_b"], ref["bound_b"]) <= 1.0
    assert worst(d_W[:5000], ref["d_W"], ref["bound_W"]) <= 1.0
    st = ops.CEHeadState(CAP, 5000, D, h.device)
    d_hc0 = torch.zeros(CAP, D, device=h.device, dtype=torch.bfloat16)
    d_W0 = torch.zeros(5000, D, device=h.device)
    fwd, bwd = (ops.ce_head_fwd, ops.ce_head_bwd) if kind == "ce" else (ops.bce_head_fwd, ops.bce_head_bwd)
    fwd(st, h, W, labels, nv)
    bwd(st, h, W, labels, nv, d_hc0, d_W0)
    torch.cuda.synchronize()
    assert float((d_W0[17] - d_W[17]).abs().max()) > 10 * float(ref["bound_W"][17].max())
