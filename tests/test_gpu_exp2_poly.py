"""ex2_poly, the polynomial exp2 that takes a fixed share of the CE passes' exponentials off the special-function unit, tested
on its own through rp_selftest_exp2 against fp64 exp2 and against ex2.approx.ftz on the same arguments."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from replay_b200 import ops as _ops

    return _ops


def _arguments():
    f32 = np.float32
    dense = np.linspace(-130.0, 130.0, 4_000_001, dtype=np.float64).astype(f32)
    # every fp32 within a few ulps of the flush edge (-126), of 0, of +127 and of the range reduction's rounding edges
    # (j +- 1/2, where round(x) changes), over the whole range
    edges = [-126.0, -127.0, 0.0, 127.0] + [j + 0.5 for j in range(-128, 128)]
    near = []
    for e in edges:
        c = f32(e)
        lo, hi = c, c
        near.append(c)
        for _ in range(4):
            lo, hi = np.nextafter(lo, f32(-np.inf)), np.nextafter(hi, f32(np.inf))
            near += [lo, hi]
    special = np.array([-np.inf, -1e30, -1000.0, -200.0, -127.5, -126.5, -1e-30, 1e-30, 1e-3, -1e-3], dtype=f32)
    rnd = np.random.default_rng(0).uniform(-127.0, 127.0, 1_000_000).astype(f32)
    return np.concatenate([dense, np.array(near, dtype=f32), special, rnd])


def test_ex2_poly_matches_exp2_and_the_flush_of_ex2(ops):
    x = _arguments()
    y_poly, y_mufu = ops.selftest_exp2(torch.from_numpy(x).cuda())
    y_poly, y_mufu = y_poly.cpu().numpy(), y_mufu.cpu().numpy()
    # the domain is x <= 127 (the fused pass's arguments stay near 100 or below); the sweep runs on to 130 all the same
    dom = x <= 127
    x, y_poly, y_mufu = x[dom], y_poly[dom], y_mufu[dom]
    assert not np.isnan(y_poly).any() and not np.isinf(y_poly).any()
    assert (np.signbit(y_poly) == 0).all()                                     # +0, never -0
    # exactly +0 wherever ex2.approx.ftz flushes, and for every x < -126 (-inf included)
    zero = y_mufu == 0
    assert zero.any() and (y_poly[zero] == 0).all(), x[zero & (y_poly != 0)][:8]
    assert (y_poly[x < -126] == 0).all(), x[(x < -126) & (y_poly != 0)][:8]
    live = x >= -126
    assert (y_poly[live] > 0).all()
    ref = np.exp2(x[live].astype(np.float64))
    rel = np.abs(y_poly[live].astype(np.float64) / ref - 1)
    assert rel.max() <= 1e-5, (rel.max(), x[live][rel.argmax()])
    # smallest normal and largest power of two are exact (the polynomial's constant term is 1)
    y, _ = ops.selftest_exp2(torch.tensor([-126.0, 0.0, 127.0], device="cuda"))
    assert y.cpu().tolist() == [2.0 ** -126, 1.0, 2.0 ** 127]
