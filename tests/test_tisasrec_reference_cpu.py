"""tests/tisasrec_reference.py without a GPU: its closed form against autograd through oracle/tisasrec.time_attention, its
interval function against oracle.time_matrix at the timestamp edges of every dtype, its dropout stream against
tests/dropout_stream.py, and its bounds' power to tell a subtly wrong kernel from a right one on the GPU tests' own input
sizes: each mistake below breaks a bound by at least ten times the GPU test's tolerance."""
import numpy as np
import pytest
import torch

import tisasrec_reference as tr
from dropout_stream import keep_draws
from oracle.tisasrec import time_attention, time_matrix
from test_gpu_tisasrec_fp64 import CTA_CASE, TOL_A, TOL_TIME

DISCRIMINATES = 10.0


@pytest.mark.parametrize("p", [0.0, 0.2])
def test_closed_form_matches_autograd_through_the_oracle(p):
    B, L, H, span = 5, 11, 2, 6
    d = H * tr.SLOT
    P = tr.make_problem(B, L, 64, H, span, p, times="edges", seed=4, seed_eff=0xABCDEF12345)
    g = torch.Generator().manual_seed(9)
    kv = (torch.randn(B * L, 2 * d, generator=g)).to(torch.bfloat16)
    ref = tr.attention_stage(P.q[:, :d], kv, P.q_in[:, :d], P.d_o[:, :d], P.times, P.pad, P.tk[:, :d], P.tv[:, :d], H, 64,
                             span, p, P.seed_eff, P.att_off)
    keep = {}
    if p > 0:
        rows = (torch.arange(B * L)[:, None] * L + torch.arange(L)[None, :])
        keep["tk"] = tr.keep(P.seed_eff, tr.SITE_TK, p, rows, torch.arange(d)).double().view(B, L, L, d) * P.ks
        keep["tv"] = tr.keep(P.seed_eff, tr.SITE_TV, p, rows, torch.arange(d)).double().view(B, L, L, d) * P.ks
        arows = torch.arange(B * H)[:, None] * P.Lp + torch.arange(L)[None, :]
        keep["att"] = tr.keep(P.seed_eff, P.att_off, p, arows, torch.arange(L)).double().view(B, H, L, L) * P.ks
    X = {"q": P.q[:, :d], "k": kv[:, :d], "v": kv[:, d:], "tk": P.tk[:, :d], "tv": P.tv[:, :d]}
    X = {k: v.double().requires_grad_(True) for k, v in X.items()}
    o = time_attention(X["q"].view(B, L, d), X["k"].view(B, L, d), X["v"].view(B, L, d), time_matrix(P.times, span),
                       X["tk"], X["tv"], P.pad, H, keep.get("att"), keep.get("tk"), keep.get("tv"))
    o = torch.where(P.pad[..., None], o, torch.zeros_like(o))
    (o * P.d_o[:, :d].double().view(B, L, d)).sum().backward()
    want = {"h": P.q_in[:, :d].double() + o.detach().reshape(B * L, d), "dQ": X["q"].grad, "dK": X["k"].grad,
            "dV": X["v"].grad, "d_time_k": X["tk"].grad, "d_time_v": X["tv"].grad}
    for k, w in want.items():
        assert torch.allclose(ref[k], w, rtol=1e-10, atol=1e-12), (k, float((ref[k] - w).abs().max()))


EDGE_VALUES = {
    torch.int64: [0, 1, 2, 7, 8, 9, -1, -8, -9, 2**62, 2**62 + 7, 2**62 + 8, 2**62 + 2**32, 2**62 + 2**32 + 7, -(2**40)],
    torch.float32: [1.7e9, 1.7e9 + 64, 1.7e9 + 128, 1.7e9 + 192, 1.7e9 + 1024, 0.0, 2.999, 3.0, 3.5, 7.999, 8.0, 9.5, -2.999,
                    -3.5],
    torch.float64: [1.7e9, 1.7e9 + 0.37, 1.7e9 + 0.74, 1.7e9 + 7.999, 1.7e9 + 8.0, 1.7e9 + 8.5, 0.0, 2.999, 3.0, 3.5, -0.5,
                    -7.25],
}


@pytest.mark.parametrize("dtype", list(EDGE_VALUES), ids=str)
@pytest.mark.parametrize("span", [1, 2, 8, 320])
def test_intervals_match_the_oracle(dtype, span):
    t = torch.tensor(EDGE_VALUES[dtype], dtype=dtype)
    assert torch.equal(tr.intervals(t, span), time_matrix(t[None], span)[0])
    for kind in ("edges", "decreasing", "unsorted", "big_int", "epoch_f32", "frac", "epoch_f64"):
        ts = tr.make_times(kind, 3, 40, span, torch.Generator().manual_seed(1), dtype)
        for b in range(3):
            assert torch.equal(tr.intervals(ts[b], span), time_matrix(ts[b:b + 1], span)[0]), kind


def test_edge_timestamps_hit_the_edges():
    g = torch.Generator().manual_seed(0)
    r = tr.intervals(tr.make_times("edges", 1, 65, 63, g)[0], 63)
    assert {62, 63} <= set(r.unique().tolist())
    t = tr.make_times("epoch_f32", 1, 65, 256, g)[0]
    assert t.dtype == torch.float32 and bool(((t[1:] - t[:-1]) % 128 == 0).all())
    t = tr.make_times("big_int", 1, 65, 63, g)[0]
    assert int(t.min()) >= 2**62 and int((t[1:] - t[:-1]).max()) >= 2**32


def test_dropout_stream_matches_the_numpy_port():
    rows = torch.tensor([0, 1, 77, 2**32 - 1, 2**32, 2**32 + 5, 3 * 2**40 + 17])
    for seed, off, p in ((0x5EED, tr.SITE_TK, 0.2), (0x5EED + 977, tr.SITE_ATT, 0.2), (2**63 + 3, tr.SITE_TV, 0.5)):
        want = keep_draws(seed, off, p, rows.numpy().astype(np.uint64), 256)
        assert torch.equal(tr.keep(seed, off, p, rows, torch.arange(256)), want)


# ------------------------------------------------------------------------------------------------ the bounds discriminate
def _fwd_problem(p=0.2):
    """the GPU forward sweep's L 65 / 2 heads / span 63 input"""
    P = tr.make_problem(5, 65, 64, 2, 63, p, seed_eff=0x5EED + 977, ld_extra=8)
    return P


def _fwd_ratio(P_ok, broken):
    ref = tr.forward(P_ok)
    return tr.ratio(broken["A"], ref["A"], ref["A_b"])


def test_bound_catches_one_pair_in_a_neighbouring_bucket():
    P = _fwd_problem()
    ref = tr.forward(P)
    for b, i, j, step in ((0, 40, 3, 1), (0, 40, 3, -1), (1, 64, 30, 1), (4, 10, 9, -1)):
        r = ref["r"].clone()
        r[b, i, j] = r[b, i, j] + step if 0 <= int(r[b, i, j]) + step <= P.span else r[b, i, j] - step
        bad = tr.forward(P, r=r)
        assert tr.ratio(bad["A"], ref["A"], ref["A_b"]) >= DISCRIMINATES * TOL_A, (b, i, j, step)


def test_bound_catches_a_missing_dropout_scale_on_the_time_terms():
    P = _fwd_problem()
    Q = tr.make_problem(5, 65, 64, 2, 63, 0.2, seed_eff=0x5EED + 977, ld_extra=8)
    Q.time_ks = 1.0
    assert _fwd_ratio(P, tr.forward(Q)) >= DISCRIMINATES * TOL_A


def test_bound_catches_swapped_time_dropout_sites():
    P = _fwd_problem()
    Q = tr.make_problem(5, 65, 64, 2, 63, 0.2, seed_eff=0x5EED + 977, ld_extra=8)
    Q.tk_off, Q.tv_off = P.tv_off, P.tk_off
    assert _fwd_ratio(P, tr.forward(Q)) >= DISCRIMINATES * TOL_A


@pytest.mark.parametrize("H", [1, 4])
def test_bound_catches_a_lost_second_sequence_of_a_backward_cta(H):
    """B = G + 1 at L 9: CTA 0 takes sequences 0 and G.  A kernel that forgets sequence G's pairs in the table gradients
    (say, it processes only b = blockIdx.x) breaks their bound."""
    G = tr.BWD_CTAS // H
    B = G + 1
    P = tr.make_problem(B, 9, CTA_CASE["head_dim"], H, CTA_CASE["span"], CTA_CASE["p"], CTA_CASE["times"], seed=B,
                        seed_eff=0x5EED + 977, ld_extra=8)
    A = tr.forward(P)["A"].to(torch.bfloat16)
    ref = tr.backward(P, A=A)
    lost = tr.make_problem(B, 9, CTA_CASE["head_dim"], H, CTA_CASE["span"], CTA_CASE["p"], CTA_CASE["times"], seed=B,
                           seed_eff=0x5EED + 977, ld_extra=8)
    lost.pad = lost.pad.clone()
    lost.pad[G] = False
    bad = tr.backward(lost, A=A)
    zero = torch.zeros_like(ref["d_time_k"])
    worst = max(tr.ratio(bad[k], ref[k], tr.table_bound(ref[k + "_b"], zero, ref[k])) for k in ("d_time_k", "d_time_v"))
    assert worst >= DISCRIMINATES * TOL_TIME, worst
