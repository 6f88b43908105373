"""TiSASRec's time-interval attention (rp_ti_attn_fwd / rp_ti_attn_bwd with the rp_gemm products around them, as
TiSasRecEngine runs them) against a float64 restatement on the same bf16 inputs, with the kernels' dropout masks replayed
on the host: the block's attention output h = q_in + o, and dQ, dK', dV' and both time tables' gradients of <h, dO>.

Sweeps sequence length across the 32-key lane and 64-key tile edges, head width 50 (padded slot) and 64, 1 / 2 / 4 heads,
time_span 1 / 8 / 256 / the kernels' largest, all-equal timestamps, gaps beyond the span and left padding.  Errors are
measured per 64-row block against the block's norm (tests/fp64_checks.py) and element-wise against the output's scale."""
import pytest
import torch

from dropout_stream import drop_keep, keep_draws
from fp64_checks import block_err
from oracle.tisasrec import time_attention, time_matrix
from replay_b200._lib import TI_MAX_SPAN
from replay_b200.engine_tisasrec import _SITE_TIME_K, _SITE_TIME_V, TiConfig, TiSasRecEngine

P_DROP = 0.2


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda")


def _times(kind, B, L, span, g):
    if kind == "equal":
        return torch.full((B, L), 12345, dtype=torch.int64)
    if kind == "gaps":   # most intervals beyond the span, some inside, some zero
        steps = torch.randint(0, 3, (B, L), generator=g) * (span + 7) + torch.randint(0, 2, (B, L), generator=g)
        return steps.cumsum(1)
    return torch.randint(0, 2 * span + 2, (B, L), generator=g).sort(1).values


def _run(dev, L, hd, H, span, drop, times_kind="mixed", seed=0):
    """(engine, inputs, reference outputs) of one forward + backward of block 0's attention."""
    B = 3
    g = torch.Generator().manual_seed(1000 * L + 10 * H + hd + span)
    cfg = TiConfig(n_items=16, d=hd * H, n_heads=H, n_blocks=1, max_len=L, dropout=drop, time_span=span)
    eng = TiSasRecEngine(cfg, B, L, dev, seed=seed)
    d, T, feat = cfg.dp, B * L, cfg.feat_index()
    pad = torch.ones(B, L, dtype=torch.bool)
    pad[1, : L // 3] = False        # left padding
    pad[2, : L - 1] = False         # one live row
    times = _times(times_kind, B, L, span, g)
    times[1, : L // 3] = 0          # padded positions carry timestamp 0
    eng.set_batch(torch.zeros(B, L, dtype=torch.int64, device=dev), pad.to(dev))
    eng.set_times(times.to(dev))
    eng._prepare(False)

    def rnd(*shape, s=1.0):
        return (torch.randn(*shape, generator=g) * s).to(torch.bfloat16)

    q, k, v, q_in, dO = (rnd(B, L, hd * H) for _ in range(5))
    dO[~pad] = 0                    # the block output of a padded row is zeroed: no gradient reaches it
    tk, tv = rnd(span + 1, hd * H, s=0.5), rnd(span + 1, hd * H, s=0.5)
    a = eng.act[0]
    for t, val in ((a["Q"], q), (a["q_in"], q_in)):
        t.zero_()
        t[:, feat] = val.reshape(T, -1).to(dev)
    a["KV"].zero_()
    a["KV"][:, feat] = k.reshape(T, -1).to(dev)
    a["KV"][:, d + feat] = v.reshape(T, -1).to(dev)
    eng.import_named("time_k", tk.float())
    eng.import_named("time_v", tv.float())
    eng.refresh_shadow()
    eng._ti_attention_forward(0, True, drop)
    eng.s["dh"].zero_()
    eng.s["dh"][:, feat] = dO.reshape(T, -1).to(dev)
    eng.grads["time_k"].zero_()
    eng.grads["time_v"].zero_()
    eng._ti_attention_backward(0, drop)
    torch.cuda.synchronize()

    keep = {}
    if drop > 0:
        seed_eff = eng.seed + int(eng.rng_counter.item())
        ks = 1.0 / (1.0 - float(torch.tensor(drop, dtype=torch.float32)))
        keep["att"] = drop_keep(seed_eff, eng._site(0, 0) << 40, drop, B, H, L, eng.Lp)
        rows = torch.arange(B * L * L).numpy()
        for name, site in (("tk", _SITE_TIME_K), ("tv", _SITE_TIME_V)):
            keep[name] = keep_draws(seed_eff, site << 40, drop, rows, d)[:, feat].double().view(B, L, L, -1) * ks
    X = {n: t.double().requires_grad_(True) for n, t in (("q", q), ("k", k), ("v", v), ("tk", tk), ("tv", tv))}
    o = time_attention(X["q"], X["k"], X["v"], time_matrix(times, span), X["tk"], X["tv"], pad, H, keep.get("att"),
                       keep.get("tk"), keep.get("tv"))
    o = torch.where(pad[..., None], o, torch.zeros_like(o))   # the kernels skip dead query rows
    (o * dO.double()).sum().backward()
    ref = {"h": q_in.double() + o.detach(), "dQ": X["q"].grad, "dK": X["k"].grad, "dV": X["v"].grad, "dTK": X["tk"].grad,
           "dTV": X["tv"].grad}
    got = {"h": a["h"][:, feat].cpu().view(B, L, -1), "dQ": eng.s["dQ"][:, feat].cpu().view(B, L, -1),
           "dK": eng.s["dKV"][:, feat].cpu().view(B, L, -1), "dV": eng.s["dKV"][:, d + feat].cpu().view(B, L, -1),
           "dTK": eng.export_named("time_k", eng.grads).cpu(), "dTV": eng.export_named("time_v", eng.grads).cpu()}
    return got, ref, pad


def _check(got, ref, pad, tol=2e-2):
    for name in ("h", "dQ", "dK", "dV"):
        g, r = got[name].double(), ref[name]
        m = pad[..., None] if name in ("h", "dQ") else torch.ones_like(pad[..., None])
        for b in range(r.shape[0]):
            err = block_err(g[b] * m[b], r[b] * m[b])
            assert err < tol, (name, b, err)
        scale = float(r.abs().max()) + 1e-6
        assert float((g - r).abs().max()) <= 2e-2 * scale + 1e-3, name
    for name in ("dTK", "dTV"):
        g, r = got[name].double(), ref[name]
        scale = float(r.abs().max()) + 1e-6
        assert float((g - r).abs().max()) <= 1e-2 * scale, (name, float((g - r).abs().max()), scale)
        if float(r.norm()) > 0:   # L 1: a single key, no softmax gradient
            assert torch.nn.functional.cosine_similarity(g.flatten(), r.flatten(), dim=0) > 0.9999, name


@pytest.mark.gpu
@pytest.mark.parametrize("L", [1, 5, 63, 64, 65, 128, 200, 256])
@pytest.mark.parametrize("drop", [0.0, P_DROP])
def test_lengths(cuda, L, drop):
    _check(*_run(cuda, L, 64, 2, 8, drop))


@pytest.mark.gpu
@pytest.mark.parametrize("hd,H", [(50, 1), (64, 1), (50, 2), (64, 2), (32, 4), (64, 4)])
@pytest.mark.parametrize("drop", [0.0, P_DROP])
def test_heads(cuda, hd, H, drop):
    _check(*_run(cuda, 77, hd, H, 16, drop))


@pytest.mark.gpu
@pytest.mark.parametrize("span", [1, 8, 256, TI_MAX_SPAN])
@pytest.mark.parametrize("times_kind", ["mixed", "equal", "gaps"])
@pytest.mark.parametrize("drop", [0.0, P_DROP])
def test_spans_and_timestamps(cuda, span, times_kind, drop):
    _check(*_run(cuda, 96, 50, 1, span, drop, times_kind))


@pytest.mark.gpu
def test_dead_rows_and_rerun(cuda):
    """A padded query row leaves h = q_in and no dQ; a rerun gives the same outputs (the time-table gradients to fp32
    rounding: their shared-memory sums are not ordered)."""
    got, ref, pad = _run(cuda, 64, 64, 2, 8, P_DROP)
    again, _, _ = _run(cuda, 64, 64, 2, 8, P_DROP)
    assert torch.equal(got["dQ"][~pad], torch.zeros_like(got["dQ"][~pad]))
    for k in ("h", "dQ", "dK", "dV"):
        assert torch.equal(got[k], again[k]), k
    for k in ("dTK", "dTV"):
        assert torch.allclose(got[k], again[k], rtol=1e-5, atol=1e-6 * float(got[k].abs().max())), k
