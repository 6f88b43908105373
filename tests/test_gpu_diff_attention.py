"""The DiffTransformer kernels against fp64 references: rp_diff_attn_fwd (outputs and saved statistics, pad rows
included), the attention backward through rp_diff_attn_softmax_bwd and the batched GEMMs (dQ, dK, dV, d rms_scale,
d lambda_*), rp_rmsnorm_fwd / _bwd at both group widths and the SwiGLU gate; two runs are bitwise identical."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda")


def _engine(cuda, hd, H, L, B, seed):
    from replay_b200.engine_diff import DiffConfig, DiffEngine

    cfg = DiffConfig(n_items=50, d=hd * H, n_heads=H, n_blocks=1, max_len=L)
    eng = DiffEngine(cfg, B, L, cuda, seed=seed)
    return eng


def _pad_mask(B, L, kind, g):
    if kind == "full":
        return torch.ones(B, L, dtype=torch.bool)
    if kind == "one":
        pm = torch.zeros(B, L, dtype=torch.bool)
        pm[:, -1] = True
        return pm
    lens = torch.randint(1, L + 1, (B,), generator=g)
    return torch.arange(L).unsqueeze(0) >= (L - lens).unsqueeze(1)


def _setup(eng, lam_target, pm, g):
    """random Q / K / V (zero in the padded slot columns), lambda_* drawn so that lambda = lam_target, random rms_scale"""
    cfg, dev = eng.cfg, eng.dev
    H, hd, vs, B, L = cfg.n_heads, cfg.head_dim, cfg.v_slot, eng.B, eng.L
    T = B * L
    q = torch.randn(T, H, 2, hd, generator=g)
    k = torch.randn(T, H, 2, hd, generator=g)
    v = torch.randn(T, H, 2 * hd, generator=g)
    qk_p = torch.zeros(T, H, 2, 64)
    QKV = torch.zeros(T, cfg.n_qkv)
    qk_p[..., :hd] = q
    QKV[:, : H * 128] = qk_p.reshape(T, -1)
    qk_p[..., :hd] = k
    QKV[:, H * 128: H * 256] = qk_p.reshape(T, -1)
    v_p = torch.zeros(T, H, vs)
    v_p[..., : 2 * hd] = v
    QKV[:, H * 256:] = v_p.reshape(T, -1)
    eng.act[0]["QKV"].copy_(QKV.to(torch.bfloat16))
    eng.in_pad[:T].copy_(pm.reshape(-1))
    from replay_b200.engine_diff import lambda_init

    li = lambda_init(0)
    # lambda = exp(a) - exp(b) + li with lq1 . lk1 = a, lq2 . lk2 = b chosen per head
    lams = torch.tensor(lam_target, dtype=torch.float64).expand(H).clone() + 0.05 * torch.arange(H)
    lq1 = torch.randn(H, hd, generator=g) * 0.3
    lk1 = lq1 / (lq1 * lq1).sum(-1, keepdim=True)   # lq1 . lk1 = 1
    a = (lq1 * lk1).sum(-1).double()
    b = torch.log(torch.exp(a) - (lams - li))
    lq2 = torch.randn(H, hd, generator=g) * 0.3
    lk2 = lq2 * (b / (lq2.double() ** 2).sum(-1)).float().unsqueeze(-1)
    for nm, t in (("q1", lq1), ("k1", lk1), ("q2", lq2), ("k2", lk2)):
        eng.params[f"b0.lambda_{nm}"].copy_(t)
    rs = torch.rand(2 * hd, generator=g) + 0.5
    eng.import_named("b0.rms_scale", rs)
    qd, kd, vd = (t.to(torch.bfloat16).double() for t in (q, k, v))
    lam = torch.exp((lq1 * lk1).double().sum(-1)) - torch.exp((lq2 * lk2).double().sum(-1)) + li
    return qd, kd, vd, lam, rs.double(), li


def _ref_attention(qd, kd, vd, lam, rs, li, pm, B, L, H, hd):
    """fp64: per head A = softmax1 - lambda softmax2 under the DiffTransformer mask, O_pre = A V, out = RMSNorm"""
    q = qd.view(B, L, H, 2, hd).permute(0, 2, 3, 1, 4)
    k = kd.view(B, L, H, 2, hd).permute(0, 2, 3, 1, 4)
    v = vd.view(B, L, H, 2 * hd).permute(0, 2, 1, 3)
    causal = torch.tril(torch.ones(L, L, dtype=torch.bool))
    vis = causal.unsqueeze(0) & (pm.unsqueeze(1) | torch.eye(L, dtype=torch.bool).unsqueeze(0))
    m = torch.where(vis, 0.0, -math.inf).double().unsqueeze(1)
    s = 1.0 / math.sqrt(hd)
    a1 = torch.softmax(q[:, :, 0] @ k[:, :, 0].transpose(-1, -2) * s + m, -1)
    a2 = torch.softmax(q[:, :, 1] @ k[:, :, 1].transpose(-1, -2) * s + m, -1)
    A = a1 - lam.view(1, H, 1, 1) * a2
    o_pre = A @ v
    o = o_pre / torch.sqrt(o_pre.pow(2).mean(-1, keepdim=True) + 1e-5) * rs * (1 - li)
    return o_pre, o, a1, a2


def _unslot(t, B, L, H, vs, w):
    return t.view(B, L, H, vs)[..., :w].permute(0, 2, 1, 3).double().cpu()


FWD = [(hd, H, L, B) for (hd, H) in ((32, 1), (48, 2), (64, 4), (32, 4), (64, 1), (48, 1))
       for (L, B) in ((1, 3), (2, 37), (63, 3), (64, 1), (65, 3), (127, 1), (128, 3), (129, 1), (200, 3), (255, 1), (256, 3))]


@pytest.mark.parametrize("hd,H,L,B", FWD)
def test_forward_and_saves(cuda, hd, H, L, B):
    g = torch.Generator().manual_seed(hd * 1000 + H * 100 + L)
    lam_t = (-0.5, 0.0, 0.2, 1.3)[(L + H) % 4]
    kind = ("full", "one", "random")[L % 3]
    eng = _engine(cuda, hd, H, L, B, 0)
    pm = _pad_mask(B, L, kind, g)
    qd, kd, vd, lam, rs, li = _setup(eng, lam_t, pm, g)
    vs, Lp = eng.cfg.v_slot, eng.Lp
    o_pre, o, a1, a2 = _ref_attention(qd, kd, vd, lam, rs, li, pm, B, L, H, hd)
    for train in (False, True):
        eng.act[0]["On"].zero_()
        eng._attention_forward(0, train)
        torch.cuda.synchronize()
        got = _unslot(eng.act[0]["On"], B, L, H, vs, 2 * hd)
        err = (got - o).abs().max()
        assert err < 3e-2 * max(1.0, float(o.abs().max())), float(err)
        if 2 * hd < vs:
            assert float(eng.act[0]["On"].view(B, L, H, vs)[..., 2 * hd:].abs().max()) == 0.0
    got_pre = _unslot(eng.act[0]["Opre"], B, L, H, vs, 2 * hd)
    assert (got_pre - o_pre).abs().max() < 2e-2 * max(1.0, float(o_pre.abs().max()))
    a = eng.act[0]
    P1 = a["e1"].view(B, H, Lp, Lp)[:, :, :L, :L].double().cpu() * a["inv1"].view(B, H, Lp)[:, :, :L, None].double().cpu()
    P2 = a["e2"].view(B, H, Lp, Lp)[:, :, :L, :L].double().cpu() * a["inv2"].view(B, H, Lp)[:, :, :L, None].double().cpu()
    assert (P1 - a1).abs().max() < 1e-2 and (P2 - a2).abs().max() < 1e-2


@pytest.mark.parametrize("hd,H,L,B", [(32, 2, 50, 3), (48, 4, 129, 2), (64, 2, 200, 2), (64, 1, 256, 1), (32, 1, 1, 5)])
def test_attention_backward(cuda, hd, H, L, B):
    g = torch.Generator().manual_seed(L + hd)
    eng = _engine(cuda, hd, H, L, B, 0)
    pm = _pad_mask(B, L, "random", g)
    qd, kd, vd, lam, rs, li = _setup(eng, 0.3, pm, g)
    vs = eng.cfg.v_slot
    eng._attention_forward(0, True)
    # upstream gradient of the normalised output, through the per-head RMSNorm backward as the engine runs it
    dO = torch.randn(B * L, H, 2 * hd, generator=g).to(torch.bfloat16)
    dOp = torch.zeros(B * L, H, vs, dtype=torch.bfloat16)
    dOp[..., : 2 * hd] = dO
    eng.s["dOn"].copy_(dOp.view(B * L, -1))
    G = eng.grads
    eng.g32.zero_()
    eng._rms_bwd(eng.s["dOn"], eng.act[0]["Opre"], eng.params["b0.rms_scale"], 1e-5, eng.s["dOpre"], G["b0.rms_scale"], B * L, vs,
                 2 * hd, alpha=1.0 - li)
    eng._attention_backward(0)
    torch.cuda.synchronize()
    # fp64 autograd of sum(out * dO) with respect to q, k, v, rms_scale and the lambda parameters
    lp = {k: eng.params[f"b0.lambda_{k}"].double().cpu().requires_grad_(True) for k in ("q1", "k1", "q2", "k2")}
    q, k, v = (t.clone().requires_grad_(True) for t in (qd, kd, vd))
    rs = rs.clone().requires_grad_(True)
    lam_t = torch.exp((lp["q1"] * lp["k1"]).sum(-1)) - torch.exp((lp["q2"] * lp["k2"]).sum(-1)) + li
    _, o, _, _ = _ref_attention(q, k, v, lam_t, rs, li, pm, B, L, H, hd)
    (o * dO.double().view(B, L, H, 2 * hd).permute(0, 2, 1, 3)).sum().backward()
    got_rs = G["b0.rms_scale"][: 2 * hd].double().cpu()
    assert (got_rs - rs.grad).abs().max() < 2e-2 * float(rs.grad.abs().max())
    dQKV = eng.s["dQKV"].double().cpu()
    T = B * L
    dq = dQKV[:, : H * 128].view(T, H, 2, 64)[..., :hd]
    dk = dQKV[:, H * 128: H * 256].view(T, H, 2, 64)[..., :hd]
    dv = dQKV[:, H * 256:].view(T, H, vs)[..., : 2 * hd]
    for got, ref in ((dq, q.grad.view(T, H, 2, hd)), (dk, k.grad.view(T, H, 2, hd)), (dv, v.grad.view(T, H, 2 * hd))):
        err = (got - ref).abs().max()
        assert err < 3e-2 * max(1.0, float(ref.abs().max())), float(err)
    for nm in ("q1", "k1", "q2", "k2"):
        ref = lp[nm].grad
        got = G[f"b0.lambda_{nm}"].double().cpu()
        assert (got - ref).abs().max() < 2e-2 * max(1e-3, float(ref.abs().max())), nm


@pytest.mark.parametrize("group,d,n_true", [(128, 128, 100), (256, 256, 256), (64, 64, 64), (64, 256, 48), (128, 256, 96)])
@pytest.mark.parametrize("gathered", [False, True])
def test_rmsnorm(cuda, group, d, n_true, gathered):
    from replay_b200._lib import check, lib

    g = torch.Generator().manual_seed(group + d + n_true)
    rows = 300
    x = torch.randn(rows, d, generator=g)
    x.view(rows, d // group, group)[..., n_true:] = 0
    x[7] = 0   # an all-zero row
    w = torch.rand(group, generator=g) + 0.5
    w[n_true:] = 0
    alpha, eps = 0.7, 1e-5
    xb = x.to(torch.bfloat16)
    gather = torch.randperm(rows, generator=g)[:150].to(torch.int32) if gathered else None
    n = 150 if gathered else rows
    y = torch.zeros(n, d, dtype=torch.bfloat16, device=cuda)
    xc, wc = xb.to(cuda), w.to(cuda)
    gc = None if gather is None else gather.to(cuda)
    L = lib()
    check(L.rp_rmsnorm_fwd(xc.data_ptr(), wc.data_ptr(), eps, alpha, n, d, group, n_true, None,
                           None if gc is None else gc.data_ptr(), y.data_ptr(), None), "rp_rmsnorm_fwd")
    xs = xb.double() if gather is None else xb.double()[gather.long()]
    xg = xs.view(n, d // group, group).clone().requires_grad_(True)
    wd = w.double().requires_grad_(True)
    ref = xg * torch.rsqrt(xg[..., :n_true].pow(2).mean(-1, keepdim=True) + eps) * wd * alpha
    torch.testing.assert_close(y.double().cpu().view(n, -1), ref.detach().view(n, -1), rtol=1e-2, atol=1e-2)
    dy = torch.randn(n, d, generator=g).to(torch.bfloat16)
    (ref * dy.double().view(n, d // group, group)).sum().backward()
    dx = torch.zeros(rows, d, dtype=torch.bfloat16, device=cuda)
    dw = torch.zeros(group, device=cuda)
    ws = torch.zeros(L.rp_rmsnorm_bwd_workspace(group), dtype=torch.uint8, device=cuda)
    dyc = dy.to(cuda)
    for _ in range(2):   # dw accumulates
        check(L.rp_rmsnorm_bwd(dyc.data_ptr(), xc.data_ptr(), wc.data_ptr(), eps, alpha, n, d, group, n_true, None,
                               None if gc is None else gc.data_ptr(), dx.data_ptr(), dw.data_ptr(), ws.data_ptr(), ws.numel(), None),
              "rp_rmsnorm_bwd")
    torch.cuda.synchronize()
    ref_dx = xg.grad.view(n, d)
    got_dx = dx.double().cpu() if gather is None else dx.double().cpu()[gather.long()]
    torch.testing.assert_close(got_dx, ref_dx, rtol=2e-2, atol=2e-2 * max(1.0, float(ref_dx.abs().max())))
    torch.testing.assert_close(dw.double().cpu(), 2 * wd.grad, rtol=1e-2, atol=1e-2 * float(wd.grad.abs().max()))
    if n_true < group:
        assert float(dx.double().cpu().view(rows, d // group, group)[..., n_true:].abs().max()) == 0.0


def test_swiglu(cuda):
    from replay_b200._lib import check, lib

    g = torch.Generator().manual_seed(0)
    T, F = 777, 384
    gl = (torch.randn(T, 2 * F, generator=g) * 3).to(torch.bfloat16)
    u = torch.zeros(T, F, dtype=torch.bfloat16, device=cuda)
    glc = gl.to(cuda)
    check(lib().rp_swiglu_fwd(glc.data_ptr(), T, F, u.data_ptr(), None), "rp_swiglu_fwd")
    x = gl.double().requires_grad_(True)
    ref = torch.nn.functional.silu(x[:, :F]) * x[:, F:]
    torch.testing.assert_close(u.double().cpu(), ref.detach(), rtol=1e-2, atol=1e-2)
    du = torch.randn(T, F, generator=g).to(torch.bfloat16)
    (ref * du.double()).sum().backward()
    dgl = torch.zeros(T, 2 * F, dtype=torch.bfloat16, device=cuda)
    check(lib().rp_swiglu_bwd(du.to(cuda).data_ptr(), glc.data_ptr(), T, F, dgl.data_ptr(), None), "rp_swiglu_bwd")
    torch.testing.assert_close(dgl.double().cpu(), x.grad, rtol=2e-2, atol=2e-2)


def test_training_step_is_deterministic(cuda):
    from replay_b200.engine_diff import DiffConfig, DiffEngine

    cfg = DiffConfig(n_items=300, d=128, n_heads=2, n_blocks=2, max_len=100, out_norm="rmsnorm")
    g = torch.Generator().manual_seed(1)
    pm = _pad_mask(8, 100, "random", g)
    ids = torch.where(pm, torch.randint(0, 300, (8, 100), generator=g), torch.full((8, 100), 300))
    labels = torch.randint(0, 300, (8, 100), generator=g)
    out = []
    for _ in range(2):
        eng = DiffEngine(cfg, 8, 100, cuda, seed=3)
        eng.set_batch(ids.to(cuda), pm.to(cuda), labels.to(cuda), pm.to(cuda))
        eng.g32.zero_()
        loss = eng.forward_train().clone()
        eng.backward()
        torch.cuda.synchronize()
        # the embedding backward and the bias column sums are SASRec's kernels, which accumulate with fp32 atomics
        shared = ("item_emb", "pos_emb", ".ff_bg", ".ff_b1", ".ff_b2")
        grads = {k: v.clone().cpu() for k, v in eng.grads.items() if not k.endswith(shared)}
        out.append((loss.cpu(), eng.x[-1].clone().cpu(), grads))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])
    for k in out[0][2]:
        assert torch.equal(out[0][2][k], out[1][2][k]), k
