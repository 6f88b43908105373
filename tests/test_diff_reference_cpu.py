"""tests/diff_reference.py without a GPU: its closed form against the forward parts and autograd gradients of
oracle/diff.diff_attention, and its bounds' power to tell a subtly wrong kernel from a right one on the GPU tests' own
input sizes: each mistake below breaks a bound by at least ten times the GPU test's tolerance."""
import math

import pytest
import torch

import diff_reference as dr
from oracle.diff import diff_attention, visible_mask
from test_gpu_diff_fp64 import LAMBDA_INIT, TOL_BWD, TOL_FWD, TOL_RMS, TOL_SWIGLU, _rows_shape

DISCRIMINATES = 10.0
H100_SMS = 132      # the warp cap of the softmax backward on an H100 SXM (the GPU tests read the device's count)


# ------------------------------------------------------------------------------------------------ agreement with the oracle
def _oracle_case(B=2, L=9, H=2, hd=5, seed=0):
    """a state dict for block 0 of oracle/diff.diff_attention, input x [B, L, d], pad with holes, dOn [B, H, L, 2 hd]"""
    g = torch.Generator().manual_seed(seed)
    d = H * hd
    sd = {f"body.encoder.layers.0.attn.{k}.weight": torch.randn(r, c, generator=g, dtype=torch.float64) / math.sqrt(c)
          for k, r, c in (("W_q", 2 * d, d), ("W_k", 2 * d, d), ("W_v", 2 * d, d), ("W_o", d, 2 * d))}
    for k in ("q1", "k1", "q2", "k2"):
        sd[f"body.encoder.layers.0.attn.lambda_{k}"] = torch.randn(H, hd, generator=g, dtype=torch.float64) * 0.3
    sd["body.encoder.layers.0.attn.rms_scale"] = 1 + 0.25 * torch.randn(2 * hd, generator=g, dtype=torch.float64)
    x = torch.randn(B, L, d, generator=g, dtype=torch.float64) * 1.5
    pad = torch.rand(B, L, generator=g) < 0.6
    pad[0, -1] = False
    dOn = torch.randn(B, H, L, 2 * hd, generator=g, dtype=torch.float64)
    return sd, x, pad, dOn


def _to_engine(q, k, v, B, L, H, hd):
    """oracle projections [B, L, 2d] (per head [x1 | x2] of hd each) -> QKV [B*L, n_qkv] in the engine's padded layout"""
    VS = dr.v_slot_of(hd)
    T = B * L
    QKV = torch.zeros(T, H * (4 * dr.SLOT + VS), dtype=torch.float64)
    for c0, t in ((0, q), (H * 2 * dr.SLOT, k)):
        blk = torch.zeros(T, H, 2, dr.SLOT, dtype=torch.float64)
        blk[..., :hd] = t.reshape(T, H, 2, hd)
        QKV[:, c0:c0 + H * 2 * dr.SLOT] = blk.reshape(T, -1)
    vb = torch.zeros(T, H, VS, dtype=torch.float64)
    vb[..., :2 * hd] = v.reshape(T, H, 2 * hd)
    QKV[:, H * 4 * dr.SLOT:] = vb.reshape(T, -1)
    return QKV


def _from_engine(dQKV, B, L, H, hd):
    """dQKV in the engine's layout -> (dq, dk, dv) [B*L, 2d] in the oracle's"""
    VS = dr.v_slot_of(hd)
    T = B * L
    dq = dQKV[:, :H * 2 * dr.SLOT].reshape(T, H, 2, dr.SLOT)[..., :hd].reshape(T, -1)
    dk = dQKV[:, H * 2 * dr.SLOT:H * 4 * dr.SLOT].reshape(T, H, 2, dr.SLOT)[..., :hd].reshape(T, -1)
    dv = dQKV[:, H * 4 * dr.SLOT:].reshape(T, H, VS)[..., :2 * hd].reshape(T, -1)
    return dq, dk, dv


def _heads_rows(t, B, L, H, VS):
    """[B, H, L, w] -> [B*L, H*VS]"""
    out = torch.zeros(B, L, H, VS, dtype=t.dtype)
    out[..., :t.shape[-1]] = t.permute(0, 2, 1, 3)
    return out.reshape(B * L, H * VS)


@pytest.mark.parametrize("H,hd", [(2, 5), (1, 8), (3, 33)])
def test_closed_form_matches_the_oracle(H, hd):
    B, L = 2, 9
    sd, x, pad, dOn = _oracle_case(B, L, H, hd, seed=H * 100 + hd)
    p = "body.encoder.layers.0.attn."
    leaves = {k: v.clone().requires_grad_(True) for k, v in sd.items() if k != p + "W_o.weight"}
    full = dict(sd, **leaves)
    _, parts = diff_attention(x, full, 0, H, visible_mask(pad), return_parts=True)
    parts["o_pre"].retain_grad()
    (parts["o"] * dOn).sum().backward()
    d, VS = H * hd, dr.v_slot_of(hd)
    xf = x.reshape(B * L, d)
    q, k, v = (xf @ sd[p + f"W_{n}.weight"].T for n in ("q", "k", "v"))
    QKV = _to_engine(q, k, v, B, L, H, hd)
    lp = [sd[p + f"lambda_{n}"] for n in ("q1", "k1", "q2", "k2")]
    rs = torch.zeros(VS, dtype=torch.float64)
    rs[:2 * hd] = sd[p + "rms_scale"]
    li = LAMBDA_INIT
    dOn_rows = _heads_rows(dOn, B, L, H, VS)
    st = dr.attention_stage(QKV, dOn_rows, pad, *lp, rs, li, H, hd)
    close = dict(rtol=1e-9, atol=1e-11)
    assert torch.allclose(st["Opre"], _heads_rows(parts["o_pre"].detach(), B, L, H, VS), **close)
    assert torch.allclose(st["On"], _heads_rows(parts["o"].detach(), B, L, H, VS), **close)
    dq, dk, dv = _from_engine(st["dQKV"], B, L, H, hd)
    for n, dx in (("q", dq), ("k", dk), ("v", dv)):
        assert torch.allclose(dx.T @ xf, leaves[p + f"W_{n}.weight"].grad, **close), n
    for n in ("q1", "k1", "q2", "k2"):
        assert torch.allclose(st["d_" + n], leaves[p + f"lambda_{n}"].grad, **close), n
    assert torch.allclose(st["d_rs"], leaves[p + "rms_scale"].grad, **close)

    # the kernel-boundary restatements: forward parts, and the softmax / lambda backward from exact saves.  They take
    # the kernels' fp32 scalars (1 / sqrt(hd), lambda_init, eps), hence the looser tolerance.
    P = dr.Attn(qkv=QKV, q_c0=0, k_c0=H * 2 * dr.SLOT, v_c0=H * 4 * dr.SLOT, pad=pad, lq1=lp[0], lk1=lp[1], lq2=lp[2],
                lk2=lp[3], li=li, rs=rs, eps=1e-5, B=B, H=H, L=L, hd=hd)
    f = dr.forward(P)
    loose = dict(rtol=1e-5, atol=1e-5)
    assert torch.allclose(f["A1"], parts["a1"].reshape(B * H, L, L), **loose)
    assert torch.allclose(f["A2"], parts["a2"].reshape(B * H, L, L), **loose)
    assert torch.allclose(f["o_pre"], st["Opre"], **loose) and torch.allclose(f["out"], st["On"], **loose)
    assert torch.allclose(f["e1"] * f["inv1"][..., None], f["A1"], **close)
    Lp = P.Lp
    sv = {}
    for kk in ("e1", "e2"):
        sv[kk] = torch.zeros(B * H, Lp, Lp, dtype=torch.float64)
        sv[kk][:, :L, :L] = f[kk]
    for kk in ("inv1", "inv2"):
        sv[kk] = torch.zeros(B * H, Lp, dtype=torch.float64)
        sv[kk][:, :L] = f[kk]
    dOpre = parts["o_pre"].grad                                        # [B, H, L, 2 hd]
    vh = v.reshape(B, L, H, 2 * hd).permute(0, 2, 1, 3)
    dA = torch.zeros(B * H, Lp, Lp, dtype=torch.float64)
    dA[:, :L, :L] = (dOpre @ vh.transpose(-1, -2)).reshape(B * H, L, L)
    sb = dr.softmax_bwd(P, sv["e1"], sv["e2"], sv["inv1"], sv["inv2"], dA, dOn_rows, f["O32"], f["O2"])
    # dQ, dK from dS1 / dS2 and dV from A: the closed form's gradients
    qh = q.reshape(B, L, H, 2, hd).permute(0, 2, 3, 1, 4).reshape(B * H, 2, L, hd)
    kh = k.reshape(B, L, H, 2, hd).permute(0, 2, 3, 1, 4).reshape(B * H, 2, L, hd)
    dq_sb = torch.stack([sb["dS1"] @ kh[:, 0], sb["dS2"] @ kh[:, 1]], 1)
    dk_sb = torch.stack([sb["dS1"].transpose(-1, -2) @ qh[:, 0], sb["dS2"].transpose(-1, -2) @ qh[:, 1]], 1)
    dv_sb = sb["A"].transpose(-1, -2) @ dOpre.reshape(B * H, L, 2 * hd)
    back = lambda t: t.reshape(B, H, 2, L, hd).permute(0, 3, 1, 2, 4).reshape(B * L, 2 * d)  # noqa: E731
    assert torch.allclose(back(dq_sb), dq, **loose), float((back(dq_sb) - dq).abs().max())
    assert torch.allclose(back(dk_sb), dk, **loose), float((back(dk_sb) - dk).abs().max())
    assert torch.allclose(dv_sb.reshape(B, H, L, 2 * hd).permute(0, 2, 1, 3).reshape(B * L, 2 * d), dv, **loose)
    dlam = torch.zeros(B * H, Lp, dtype=torch.float64)
    dlam[:, :L] = sb["dlam"]
    lb = dr.lambda_bwd(dlam, B, H, L, *lp, li)
    for n in ("q1", "k1", "q2", "k2"):
        assert torch.allclose(lb["g_" + n], leaves[p + f"lambda_{n}"].grad, **loose), n
    rb = dr.rmsnorm_bwd(dOn_rows, f["o_pre"], rs, 1e-5, 1 - li, B * L, H * VS, VS, 2 * hd)
    assert torch.allclose(rb["dw"][:2 * hd], leaves[p + "rms_scale"].grad, **loose)


def test_rmsnorm_and_swiglu_match_autograd():
    x, w, dy, n_true = dr.make_rms(40, 256, 128, "slots", seed=3, zero_row=7)
    xd = x.double().requires_grad_(True)
    wd = w.double().requires_grad_(True)
    xv = xd.view(40, 2, 128)
    y = xv * torch.rsqrt(xv.pow(2).sum(-1, keepdim=True) / n_true + dr.f32(1e-5)) * wd * dr.f32(0.7)
    (y.reshape(40, 256) * dy.double()).sum().backward()
    ry, _, _ = dr.rmsnorm_fwd(x, w, 1e-5, 0.7, 40, 256, 128, n_true)
    rb = dr.rmsnorm_bwd(dy, x, w, 1e-5, 0.7, 40, 256, 128, n_true)
    assert torch.allclose(ry, y.detach().reshape(40, 256), rtol=1e-12, atol=1e-14)
    assert torch.allclose(rb["dx"], xd.grad, rtol=1e-10, atol=1e-12)
    assert torch.allclose(rb["dw"], wd.grad, rtol=1e-10, atol=1e-12)
    assert torch.allclose(rb["dw_parts"].sum(0), rb["dw"], rtol=1e-12, atol=1e-14)
    gl, du = dr.make_swiglu(50, 33, seed=1)
    gd = gl[:50].double().requires_grad_(True)
    u = torch.nn.functional.silu(gd[:, :33]) * gd[:, 33:]
    (u * du[:50].double()).sum().backward()
    ru, _ = dr.swiglu_fwd(gl, 50, 33)
    rd, _ = dr.swiglu_bwd(du, gl, 50, 33)
    assert torch.allclose(ru, u.detach(), rtol=1e-12, atol=1e-300)
    assert torch.allclose(rd, gd.grad, rtol=1e-10, atol=1e-300)


def test_inputs_hit_their_targets():
    P = dr.make_attn(3, 40, 33, 4, pad="left", lam_target=0.999, li=LAMBDA_INIT, identical=True, seed=1)
    lam = P.lam()["lam"]
    assert abs(float(lam[0]) - 0.999) < 1e-5 and float((lam[1:] - lam[:-1]).abs().min()) > 0.04
    q, k, _ = P.heads(0)
    assert torch.equal(q[:, 0], q[:, 1]) and torch.equal(k[:, 0], k[:, 1])
    # the slot padding q / k [hd, 64) and v [2 hd, v_slot) is zero
    X = P.qkv.float()
    assert float(X[:, :4 * 4 * dr.SLOT].reshape(-1, 16, dr.SLOT)[..., 33:].abs().max()) == 0
    assert float(X[:, 16 * dr.SLOT:P.n_qkv].reshape(-1, 4, 128)[..., 66:].abs().max()) == 0
    gl, _ = dr.make_swiglu(100, 64, seed=0)
    gates = gl[:100, :64].float()
    assert float(gates.min()) <= -88.5 and float(gates.max()) >= 88.5
    assert set(dr.EDGE_GATES) <= set(gates.reshape(-1).tolist())


# ------------------------------------------------------------------------------------------------ the bounds discriminate
def _gpu_attn(hd, H, L, pad, lam, B=3, **kw):
    """test_attention's input for one case (same seed)"""
    seed = hd * 1000 + H * 300 + L
    return dr.make_attn(B, L, hd, H, pad=pad, lam_target=lam, li=LAMBDA_INIT, seed=seed, **kw)


def test_bound_catches_the_neighbouring_heads_lambda():
    P = _gpu_attn(32, 3, 100, "holes", LAMBDA_INIT)
    ref = dr.forward(P)
    lam = {k: v.roll(1, 0) for k, v in P.lam().items()}
    bad = dr.forward(P, lam=lam)
    for name in ("o_pre", "out"):
        assert dr.ratio(bad[name], ref[name], ref[name + "_b"]) >= DISCRIMINATES * TOL_FWD, name


def test_bound_catches_a_missing_output_scale():
    P = _gpu_attn(64, 2, 100, "holes", 0.3)
    ref = dr.forward(P)
    bad = dr.forward(P, alpha=1.0)
    assert dr.ratio(bad["out"], ref["out"], ref["out_b"]) >= DISCRIMINATES * TOL_FWD


@pytest.mark.parametrize("mistake", ["no_diagonal", "padded_keys_visible"])
def test_bound_catches_a_wrong_mask(mistake):
    P = _gpu_attn(48, 2, 33, "holes", 0.3)
    ref = dr.forward(P)
    causal = torch.ones(P.L, P.L, dtype=torch.bool).tril()
    eye = torch.eye(P.L, dtype=torch.bool)

    def vis(b):
        if mistake == "padded_keys_visible":
            return causal
        return causal & P.pad[b][None, :]      # a padded query row loses its own key

    bad = dr.forward(P, visible=vis)
    assert not bool(P.pad.all()) and bool((causal & eye).any())
    got = torch.nan_to_num(bad["o_pre"], nan=0.0)   # a row left without keys: whatever the kernel writes, not the ref
    assert dr.ratio(got, ref["o_pre"], ref["o_pre_b"]) >= DISCRIMINATES * TOL_FWD


def _bwd_problem(P, seed=1):
    f = dr.forward(P)
    s = dr.saves_from_reference(P, f)
    dA, d_on = dr.bwd_inputs(P, s, seed)
    return s, dA, d_on


def test_bound_catches_r2_from_the_bf16_dO_pre():
    """the kernel recomputes dO_pre in fp32; the bf16 dO_pre the dV GEMM uses would lose r2 to cancellation"""
    P = _gpu_attn(64, 2, 100, "holes", 0.3)
    s, dA, d_on = _bwd_problem(P)
    ref = dr.softmax_bwd(P, s["e1"], s["e2"], s["inv1"], s["inv2"], dA, d_on, s["o32"], s["o2"])
    B, H, L, VS, hd = P.B, P.H, P.L, P.VS, P.hd
    x = s["o32"][:, :H * VS].double().reshape(B * L, H, VS)
    o2 = s["o2"][:, :H * VS].double().reshape(B * L, H, VS)
    gw = d_on[:, :H * VS].double().reshape(B * L, H, VS) * P.rs.double() * (1 - dr.f32(P.li))
    n = 2 * hd
    r = 1 / torch.sqrt(x.pow(2).sum(-1, keepdim=True) / n + dr.f32(P.eps))
    dOpre = r * gw - x * r ** 3 * (gw * x).sum(-1, keepdim=True) / n
    r2_bad = (dOpre.to(torch.bfloat16).double() * o2).sum(-1)         # [B*L, H]
    bad = -r2_bad.reshape(B, L, H).permute(0, 2, 1).reshape(B * H, L)
    assert dr.ratio(bad, ref["dlam"], ref["dlam_b"]) >= DISCRIMINATES * TOL_BWD


def test_bound_catches_a_warp_keeping_its_first_rows_lambda():
    """B * H * L = 4 x the warp cap (SMs * 128 rows) with 4 heads: a warp's rows are cap apart, and cap / L sequences of 4
    heads put them in other heads.  A kernel that reads lambda once per warp breaks A's and dS2's bounds."""
    cap = H100_SMS * dr.BWD_WARPS_PER_SM
    B, H, L = _rows_shape(4 * cap)
    assert H == 4
    P = dr.make_attn(B, L, 64, H, pad="left", lam_target=0.3, li=LAMBDA_INIT, seed=4 * cap)
    s, dA, d_on = _bwd_problem(P)
    ref = dr.softmax_bwd(P, s["e1"], s["e2"], s["inv1"], s["inv2"], dA, d_on, s["o32"], s["o2"])
    lam = P.lam()["lam"]
    row = torch.arange(B * H * L)
    first_head = ((row % cap) // L) % H
    lam_bad = lam[first_head].reshape(B * H, L, 1)
    A_bad = ref["A1"] - lam_bad * ref["A2"]
    assert dr.ratio(A_bad, ref["A"], ref["A_b"]) >= DISCRIMINATES * TOL_BWD


def test_bound_catches_rmsnorm_dividing_by_the_group():
    x, w, dy, n_true = dr.make_rms(300, 256, 64, "slots", seed=1)
    assert n_true == 50
    y, yb, _ = dr.rmsnorm_fwd(x, w, 1e-5, 0.7, 300, 256, 64, n_true)
    bad, _, _ = dr.rmsnorm_fwd(x, w, 1e-5, 0.7, 300, 256, 64, 64)
    assert dr.ratio(bad, y, yb) >= DISCRIMINATES * TOL_RMS
    rb = dr.rmsnorm_bwd(dy, x, w, 1e-5, 0.7, 300, 256, 64, n_true)
    bb = dr.rmsnorm_bwd(dy, x, w, 1e-5, 0.7, 300, 256, 64, 64)
    assert dr.ratio(bb["dx"], rb["dx"], rb["dx_b"]) >= DISCRIMINATES * TOL_RMS


@pytest.mark.parametrize("items", [1025, 20000])
def test_bound_catches_a_dropped_dw_partial(items):
    x, w, dy, n_true = dr.make_rms(items, 64, 64, "slots", seed=2)
    rb = dr.rmsnorm_bwd(dy, x, w, 1e-5, 1.0, items, 64, 64, n_true)
    start = torch.randn(64, generator=torch.Generator().manual_seed(0))
    bound = dr.dw_bound(rb, start)
    worst = max(dr.ratio(rb["dw"] - rb["dw_parts"][p], rb["dw"], bound, w > 0) for p in (0, 1, 511, 1023))
    assert worst >= DISCRIMINATES * TOL_RMS
    # every single partial matters somewhere
    each = ((rb["dw_parts"][:, w > 0]).abs() / bound[w > 0]).amax(1)
    assert float(each.min()) >= DISCRIMINATES * TOL_RMS, float(each.min())


def test_bound_catches_swiglu_without_the_silu_slope():
    gl, du = dr.make_swiglu(777, 384, seed=5)
    ref, bound = dr.swiglu_bwd(du, gl, 777, 384)
    bad, _ = dr.swiglu_bwd(du, gl, 777, 384, with_silu_slope=False)
    assert dr.ratio(bad, ref, bound) >= DISCRIMINATES * TOL_SWIGLU
