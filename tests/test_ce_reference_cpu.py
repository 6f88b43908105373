"""The float64 CE-head reference of the GPU tests (tests/ce_reference.py), without a GPU: it matches the oracle's per-row
losses (oracle/sampled.py::row_loss, pinned against the real reference classes by tests/golden/row_losses.npz) and its own
autograd; a simulation of the kernel's arithmetic (fp32 logits and sums, G rounded to bf16, bf16 d_hc) stays within every
bound at the GPU file's shapes; and each planted mistake of the head leaves the bounds by a clear margin."""
import pytest
import torch

import ce_reference as cr
from oracle.sampled import row_loss

MARGIN = 3.0   # a planted mistake must leave its bound by at least this factor


def _oracle(kind, weights=None, log_eps=1e-6, clamp=100.0, seed=0):
    """fp64 autograd of row_loss on a [B, L] batch with gaps in the target mask, and the same batch compacted for reference()"""
    g = torch.Generator().manual_seed(seed)
    B, L, d, I = 3, 7, 16, 40
    hidden = (torch.randn(B, L, d, generator=g) * 0.8).double().requires_grad_(True)
    table = (torch.randn(I, d, generator=g) * 0.6).double().requires_grad_(True)
    labels = torch.randint(0, I, (B, L), generator=g)
    tm = torch.rand(B, L, generator=g) > 0.3
    w = torch.rand(B, L, 1, generator=g, dtype=torch.float64) * 3 if weights else None
    loss = row_loss(hidden, table, labels, tm, kind, w, log_eps=log_eps, clamp=clamp)
    loss.backward()
    n = int(tm.sum())
    ref = cr.reference(hidden.detach()[tm], table.detach(), None, labels[tm], n,
                       row_weight=w[..., 0][tm] if weights else None, loss_kind=1 if kind == "login" else 0,
                       log_eps=log_eps, clamp=clamp)
    return loss.detach(), hidden.grad[tm], table.grad, ref


@pytest.mark.parametrize("kind,weights,log_eps,clamp", [("logout", False, 1e-6, 100.0), ("logout_weighted", True, 1e-6, 100.0),
                                                        ("login", False, 1e-6, 100.0), ("login", False, 1e-2, 3.2)])
def test_reference_matches_oracle_row_losses(kind, weights, log_eps, clamp):
    loss, gh, gW, ref = _oracle(kind, weights, log_eps, clamp)
    if clamp < 100:
        assert (~ref["gate"]).any() and ref["gate"].any(), "the clamp should be active on some rows and not on others"
    torch.testing.assert_close(ref["loss"], loss, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(ref["d_h"], gh, rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(ref["d_W"], gW, rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("kind", ["plain", "login_w", "login_hi"])
def test_reference_matches_its_autograd_with_bias(kind):
    """CE with a bias, LogInCE with row weights and an active clamp: the closed-form gradients are those of the loss"""
    c = cr.make_case(200, 150, 97, 64, bias=True, kind=kind, seed=3)
    ref = cr.case_reference(c, 150)
    h = c["h"][:150].double().requires_grad_(True)
    W = c["W"].double().requires_grad_(True)
    b = c["b"].double().requires_grad_(True)
    x = h @ W.T + b
    y = c["labels"][:150]
    lp = x.gather(1, y[:, None])[:, 0] - torch.logsumexp(x, -1)
    w = c["row_weight"][:150].double() if c["row_weight"] is not None else torch.ones(150, dtype=torch.float64)
    if c["loss_kind"] == 0:
        lt = -lp
    else:
        lt = -torch.clamp(torch.log(lp.exp() + c["log_eps"]), -c["clamp"], c["clamp"])
        assert (~ref["gate"]).any() and ref["gate"].any()
    loss = (w * lt).mean()
    loss.backward()
    torch.testing.assert_close(ref["loss"], loss.detach(), rtol=1e-12, atol=1e-12)
    for got, want in ((ref["d_h"], h.grad), (ref["d_W"], W.grad), (ref["d_b"], b.grad)):
        torch.testing.assert_close(got, want, rtol=1e-9, atol=1e-13)


def _simulate(c, n_valid):
    """the kernel's arithmetic: fp32 logits, lse, target logit and row terms; G = exp(x - lse) wg / T_v rounded to bf16; fp32
    GEMMs and one-hot terms; d_hc stored in bf16"""
    T = n_valid
    h, W = c["h"][:T].float(), c["W"].float()
    y = c["labels"][:T]
    x = h @ W.T
    if c["b"] is not None:
        x = x + c["b"].float()[None, :]
    lse = torch.logsumexp(x, -1)
    zy = x.gather(1, y[:, None])[:, 0]
    w = c["row_weight"][:T].float() if c["row_weight"] is not None else torch.ones(T)
    if c["loss_kind"] == 0:
        lt, wg = lse - zy, w
    else:
        p = torch.exp(zy - lse)
        lg = torch.log(p + c["log_eps"])
        lt = -lg.clamp(-c["clamp"], c["clamp"])
        wg = w * torch.where((lg > -c["clamp"]) & (lg < c["clamp"]), p / (p + c["log_eps"]), torch.zeros_like(p))
    inv = torch.tensor(1.0 / max(T, 1), dtype=torch.float32)
    cw = wg * inv
    G = (torch.exp(x - lse[:, None]) * cw[:, None]).to(torch.bfloat16).float()
    d_h = (G @ W - cw[:, None] * W[y]).to(torch.bfloat16)
    d_W = (G.T @ h).index_add_(0, y, -cw[:, None] * h)
    d_b = G.sum(0).index_add_(0, y, -cw)
    return dict(loss=(w * lt).sum() * inv, d_h=d_h, d_W=d_W, d_b=d_b)


def _worst_all(got, ref):
    return max(cr.worst(got["loss"].reshape(()), ref["loss"], ref["bound_loss"]),
               cr.worst(got["d_h"], ref["d_h"], ref["bound_h"]), cr.worst(got["d_W"], ref["d_W"], ref["bound_W"]), cr.worst(got["d_b"], ref["d_b"], ref["bound_b"]))


# shapes of tests/test_gpu_ce_head_fp64.py (layout() at 132 SMs): (capacity, n_valid, n_items, d, bias, kind, scale_h, scale_e)
SHAPES = [
    (16896, 635, 623, 128, True, "weighted", 0.5, 0.3),       # fused, P == 1 (layout(NSTAGE + 1, 128, "P1"))
    (128, 123, 20001, 256, True, "login_w", 0.5, 0.3),        # fused, P > 1, large catalog
    (128, 123, 20001, 64, False, "plain", 0.5, 0.3),
    (16896, 315, 303, 256, True, "login_lo", 2.0, 1.0),       # behind the two-pass forward
    (1152, 1147, 1135, 64, True, "login_hi", 0.5, 0.3),       # un-fused (layout(NSTAGE + 1, 64, "twopass"))
    (384, 300, 5003, 512, True, "weighted", 0.5, 0.3),        # d = 512
    (300, 298, 65, 128, True, "login", 0.5, 0.3),             # capacity off the 128-row grid
    (256, 200, 20001, 128, True, "weighted", 0.5, 0.3),       # the largest catalog of the edge cases
]


@pytest.mark.parametrize("shape", SHAPES, ids=[f"{s[1]}x{s[2]}d{s[3]}{s[5]}" for s in SHAPES])
def test_kernel_arithmetic_stays_within_bounds(shape):
    cap, nv, I, d, bias, kind, sh, se = shape
    c = cr.make_case(cap, nv, I, d, bias=bias, kind=kind, scale_h=sh, scale_e=se)
    ref = cr.case_reference(c, nv)
    got = _simulate(c, nv)
    assert _worst_all(got, ref) <= 1.0


def test_kernel_arithmetic_stays_within_bounds_with_the_bias_trap():
    c = cr.make_case(256, 200, 5003, 128, bias=True, kind="weighted", bias_trap=True)
    assert (c["b"] == -60).sum() == 1
    assert _worst_all(_simulate(c, 200), cr.case_reference(c, 200)) <= 1.0


def _mistakes(c, ref, nv, cap):
    """the fp64 result with one mistake of the head planted at a time: name -> outputs"""
    h, W = c["h"][:nv].double(), c["W"].double()
    y = c["labels"][:nv].long()
    w = c["row_weight"][:nv].double() if c["row_weight"] is not None else torch.ones(nv, dtype=torch.float64)
    base = dict(loss=ref["loss"], d_h=ref["d_h"], d_W=ref["d_W"], d_b=ref["d_b"])
    out = {}
    if c["row_weight"] is not None:   # the label scatter subtracts h / T_v and 1 / T_v whatever the row's weight
        d_W = ref["d_W"].clone().index_add_(0, y, ((ref["wg"] - 1) * ref["inv"])[:, None] * h)
        d_b = ref["d_b"].clone().index_add_(0, y, (ref["wg"] - 1) * ref["inv"])
        out["scatter_ignores_weight"] = dict(base, d_W=d_W, d_b=d_b)
    if c["loss_kind"] == 1:
        p, py, eps = ref["p"], ref["py"], c["log_eps"]
        if (~ref["gate"]).any():   # a clamped row keeps its gradient
            wg = w * py / (py + eps)
            d_h, d_W, d_b = cr.grads(p, y, wg * ref["inv"], h, W)
            out["clamped_row_keeps_gradient"] = dict(base, d_h=d_h, d_W=d_W, d_b=d_b)
        if eps >= 1e-3:   # with eps = 1e-6 the weight differs from 1 by less than G's rounding unless p_y < 1e-3
            wg = w * ref["gate"].double()   # p / (p + eps) replaced by 1
            d_h, d_W, d_b = cr.grads(p, y, wg * ref["inv"], h, W)
            out["login_weight_is_one"] = dict(base, d_h=d_h, d_W=d_W, d_b=d_b)
    # a row of median gradient among those the logits do not already fit (p_y < 1/2: with p_y near 1 the softmax and one-hot
    # parts cancel, and the whole row's gradient is smaller than the rounding of its terms)
    live = ((ref["wg"] != 0) & (ref["py"] < 0.5)).nonzero()[:, 0]
    if len(live):
        t = live[ref["d_h"][live].norm(dim=1).argsort()[len(live) // 2]]
        d_W = ref["d_W"].clone()
        d_W[y[t]] = 0
        out["table_row_zeroed"] = dict(base, d_W=d_W)
        d_h = ref["d_h"].clone()
        d_h[t] = 0
        out["token_row_zeroed"] = dict(base, d_h=d_h)
    if cap >= 1.1 * nv:   # closer, the change hides below the bf16 rounding of G
        s = nv / cap
        out["normalised_by_capacity"] = dict(loss=ref["loss"] * s, d_h=ref["d_h"] * s, d_W=ref["d_W"] * s, d_b=ref["d_b"] * s)
    if c["b"] is not None:
        if c["loss_kind"] == 0:   # every row loss grows by its target's bias
            out["bias_dropped_from_zy"] = dict(base, loss=ref["loss"] + (w * c["b"].double()[y]).sum() * ref["inv"])
        else:
            p, eps = ref["p"], c["log_eps"]
            lp = ref["py"].log() - c["b"].double()[y]
            lg = torch.log(lp.exp() + eps)
            gate = (lg > -c["clamp"]) & (lg < c["clamp"])
            wg = w * torch.where(gate, lp.exp() / (lp.exp() + eps), torch.zeros_like(lp))
            d_h, d_W, d_b = cr.grads(p, y, wg * ref["inv"], h, W)
            out["bias_dropped_from_zy"] = dict(loss=(-w * lg.clamp(-c["clamp"], c["clamp"])).sum() * ref["inv"], d_h=d_h,
                                               d_W=d_W, d_b=d_b)
    return out


@pytest.mark.parametrize("shape", SHAPES, ids=[f"{s[1]}x{s[2]}d{s[3]}{s[5]}" for s in SHAPES])
def test_planted_mistakes_leave_the_bounds(shape):
    cap, nv, I, d, bias, kind, sh, se = shape
    c = cr.make_case(cap, nv, I, d, bias=bias, kind=kind, scale_h=sh, scale_e=se)
    ref = cr.case_reference(c, nv)
    seen = {}
    for name, got in _mistakes(c, ref, nv, cap).items():
        seen[name] = _worst_all(got, ref)
    print(shape, {k: f"{v:.3g}" for k, v in seen.items()})
    assert seen and min(seen.values()) > MARGIN, seen


def test_every_planted_mistake_is_planted_somewhere():
    names = set()
    for shape in SHAPES:
        cap, nv, I, d, bias, kind, sh, se = shape
        c = cr.make_case(cap, nv, I, d, bias=bias, kind=kind, scale_h=sh, scale_e=se)
        names |= set(_mistakes(c, cr.case_reference(c, nv), nv, cap))
    assert names == {"scatter_ignores_weight", "clamped_row_keeps_gradient", "login_weight_is_one", "table_row_zeroed",
                     "token_row_zeroed", "normalised_by_capacity", "bias_dropped_from_zy"}
