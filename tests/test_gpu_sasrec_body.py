"""SASRec's fused block kernels (csrc/rp_block_fused.cu: rp_ln_qkv_fused, rp_post_attn_train, rp_post_attn_fused,
rp_post_attn_bwd, rp_pre_attn_bwd; csrc/rp_wgrad.cu: rp_wgrad_group) and SasRecEngine's training step, each
against a float64 reference computed from the same bf16 inputs, at the config-2 shape (L = 200, d = 128, H = 2, two blocks,
dropout 0.2, T = 102 400 tokens) and at the edges where these kernels change behaviour.

Kernels are called through the C ABI with the argument patterns of engine.py.  Dropout masks come from the Python port of
rp_philox.cuh (tests/dropout_stream.py) and are compared with the kernels' zero patterns bit for bit; values are compared
element-wise in half-ulp units (ulp_err) where an output is one rounding away from the exact value, and per 64-row block
(block_err) for reductions and gradients.  Buffers have 64 sentinel rows past T that no kernel may write.

Kernel matrix (T, d, hd_valid, dropout, row mask):
    T = 1 (one partial tile), 129 (a ragged second tile), 1400 (the step test's T), 102 400 and 102 363 (config 2's T,
    ~6 tiles per CTA through the TMA double buffer, full and ragged);
    d = 64 and 128 at T = 1400 and at the large T; hd_valid 32 and 48 at d = 128, 50 at d = 64 (padded feature slots);
    dropout 0 and 0.2 with a non-zero counter behind seed_ptr; row mask on and off.
Every input mixes rows at unit scale, rows with a common offset of up to 50x their spread, and rows at 1e-4 to 1e-3
scale, where the LayerNorm eps (1e-8) matters.
Run with -s to print the worst error of each family.
"""
import math
import os

import numpy as np
import pytest
import torch

from dropout_stream import keep_draws
from fp64_checks import WorstErrors, block_err, feat_mask, ln_bwd_ref, ln_ref, seq_block_err, ulp_err
from replay_b200._lib import WgradPair, check, lib
from sasrec_fp64 import (CTR, EPS, P_DROP, SEED, _bf, _Case, _gen, _ks, _leaves, _map, _site, engine_keeps,
                         ref_loss_and_grads, step_batch, unit_keeps)

SENT = -3.25                           # sentinel for memory a kernel must not write (exact in bf16)
HALF_ULP_SLACK = 2.0 ** -21            # fp32 accumulation slack, times sum_k |a_k b_k|

# Tolerances.  Each bound is about 3x the worst error observed over every case of this file on one H100 80GB HBM3
# (400 W power limit); the element-wise ones are in units of half a bf16 ulp, where rounding to nearest alone gives 1.
TOL_ULP = 3.5            # outputs one rounding from fp64 (GEMM epilogues, LayerNorm y, h): element-wise; worst seen 1.18
TOL_ULP_EVAL = 4.0       # eval kernels, whose y / u are rounded to bf16 inside: element-wise; worst seen 1.29
TOL_MEAN = 2.5e-7        # fused LayerNorm mean, relative to the row's RMS; worst seen 8.1e-8
TOL_RSTD = 9e-4          # fused LayerNorm rstd, relative: the kernels' one-pass E[x^2] - mean^2 loses precision on rows with
                         # a common offset, (mean / std)^2 x fp32 eps; worst seen 3.0e-4 (offset 50x, 50 features)
TOL_BWD = 1.1e-2         # d_t, du, dh, d_o, dx (bf16): per 64-row block norm-relative; worst seen 3.6e-3 (d_o)
TOL_LN_GRAD = 7e-3       # dln_w / dln_b of the fused backward kernels: norm-relative; worst seen 2.2e-3 (post_attn_bwd)
TOL_SPLITK = 1.5e-5      # rp_wgrad_group dW: per 64-row block norm-relative; worst seen 5.1e-6
TOL_SUM = 6e-7           # rp_wgrad_group db (fp32 column sums): norm-relative; worst seen 2.0e-7
TOL_LOSS = 6e-5          # SASRec step: relative loss error; worst seen 1.9e-5
TOL_HID = 2.2e-2         # SASRec step: x[-1] of real rows, per (sequence, 64-row block); worst seen 7.2e-3
TOL_GRAD = 0.22          # SASRec step: parameter gradients, per 64-row block; worst seen 7.4e-2 (in_w, d 192 / 4 heads)

_worst = WorstErrors()
_note = _worst.note


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    _worst.report()


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda")


def _stream():
    return torch.cuda.current_stream().cuda_stream


_CASES = {"c2": ("new", 128, 2, True), "c2_unfused": ("new", 128, 2, False), "d64h2": ("new", 64, 2, True),
          "legacy_d50h1": ("legacy", 50, 1, True), "d192h4": ("new", 192, 4, True)}


def _model_errs(a, b, real):
    """(loss, x[-1], gradient) errors of result ``a`` against ``b`` in units of their tolerances."""
    la, xa, _, Ga = a
    lb, xb, _, Gb = b
    e_loss = abs(float(la - lb)) / abs(float(lb)) / TOL_LOSS
    e_hid = seq_block_err(xa, xb, real) / TOL_HID
    e_grad = max(_name_err(Ga[k], Gb[k]) for k in Gb) / TOL_GRAD
    return e_loss, e_hid, e_grad


def _name_err(got, ref):
    return block_err(got.reshape(got.shape[0], -1) if got.dim() > 1 else got.view(-1, 1),
                     ref.reshape(ref.shape[0], -1) if ref.dim() > 1 else ref.view(-1, 1))


# ======================================================================================================================
# CPU: the reference
# ======================================================================================================================
_GOLDENS = [("sasrec_new_tiny.npz", "new"), ("sasrec_new_small.npz", "new"), ("sasrec_legacy_tiny.npz", "legacy"),
            ("sasrec_new_d192h4.npz", "new"), ("sasrec_new_d64h2.npz", "new"), ("sasrec_legacy_d50h1.npz", "legacy")]


@pytest.mark.parametrize("name,variant", _GOLDENS)
def test_reference_with_unit_keeps_matches_oracle_and_golden(golden_dir, name, variant):
    """With every keep mask equal to 1 the dropout restatement is oracle.sasrec.train_loss / loss_and_grads, and it
    reproduces the golden loss, hidden states and gradients of the real reference."""
    from oracle import sasrec as osr

    z = np.load(os.path.join(golden_dir, name))
    conv = osr.params_from_new_state_dict if variant == "new" else osr.params_from_legacy_state_dict
    P = conv({k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd::")})
    Gz = conv({k[6:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("grad::")})
    ids, pad, labels, tmask = (torch.from_numpy(z[k]) for k in ("ids", "pad_mask", "labels", "target_mask"))
    B, L = ids.shape
    d, H = int(z["d"]), int(z["H"])
    lnf_eps = 1e-5 if variant == "new" else 1e-8
    keeps = unit_keeps(B, L, d, H, len(P["blocks"]))
    loss, x, hid, G = ref_loss_and_grads(P, ids, pad, labels, tmask, H, variant, lnf_eps, keeps)
    P64 = osr.params_to(P, torch.float64)
    o_loss, o_G = osr.loss_and_grads(P64, ids, pad, labels, tmask, H, variant)
    torch.testing.assert_close(loss, o_loss, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(hid, osr.sasrec_body(P64, ids, pad, H, variant), rtol=1e-12, atol=1e-12)
    for (k, _), og in zip(_leaves(P), osr.flat_param_list(o_G)):
        torch.testing.assert_close(G[k], og, rtol=1e-10, atol=1e-12, msg=k)
    # the real reference (fp32) on the same inputs
    torch.testing.assert_close(loss.float(), torch.tensor(float(z["train_loss"])), rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(hid.float(), torch.from_numpy(z["train_hidden"]), rtol=2e-5, atol=2e-5)
    for (k, g_ref) in _leaves(Gz):
        torch.testing.assert_close(G[k].float(), g_ref, rtol=1e-4, atol=1e-6, msg=k)


def test_reference_dropout_is_exact_under_its_masks():
    """keep = 0 at a site removes exactly what it should: without the last block's FFN output x[-1] is LayerNorm2's
    output (each row normalised before ln2_w / ln2_b); without block 0's attention probabilities its out_w and the
    Q / K rows of in_w get no gradient.  Keep rates are 1 - p and the sites draw different masks."""
    case = _Case("new", 64, 2, L=24, I=50)
    B, L = 3, 24
    P = _map(case.params(3), lambda k, v: v.double())
    ids, pad, labels, tmask = step_batch(B, L, case.I, 4)
    keeps = engine_keeps(SEED + CTR, P_DROP, B, L, case.cfg)
    keeps["blocks"][1]["ffn2"].zero_()
    _, x, _, _ = ref_loss_and_grads(P, ids, pad, labels, tmask, 2, "new", 1e-5, keeps)
    blk = P["blocks"][1]
    xh = (x - blk["ln2_b"]) / blk["ln2_w"]
    assert float(xh.mean(-1).abs().max()) < 1e-9 and float((xh.var(-1, unbiased=False) - 1).abs().max()) < 1e-6
    keeps = engine_keeps(SEED + CTR, P_DROP, B, L, case.cfg)
    keeps["blocks"][0]["attn"].zero_()
    _, _, _, G = ref_loss_and_grads(P, ids, pad, labels, tmask, 2, "new", 1e-5, keeps)
    assert float(G["b0.out_w"].abs().max()) == 0.0 and float(G["b0.in_w"].abs().max()) == 0.0
    keeps = engine_keeps(SEED + CTR, P_DROP, 7, 200, _Case("new", 128, 2).cfg)
    for site in ("emb", "ffn1", "ffn2"):
        t = keeps[site] if site == "emb" else keeps["blocks"][1][site]
        assert abs(float((t > 0).double().mean()) - (1 - P_DROP)) < 0.01, site
    assert abs(float((keeps["blocks"][0]["attn"] > 0).double().mean()) - (1 - P_DROP)) < 0.01
    b = keeps["blocks"]
    assert not torch.equal(b[0]["ffn1"], b[0]["ffn2"]) and not torch.equal(b[0]["ffn2"], b[1]["ffn1"])
    assert not torch.equal(keeps["emb"], b[0]["ffn1"])


# ----------------------------------------------------------------------------------------------------------------------
# CPU: every plausible mistake moves what the GPU tests compare by >= 10x the tolerance
# ----------------------------------------------------------------------------------------------------------------------
_MISTAKES = {"site_off_by_one": "c2", "ffn_drop_after_residual": "c2", "no_scale": "c2", "ln_padded_width": "d64h2",
             "no_row_mask": "legacy_d50h1", "kv_from_normed": "c2", "pos_first_rows": "c2"}


@pytest.mark.parametrize("mistake", sorted(_MISTAKES))
def test_step_tolerances_discriminate_perturbed_references(mistake):
    """At the GPU step test's shape (B = 7, L = 200, I = 2000, dropout 0.2) and tolerances: a dropout site number off by
    one, the FFN-output dropout applied after the residual add, the 1/(1-p) scale missing, LayerNorm statistics over the
    padded width (d 64 in 128 columns), the legacy row mask dropped, K and V computed from the normalised x, and the new
    path's positional window taken from the first L rows (max_len 210) each move the loss, x[-1] or a gradient by >= 10x
    its tolerance."""
    case = _Case(*_CASES[_MISTAKES[mistake]])
    B, L, H = 7, case.L, case.H
    P = case.params(11)
    ids, pad, labels, tmask = step_batch(B, L, case.I, 12)
    keeps = engine_keeps(SEED + CTR, P_DROP, B, L, case.cfg)
    args = (ids, pad, labels, tmask, H, case.variant, case.lnf_eps)
    ref = ref_loss_and_grads(P, *args, keeps)
    if mistake == "site_off_by_one":
        bad = ref_loss_and_grads(P, *args, engine_keeps(SEED + CTR, P_DROP, B, L, case.cfg, site_shift=1))
    elif mistake == "no_scale":
        unscaled = {"emb": (keeps["emb"] > 0).double(),
                    "blocks": [{k: (v > 0).double() for k, v in blk.items()} for blk in keeps["blocks"]]}
        bad = ref_loss_and_grads(P, *args, unscaled)
    else:
        bad = ref_loss_and_grads(P, *args, keeps, mistake=mistake, dp=case.cfg.dp)
    errs = _model_errs(bad, ref, pad)
    print(mistake, "loss / x[-1] / grad error in tolerances:", [round(e, 1) for e in errs])
    assert max(errs) >= 10, errs


# ======================================================================================================================
# kernel-level inputs and references (float64, in the padded layout the kernels see)
# ======================================================================================================================
def _row_scales(T, g):
    """Per-row (scale, offset): 70 % at unit scale (0.3 .. 3), 15 % with a common offset of up to 50x the row's spread,
    15 % at 1e-4 .. 1e-3 (the LayerNorm eps 1e-8 is comparable to their variance)."""
    u = torch.rand(T, 1, generator=g)
    scale = torch.exp(torch.empty(T, 1).uniform_(math.log(0.3), math.log(3.0), generator=g))
    small = torch.exp(torch.empty(T, 1).uniform_(math.log(1e-4), math.log(1e-3), generator=g))
    offset = torch.empty(T, 1).uniform_(-50.0, 50.0, generator=g)
    is_off, is_small = (u >= 0.7) & (u < 0.85), u >= 0.85
    return torch.where(is_small, small, scale), torch.where(is_off, offset, torch.zeros_like(offset)), is_small


def _weights(n_out, n_in, v_out, v_in, g, scale=1.0):
    """bf16 [n_out, n_in] with zero padded rows / columns (the padded layout's invariant)."""
    w = torch.randn(n_out, n_in, generator=g) * scale / math.sqrt(float(v_in.sum()))
    return _bf(w * v_out[:, None] * v_in[None, :])


def _vec(n, v, g, scale, base=0.0):
    return ((base + scale * torch.randn(n, generator=g)) * v).float()


def _dev(ts, dev):
    return [t.to(dev) if t is not None else None for t in ts]


def _sent(rows, cols, dev, dtype=torch.bfloat16):
    return torch.full((rows + 64, cols), SENT, dtype=dtype, device=dev) if cols else \
        torch.full((rows + 64,), SENT, dtype=dtype, device=dev)


def _untouched(buf, T, what):
    assert (buf[T:] == SENT).all(), f"{what} written past row T"


def _ln_fwd_atol(x, mean, rstd, w):
    """fp32 slack of y = (x - mean) * rstd * w + b: a few ulps of the fp32 terms."""
    return 4e-7 * ((x.abs() + mean.abs()[:, None]) * rstd[:, None] * w.abs() + 1.0) + 1e-30


def _check_stats(mean, rstd, m_ref, r_ref, x, valid):
    rms = (x.double() * valid.to(x.device)).square().sum(-1).div(float(valid.sum())).sqrt().clamp_min(1e-30)
    assert _note("fused ln mean", ((mean.double() - m_ref).abs() / rms).max()) < TOL_MEAN
    assert _note("fused ln rstd", ((rstd.double() - r_ref).abs() / r_ref).max()) < TOL_RSTD


def _assert_keep_pattern(out, keep, exact, slack, what):
    """Dropped elements are exactly zero, bit for bit against the ported mask; kept ones are non-zero unless their exact
    value is within the accumulation slack of zero."""
    nz = out != 0
    leak = int((nz & ~keep).sum())
    assert leak == 0, f"{what}: {leak} dropped elements are not zero"
    bad = int(((exact.abs() > slack) & keep & ~nz).sum())
    assert bad == 0, f"{what}: {bad} kept elements are zero"


def _post_attn_inputs(T, d, hdv, seed, dev):
    """O, q_in (bf16 [T, d]) and the block's weights for the part after the attention.  h = O Wo^T + bo + q_in gets the
    row mix of _row_scales: offset rows through q_in, small rows by scaling O and cancelling bo in q_in."""
    g = _gen(seed)
    v = feat_mask(d, hdv)
    scale, offset, small = _row_scales(T, g)
    Wo, W1, W2 = (_weights(d, d, v, v, g) for _ in range(3))
    bo, b1, b2 = _vec(d, v, g, 0.1), _vec(d, v, g, 0.3), _vec(d, v, g, 0.1)
    lw, lb = _vec(d, v, g, 0.2, 1.0), _vec(d, v, g, 0.1)
    O = _bf(torch.randn(T, d, generator=g) * 0.7 * scale * v)
    q = (torch.randn(T, d, generator=g) * 0.7 + offset) * scale - torch.where(small, bo[None, :], torch.zeros(1, d))
    q_in = _bf(q * v)
    return _dev([O, q_in, Wo, bo, lw, lb, W1, b1, W2, b2], dev) + [v.to(dev)]


def _x_rows(T, d, hdv, seed, dev):
    g = _gen(seed)
    v = feat_mask(d, hdv)
    scale, offset, _ = _row_scales(T, g)
    return _bf((torch.randn(T, d, generator=g) + offset) * scale * v).to(dev), v.to(dev), g


def post_attn_train_ref(O, q_in, Wo, bo, lw, lb, W1, b1, W2, b2, valid, keep1, keep2, rm, ks, got=None, mistake=None):
    """Step by step fp64 reference of rp_post_attn_train.  Each stage starts from the kernel's own bf16 output of the
    stage before (``got`` = dict h, y, u), or from the rounded reference when ``got`` is None; returns {name: (ref, atol)}
    plus the statistics.  ``mistake``: 'h_fp32_stats' (LayerNorm of the unrounded h), 'site1_off2' (keep2 at site 1)."""
    D = lambda t: t.double()  # noqa: E731
    r = {}
    h = D(O) @ D(Wo).T + D(bo) + D(q_in)
    r["h"] = (h, HALF_ULP_SLACK * (D(O).abs() @ D(Wo).abs().T + D(bo).abs() + D(q_in).abs()) + 1e-30)
    h_k = D(got["h"]) if got else D(_bf(h))
    y, mean, rstd = ln_ref(h if mistake == "h_fp32_stats" else h_k, D(lw), D(lb), EPS, valid)
    r["y"] = (y, _ln_fwd_atol(h_k, mean, rstd, D(lw)))
    y_k = D(got["y"]) if got else D(_bf(y))
    pre1 = y_k @ D(W1).T + D(b1)
    k1 = keep2 if mistake == "site1_off2" else keep1
    r["u"] = (torch.relu(pre1) * D(k1) * ks, ks * HALF_ULP_SLACK * (y_k.abs() @ D(W1).abs().T + D(b1).abs()) + 1e-30)
    r["u_exact"] = torch.relu(pre1) * ks
    u_k = D(got["u"]) if got else D(_bf(r["u"][0]))
    pre2 = u_k @ D(W2).T + D(b2)
    out = (y_k + pre2 * D(keep2) * ks) * D(rm)[:, None]
    r["out"] = (out, ks * HALF_ULP_SLACK * (u_k.abs() @ D(W2).abs().T + D(b2).abs()) + 2e-7 * y_k.abs() + 1e-30)
    return r, mean, rstd


def _post_attn_keeps(T, d, drop, seed_eff, dev, off1, off2):
    if drop == 0:
        one = torch.ones(T, d, dtype=torch.bool, device=dev)
        return one, one
    rows = np.arange(T)
    return (keep_draws(seed_eff, off1, drop, rows, d).to(dev), keep_draws(seed_eff, off2, drop, rows, d).to(dev))


@pytest.mark.parametrize("mistake", ["h_fp32_stats", "site1_off2"])
def test_post_attn_tolerance_discriminates_mistakes(mistake):
    """At the kernel test's inputs (T = 1400, d = 128, rows with a large common offset) and element-wise tolerance:
    LayerNorm statistics of the fp32 h instead of the bf16 h the kernel saves move y, and site 1 drawn with site 2's
    offset moves u, by >= 10x TOL_ULP."""
    T, d = 1400, 128
    O, q_in, Wo, bo, lw, lb, W1, b1, W2, b2, v = _post_attn_inputs(T, d, 0, 5, None)
    off1, off2 = _site(1, 1) << 40, _site(1, 2) << 40
    k1, k2 = _post_attn_keeps(T, d, P_DROP, SEED + CTR, None, off1, off2)
    rm = torch.ones(T, dtype=torch.uint8)
    args = (O, q_in, Wo, bo, lw, lb, W1, b1, W2, b2, v, k1, k2, rm, _ks(P_DROP))
    ref, _, _ = post_attn_train_ref(*args)
    bad, _, _ = post_attn_train_ref(*args, mistake=mistake)
    key = "y" if mistake == "h_fp32_stats" else "u"
    e = ulp_err(_bf(bad[key][0]).double(), ref[key][0], ref[key][1])
    print(mistake, f"{key} error in TOL_ULP:", round(e / TOL_ULP, 1))
    assert e >= 10 * TOL_ULP


# ======================================================================================================================
# GPU 1: rp_ln_qkv_fused (full and K | V-only) and rp_pre_attn_bwd fed from its statistics
# ======================================================================================================================
_PRE_SHAPES = [(1, 128, 0), (129, 64, 0), (1400, 128, 0), (1400, 64, 50), (1400, 128, 32), (1400, 128, 48),
               (102400, 128, 0), (102363, 64, 0), (102363, 128, 48)]


def _ln_qkv(x, lw, lb, w_in, b_in, T, d, q_in, Q, KV, mean, rstd, hdv):
    p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    check(lib().rp_ln_qkv_fused(x.data_ptr(), p(lw), p(lb), EPS, w_in.data_ptr(), b_in.data_ptr(), T, d, p(q_in), p(Q),
                                KV.data_ptr(), p(mean), p(rstd), hdv, _stream()), "rp_ln_qkv_fused")


@pytest.mark.gpu
@pytest.mark.parametrize("T,d,hdv", _PRE_SHAPES)
def test_ln_qkv_fused_and_pre_attn_bwd(cuda, T, d, hdv):
    """rp_ln_qkv_fused: q_in = LN1(x) over the real features, Q = q_in Wq^T + bq from the bf16 q_in, [K | V] = x Wkv^T +
    bkv, mean / rstd - element-wise against fp64; with NULL statistics pointers the outputs are bit-identical; the K | V-
    only mode (q_in = Q = NULL, predict's final block) writes the same KV and nothing else.  rp_pre_attn_bwd, fed with the
    forward's own statistics: dx = [dK | dV] Wkv + LN1-backward(dQ Wq + dh), dln_w / dln_b accumulated onto preset values,
    padded inputs get exactly zero gradient."""
    x, v, g = _x_rows(T, d, hdv, T + d + hdv, cuda)
    vc = v.cpu()
    v3 = torch.cat([vc] * 3)
    w_in = _weights(3 * d, d, v3, vc, g).to(cuda)
    b_in = _vec(3 * d, v3, g, 0.1).to(cuda)
    lw, lb = _vec(d, vc, g, 0.2, 1.0).to(cuda), _vec(d, vc, g, 0.1).to(cuda)
    q_in, Q, KV = _sent(T, d, cuda), _sent(T, d, cuda), _sent(T, 2 * d, cuda)
    mean, rstd = _sent(T, 0, cuda, torch.float32), _sent(T, 0, cuda, torch.float32)
    _ln_qkv(x, lw, lb, w_in, b_in, T, d, q_in, Q, KV, mean, rstd, hdv)
    torch.cuda.synchronize()
    for buf, what in ((q_in, "q_in"), (Q, "Q"), (KV, "KV"), (mean, "mean"), (rstd, "rstd")):
        _untouched(buf, T, what)
    X, W, Bv = x.double(), w_in.double(), b_in.double()
    y_ref, m_ref, r_ref = ln_ref(X, lw.double(), lb.double(), EPS, v)
    assert (q_in[:T][:, ~v] == 0).all(), "padded features of q_in must be 0"
    assert _note("ln_qkv q_in ulp", ulp_err(q_in[:T], y_ref, _ln_fwd_atol(X, m_ref, r_ref, lw.double()))) < TOL_ULP
    _check_stats(mean[:T], rstd[:T], m_ref, r_ref, x, v)
    q16 = q_in[:T].double()
    Q_ref = q16 @ W[:d].T + Bv[:d]
    assert _note("ln_qkv Q ulp", ulp_err(Q[:T], Q_ref, HALF_ULP_SLACK * (q16.abs() @ W[:d].abs().T + Bv[:d].abs()) + 1e-30)) < TOL_ULP
    KV_ref = X @ W[d:].T + Bv[d:]
    KV_atol = HALF_ULP_SLACK * (X.abs() @ W[d:].abs().T + Bv[d:].abs()) + 1e-30
    assert _note("ln_qkv KV ulp", ulp_err(KV[:T], KV_ref, KV_atol)) < TOL_ULP
    # no statistics: the same outputs
    q2, Q2, KV2 = _sent(T, d, cuda), _sent(T, d, cuda), _sent(T, 2 * d, cuda)
    _ln_qkv(x, lw, lb, w_in, b_in, T, d, q2, Q2, KV2, None, None, hdv)
    torch.cuda.synchronize()
    assert torch.equal(q2, q_in) and torch.equal(Q2, Q) and torch.equal(KV2, KV)
    # K | V only
    KV3 = _sent(T, 2 * d, cuda)
    _ln_qkv(x, None, None, w_in, b_in, T, d, None, None, KV3, None, None, hdv)
    torch.cuda.synchronize()
    assert torch.equal(KV3, KV), "the K | V-only mode must write the full mode's KV"

    # ---- rp_pre_attn_bwd from the forward's own statistics
    gb = _gen(T * 3 + d)
    dQ = _bf(torch.randn(T, d, generator=gb) * 0.3 * vc).to(cuda)
    dKV = _bf(torch.randn(T, 2 * d, generator=gb) * 0.3 * torch.cat([vc, vc])).to(cuda)
    dh = _bf(torch.randn(T, d, generator=gb) * 0.3 * vc).to(cuda)
    dw0, db0 = torch.randn(d, generator=gb).to(cuda), torch.randn(d, generator=gb).to(cuda)
    dw, db = dw0.clone(), db0.clone()
    dx = _sent(T, d, cuda)
    check(lib().rp_pre_attn_bwd(dQ.data_ptr(), dKV.data_ptr(), dh.data_ptr(), x.data_ptr(), mean.data_ptr(),
                                rstd.data_ptr(), lw.data_ptr(), w_in.data_ptr(), T, d, dx.data_ptr(), dw.data_ptr(),
                                db.data_ptr(), hdv, _stream()), "rp_pre_attn_bwd")
    torch.cuda.synchronize()
    _untouched(dx, T, "dx")
    dq = dQ.double() @ W[:d] + dh.double()
    t, dw_ref, db_ref = ln_bwd_ref(dq, X, lw.double(), m_ref, r_ref, v)
    dx_ref = dKV.double() @ W[d:] + t
    assert (dx[:T][:, ~v] == 0).all(), "padded inputs must get exactly zero gradient"
    assert _note("pre_attn_bwd dx block", block_err(dx[:T], dx_ref)) < TOL_BWD
    assert _note("pre_attn_bwd dln_w", block_err((dw - dw0).double().view(-1, 1), dw_ref.view(-1, 1))) < TOL_LN_GRAD
    assert _note("pre_attn_bwd dln_b", block_err((db - db0).double().view(-1, 1), db_ref.view(-1, 1))) < TOL_LN_GRAD
    assert torch.equal(dw[~v], dw0[~v]) and torch.equal(db[~v], db0[~v])


# ======================================================================================================================
# GPU 2: rp_post_attn_train and rp_post_attn_bwd fed from its saved activations (a round trip)
# ======================================================================================================================
_POST_CASES = [(1, 128, 0, P_DROP, True), (129, 64, 0, P_DROP, False), (1400, 128, 0, P_DROP, True),
               (1400, 128, 0, 0.0, False), (1400, 64, 50, P_DROP, True), (1400, 128, 32, 0.0, True),
               (1400, 128, 48, P_DROP, False), (102400, 128, 0, P_DROP, False), (102363, 128, 0, P_DROP, True),
               (102363, 64, 0, 0.0, False), (102400, 64, 50, P_DROP, True)]


def _rowmask(T, masked, seed, dev):
    if not masked:
        return None
    return (torch.rand(T, generator=_gen(seed)) > 0.3).to(torch.uint8).to(dev)


def post_attn_bwd_ref(dz, h_k, u_k, lw, lb, W1, W2, Wo, b1, b2, valid, keep2, rm, ks):
    """fp64 autograd of the forward formula z = (y + drop2(drop1(relu(y W1^T + b1)) W2^T + b2)) * rm, y = LN2(h), under
    the kernel's masks (site 1 and the ReLU from the zeros of the saved u): d_t, du, dh, d_o = dh Wo, dln_w, dln_b."""
    D = lambda t: t.double()  # noqa: E731
    h = D(h_k).requires_grad_(True)
    w, b = D(lw).requires_grad_(True), D(lb).requires_grad_(True)
    y = ln_ref(h, w, b, EPS, valid)[0]
    pre1 = y @ D(W1).T + D(b1)
    pre1.retain_grad()
    u = pre1 * (u_k != 0).double() * ks
    pre2 = u @ D(W2).T + D(b2)
    pre2.retain_grad()
    z = (y + pre2 * D(keep2) * ks) * D(rm)[:, None]
    z.backward(D(dz))
    return pre2.grad, pre1.grad, h.grad, h.grad @ D(Wo), w.grad, b.grad


@pytest.mark.gpu
@pytest.mark.parametrize("T,d,hdv,drop,masked", _POST_CASES)
def test_post_attn_train_and_bwd(cuda, T, d, hdv, drop, masked):
    """rp_post_attn_train: h = O Wo^T + bo + q_in rounded to bf16, y = LN2(h) over the real features of that bf16 h,
    u = drop1(relu(y W1^T + b1)), out = (y + drop2(u W2^T + b2)) * rowmask; saved h, y, u, mean, rstd and out element-wise
    against fp64; u's zeros are the ported site-1 mask (and the ReLU), out equals y bit for bit where site 2 dropped, rows
    with row mask 0 are exactly 0.  rp_post_attn_bwd on the kernel's own h, u, mean and rstd: d_t, du, dh, d_o per 64-row
    block against fp64 autograd under the same masks, dln_w / dln_b accumulated onto preset values, padded columns of dh
    and d_o exactly 0, and d_t = NULL when there is neither dropout nor a row mask."""
    O, q_in, Wo, bo, lw, lb, W1, b1, W2, b2, v = _post_attn_inputs(T, d, hdv, T + d + hdv + int(masked), cuda)
    rm = _rowmask(T, masked, T + 1, cuda)
    rm1 = rm if rm is not None else torch.ones(T, dtype=torch.uint8, device=cuda)
    ctr = torch.tensor([CTR], dtype=torch.int64, device=cuda)
    off1, off2 = _site(1, 1) << 40, _site(1, 2) << 40
    ks = _ks(drop) if drop > 0 else 1.0
    k1, k2 = _post_attn_keeps(T, d, drop, SEED + CTR, cuda, off1, off2)
    bufs = {k: _sent(T, d, cuda) for k in ("h", "y", "u", "out")}
    mean, rstd = _sent(T, 0, cuda, torch.float32), _sent(T, 0, cuda, torch.float32)
    ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    check(lib().rp_post_attn_train(O.data_ptr(), q_in.data_ptr(), Wo.data_ptr(), bo.data_ptr(), lw.data_ptr(), lb.data_ptr(),
                                   EPS, W1.data_ptr(), b1.data_ptr(), W2.data_ptr(), b2.data_ptr(), ptr(rm), T, d, drop, SEED,
                                   off1, off2, ctr.data_ptr(), bufs["h"].data_ptr(), bufs["y"].data_ptr(),
                                   bufs["u"].data_ptr(), mean.data_ptr(), rstd.data_ptr(), bufs["out"].data_ptr(), hdv,
                                   _stream()), "rp_post_attn_train")
    torch.cuda.synchronize()
    for k, b in list(bufs.items()) + [("mean", mean), ("rstd", rstd)]:
        _untouched(b, T, k)
    got = {k: b[:T] for k, b in bufs.items()}
    ref, m_ref, r_ref = post_attn_train_ref(O, q_in, Wo, bo, lw, lb, W1, b1, W2, b2, v, k1, k2, rm1, ks, got=got)
    for k in ("h", "y", "u", "out"):
        assert (got[k][:, ~v] == 0).all(), f"padded features of {k} must be 0"
    assert _note("post_attn h ulp", ulp_err(got["h"], *ref["h"])) < TOL_ULP
    assert _note("post_attn y ulp", ulp_err(got["y"], *ref["y"])) < TOL_ULP
    _check_stats(mean[:T], rstd[:T], m_ref, r_ref, got["h"], v)
    _assert_keep_pattern(got["u"][:, v], k1[:, v], ref["u_exact"][:, v], ref["u"][1][:, v], "u (site 1)")
    assert _note("post_attn u ulp", ulp_err(got["u"], *ref["u"])) < TOL_ULP
    assert _note("post_attn out ulp", ulp_err(got["out"], *ref["out"])) < TOL_ULP
    on = rm1.bool()
    assert (got["out"][~on] == 0).all(), "rows with row mask 0 must be exactly 0"
    dropped = ~k2 & on[:, None] & v[None, :]
    assert torch.equal(got["out"][dropped], got["y"][dropped]), "where site 2 dropped, out must be y"

    # ---- rp_post_attn_bwd from the saved activations
    gb = _gen(T * 7 + d)
    dz = _bf(torch.randn(T, d, generator=gb) * 0.5 * v.cpu()).to(cuda)
    dz = torch.where((dz == 0) & v, torch.full_like(dz, 0.25), dz)      # never exactly zero on the real features
    dw0, db0 = torch.randn(d, generator=gb).to(cuda), torch.randn(d, generator=gb).to(cuda)
    masked_t = drop > 0 or masked
    for with_dt in ([True] if masked_t else [True, False]):
        o = {k: _sent(T, d, cuda) for k in ("d_t", "du", "dh", "d_o")}
        dw, db = dw0.clone(), db0.clone()
        check(lib().rp_post_attn_bwd(dz.data_ptr(), bufs["u"].data_ptr(), bufs["h"].data_ptr(), mean.data_ptr(),
                                     rstd.data_ptr(), lw.data_ptr(), W2.data_ptr(), W1.data_ptr(), Wo.data_ptr(), ptr(rm), T, d,
                                     drop, SEED, off2, ctr.data_ptr(), o["d_t"].data_ptr() if with_dt else None,
                                     o["du"].data_ptr(), o["dh"].data_ptr(), o["d_o"].data_ptr(), dw.data_ptr(),
                                     db.data_ptr(), hdv, _stream()), "rp_post_attn_bwd")
        torch.cuda.synchronize()
        for k, b in o.items():
            if with_dt or k != "d_t":
                _untouched(b, T, k)
        if not with_dt:
            assert (o["d_t"] == SENT).all()
            assert torch.equal(o["du"], first["du"]) and torch.equal(o["dh"], first["dh"]) and torch.equal(o["d_o"], first["d_o"])
            # dln_w / dln_b add one fp32 atomic per column and CTA: the order, and so the last bits, may differ
            assert _note("post_attn_bwd dln_w", block_err((dw - dw0).double().view(-1, 1), first["r_dw"])) < TOL_LN_GRAD
            assert _note("post_attn_bwd dln_b", block_err((db - db0).double().view(-1, 1), first["r_db"])) < TOL_LN_GRAD
            continue
        r_dt, r_du, r_dh, r_do, r_dw, r_db = post_attn_bwd_ref(dz, got["h"], got["u"], lw, lb, W1, W2, Wo, b1, b2, v, k2, rm1, ks)
        assert torch.equal(o["d_t"][:T] != 0, (k2 & on[:, None] & v[None, :])), "d_t's zeros must be site 2's mask and the row mask"
        assert _note("post_attn_bwd d_t block", block_err(o["d_t"][:T], r_dt)) < TOL_BWD
        assert _note("post_attn_bwd du block", block_err(o["du"][:T], r_du)) < TOL_BWD
        assert _note("post_attn_bwd dh block", block_err(o["dh"][:T], r_dh)) < TOL_BWD
        assert _note("post_attn_bwd d_o block", block_err(o["d_o"][:T], r_do)) < TOL_BWD
        assert (o["dh"][:T][:, ~v] == 0).all() and (o["d_o"][:T][:, ~v] == 0).all(), "padded columns of dh / d_o must be 0"
        assert _note("post_attn_bwd dln_w", block_err((dw - dw0).double().view(-1, 1), r_dw.view(-1, 1))) < TOL_LN_GRAD
        assert _note("post_attn_bwd dln_b", block_err((db - db0).double().view(-1, 1), r_db.view(-1, 1))) < TOL_LN_GRAD
        assert torch.equal(dw[~v], dw0[~v]) and torch.equal(db[~v], db0[~v])
        first = {"du": o["du"], "dh": o["dh"], "d_o": o["d_o"], "r_dw": r_dw.view(-1, 1), "r_db": r_db.view(-1, 1)}


# ======================================================================================================================
# GPU 3: the eval kernel rp_post_attn_fused
# ======================================================================================================================
_EVAL_CASES = [(1, 128, 0, True), (129, 64, 0, False), (1400, 128, 0, True), (1400, 64, 50, True), (1400, 128, 32, False),
               (1400, 128, 48, True), (102400, 128, 0, False), (102363, 64, 0, True), (102363, 128, 48, False)]


def _eval_atol(y, u, W1, W2, S2):
    """Slack of out = y + u W2^T + b2 when y and u are rounded to bf16 inside the kernel: the fp32 accumulation, one
    rounding flip of the residual y, and one flip of u (directly, and through y's flip into the FFN) per row."""
    ulp = lambda t: torch.exp2(torch.floor(torch.log2(t.abs().clamp_min(1e-300))) - 7)  # noqa: E731
    w2max = W2.double().abs().amax(-1)[None, :]
    u_flip = ulp(u).amax(-1, keepdim=True) + ulp(y).amax(-1, keepdim=True) * W1.double().abs().max()
    return HALF_ULP_SLACK * S2 + ulp(y) + u_flip * w2max + 1e-30


@pytest.mark.gpu
@pytest.mark.parametrize("T,d,hdv,masked", _EVAL_CASES)
def test_post_attn_fused(cuda, T, d, hdv, masked):
    """rp_post_attn_fused (predict: h = O Wo^T + bo + q_in in fp32, y = LN2(h) over the real features, out = (y +
    relu(y W1^T + b1) W2^T + b2) * rowmask) element-wise against fp64 with the internal bf16 roundings of y and u allowed
    one flip; rows with row mask 0 exactly 0; nothing written past T."""
    O, q_in, Wo, bo, lw, lb, W1, b1, W2, b2, v = _post_attn_inputs(T, d, hdv, T + d + hdv + 17, cuda)
    rm = _rowmask(T, masked, T + 2, cuda)
    on = (rm if rm is not None else torch.ones(T, dtype=torch.uint8, device=cuda)).bool()
    ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    out = _sent(T, d, cuda)
    check(lib().rp_post_attn_fused(O.data_ptr(), q_in.data_ptr(), Wo.data_ptr(), bo.data_ptr(), lw.data_ptr(), lb.data_ptr(),
                                   EPS, W1.data_ptr(), b1.data_ptr(), W2.data_ptr(), b2.data_ptr(), ptr(rm), T, d,
                                   out.data_ptr(), hdv, _stream()), "rp_post_attn_fused")
    torch.cuda.synchronize()
    _untouched(out, T, "out")
    Dd = lambda t: t.double()  # noqa: E731
    h = Dd(O) @ Dd(Wo).T + Dd(bo) + Dd(q_in)
    y = ln_ref(h, Dd(lw), Dd(lb), EPS, v)[0]
    yb = Dd(_bf(y))
    u = torch.relu(yb @ Dd(W1).T + Dd(b1))
    ub = Dd(_bf(u))
    ref = (yb + ub @ Dd(W2).T + Dd(b2)) * on[:, None]
    S2 = ub.abs() @ Dd(W2).abs().T + Dd(b2).abs() + yb.abs()
    assert (out[:T][~on] == 0).all(), "rows with row mask 0 must be exactly 0"
    assert (out[:T][:, ~v] == 0).all(), "padded features must be 0"
    assert _note("post_attn_fused out ulp", ulp_err(out[:T], ref, _eval_atol(y, u, W1, W2, S2))) < TOL_ULP_EVAL


# ======================================================================================================================
# GPU 4: rp_wgrad_group on one block's five pairs
# ======================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 65, 102400])
def test_wgrad_group_block_pairs(cuda, T):
    """rp_wgrad_group as SasRecEngine._wgrad_group runs it at d = 128: (d_t, u) -> w2 / b2, (du, y) -> w1 / b1, (dh, O) ->
    out_w / out_b, (dQ, q_in) -> in_w[:d] / in_b[:d], (dKV 2d wide, x) -> in_w[d:] / in_b[d:], accumulated onto preset
    values (T = 1 and 65 give more splits than token chunks); a rerun is bit-identical."""
    d = 128
    g = _gen(T + 5)
    bf = lambda n: _bf(torch.randn(T, n, generator=g) * 0.5).to(cuda)  # noqa: E731
    ops_ = [(bf(d), bf(d)) for _ in range(4)] + [(bf(2 * d), bf(d))]
    gw = {k: torch.randn(*s, generator=g).to(cuda) for k, s in
          (("w2", (d, d)), ("w1", (d, d)), ("out_w", (d, d)), ("in_w", (3 * d, d)))}
    gb = {k: torch.randn(n, generator=g).to(cuda) for k, n in (("b2", d), ("b1", d), ("out_b", d), ("in_b", 3 * d))}

    def run():
        W = {k: t.clone() for k, t in gw.items()}
        Bb = {k: t.clone() for k, t in gb.items()}
        dst = [(W["w2"], Bb["b2"]), (W["w1"], Bb["b1"]), (W["out_w"], Bb["out_b"]), (W["in_w"][:d], Bb["in_b"][:d]),
               (W["in_w"][d:], Bb["in_b"][d:])]
        arr = (WgradPair * 5)()
        for k, ((dY, X), (dW, db)) in enumerate(zip(ops_, dst)):
            arr[k].dY, arr[k].dy_ld, arr[k].n_out = dY.data_ptr(), dY.stride(0), dW.shape[0]
            arr[k].X, arr[k].x_ld, arr[k].n_in = X.data_ptr(), X.stride(0), dW.shape[1]
            arr[k].dW, arr[k].dw_ld, arr[k].db = dW.data_ptr(), dW.stride(0), db.data_ptr()
        need = lib().rp_wgrad_group_workspace(arr, 5)
        assert need > 0
        ws = torch.zeros(need, device=cuda, dtype=torch.uint8)
        check(lib().rp_wgrad_group(arr, 5, T, 1, ws.data_ptr(), need, _stream()), "rp_wgrad_group")
        torch.cuda.synchronize()
        return dst

    dst = run()
    pre_w = [gw["w2"], gw["w1"], gw["out_w"], gw["in_w"][:d], gw["in_w"][d:]]
    pre_b = [gb["b2"], gb["b1"], gb["out_b"], gb["in_b"][:d], gb["in_b"][d:]]
    for (dY, X), (dW, db), w0, b0 in zip(ops_, dst, pre_w, pre_b):
        ref = dY.double().T @ X.double()
        assert _note("wgrad_group dW block", block_err(dW.double() - w0.double(), ref)) < TOL_SPLITK
        rb = dY.double().sum(0)
        assert _note("wgrad_group db", block_err((db.double() - b0.double()).view(-1, 1), rb.view(-1, 1))) < TOL_SUM
    again = run()
    for (a, b), (c, e) in zip(dst, again):
        assert torch.equal(a, c) and torch.equal(b, e), "rp_wgrad_group reruns must be bit-identical"


# ======================================================================================================================
# GPU 5: the SASRec training step against the fp64 reference
# ======================================================================================================================
def _run_step(case, B, drop, cuda, monkeypatch, seed):
    from replay_b200.engine import EncoderConfig, SasRecEngine

    monkeypatch.setenv("RP_FUSED_BODY", "1" if case.fused else "0")
    cfg = EncoderConfig(n_items=case.I, d=case.d, n_heads=case.H, n_blocks=2, max_len=case.max_len, dropout=drop,
                        variant=case.variant)
    P = case.params(seed)
    ids, pad, labels, tmask = step_batch(B, case.L, case.I, seed + 1)
    eng = SasRecEngine(cfg, B, case.L, cuda, seed=SEED)
    assert eng.fused_post_attn_train == case.fused
    eng.load_canonical(P)
    if drop > 0:
        eng.tick_rng()
    ctr = int(eng.rng_counter.item())
    assert (ctr != 0) == (drop > 0)
    eng.set_batch(ids.to(cuda), pad.to(cuda), labels.to(cuda), tmask.to(cuda))
    loss = float(eng.forward_train()[0])
    torch.cuda.synchronize()
    x = eng.unpad_features(eng.x[-1]).view(B, case.L, case.d).double()
    eng.g32.zero_()
    eng.backward()
    torch.cuda.synchronize()
    G = {k: v for k, v in _leaves(eng.export_canonical(eng.grads))}
    Pe = _map(P, lambda k, v: v.to(cuda))
    keeps = engine_keeps(eng.seed + ctr, drop, B, case.L, cfg, dev=cuda) if drop > 0 else None
    ref = ref_loss_and_grads(Pe, ids.to(cuda), pad.to(cuda), labels.to(cuda), tmask.to(cuda), case.H, case.variant,
                             case.lnf_eps, keeps)
    return loss, x, G, ref, pad.to(cuda)


def _check_step(case, loss, x, G, ref, pad, tag=""):
    r_loss, r_x, _, r_G = ref
    d = case.d
    assert _note(f"step loss rel{tag}", abs(loss - float(r_loss)) / float(r_loss)) < TOL_LOSS
    assert _note(f"step x[-1] block{tag}", seq_block_err(x, r_x, pad)) < TOL_HID
    bad = []
    for name, g in G.items():
        g, r = g.to(r_x.device).double(), r_G[name]
        if name.endswith("in_b"):
            # a key bias cannot change a softmax: the exact gradient of in_b's key third is 0, the kernels' is round-off
            assert float(r[d:2 * d].norm()) < 1e-9 * float(r.norm())
            assert _note("step grad in_b key third", g[d:2 * d].norm() / r.norm()) < TOL_GRAD, name
            g, r = torch.cat([g[:d], g[2 * d:]]), torch.cat([r[:d], r[2 * d:]])
        e = _note(f"step grad {name.split('.')[-1]}{tag}", _name_err(g, r))
        if e >= TOL_GRAD:
            bad.append((name, round(e, 4)))
    assert not bad, bad


@pytest.mark.gpu
@pytest.mark.parametrize("drop", [0.0, P_DROP])
@pytest.mark.parametrize("name", list(_CASES))
def test_sasrec_step_matches_fp64_reference(cuda, monkeypatch, name, drop):
    """SasRecEngine with two blocks at L = 200, B = 7 left-padded histories (lengths 200, 200, 150, 57, 13, 1, 120),
    I = 2000, the new path with max_len 210 (offset positional window), the dropout counter ticked once: config 2 on the
    fused body and on the launch-per-GEMM body (RP_FUSED_BODY=0), d 64 / 2 heads in 128 columns, the legacy d 50 / 1
    head (row mask, causal-only attention) and d 192 / 4 heads in 256 columns.  Loss, x[-1] of the real rows and every
    parameter gradient against the fp64 reference under the ported masks."""
    case = _Case(*_CASES[name])
    loss, x, G, ref, pad = _run_step(case, 7, drop, cuda, monkeypatch, seed=case.d + case.H)
    _check_step(case, loss, x, G, ref, pad)


@pytest.mark.gpu
def test_c2_full_batch_step_matches_fp64_reference(cuda, monkeypatch):
    """Config 2 at the bench's batch: B = 512 (T = 102 400), dropout 0.2, I = 2000; the reference in float64 on the GPU."""
    case = _Case(*_CASES["c2"])
    loss, x, G, ref, pad = _run_step(case, 512, P_DROP, cuda, monkeypatch, seed=77)
    _check_step(case, loss, x, G, ref, pad, tag=" B512")
