"""BERT4Rec's training step and the un-fused transformer-body kernels it runs on (rp_gemm's epilogue features and split-K,
LayerNorm, the two embeddings, column sums, row gather / scatter, dropout backward, batch preparation), each against a
float64 reference computed from the same bf16 inputs, at the config-3 shape (L = 200, d = 256, 4d = 1024 FFN columns,
dropout 0.1) and at the edges where these kernels change behaviour.

Kernels are called through the C ABI with the argument patterns of engine_bert.py / engine.py.  Dropout masks come from
the Python port of rp_philox.cuh (tests/dropout_stream.py) and are compared with the kernels' zero patterns bit for bit,
on inputs that are never exactly zero; the values are then compared against a tolerance:
- an element-wise one in units of half a bf16 ulp of the reference (what rounding the fp32 result to bf16 costs), plus an
  absolute slack for the fp32 accumulation and the fp32 erf / exp, for outputs that are one rounding away from the exact
  value;
- a per-64-row-block norm-relative one for reductions and for the whole training step, so that one wrong block cannot
  hide in a global norm.
Run with -s to print the worst error of each family.
"""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from dropout_stream import drop_keep, keep_draws
from fp64_checks import WorstErrors, block_err, feat_mask, ln_bwd_ref, ln_ref, seq_block_err, ulp_err
from replay_b200._lib import check, lib

SENT = -3.25                       # sentinel for memory a kernel must not write (exact in bf16)
SEED, CTR = 0x5EED1234ABC, 987654321   # dropout stream of the kernel-level tests (seed_ptr holds CTR)
P_DROP = 0.1                       # config 3
HALF_ULP_SLACK = 2.0 ** -21        # fp32 accumulation slack, times sum_k |a_k b_k|

# Tolerances.  Each bound is about 3x the worst error observed over every case of this file on one H100 80GB HBM3
# (400 W power limit); the element-wise ones are in units of half a bf16 ulp, where rounding to nearest alone gives 1.
TOL_ULP = 3.0            # GEMM epilogue outputs, LayerNorm y, embeddings: element-wise; worst seen 1.0
TOL_SPLITK = 2e-5        # split-K weight gradients: per 64-row block norm-relative; worst seen 6.3e-6 (K = 51 200)
TOL_SUM = 1.8e-6         # fp32 sums (colsum, LayerNorm dw / db, embedding backward): norm-relative; worst seen 6.0e-7
TOL_LN_DX = 6e-3         # LayerNorm dx (bf16): per 64-row block norm-relative; worst seen 1.9e-3
TOL_LN_STAT = 5e-7       # LayerNorm mean (relative to the row's RMS) and rstd (relative); worst seen 1.7e-7
TOL_LOSS = 2e-4          # BERT4Rec step: relative loss error; worst seen 6.1e-5
TOL_HID = 1.6e-2         # BERT4Rec step: hidden states, per (sequence, 64-row block); worst seen 5.3e-3
TOL_GRAD = 5e-2          # BERT4Rec step: parameter gradients, per 64-row block; worst seen 1.6e-2 (in_b)
TOL_LAST = 1.6e-2        # forward_last_hidden: per-row norm-relative; worst seen 5.2e-3


def _ru(x, m):
    return (x + m - 1) // m * m


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


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _bf(x):
    return x.to(torch.bfloat16)


def _ks(p):
    return 1.0 / (1.0 - float(np.float32(p)))


# ----------------------------------------------------------------------------------------------------------------------
# float64 references: GELU
# ----------------------------------------------------------------------------------------------------------------------
_C_TANH = math.sqrt(2.0 / math.pi)


def gelu_erf(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def gelu_erf_grad(z):
    return 0.5 * (1.0 + torch.erf(z / math.sqrt(2.0))) + z * torch.exp(-0.5 * z * z) / math.sqrt(2.0 * math.pi)


def gelu_tanh(x):
    return 0.5 * x * (1.0 + torch.tanh(_C_TANH * (x + 0.044715 * x ** 3)))


def gelu_tanh_grad(x):
    t = torch.tanh(_C_TANH * (x + 0.044715 * x ** 3))
    return 0.5 * (1.0 + t) + 0.5 * x * (1.0 - t * t) * _C_TANH * (1.0 + 3 * 0.044715 * x * x)


class _GeluTanhGrad(torch.autograd.Function):
    """erf GELU forward with the tanh form's derivative (a plausible backward mistake)."""

    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return gelu_erf(x)

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        return g * gelu_tanh_grad(x)


# ----------------------------------------------------------------------------------------------------------------------
# float64 reference of the BERT4Rec training loss with every dropout site
# ----------------------------------------------------------------------------------------------------------------------
def _site(blk, k):
    """SasRecEngine._site (both engines): dropout site k of block blk (offset = site << 40; the embedding is site 0)."""
    return 1 + blk * 8 + k


def engine_keeps(seed_eff, p, B, L, d, H, n_blocks, site_shift=0, dev=None):
    """Keep masks (0 or 1/(1-p), float64) of every dropout site of Bert4RecEngine's training body: the embedding at
    offset 0; per block k = 0 attention probabilities (row key bz*Lp + i), 1 out-projection, 2 GELU output, 3 FFN output,
    4 block output, at offset _site(i, k) << 40.  ``site_shift`` moves every block site number (a plausible mistake)."""
    T, Lp, ks = B * L, _ru(L, 64), _ks(p)
    rows = np.arange(T)

    def tok(off, n):
        return (keep_draws(seed_eff, off, p, rows, n).double() * ks).view(B, L, n).to(dev)

    out = {"emb": tok(0, d), "blocks": []}
    for i in range(n_blocks):
        s = lambda k: (_site(i, k) + site_shift) << 40  # noqa: E731
        out["blocks"].append({"attn": drop_keep(seed_eff, s(0), p, B, H, L, Lp).to(dev), "out": tok(s(1), d),
                              "gelu": tok(s(2), 4 * d), "ffn": tok(s(3), d), "blk": tok(s(4), d)})
    return out


def _ln64(x, w, b, eps):
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + eps) * w + b


def bert_ref(P, ids, pad, tok, labels, H, keeps=None, mistake=None, n_items=None):
    """oracle.bert4rec.train_loss restated with a keep mask at every dropout site -> (loss, hidden [B, L, d]).
    ``mistake`` (a plausible kernel / engine error, for the tolerance checks): 'drop_before_gelu', 'post_no_scale'
    (the block-output site without 1/(1-p)), 'no_add_to' (the residual gradient of y = x + a dropped)."""
    B, L = ids.shape
    d = P["pos_emb"].shape[1]
    hd = d // H
    x = torch.where(tok[..., None], P["item_emb"][ids], P["mask_emb"].expand(B, L, d)) + P["pos_emb"][:L]
    if keeps is not None:
        x = x * keeps["emb"]
    vis = pad[:, None, None, :]
    for i, blk in enumerate(P["blocks"]):
        kb = keeps["blocks"][i] if keeps is not None else None
        xn = _ln64(x, blk["ln1_w"], blk["ln1_b"], 1e-5)
        qkv = xn @ blk["in_w"].T + blk["in_b"]
        q, k, v = (qkv[..., j * d:(j + 1) * d].reshape(B, L, H, hd).transpose(1, 2) for j in range(3))
        s = (q @ k.transpose(-1, -2)) / math.sqrt(hd)
        s = s.masked_fill(~vis, float("-inf"))
        m = s.detach().amax(-1, keepdim=True)
        m = torch.where(torch.isinf(m), torch.zeros_like(m), m)
        e = torch.exp(s - m)
        den = e.sum(-1, keepdim=True)
        pr = torch.where(den > 0, e / den.clamp_min(1e-300), torch.zeros_like(e))
        if kb is not None:
            pr = pr * kb["attn"]
        o = (pr @ v).transpose(1, 2).reshape(B, L, d)
        a = o @ blk["out_w"].T + blk["out_b"]
        if kb is not None:
            a = a * kb["out"]
        y = (x.detach() if mistake == "no_add_to" else x) + a
        yn = _ln64(y, blk["ln2_w"], blk["ln2_b"], 1e-5)
        pre = yn @ blk["w1"].T + blk["b1"]
        if kb is not None and mistake == "drop_before_gelu":
            u = gelu_erf(pre * kb["gelu"])
        else:
            u = gelu_erf(pre)
            if kb is not None:
                u = u * kb["gelu"]
        t = u @ blk["w2"].T + blk["b2"]
        if kb is not None:
            t = t * kb["ffn"]
        z = y + t
        if kb is not None:
            z = z * ((kb["blk"] > 0).to(z.dtype) if mistake == "post_no_scale" else kb["blk"])
        x = z
    w = P["head_w"] if "head_w" in P else P["item_emb"]
    b = P["head_b"]
    sel = pad & ~tok
    if n_items is not None:
        sel = sel & (labels >= 0) & (labels < n_items)
    logits = x[sel] @ w.T + b
    y = labels[sel]
    loss = (torch.logsumexp(logits, -1) - logits.gather(1, y[:, None])[:, 0]).mean()
    return loss, x


def _leaves(P):
    """[(name, tensor)] of a canonical parameter dict in Bert4RecEngine's naming."""
    out = [("item_emb", P["item_emb"]), ("mask_emb", P["mask_emb"]), ("pos_emb", P["pos_emb"])]
    for i, blk in enumerate(P["blocks"]):
        out += [(f"b{i}.{k}", blk[k]) for k in ("ln1_w", "ln1_b", "in_w", "in_b", "out_w", "out_b", "ln2_w", "ln2_b",
                                                  "w1", "b1", "w2", "b2")]
    if "head_w" in P:
        out.append(("head_w", P["head_w"]))
    out.append(("head_b", P["head_b"]))
    return out


def _map(P, f):
    Q = {k: f(k, v) for k, v in P.items() if k != "blocks"}
    Q["blocks"] = [{k: f(f"b{i}.{k}", v) for k, v in blk.items()} for i, blk in enumerate(P["blocks"])]
    return Q


def ref_loss_and_grads(P, ids, pad, tok, labels, H, keeps=None, mistake=None, n_items=None):
    """float64 loss, hidden states and autograd gradients {name: tensor}."""
    Q = _map(P, lambda k, v: v.detach().double().clone().requires_grad_(True))
    loss, h = bert_ref(Q, ids, pad, tok, labels, H, keeps, mistake, n_items)
    leaves = _leaves(Q)
    grads = torch.autograd.grad(loss, [t for _, t in leaves])
    return loss.detach(), h.detach(), {k: g for (k, _), g in zip(leaves, grads)}


# the bf16-consumed parameters of Bert4RecEngine (the kernels read their bf16 shadow): the reference uses them rounded
_BF16_PARAMS = ("item_emb", "mask_emb", "head_w", "in_w", "out_w", "w1", "w2")


def random_params(I, d, L, n_blocks, tied, seed):
    g = _gen(seed)
    r = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    P = {"item_emb": r(I, d) * 0.5, "mask_emb": r(1, d) * 0.5, "pos_emb": r(L, d) * 0.3, "blocks": []}
    for _ in range(n_blocks):
        P["blocks"].append({"ln1_w": 1 + 0.1 * r(d), "ln1_b": 0.1 * r(d), "in_w": r(3 * d, d) / math.sqrt(d),
                            "in_b": 0.05 * r(3 * d), "out_w": r(d, d) / math.sqrt(d), "out_b": 0.05 * r(d),
                            "ln2_w": 1 + 0.1 * r(d), "ln2_b": 0.1 * r(d), "w1": r(4 * d, d) / math.sqrt(d),
                            "b1": 0.05 * r(4 * d), "w2": r(d, 4 * d) / math.sqrt(4 * d), "b2": 0.05 * r(d)})
    if not tied:
        P["head_w"] = r(I, d) / math.sqrt(d)
    P["head_b"] = 0.5 * r(I)
    return P


def engine_view(P):
    """The parameters as Bert4RecEngine computes with them: bf16-consumed ones rounded to bf16, the rest fp32."""
    return _map(P, lambda k, v: (_bf(v).float() if k.split(".")[-1] in _BF16_PARAMS else v.float()))


def step_batch(B, L, I, seed, mask_prob=0.2):
    """Left-padded histories of several lengths (full, short, one token) and a uniform_masker token mask."""
    from oracle.bert4rec import uniform_masker

    g = _gen(seed)
    lengths = [L, L, 150, 57, 13, 1, 120][:B] + [L] * max(0, B - 7)
    pad = torch.zeros(B, L, dtype=torch.bool)
    for b, n in enumerate(lengths):
        pad[b, L - min(n, L):] = True
    items = torch.randint(0, I, (B, L), generator=g)
    tok = uniform_masker(pad, mask_prob, g)
    tok[B // 2:, -1] = False                # the short histories have a masked token
    ids = torch.where(pad, items, torch.zeros_like(items))
    labels = torch.where(pad & ~tok, items, torch.zeros_like(items))
    return ids, pad, tok, labels


# ----------------------------------------------------------------------------------------------------------------------
# kernel calls
# ----------------------------------------------------------------------------------------------------------------------
def _gemm(*args, **kw):
    from replay_b200 import ops

    ops.gemm(*args, **kw)


def _ln_fwd(x, w, b, eps, n_rows, d, y, mean, rstd, hdv=0, gather=None, n_dev=None):
    check(lib().rp_layernorm_fwd(x.data_ptr(), w.data_ptr(), b.data_ptr(), eps, n_rows, d,
                                 None if n_dev is None else n_dev.data_ptr(), None if gather is None else gather.data_ptr(),
                                 y.data_ptr(), mean.data_ptr(), rstd.data_ptr(), hdv, _stream()), "rp_layernorm_fwd")


def _ln_bwd(dy, x, w, mean, rstd, n_rows, d, dx, dw, db, hdv=0, gather=None, n_dev=None, add_to=None):
    check(lib().rp_layernorm_bwd(dy.data_ptr(), x.data_ptr(), w.data_ptr(), mean.data_ptr(), rstd.data_ptr(), n_rows, d,
                                 None if n_dev is None else n_dev.data_ptr(), None if gather is None else gather.data_ptr(),
                                 None if add_to is None else add_to.data_ptr(), dx.data_ptr(), dw.data_ptr(), db.data_ptr(),
                                 hdv, _stream()), "rp_layernorm_bwd")


# ======================================================================================================================
# CPU: the reference
# ======================================================================================================================
def _golden(golden_dir, name):
    from oracle import bert4rec as ob

    z = np.load(os.path.join(golden_dir, name))
    P = ob.params_from_state_dict({k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd::")})
    Gref = ob.params_from_state_dict({k[6:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("grad::")})
    ids, pad, tok, labels = (torch.from_numpy(z[k]) for k in ("ids", "pad_mask", "token_mask", "labels"))
    return z, P, Gref, ids, pad, tok, labels


@pytest.mark.parametrize("name", ["bert4rec_tiny.npz", "bert4rec_tiny_tied.npz"])
def test_reference_with_unit_keeps_matches_oracle_and_golden(golden_dir, name):
    """With every keep mask equal to 1 the dropout restatement is oracle.bert4rec.train_loss and its fp64 autograd
    gradients, and it reproduces the golden loss, hidden states and gradients of the real reference."""
    from oracle import bert4rec as ob

    z, P, Gref, ids, pad, tok, labels = _golden(golden_dir, name)
    B, L = ids.shape
    d, H = int(z["d"]), int(z["H"])
    ones = lambda *s: torch.ones(*s, dtype=torch.float64)  # noqa: E731
    keeps = {"emb": ones(B, L, d), "blocks": [{"attn": ones(B, H, L, L), "out": ones(B, L, d), "gelu": ones(B, L, 4 * d),
                                                "ffn": ones(B, L, d), "blk": ones(B, L, d)} for _ in P["blocks"]]}
    loss, h, G = ref_loss_and_grads(P, ids, pad, tok, labels, H, keeps)
    Q = _map(P, lambda k, v: v.detach().double().clone().requires_grad_(True))
    o_loss = ob.train_loss(Q, ids, pad, tok, labels, H)
    leaves = _leaves(Q)
    o_grads = torch.autograd.grad(o_loss, [t for _, t in leaves])
    torch.testing.assert_close(loss, o_loss.detach(), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(h, ob.bert4rec_body(_map(P, lambda k, v: v.double()), ids, pad, tok, H), rtol=1e-12, atol=1e-12)
    for (k, _), og in zip(leaves, o_grads):
        torch.testing.assert_close(G[k], og, rtol=1e-10, atol=1e-12, msg=k)
    # the real reference (fp32) on the same inputs
    torch.testing.assert_close(loss.float(), torch.from_numpy(z["train_loss"]), rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(h.float(), torch.from_numpy(z["train_hidden"]), rtol=2e-5, atol=2e-6)
    for (k, g_ref) in _leaves(Gref):
        torch.testing.assert_close(G[k].float(), g_ref, rtol=1e-4, atol=1e-6, msg=k)


def test_reference_dropout_is_exact_under_its_masks():
    """keep = 0 at a site removes exactly what it should: dropping the whole block-output site of the last block makes
    the hidden states zero, and dropping every embedding element makes the first block see only its biases."""
    B, L, d, H, I = 2, 8, 64, 2, 40
    P = _map(random_params(I, d, L, 2, False, 3), lambda k, v: v.double())
    ids, pad, tok, labels = step_batch(B, L, I, 4)
    keeps = engine_keeps(SEED + CTR, P_DROP, B, L, d, H, 2)
    keeps["blocks"][1]["blk"] = torch.zeros(B, L, d, dtype=torch.float64)
    _, h = bert_ref(P, ids, pad, tok, labels, H, keeps)
    assert (h == 0).all()
    keeps = engine_keeps(SEED + CTR, P_DROP, B, L, d, H, 2)
    rate = float((keeps["blocks"][0]["gelu"] > 0).double().mean())
    assert abs(rate - (1 - P_DROP)) < 0.02
    assert not torch.equal(keeps["blocks"][0]["ffn"], keeps["blocks"][0]["blk"]), "sites must draw independent masks"


# ----------------------------------------------------------------------------------------------------------------------
# CPU: every plausible mistake moves what the GPU tests compare by >= 10x the tolerance
# ----------------------------------------------------------------------------------------------------------------------
def _model_case(d, H, tied, seed=11, B=7, L=200, I=2000):
    P = engine_view(random_params(I, d, L, 2, tied, seed))
    ids, pad, tok, labels = step_batch(B, L, I, seed + 1)
    return P, ids, pad, tok, labels


def _model_errs(a, b, real):
    """(loss, hidden, gradient) errors of result ``a`` against ``b`` in units of their tolerances."""
    la, ha, Ga = a
    lb, hb, Gb = b
    e_loss = abs(float(la - lb)) / abs(float(lb)) / TOL_LOSS
    e_hid = seq_block_err(ha, hb, real) / TOL_HID
    e_grad = max(block_err(Ga[k], Gb[k]) for k in Gb) / TOL_GRAD
    return e_loss, e_hid, e_grad


@pytest.mark.parametrize("mistake", ["site_off_by_one", "drop_before_gelu", "post_no_scale", "no_add_to"])
def test_step_tolerances_discriminate_perturbed_references(mistake):
    """At the GPU step test's shape and tolerances (d = 256, H = 4, dropout 0.1): a dropout site number off by one, the
    GELU-output dropout applied to the pre-activation, the block-output site without its 1/(1-p), and the residual
    gradient of y = x + attn dropped each move the loss, the hidden states or a gradient by >= 10x its tolerance."""
    d, H = 256, 4
    P, ids, pad, tok, labels = _model_case(d, H, False)
    B, L = ids.shape
    keeps = engine_keeps(SEED + CTR, P_DROP, B, L, d, H, 2)
    ref = ref_loss_and_grads(P, ids, pad, tok, labels, H, keeps)
    if mistake == "site_off_by_one":
        bad = ref_loss_and_grads(P, ids, pad, tok, labels, H, engine_keeps(SEED + CTR, P_DROP, B, L, d, H, 2, site_shift=1))
    else:
        bad = ref_loss_and_grads(P, ids, pad, tok, labels, H, keeps, mistake=mistake)
    assert max(_model_errs(bad, ref, pad)) >= 10


def _ffn_in_case(M, seed, dev=None):
    """Inputs of the FFN-in GEMM (K = 256, N = 1024): pre-activations ~ N(0, 0.8^2), never beyond the range where
    gelu(pre) would round to zero in fp32."""
    g = _gen(seed)
    N, K = 1024, 256
    A = _bf(torch.randn(M, K, generator=g) * 0.25)
    W = _bf(torch.randn(N, K, generator=g) * 0.2)
    bias = torch.randn(N, generator=g) * 0.1
    if dev is not None:
        A, W, bias = A.to(dev), W.to(dev), bias.to(dev)
    pre = A.double() @ W.double().T + bias.double()
    S = A.double().abs() @ W.double().abs().T + bias.double().abs()
    return A, W, bias, pre, S


def _ffn_in_ref(pre, S, keep, ks, gelu=gelu_erf, drop_before=False):
    """u = drop(gelu(pre)) and the element-wise slack: fp32 accumulation (through gelu') and fp32 erf (~1e-7 |pre|)."""
    u = gelu(pre * keep * ks) if drop_before else gelu(pre) * keep * ks
    atol = ks * (HALF_ULP_SLACK * S * gelu_erf_grad(pre).abs() + 1.5e-7 * pre.abs()) + 1e-30
    return u, atol


def _ffn_in_bwd_case(M, seed, dev=None):
    g = _gen(seed)
    d = 256
    dT = _bf(torch.randn(M, d, generator=g))
    W2 = _bf(torch.randn(d, 4 * d, generator=g) / 16)
    pre = _bf(torch.randn(M, 4 * d, generator=g))
    if dev is not None:
        dT, W2, pre = dT.to(dev), W2.to(dev), pre.to(dev)
    acc = dT.double() @ W2.double()
    S = dT.double().abs() @ W2.double().abs()
    return dT, W2, pre, acc, S


def _ffn_in_bwd_ref(acc, S, pre, keep, ks, grad=gelu_erf_grad):
    """du = (d_t W2) * keep/(1-p) * gelu'(pre): ``pre`` is the bf16 pre-activation the forward stored (C2), so the
    reference evaluates gelu' at that rounded value, as the kernel does."""
    z = pre.double()
    gz = grad(z)
    du = acc * keep * ks * gz
    atol = ks * (HALF_ULP_SLACK * S * gz.abs() + 4e-7 * acc.abs()) + 1e-30
    return du, atol


@pytest.mark.parametrize("mistake", ["gelu_tanh_fwd", "drop_before_gelu", "gelu_tanh_bwd"])
def test_gemm_tolerance_discriminates_gelu_mistakes(mistake):
    """At the FFN-in GEMM test's inputs (M = 600) and element-wise tolerance, the tanh GELU in the forward or in gelu',
    and dropout applied before the GELU, move the output by >= 10x TOL_ULP."""
    M = 600
    keep = keep_draws(SEED + CTR, _site(0, 2) << 40, P_DROP, np.arange(M), 1024).double()
    ks = _ks(P_DROP)
    if mistake == "gelu_tanh_bwd":
        _, _, pre, acc, S = _ffn_in_bwd_case(M, 5)
        ref, atol = _ffn_in_bwd_ref(acc, S, pre, keep, ks)
        bad, _ = _ffn_in_bwd_ref(acc, S, pre, keep, ks, grad=gelu_tanh_grad)
    else:
        _, _, _, pre, S = _ffn_in_case(M, 3)
        ref, atol = _ffn_in_ref(pre, S, keep, ks)
        bad, _ = _ffn_in_ref(pre, S, keep, ks, gelu=gelu_tanh if mistake == "gelu_tanh_fwd" else gelu_erf,
                             drop_before=mistake == "drop_before_gelu")
    assert ulp_err(_bf(bad).double(), ref, atol) >= 10 * TOL_ULP


def _ln_case(T, d, hdv, seed, dev=None):
    """Rows at scales from 1e-3 to 10 (so that eps matters on the small ones), padded features zero, w / b zero there."""
    g = _gen(seed)
    valid = feat_mask(d, hdv)
    scale = torch.exp(torch.empty(T, 1).uniform_(math.log(1e-3), math.log(10.0), generator=g))
    x = _bf((torch.randn(T, d, generator=g) * scale + 0.3 * scale) * valid)
    w = (1 + 0.2 * torch.randn(d, generator=g)) * valid
    b = 0.1 * torch.randn(d, generator=g) * valid
    dy = _bf(torch.randn(T, d, generator=g) * valid)
    add = _bf(torch.randn(T, d, generator=g) / scale * valid)    # a residual gradient of dx's size (dx ~ rstd ~ 1/scale)
    out = [x, w, b, dy, add, valid]
    return [t.to(dev) for t in out] if dev is not None else out


def _ln_fwd_atol(x, mean, rstd, w):
    """fp32 slack of y = (x - mean) * rstd * w + b: a few ulps of the fp32 terms."""
    return 4e-7 * ((x.abs() + mean.abs()[:, None]) * rstd[:, None] * w.abs() + 1.0) + 1e-30


@pytest.mark.parametrize("mistake", ["eps", "no_add_to"])
def test_layernorm_tolerances_discriminate_mistakes(mistake):
    """eps 1e-8 in place of 1e-5 moves y on the small-scale rows, and dropping add_to moves dx, by >= 10x the tolerance."""
    x, w, b, dy, add, valid = _ln_case(1400, 256, 0, 7)
    x64, w64, b64 = x.double(), w.double(), b.double()
    y, mean, rstd = ln_ref(x64, w64, b64, 1e-5, valid)
    if mistake == "eps":
        bad = ln_ref(x64, w64, b64, 1e-8, valid)[0]
        assert ulp_err(_bf(bad).double(), y, _ln_fwd_atol(x64, mean, rstd, w64)) >= 10 * TOL_ULP
    else:
        dx = ln_bwd_ref(dy.double(), x64, w64, mean, rstd, valid)[0]
        assert block_err(dx, dx + add.double()) >= 10 * TOL_LN_DX


def _bert_embed_bwd_ref(dx, ids, pad, tok, keep, I, include_pad_mask=False):
    """d_table, d_mask_emb, d_pos of the BERT4Rec embedding: real unmasked tokens -> their item row, real masked tokens ->
    mask_emb (pads take the gradient of nothing: their dx is exactly zero in the model), every real token -> its position."""
    B, L = pad.shape
    d = dx.shape[1]
    gx = dx.double() * keep
    real, tk = pad.reshape(-1), tok.reshape(-1)
    d_table = torch.zeros(I, d, dtype=torch.float64).index_add_(0, ids[real & tk].long(), gx[real & tk])
    to_mask = (~tk) if include_pad_mask else (real & ~tk)
    d_mask = gx[to_mask].sum(0, keepdim=True)
    d_pos = (gx * real[:, None]).view(B, L, d).sum(0)
    return d_table, d_mask, d_pos


def test_embedding_tolerance_discriminates_mask_emb_of_pads():
    B, L, d, I = 3, 200, 256, 300
    g = _gen(1)
    ids, pad, tok = _embed_batch(B, L, I, g)
    dx = _bf(torch.randn(B * L, d, generator=g))
    keep = keep_draws(SEED + CTR, 0, P_DROP, np.arange(B * L), d).double() * _ks(P_DROP)
    ref = _bert_embed_bwd_ref(dx, ids, pad, tok, keep, I)[1]
    bad = _bert_embed_bwd_ref(dx, ids, pad, tok, keep, I, include_pad_mask=True)[1]
    assert block_err(bad, ref) >= 10 * TOL_SUM


def _embed_batch(B, L, I, g):
    """ids int32 with many repeats (the atomics must add up), left-padded rows, ~20 % masked real tokens."""
    pad = torch.zeros(B, L, dtype=torch.bool)
    for b in range(B):
        pad[b, int(torch.randint(0, L - 1, (1,), generator=g)) if b % 2 else 0:] = True
    ids = torch.randint(0, min(I, 40), (B, L), generator=g).to(torch.int32)
    tok = (torch.rand(B, L, generator=g) > 0.2) & pad
    return ids.reshape(-1), pad, tok


# ======================================================================================================================
# GPU 1: rp_gemm epilogue features
# ======================================================================================================================
def _sent_buf(rows, cols, dev, dtype=torch.bfloat16):
    return torch.full((rows + 64, cols + 64), SENT, dtype=dtype, device=dev)


def _check_sentinels(buf, rows, cols, what):
    assert (buf[rows:] == SENT).all() and (buf[:, cols:] == SENT).all(), f"{what} written outside [{rows}, {cols})"


def _assert_keep_pattern(out, keep, exact, slack, what):
    """Dropped elements are exactly zero, bit for bit against the ported mask; kept ones are non-zero unless their exact
    value is within the accumulation slack of zero (an fp32 accumulator of bf16 products cancels to exactly 0 about once
    in 5e7 elements)."""
    nz = out != 0
    leak = int((nz & ~keep).sum())
    assert leak == 0, f"{what}: {leak} dropped elements are not zero"
    lost = keep & ~nz
    bad = int(((exact.abs() > slack) & lost).sum())
    assert bad == 0, f"{what}: {bad} of {int(lost.sum())} kept elements are zero"


def _like_c(t):
    """``t`` [rows, cols] copied into a view with the row pitch of a _sent_buf output: gate and residual are read with
    the output's geometry."""
    rows, cols = t.shape
    buf = torch.zeros(rows + 64, cols + 64, dtype=t.dtype, device=t.device)
    buf[:rows, :cols] = t
    return buf[:rows, :cols]


@pytest.mark.gpu
@pytest.mark.parametrize("M", [600, 51200])
def test_gemm_ffn_in_forward_gelu_dropout_c2(cuda, M):
    """u = drop(gelu(yn W1^T + b1)) with C2 = the pre-activation before the GELU and the dropout (K = 256, N = 1024; 600
    rows end in a ragged tile, 51 200 is config 3's token count): the zero pattern is the ported keep mask bit for bit,
    the values are one rounding from fp64, C2 is the rounded pre-activation everywhere, nothing is written outside."""
    N, K = 1024, 256
    off = _site(1, 2) << 40
    A, W, bias, pre, S = _ffn_in_case(M, 3 if M == 600 else 4, dev=cuda)
    ctr = torch.tensor([CTR], dtype=torch.int64, device=cuda)
    C, C2 = _sent_buf(M, N, cuda), _sent_buf(M, N, cuda)
    _gemm(A, W, C[:M, :N], M, N, K, bias=bias, act=2, drop_p=P_DROP, drop_offset=off, seed=SEED, seed_ptr=ctr.data_ptr(),
          C2=C2[:M, :N])
    torch.cuda.synchronize()
    _check_sentinels(C, M, N, "u")
    _check_sentinels(C2, M, N, "C2")
    keep = keep_draws(SEED + CTR, off, P_DROP, np.arange(M), N).to(cuda)
    u = C[:M, :N]
    ref, atol = _ffn_in_ref(pre, S, keep.double(), _ks(P_DROP))
    _assert_keep_pattern(u, keep, gelu_erf(pre) * _ks(P_DROP), atol, "u")
    assert _note("gemm gelu+drop ulp", ulp_err(u, ref, atol)) < TOL_ULP
    assert _note("gemm C2 ulp", ulp_err(C2[:M, :N], pre, HALF_ULP_SLACK * S + 1e-30)) < TOL_ULP


@pytest.mark.gpu
@pytest.mark.parametrize("M", [600, 51200])
def test_gemm_ffn_in_backward_gelu_grad_dropout(cuda, M):
    """du = (d_t W2) * keep/(1-p) * gelu'(pre) (b_mn, gate_mode 1), and SASRec's un-fused ReLU backward
    du = (d_t W2) * (gate != 0 ? 1/(1-p) : 0) (gate_mode 0, gate = the dropped ReLU output)."""
    d = 256
    off = _site(0, 2) << 40
    dT, W2, pre, acc, S = _ffn_in_bwd_case(M, 5 if M == 600 else 6, dev=cuda)
    ctr = torch.tensor([CTR], dtype=torch.int64, device=cuda)
    ks = _ks(P_DROP)
    keep = keep_draws(SEED + CTR, off, P_DROP, np.arange(M), 4 * d).to(cuda)
    C = _sent_buf(M, 4 * d, cuda)
    _gemm(dT, W2, C[:M, :4 * d], M, 4 * d, d, b_mn=True, drop_p=P_DROP, drop_offset=off, seed=SEED, seed_ptr=ctr.data_ptr(),
          gate=_like_c(pre), gate_mode=1, gate_scale=1.0)
    torch.cuda.synchronize()
    _check_sentinels(C, M, 4 * d, "du")
    du = C[:M, :4 * d]
    ref, atol = _ffn_in_bwd_ref(acc, S, pre, keep.double(), ks)
    _assert_keep_pattern(du, keep, acc * ks * gelu_erf_grad(pre.double()), atol, "du")
    assert _note("gemm gelu' ulp", ulp_err(du, ref, atol)) < TOL_ULP
    # gate_mode 0: gate = relu(pre) * keep / (1-p), zero where ReLU or dropout zeroed it
    gate = _bf(torch.relu(pre.float()) * keep.float() * ks)
    C = _sent_buf(M, 4 * d, cuda)
    _gemm(dT, W2, C[:M, :4 * d], M, 4 * d, d, b_mn=True, gate=_like_c(gate), gate_scale=ks)
    torch.cuda.synchronize()
    _check_sentinels(C, M, 4 * d, "du (relu)")
    du = C[:M, :4 * d]
    atol = ks * HALF_ULP_SLACK * S + 1e-30
    _assert_keep_pattern(du, gate != 0, acc * ks, atol, "du (relu)")
    on = (gate != 0).double()
    assert _note("gemm relu' ulp", ulp_err(du, acc * on * ks, atol)) < TOL_ULP


def _block_out_case(M, seed, dev):
    g = _gen(seed)
    d = 256
    U = _bf(torch.randn(M, 4 * d, generator=g) * 0.5).to(dev)
    W2 = _bf(torch.randn(d, 4 * d, generator=g) / 32).to(dev)
    b2 = (0.1 * torch.randn(d, generator=g)).to(dev)
    y = _bf(torch.randn(M, d, generator=g) + 0.05).to(dev)
    y = torch.where(y == 0, torch.full_like(y, 0.5), y)          # the residual is never exactly zero
    t = U.double() @ W2.double().T + b2.double()
    S = U.double().abs() @ W2.double().abs().T + b2.double().abs()
    return U, W2, b2, y, t, S


@pytest.mark.gpu
@pytest.mark.parametrize("M", [600, 51200])
def test_gemm_block_output_two_dropout_sites(cuda, M):
    """x_next = drop4(y + drop3(u W2^T + b2)) with seed_ptr at a non-zero counter: the outer zero pattern is site 4's mask;
    with a zero residual it is site 3's AND site 4's, so both sites draw their own masks and both add the counter;
    values against fp64; a row mask applied after everything zeroes its rows exactly and leaves the others bit-identical."""
    d, K = 256, 1024
    off3, off4 = _site(1, 3) << 40, _site(1, 4) << 40
    U, W2, b2, y, t, S = _block_out_case(M, 7 if M == 600 else 8, cuda)
    ctr = torch.tensor([CTR], dtype=torch.int64, device=cuda)
    ks = _ks(P_DROP)
    k3 = keep_draws(SEED + CTR, off3, P_DROP, np.arange(M), d).to(cuda)
    k4 = keep_draws(SEED + CTR, off4, P_DROP, np.arange(M), d).to(cuda)
    both = float((k3 & k4).double().mean())
    assert abs(both - (1 - P_DROP) ** 2) < 0.01, "the two sites must be independent draws"

    def run(res, rowmask=None):
        C = _sent_buf(M, d, cuda)
        _gemm(U, W2, C[:M, :d], M, d, K, bias=b2, drop_p=P_DROP, drop_offset=off3, seed=SEED, seed_ptr=ctr.data_ptr(),
              residual=_like_c(res), post_drop_p=P_DROP, post_drop_offset=off4, rowmask=rowmask)
        torch.cuda.synchronize()
        _check_sentinels(C, M, d, "x_next")
        return C[:M, :d].clone()

    out = run(y)
    inner = y.double() + t * k3.double() * ks
    atol = ks * ks * HALF_ULP_SLACK * S + 2e-7 * (y.double().abs() + t.abs() * ks) * ks + 1e-30
    _assert_keep_pattern(out, k4, inner * ks, atol, "x_next")
    assert _note("gemm residual+2 drops ulp", ulp_err(out, inner * k4.double() * ks, atol)) < TOL_ULP
    zero = torch.zeros_like(y)
    out0 = run(zero)
    atol0 = ks * ks * HALF_ULP_SLACK * S + 1e-30
    _assert_keep_pattern(out0, k3 & k4, t * ks * ks, atol0, "x_next with a zero residual (site 3 AND site 4)")
    ref0 = t * k3.double() * k4.double() * ks * ks
    assert _note("gemm 2 drops ulp", ulp_err(out0, ref0, atol0)) < TOL_ULP
    rm = (torch.rand(M, generator=_gen(M)) > 0.3).to(torch.uint8).to(cuda)
    outm = run(y, rm)
    assert (outm[rm == 0] == 0).all(), "rows with mask 0 must be exactly zero"
    assert torch.equal(outm[rm != 0], out[rm != 0])


# ----------------------------------------------------------------------------------------------------------------------
# GPU 1b: split-K weight gradients (the _wgrad recipe) and atomic split-K
# ----------------------------------------------------------------------------------------------------------------------
def _splits_empty(K, split):
    chunks = (K + 63) // 64
    return [(chunks * s) // split == (chunks * (s + 1)) // split for s in range(split)]


def _wgrad_case(M, N, K, seed, dev):
    g = _gen(seed)
    dY = _bf(torch.randn(K, M, generator=g)).to(dev)
    X = _bf(torch.randn(K, N, generator=g)).to(dev)
    preset = torch.randn(M, N, generator=g).to(dev)
    ref = dY.double().T @ X.double()
    return dY, X, preset, ref


@pytest.mark.gpu
@pytest.mark.parametrize("M,K,split", [(1024, 1400, 1), (1024, 1400, 2), (1024, 1400, 9), (256, 1400, 9), (1024, 1400, 23),
                                       (256, 1400, 100), (1024, 51200, 9), (256, 51200, 100), (1024, 51200, 100)])
def test_wgrad_split_k_partials_and_reduction(cuda, M, K, split):
    """dW[M, 256] += dY[K, M]^T X[K, 256] as Bert4RecEngine._wgrad runs it (both operands MN-major, out_mode 3 partials
    at c_split_stride, rp_reduce_splits accumulating onto preset values): 9 splits is what _wgrad picks at config 3 on
    132 SMs; 23 > the 22 chunks of K = 1400 and 100 leave splits empty, whose partials must be exactly 0.  Reruns are
    bit-identical; atomic split-K (out_mode 1) matches the same reference."""
    N = 256
    n = M * N
    dY, X, preset, ref = _wgrad_case(M, N, K, M + K + split, cuda)

    def run():
        ws = torch.full((split * n + 64,), 7.0, device=cuda)
        _gemm(dY, X, ws, M, N, K, a_mn=True, b_mn=True, out_mode=3, split_k=split, c_geom=(N, 0, 0, 0), c_split_stride=n)
        dW = preset.clone()
        check(lib().rp_reduce_splits(ws.data_ptr(), split, n, n, dW.data_ptr(), 1, _stream()), "rp_reduce_splits")
        torch.cuda.synchronize()
        return ws, dW

    ws, dW = run()
    assert (ws[split * n:] == 7.0).all(), "partials written past the last split"
    parts = ws[:split * n].view(split, M, N)
    for s, empty in enumerate(_splits_empty(K, split)):
        if empty:
            assert (parts[s] == 0).all(), f"empty split {s} must store exact zeros"
    psum = parts.double().sum(0)
    assert _note("split-K partial sum", block_err(psum, ref)) < TOL_SPLITK
    assert _note("split-K reduced", block_err(dW.double() - preset.double(), ref)) < TOL_SPLITK
    ws2, dW2 = run()
    assert torch.equal(ws, ws2) and torch.equal(dW, dW2), "split-K reruns must be bit-identical"
    if split in (1, 9, 23):
        C = preset.clone()
        _gemm(dY, X, C, M, N, K, a_mn=True, b_mn=True, out_mode=1, split_k=split, c_geom=(N, 0, 0, 0))
        torch.cuda.synchronize()
        assert _note("split-K atomic", block_err(C.double() - preset.double(), ref)) < TOL_SPLITK


# ======================================================================================================================
# GPU 2: LayerNorm
# ======================================================================================================================
def _ln_check_fwd(y, mean, rstd, x, w, b, eps, valid, rows):
    y_ref, m_ref, r_ref = ln_ref(x.double(), w.double(), b.double(), eps, valid)
    y_ref, m_ref, r_ref = y_ref[rows], m_ref[rows], r_ref[rows]
    assert (y.double()[:, ~valid.to(y.device)] == 0).all(), "padded features of y must be 0"
    atol = _ln_fwd_atol(x.double()[rows], m_ref, r_ref, w.double())
    assert _note("ln y ulp", ulp_err(y, y_ref, atol)) < TOL_ULP
    rms = x.double()[rows].square().mean(-1).sqrt().clamp_min(1e-30)
    assert _note("ln mean", ((mean.double() - m_ref).abs() / rms).max()) < TOL_LN_STAT
    assert _note("ln rstd", ((rstd.double() - r_ref).abs() / r_ref).max()) < TOL_LN_STAT


@pytest.mark.gpu
@pytest.mark.parametrize("eps", [1e-5, 1e-8])
@pytest.mark.parametrize("d,T,hdv", [(64, 1400, 0), (128, 1400, 0), (256, 1400, 0), (512, 1400, 0), (256, 51200, 0),
                                     (128, 1400, 48), (128, 1400, 50), (256, 1400, 50), (128, 1400, 96), (256, 1400, 96)])
def test_layernorm_fwd_bwd_plain_rows(cuda, d, T, hdv, eps):
    """rp_layernorm_fwd / _bwd on every row (T = 51 200 wraps both grid-stride loops): y, mean, rstd against fp64 with
    statistics over the real features only (hd_valid), dx with add_to, padded inputs get exactly zero gradient (add_to
    is zero there), dw / db accumulate on top of preset values."""
    x, w, b, dy, add, valid = _ln_case(T, d, hdv, seed=d + T + hdv, dev=cuda)
    y = torch.full((T + 8, d), SENT, dtype=torch.bfloat16, device=cuda)
    mean = torch.full((T + 8,), SENT, device=cuda)
    rstd = torch.full((T + 8,), SENT, device=cuda)
    _ln_fwd(x, w, b, eps, T, d, y, mean, rstd, hdv)
    torch.cuda.synchronize()
    assert (y[T:] == SENT).all() and (mean[T:] == SENT).all() and (rstd[T:] == SENT).all()
    _ln_check_fwd(y[:T], mean[:T], rstd[:T], x, w, b, eps, valid, slice(None))
    g = _gen(d)
    dw0, db0 = torch.randn(d, generator=g).to(cuda), torch.randn(d, generator=g).to(cuda)
    dx = torch.full((T + 8, d), SENT, dtype=torch.bfloat16, device=cuda)
    dw, db = dw0.clone(), db0.clone()
    _ln_bwd(dy, x, w, mean, rstd, T, d, dx, dw, db, hdv, add_to=add)
    torch.cuda.synchronize()
    assert (dx[T:] == SENT).all()
    dx_ref, dw_ref, db_ref = ln_bwd_ref(dy.double(), x.double(), w.double(), mean.double()[:T], rstd.double()[:T], valid)
    dx_ref = dx_ref + add.double()
    assert (dx[:T, ~valid.to(cuda)] == 0).all(), "padded inputs must get exactly zero gradient"
    assert _note("ln dx block", block_err(dx[:T], dx_ref)) < TOL_LN_DX
    assert _note("ln dw", block_err((dw.double() - dw0.double()).view(-1, 1), dw_ref.view(-1, 1))) < TOL_SUM
    assert _note("ln db", block_err((db.double() - db0.double()).view(-1, 1), db_ref.view(-1, 1))) < TOL_SUM
    assert (dw[~valid.to(cuda)] == dw0[~valid.to(cuda)]).all() and (db[~valid.to(cuda)] == db0[~valid.to(cuda)]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("d", [64, 128, 256, 512])
@pytest.mark.parametrize("n_dev", [0, 517])
def test_layernorm_gather_with_device_row_count(cuda, d, n_dev):
    """gather + n_rows_dev (the valid-target compaction): output row r < *n_rows_dev reads input row gather[r]; rows past
    the device count keep their sentinels; the backward scatters dx into the gathered rows only and accumulates
    dw / db over the gathered rows; a device count of 0 writes nothing and leaves dw / db unchanged."""
    T, n_max, eps = 1400, 900, 1e-5
    x, w, b, dy, add, valid = _ln_case(T, d, 0, seed=d + n_dev, dev=cuda)
    perm = torch.randperm(T, generator=_gen(d))[:n_max].sort().values
    gather = perm.to(torch.int32).to(cuda)
    nd = torch.tensor([n_dev], dtype=torch.int32, device=cuda)
    y = torch.full((n_max, d), SENT, dtype=torch.bfloat16, device=cuda)
    mean = torch.full((n_max,), SENT, device=cuda)
    rstd = torch.full((n_max,), SENT, device=cuda)
    _ln_fwd(x, w, b, eps, n_max, d, y, mean, rstd, gather=gather, n_dev=nd)
    torch.cuda.synchronize()
    assert (y[n_dev:] == SENT).all() and (mean[n_dev:] == SENT).all() and (rstd[n_dev:] == SENT).all()
    rows = gather[:n_dev].long()
    if n_dev:
        _ln_check_fwd(y[:n_dev], mean[:n_dev], rstd[:n_dev], x, w, b, eps, valid, rows)
    dyc = dy[:n_max].contiguous()
    dx = torch.full((T, d), SENT, dtype=torch.bfloat16, device=cuda)
    dw0 = torch.randn(d, generator=_gen(1)).to(cuda)
    db0 = torch.randn(d, generator=_gen(2)).to(cuda)
    dw, db = dw0.clone(), db0.clone()
    _ln_bwd(dyc, x, w, mean, rstd, n_max, d, dx, dw, db, gather=gather, n_dev=nd)
    torch.cuda.synchronize()
    untouched = torch.ones(T, dtype=torch.bool, device=cuda)
    untouched[rows] = False
    assert (dx[untouched] == SENT).all(), "rows not gathered must keep their sentinels"
    if n_dev == 0:
        assert torch.equal(dw, dw0) and torch.equal(db, db0)
        return
    dx_ref, dw_ref, db_ref = ln_bwd_ref(dyc[:n_dev].double(), x.double()[rows], w.double(), mean[:n_dev].double(),
                                        rstd[:n_dev].double(), valid)
    assert _note("ln dx block", block_err(dx[rows], dx_ref)) < TOL_LN_DX
    assert _note("ln dw", block_err((dw.double() - dw0.double()).view(-1, 1), dw_ref.view(-1, 1))) < TOL_SUM
    assert _note("ln db", block_err((db.double() - db0.double()).view(-1, 1), db_ref.view(-1, 1))) < TOL_SUM


# ======================================================================================================================
# GPU 3: embeddings
# ======================================================================================================================
_EMB_SHAPES = [(B, L, d) for B in (1, 3, 9) for L in (16, 200) for d in (64, 128, 256, 512)]


@pytest.mark.gpu
@pytest.mark.parametrize("B,L,d", _EMB_SHAPES)
def test_bert_embedding_fwd_bwd(cuda, B, L, d):
    """rp_bert_embed_fwd / _bwd (B not a multiple of the 4- / 8-token groups): <MASK> and pad positions read mask_emb,
    dropout at site offset 0 with the counter; the backward adds repeated ids up, gives d_mask_emb the gradient of the
    real masked tokens only, d_pos the real tokens', leaves untouched table rows at their preset values."""
    I = 300
    g = _gen(B * 1000 + L + d)
    ids, pad, tok = _embed_batch(B, L, I, g)
    T = B * L
    table = _bf(torch.randn(I, d, generator=g))
    mask_emb = _bf(torch.randn(1, d, generator=g))
    pos = torch.randn(L, d, generator=g) * 0.3 + 0.01
    dx = _bf(torch.randn(T, d, generator=g))
    ctr = torch.tensor([CTR], dtype=torch.int64, device=cuda)
    ks = _ks(P_DROP)
    keep = keep_draws(SEED + CTR, 0, P_DROP, np.arange(T), d)
    idd, tokd, padd = ids.to(cuda), tok.reshape(-1).to(torch.uint8).to(cuda), pad.reshape(-1).to(torch.uint8).to(cuda)
    table_d, mask_d, pos_d, dx_d = table.to(cuda), mask_emb.to(cuda), pos.to(cuda), dx.to(cuda)
    for drop in (0.0, P_DROP):
        out = torch.full((T + 8, d), SENT, dtype=torch.bfloat16, device=cuda)
        check(lib().rp_bert_embed_fwd(table_d.data_ptr(), mask_d.data_ptr(), pos_d.data_ptr(), idd.data_ptr(), tokd.data_ptr(),
                                      T, L, d, drop, SEED, 0, ctr.data_ptr(), out.data_ptr(), _stream()), "rp_bert_embed_fwd")
        torch.cuda.synchronize()
        assert (out[T:] == SENT).all()
        kp = keep.double() * ks if drop > 0 else torch.ones(T, d, dtype=torch.float64)
        v = torch.where(tok.reshape(-1, 1), table.double()[ids.long()], mask_emb.double()) + pos.double().repeat(B, 1)
        ref = v * kp
        got = out[:T].cpu()
        if drop > 0:
            assert torch.equal(got != 0, keep)
        atol = 2e-7 * (table.double()[ids.long()].abs() + mask_emb.double().abs() + pos.double().abs().repeat(B, 1)) * ks
        assert _note("embed fwd ulp", ulp_err(got, ref, atol)) < TOL_ULP
        d_table0 = torch.randn(I, d, generator=g)
        d_mask0, d_pos0 = torch.randn(1, d, generator=g), torch.randn(L, d, generator=g)
        dt, dm, dp = d_table0.to(cuda), d_mask0.to(cuda), d_pos0.to(cuda)
        check(lib().rp_bert_embed_bwd(dx_d.data_ptr(), idd.data_ptr(), padd.data_ptr(), tokd.data_ptr(), B, L, d, drop,
                                      SEED, 0, ctr.data_ptr(), dt.data_ptr(), dm.data_ptr(), dp.data_ptr(), _stream()),
              "rp_bert_embed_bwd")
        torch.cuda.synchronize()
        r_table, r_mask, r_pos = _bert_embed_bwd_ref(dx, ids, pad, tok, kp, I)
        dt, dm, dp = dt.cpu().double(), dm.cpu().double(), dp.cpu().double()
        used = torch.zeros(I, dtype=torch.bool)
        used[ids[(pad & tok).reshape(-1)].long()] = True
        assert torch.equal(dt[~used], d_table0.double()[~used]), "table rows without a real unmasked token were written"
        assert _note("embed d_table", block_err(dt[used] - d_table0.double()[used], r_table[used])) < TOL_SUM
        assert _note("embed d_mask_emb", block_err(dm - d_mask0.double(), r_mask)) < TOL_SUM
        assert _note("embed d_pos", block_err(dp - d_pos0.double(), r_pos)) < TOL_SUM


@pytest.mark.gpu
@pytest.mark.parametrize("zero_pad_rows", [0, 1])
@pytest.mark.parametrize("B,L", [(1, 200), (3, 16), (9, 200)])
@pytest.mark.parametrize("d", [64, 128, 256, 512])
def test_sasrec_embedding_fwd_bwd(cuda, d, B, L, zero_pad_rows):
    """rp_embed_fwd / _bwd: x = E[id] * sqrt(d) + P[pos0 + t % L] (pos0 = 37: the right-aligned window of a longer
    max_len) -> dropout -> pad rows zeroed or not; the backward scales by sqrt(d), freezes the pad row, takes pad tokens'
    position gradient only when their rows are not zeroed."""
    I, pad_id, pos0, max_len = 300, 300, 37, L + 37
    g = _gen(d * 7 + B * 100 + L + zero_pad_rows)
    ids, pad, _ = _embed_batch(B, L, I, g)
    ids = torch.where(pad.reshape(-1), ids, torch.full_like(ids, pad_id))   # rp_prepare_batch's pad replacement
    T = B * L
    scale = math.sqrt(d)
    table = _bf(torch.randn(I + 1, d, generator=g) * 0.1)
    pos = torch.randn(max_len, d, generator=g) * 0.3 + 0.01
    dx = _bf(torch.randn(T, d, generator=g))
    ctr = torch.tensor([CTR], dtype=torch.int64, device=cuda)
    ks = _ks(P_DROP)
    keep = keep_draws(SEED + CTR, 0, P_DROP, np.arange(T), d)
    kp = keep.double() * ks
    idd, padd = ids.to(cuda), pad.reshape(-1).to(torch.uint8).to(cuda)
    table_d, pos_d, dx_d = table.to(cuda), pos.to(cuda), dx.to(cuda)
    out = torch.full((T + 8, d), SENT, dtype=torch.bfloat16, device=cuda)
    check(lib().rp_embed_fwd(table_d.data_ptr(), pos_d.data_ptr(), idd.data_ptr(), padd.data_ptr(), T, L, d, pos0, scale,
                             zero_pad_rows, P_DROP, SEED, 0, ctr.data_ptr(), out.data_ptr(), _stream()), "rp_embed_fwd")
    torch.cuda.synchronize()
    assert (out[T:] == SENT).all()
    real = pad.reshape(-1, 1).double() if zero_pad_rows else torch.ones(T, 1, dtype=torch.float64)
    v = table.double()[ids.long()] * scale + pos.double()[pos0:pos0 + L].repeat(B, 1)
    got = out[:T].cpu()
    assert torch.equal(got != 0, keep & (real > 0)), "zero pattern: dropout mask and zeroed pad rows"
    atol = 2e-7 * (table.double()[ids.long()].abs() * scale + pos.double()[pos0:pos0 + L].abs().repeat(B, 1)) * ks
    assert _note("embed fwd ulp", ulp_err(got, v * kp * real, atol)) < TOL_ULP
    d_table0, d_pos0 = torch.randn(I + 1, d, generator=g), torch.randn(max_len, d, generator=g)
    dt, dp = d_table0.to(cuda), d_pos0.to(cuda)
    check(lib().rp_embed_bwd(dx_d.data_ptr(), idd.data_ptr(), padd.data_ptr(), B, L, d, pad_id, pos0, scale,
                             zero_pad_rows, P_DROP, SEED, 0, ctr.data_ptr(), dt.data_ptr(), dp.data_ptr(), _stream()),
          "rp_embed_bwd")
    torch.cuda.synchronize()
    gx = dx.double() * kp * real
    on = ids != pad_id
    r_table = torch.zeros(I + 1, d, dtype=torch.float64).index_add_(0, ids[on].long(), gx[on] * scale)
    r_pos = gx.view(B, L, d).sum(0)
    dt, dp = dt.cpu().double(), dp.cpu().double()
    assert torch.equal(dt[pad_id], d_table0.double()[pad_id]), "the pad row must receive no gradient"
    used = torch.zeros(I + 1, dtype=torch.bool)
    used[ids[on].long()] = True
    assert torch.equal(dt[~used], d_table0.double()[~used])
    assert _note("embed d_table", block_err(dt[used] - d_table0.double()[used], r_table[used])) < TOL_SUM
    assert torch.equal(dp[:pos0], d_pos0.double()[:pos0]), "positions before pos0 were written"
    assert _note("embed d_pos", block_err(dp[pos0:] - d_pos0.double()[pos0:], r_pos)) < TOL_SUM


# ======================================================================================================================
# GPU 4: column sums, row gather / scatter, dropout backward, batch preparation
# ======================================================================================================================
def _colsum_err(got, preset, y):
    """|db - preset - sum_r y| / sum_r |y| per column (the fp32 summation error in units of the sum of magnitudes)."""
    y = y.double()
    return float(((got.double() - preset.double() - y.sum(0)).abs() / y.abs().sum(0).clamp_min(1e-30)).max())


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [3, 1400, 51200])
@pytest.mark.parametrize("cols", [64, 192, 256, 768, 1024])
def test_colsum_and_colsum_multi(cuda, cols, rows):
    """db += column sums of a column view (ld > cols, like the in_b slice of dQKV) for rows below and far above the
    block's row lanes (256 / (cols / 4)); rp_colsum_multi over five tensors of different widths sharing the rows."""
    g = _gen(cols + rows)
    big = _bf(torch.randn(rows, 3 * cols + 64, generator=g)).to(cuda)
    view = big[:, cols:2 * cols]
    db0 = torch.randn(cols + 4, generator=g).to(cuda)
    db = db0.clone()
    check(lib().rp_colsum(view.data_ptr(), rows, cols, view.stride(0), db.data_ptr(), _stream()), "rp_colsum")
    torch.cuda.synchronize()
    assert torch.equal(db[cols:], db0[cols:]), "colsum wrote past cols"
    assert _note("colsum", _colsum_err(db[:cols], db0[:cols], view)) < TOL_SUM
    widths = [cols, 1024, 768, 192, 64]
    ys = [big[:, :w] if w <= 3 * cols + 64 else _bf(torch.randn(rows, w, generator=g)).to(cuda) for w in widths]
    dbs0 = [torch.randn(w + 4, generator=g).to(cuda) for w in widths]
    dbs = [t.clone() for t in dbs0]
    n = len(widths)
    dy_p = (ctypes.c_void_p * n)(*[y.data_ptr() for y in ys])
    db_p = (ctypes.c_void_p * n)(*[t.data_ptr() for t in dbs])
    cols_p = (ctypes.c_int * n)(*widths)
    ld_p = (ctypes.c_longlong * n)(*[y.stride(0) for y in ys])
    check(lib().rp_colsum_multi(n, dy_p, cols_p, ld_p, db_p, rows, _stream()), "rp_colsum_multi")
    torch.cuda.synchronize()
    for w, y, t, t0 in zip(widths, ys, dbs, dbs0):
        assert torch.equal(t[w:], t0[w:])
        assert _note("colsum_multi", _colsum_err(t[:w], t0[:w], y)) < TOL_SUM


@pytest.mark.gpu
@pytest.mark.parametrize("d", [64, 256, 512])
@pytest.mark.parametrize("scatter", [0, 1])
@pytest.mark.parametrize("n_dev", [None, 0, 333])
def test_gather_rows(cuda, d, scatter, n_dev):
    """rp_gather_rows: dst[r] = src[idx[r]] (gather) or dst[idx[r]] = src[r] (scatter) for r < min(n_max, *n_dev), bit
    exact; every other dst row keeps its sentinel."""
    T, n_max = 1400, 700
    g = _gen(d + scatter)
    src = _bf(torch.randn(T if not scatter else n_max, d, generator=g)).to(cuda)
    idx = torch.randperm(T, generator=g)[:n_max].to(torch.int32).to(cuda)
    nd = None if n_dev is None else torch.tensor([n_dev], dtype=torch.int32, device=cuda)
    dst = torch.full((n_max if not scatter else T, d), SENT, dtype=torch.bfloat16, device=cuda)
    check(lib().rp_gather_rows(src.data_ptr(), idx.data_ptr(), n_max, None if nd is None else nd.data_ptr(), d,
                               dst.data_ptr(), scatter, _stream()), "rp_gather_rows")
    torch.cuda.synchronize()
    n = n_max if n_dev is None else n_dev
    ref = torch.full_like(dst, SENT)
    if scatter:
        ref[idx[:n].long()] = src[:n]
    else:
        ref[:n] = src[idx[:n].long()]
    assert torch.equal(dst, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("cols", [256, 1024])
def test_dropout_bwd_with_row_mask(cuda, cols):
    """rp_dropout_bwd: out = in * keep / (1-p) (fp32 product rounded to bf16: exact), rows with mask 0 exactly zero;
    the in-place row-mask-only form the legacy backward uses."""
    rows, off = 1400, _site(1, 4) << 40
    g = _gen(cols)
    x = _bf(torch.randn(rows, cols, generator=g)).to(cuda)
    rm = (torch.rand(rows, generator=g) > 0.3).to(torch.uint8).to(cuda)
    ctr = torch.tensor([CTR], dtype=torch.int64, device=cuda)
    out = torch.empty_like(x)
    check(lib().rp_dropout_bwd(x.data_ptr(), out.data_ptr(), rows, cols, rm.data_ptr(), P_DROP, SEED, off, ctr.data_ptr(),
                               _stream()), "rp_dropout_bwd")
    torch.cuda.synchronize()
    keep = keep_draws(SEED + CTR, off, P_DROP, np.arange(rows), cols).to(cuda)
    ks32 = torch.tensor(1.0, dtype=torch.float32) / (1.0 - torch.tensor(P_DROP, dtype=torch.float32))
    ref = _bf(x.float() * keep.float() * ks32.to(cuda) * rm[:, None].float())
    assert torch.equal(out, ref)
    y = x.clone()
    check(lib().rp_dropout_bwd(y.data_ptr(), y.data_ptr(), rows, cols, rm.data_ptr(), 0.0, 0, 0, None, _stream()),
          "rp_dropout_bwd")
    torch.cuda.synchronize()
    assert torch.equal(y, x * rm[:, None].to(x.dtype))


@pytest.mark.gpu
@pytest.mark.parametrize("with_targets", [True, False])
def test_prepare_batch_two_blocks(cuda, with_targets):
    """rp_prepare_batch over T = 2500 tokens (three 1024-token blocks): ids -> int32 with pads and out-of-range ids
    replaced by pad_id, the valid targets (target mask and 0 <= label < n_items) compacted in ascending token order
    with their labels, n_valid exact; entries past n_valid keep their sentinels."""
    T, I, pad_id = 2500, 1000, 0
    g = _gen(T)
    ids = torch.randint(-5, I + 5, (T,), generator=g)
    pad = torch.rand(T, generator=g) > 0.3
    labels = torch.randint(-3, I + 3, (T,), generator=g)
    tmask = (torch.rand(T, generator=g) > 0.6) & pad
    tmask[1000:1100] = False                                     # a run without targets across a block edge
    dev = lambda t: t.to(cuda)  # noqa: E731
    ids32 = torch.full((T,), -7, dtype=torch.int32, device=cuda)
    vidx = torch.full((T,), -7, dtype=torch.int32, device=cuda)
    lab_c = torch.full((T,), -7, dtype=torch.int32, device=cuda)
    nv = torch.full((1,), -7, dtype=torch.int32, device=cuda)
    scratch = torch.zeros((T + 1023) // 1024 + 1, dtype=torch.int32, device=cuda)
    idsd, padd, labd, tmd = dev(ids), dev(pad), dev(labels), dev(tmask)
    check(lib().rp_prepare_batch(idsd.data_ptr(), padd.data_ptr(), labd.data_ptr() if with_targets else None,
                                 tmd.data_ptr() if with_targets else None, T, pad_id, I, ids32.data_ptr(), vidx.data_ptr(),
                                 lab_c.data_ptr(), nv.data_ptr(), scratch.data_ptr(), _stream()), "rp_prepare_batch")
    torch.cuda.synchronize()
    ref_ids = [int(i) if (p and 0 <= i < I) else pad_id for i, p in zip(ids.tolist(), pad.tolist())]
    assert ids32.cpu().tolist() == ref_ids
    if not with_targets:
        assert (vidx == -7).all() and (nv == -7).all()
        return
    valid = [t for t in range(T) if tmask[t] and 0 <= int(labels[t]) < I]
    n = len(valid)
    assert int(nv.item()) == n
    assert vidx[:n].cpu().tolist() == valid
    assert lab_c[:n].cpu().tolist() == [int(labels[t]) for t in valid]
    assert (vidx[n:] == -7).all() and (lab_c[n:] == -7).all()


# ======================================================================================================================
# GPU 5: the BERT4Rec training step at the config-3 shape
# ======================================================================================================================
def _block_name_err(got, ref):
    return block_err(got.reshape(got.shape[0], -1) if got.dim() > 1 else got.view(-1, 1),
                     ref.reshape(ref.shape[0], -1) if ref.dim() > 1 else ref.view(-1, 1))


@pytest.mark.gpu
@pytest.mark.parametrize("drop", [0.0, P_DROP])
@pytest.mark.parametrize("d,H,tied", [(256, 4, False), (256, 2, False), (128, 2, True)])
def test_bert4rec_step_matches_fp64_reference(cuda, d, H, tied, drop):
    """Bert4RecEngine at L = 200 with B = 7 (T = 1400: rp_prepare_batch spans two blocks, 128-row tiles cross sequence
    boundaries), 2 blocks, 2000 items, left-padded short histories and uniform_masker's masked tokens: head_dim 64 runs
    the fused attention backward, head_dim 128 the un-fused one.  With dropout the counter is ticked first and the
    reference takes the ported keep masks at the engine's site numbers.  Checked: loss, hidden states of real rows,
    n_valid, every parameter gradient (mask_emb, head_b, and the tied item_emb's CE + embedding parts), the direction of
    one Adam step, forward_last_hidden on the shifted window against the eval body, and the fused top-10 with the bias."""
    from oracle import bert4rec as ob
    from replay_b200 import ops
    from replay_b200.engine_bert import Bert4RecEngine, BertConfig

    B, L, I, nb = 7, 200, 2000, 2
    P = random_params(I, d, L, nb, tied, seed=d + H)
    ids, pad, tok, labels = step_batch(B, L, I, seed=d + H + 1)
    cfg = BertConfig(n_items=I, d=d, n_heads=H, n_blocks=nb, max_len=L, dropout=drop, tying=tied)
    eng = Bert4RecEngine(cfg, B, L, cuda, seed=SEED)
    assert eng.fused_attn_bwd == (d // H == 64)
    eng.load_canonical(P)
    if drop > 0:
        eng.tick_rng()
    ctr = int(eng.rng_counter.item())
    assert (ctr != 0) == (drop > 0)
    eng.set_batch(ids.to(cuda), pad.to(cuda), tok.to(cuda), labels.to(cuda))
    loss = eng.forward_train()
    torch.cuda.synchronize()
    assert int(eng.n_valid.item()) == int((pad & ~tok).sum())
    hid = eng.x[-1].view(B, L, d).double()
    p0 = eng.export_canonical()
    eng.g32.zero_()
    eng.backward()
    torch.cuda.synchronize()
    G = eng.export_canonical(eng.grads)

    Pe = _map(engine_view(P), lambda k, v: v.to(cuda))
    keeps = engine_keeps(eng.seed + ctr, drop, B, L, d, H, nb, dev=cuda) if drop > 0 else None
    r_loss, r_h, r_G = ref_loss_and_grads(Pe, ids.to(cuda), pad.to(cuda), tok.to(cuda), labels.to(cuda), H, keeps)
    assert _note("step loss rel", abs(loss[0].item() - float(r_loss)) / float(r_loss)) < TOL_LOSS
    assert _note("step hidden block", seq_block_err(hid, r_h, pad.to(cuda))) < TOL_HID
    bad = []
    for name, g in _leaves(G):
        g, r = g.to(cuda).double(), r_G[name]
        if name.endswith("in_b"):
            # a key bias cannot change a softmax: the exact gradient of in_b's key third is 0, the kernels' is round-off
            assert float(r[d:2 * d].norm()) < 1e-9 * float(r.norm())
            assert _note("step grad in_b key third", g[d:2 * d].norm() / r.norm()) < TOL_GRAD, name
            g, r = torch.cat([g[:d], g[2 * d:]]), torch.cat([r[:d], r[2 * d:]])
        e = _note(f"step grad {name.split('.')[-1]}", _block_name_err(g, r))
        if e >= TOL_GRAD:
            bad.append((name, round(e, 4)))
    assert not bad, bad

    # one Adam step (lr 1e-3): every element moves by at most lr, against the sign of the fp64 gradient where it is not ~0
    eng.optimizer_step()
    torch.cuda.synchronize()
    p1 = eng.export_canonical()
    for (name, a), (_, b) in zip(_leaves(p0), _leaves(p1)):
        du, gr = (b - a).to(cuda).double(), r_G[name]
        assert du.abs().max() <= 1.001e-3 + 1e-7, name
        big = gr.abs() > 0.05 * gr.abs().max()
        if big.any():
            agree = float((torch.sign(du[big]) == -torch.sign(gr[big])).double().mean())
            assert agree > 0.98, (name, agree)

    # predict: the shifted window through the eval body (no dropout), then the fused top-10 with the head bias
    eng.load_canonical(P)
    sids, spm, stm = ob.shift_for_predict(ids, pad, pad)   # prediction batches carry token_mask = pad_mask
    eng.set_batch(sids.to(cuda), spm.to(cuda), stm.to(cuda))
    hq = eng.forward_last_hidden()
    torch.cuda.synchronize()
    r_last = ob.bert4rec_body(_map(Pe, lambda k, v: v.double()), sids.to(cuda), spm.to(cuda), stm.to(cuda), H)[:, -1]
    err = ((hq.double() - r_last).norm(dim=-1) / r_last.norm(dim=-1)).max()
    assert _note("last hidden row", err) < TOL_LAST
    W16, bias = eng.head_for_scoring()
    ids_k, sc_k = ops.score_topk(hq, W16, 10, None, bias=bias)
    logits = hq.double() @ W16.double().T + bias[:I].double()
    ref_ids = torch.argsort(-logits, dim=1, stable=True)[:, :10]
    got_sc = torch.gather(logits, 1, ids_k)
    assert (sc_k.double() - got_sc).abs().max() < 1e-4 * (1 + logits.abs().max())
    mism = ids_k != ref_ids
    if mism.any():   # adjudicate in fp64: a swap is only acceptable between scores closer than fp32 accumulation noise
        gap = (got_sc - torch.gather(logits, 1, ref_ids)).abs()
        assert (gap[mism] < 1e-5 * (1 + logits.abs().max())).all(), f"{int(mism.sum())} top-10 mismatches beyond fp32 noise"
