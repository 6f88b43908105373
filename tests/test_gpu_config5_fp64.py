"""SasRecEngine's training step at the config-5 shape (new path, L = 512, d = 512, 8 heads, two blocks, dropout 0.2, a
million items, 32 sequences) against a float64 reference, with every dropout mask ported from csrc/rp_philox.cuh.

At d = 512 no fused block kernel runs: the body is rp_layernorm_fwd / _bwd, rp_gemm with dropout, gate and residual
epilogues, rp_dropout_bwd, and the weight gradients go through SasRecEngine._wgrad (split-K out_mode 3 partials,
rp_reduce_splits, rp_colsum_multi).  At L = 512 the attention backward is un-fused (dO.V^T, rp_attn_softmax_bwd over the
saved probabilities, three batched GEMMs).  The CE head at d = 512 runs the two-pass forward and the chunked
materialised-G backward (wide_bwd in csrc/rp_ce_head.cu).

- the step: loss, x[-1] of the real rows per (sequence, 64-row block), every parameter gradient per 64-row block;
- stage checks on the engine's own bf16 operands of block 0 (whose backward runs last, so its buffers still hold its
  values): every stage recomputed in float64 from the same inputs, so upstream rounding cannot hide an error;
- the d = 512 CE head at 16 384 rows x 1 000 000 items directly, at the chunk edges, both dH split choices, 128-row
  chunks and with stale G rows left by an earlier call;
- the eval body (forward_hidden_all, forward_last_hidden);
- CPU: the chunked reference head against the unchunked one, and every plausible mistake moves a compared quantity by
  >= 10x its tolerance.

The references for a million items run in float64 on the GPU with the CE head in row chunks; the file's largest case
(c5_full) peaks at about 45 GiB of device memory.  Run with -s to print the worst error of each family.
"""
import math

import numpy as np
import pytest
import torch

from fp64_checks import WorstErrors, block_err, ln_bwd_ref, seq_block_err, ulp_err
from sasrec_fp64 import (P_DROP, SEED, _bf, _Case, _gen, _leaves, _map, _ru, _site, ce_head_chunked, engine_keeps,
                         ref_loss_and_grads, ref_loss_and_grads_chunked, sasrec_body_ref, step_batch)

HALF_ULP_SLACK = 2.0 ** -21      # fp32 accumulation slack, times sum_k |a_k b_k|
SENT = -3.25                     # sentinel for memory a kernel must not write
C5_LENGTHS = [512, 511, 257, 256, 255, 129, 64, 1]

# Tolerances.  Each bound is about 3x the worst error observed over every case of this file on one H100 80GB HBM3
# (700 W power limit); the element-wise ones are in units of half a bf16 ulp, where rounding to nearest alone gives 1.
TOL_LOSS = 4e-5          # step: relative loss error; worst seen 1.2e-5 (d 256 / 2 heads)
TOL_HID = 1.8e-2         # step: x[-1] of real rows, per (sequence, 64-row block); worst seen 5.8e-3 (c5_full)
TOL_GRAD = 0.25          # step: parameter gradients, per 64-row block; worst seen 8.3e-2 (b1, d 256 / 2 heads)
TOL_GRAD_TABLE = 0.6     # step: item_emb's gradient at a million items, per 64-row block: a block holds about one input
                         # token's gradient through both blocks, where the smaller catalogs average dozens; worst seen 0.19
TOL_ULP = 3.0            # stage: bf16 outputs one rounding from fp64 of the kernel's own inputs (GEMM epilogues,
                         # rp_dropout_bwd), element-wise; worst seen 1.0
TOL_BWD = 2.5e-2         # stage: LayerNorm backward dx, the attention's Pd / dS / dQ / dK / dV against fp64 of Q, KV and
                         # d_o, per 64-row block norm-relative; worst seen 8.5e-3 (dQ, c5_full)
TOL_LN_GRAD = 7e-7       # stage: dln_w / dln_b, norm-relative; worst seen 2.2e-7
TOL_SPLITK = 5.5e-6      # stage: dW of the split-K weight gradients, per 64-row block norm-relative; worst seen 1.8e-6
TOL_SUM = 4.5e-7         # stage: db (fp32 column sums), norm-relative; worst seen 1.5e-7
TOL_HEAD_LOSS = 2.5e-6   # head: relative loss error; worst seen 8.4e-7
TOL_LSE = 2e-5           # head: lse, absolute; worst seen 6.9e-6
TOL_HEAD_DH = 5e-3       # head: d_hc, per 64-row block; worst seen 1.7e-3
TOL_HEAD_DE = 1.1e-2     # head: d_table, per 64-row block; worst seen 3.6e-3
TOL_EVAL = 1.9e-2        # eval: hidden states per (sequence, 64-row block), last hidden state per row; worst seen 6.3e-3

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


# name: (variant, d, H, L, max_len, I)
_CASES = {"c5": ("new", 512, 8, 512, 512, 3000), "c5_legacy": ("legacy", 512, 8, 512, 512, 3000),
          "d256h2_L512": ("new", 256, 2, 512, 520, 3000), "c5_full": ("new", 512, 8, 512, 512, 1_000_000)}


def _case(name):
    variant, d, H, L, max_len, I = _CASES[name]
    return _Case(variant, d, H, fused=True, L=L, I=I, max_len=max_len)


def _name_err(got, ref):
    return block_err(got.reshape(got.shape[0], -1) if got.dim() > 1 else got.view(-1, 1),
                     ref.reshape(ref.shape[0], -1) if ref.dim() > 1 else ref.view(-1, 1))


def _rel(got, ref):
    return float((got.double() - ref).norm() / ref.norm().clamp_min(1e-300))


def _model_errs(a, b, real):
    """(loss, x[-1], gradient) errors of result ``a`` against ``b`` in units of their tolerances."""
    la, xa, _, Ga = a
    lb, xb, _, Gb = b
    e_loss = abs(float(la - lb)) / abs(float(lb)) / TOL_LOSS
    e_hid = seq_block_err(xa, xb, real) / TOL_HID
    e_grad = max(_name_err(Ga[k], Gb[k]) for k in Gb) / TOL_GRAD
    return e_loss, e_hid, e_grad


def _wgrad_split_rows(T, split):
    """Row ranges of the split-K partials of SasRecEngine._wgrad: split s takes 64-row chunks [C s / split, C (s+1) /
    split) of the C = ceil(T / 64) chunks (csrc/rp_gemm.cu)."""
    C = (T + 63) // 64
    return [(64 * (C * s // split), min(T, 64 * (C * (s + 1) // split))) for s in range(split)]


# ======================================================================================================================
# CPU: the chunked head is the unchunked one; every plausible mistake moves what the GPU tests compare by >= 10x
# ======================================================================================================================
def test_chunked_head_reference_matches_unchunked():
    """ref_loss_and_grads_chunked (the CE head in 7-row chunks, the body's gradients from d(hidden)) equals
    ref_loss_and_grads to 1e-12, with dropout, on the new path and the legacy one."""
    for variant in ("new", "legacy"):
        case = _Case(variant, 64, 2, L=24, I=50)
        B = 3
        P = _map(case.params(21), lambda k, v: v.double())
        ids, pad, labels, tmask = step_batch(B, case.L, case.I, 22, lengths=[24, 13, 1])
        keeps = engine_keeps(SEED + 5, P_DROP, B, case.L, case.cfg)
        args = (P, ids, pad, labels, tmask, case.H, variant, case.lnf_eps, keeps)
        ref = ref_loss_and_grads(*args)
        got = ref_loss_and_grads_chunked(*args, rows=7)
        torch.testing.assert_close(got[0], ref[0], rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(got[1], ref[1], rtol=1e-12, atol=1e-12)
        for k in ref[3]:
            torch.testing.assert_close(got[3][k], ref[3][k], rtol=1e-12, atol=1e-12, msg=k)


_MISTAKES = ("site_off_by_one", "no_scale", "ffn_drop_after_residual", "attn_keep_transposed")


@pytest.fixture(scope="module")
def cpu_c5():
    """The step reference at a CPU-sized config-5 shape: B = 3 (lengths 512, 511, 257), L = 512, d = 512, H = 8,
    I = 500, dropout 0.2."""
    case = _Case("new", 512, 8, L=512, I=500, max_len=512)
    B = 3
    P = case.params(31)
    ids, pad, labels, tmask = step_batch(B, case.L, case.I, 32, lengths=C5_LENGTHS)
    keeps = engine_keeps(SEED + 9, P_DROP, B, case.L, case.cfg)
    args = (ids, pad, labels, tmask, case.H, case.variant, case.lnf_eps)
    return case, P, args, keeps, pad, ref_loss_and_grads(P, *args, keeps)


@pytest.mark.parametrize("mistake", _MISTAKES)
def test_step_tolerances_discriminate_perturbed_references(cpu_c5, mistake):
    """At a CPU-sized config-5 shape and the step tolerances: a dropout site number off by one, the 1/(1-p) scale missing,
    the FFN-output dropout applied after the residual add and the attention keep mask transposed each move the loss,
    x[-1] or a gradient by >= 10x its tolerance."""
    case, P, args, keeps, pad, ref = cpu_c5
    B, L = pad.shape
    if mistake == "site_off_by_one":
        bad = ref_loss_and_grads(P, *args, engine_keeps(SEED + 9, P_DROP, B, L, case.cfg, site_shift=1))
    elif mistake == "no_scale":
        unscaled = {"emb": (keeps["emb"] > 0).double(),
                    "blocks": [{k: (v > 0).double() for k, v in blk.items()} for blk in keeps["blocks"]]}
        bad = ref_loss_and_grads(P, *args, unscaled)
    else:
        bad = ref_loss_and_grads(P, *args, keeps, mistake=mistake)
    errs = _model_errs(bad, ref, pad)
    print(mistake, "loss / x[-1] / grad error in tolerances:", [round(e, 1) for e in errs])
    assert max(errs) >= 10, errs


@pytest.mark.parametrize("T", [7 * 512, 32 * 512])
def test_wgrad_tolerance_discriminates_a_missing_split(T):
    """At the stage checks' T (B = 7 and B = 32 rows of 512) and the split count _wgrad picks on a 132-SM H100 for a
    d x d weight: leaving out any one split's row slice moves dW by >= 10x TOL_SPLITK."""
    d = 512
    split = max(1, min((T + 63) // 64 // 8, (132 + 15) // 16))
    g = _gen(T)
    dY, X = _bf(torch.randn(T, d, generator=g) * 0.3).double(), _bf(torch.randn(T, d, generator=g)).double()
    ref = dY.T @ X
    worst = float("inf")
    for r0, r1 in _wgrad_split_rows(T, split):
        worst = min(worst, block_err(ref - dY[r0:r1].T @ X[r0:r1], ref))
    print(f"T {T}, {split} splits: smallest error in TOL_SPLITK", round(worst / TOL_SPLITK, 1))
    assert worst >= 10 * TOL_SPLITK


def test_head_tolerance_discriminates_a_missing_g_chunk():
    """16 384 rows in the head test's value ranges, G chunks of 4224 rows (the default budget at a million items): d_table
    without one chunk's rows moves by >= 10x TOL_HEAD_DE (at I = 2000, so that the reference fits a CPU)."""
    n, I, d = 16384, 2000, 512
    g = _gen(41)
    h = _bf(torch.randn(n, d, generator=g) * 0.7).double()
    E = _bf(torch.randn(I, d, generator=g) * 0.15).double()
    y = torch.randint(0, I, (n,), generator=g)
    _, _, _, ref = ce_head_chunked(h, E, y, rows=4224)
    _, _, _, bad = ce_head_chunked(h, E, y, rows=4224, skip=(4224, 8448))
    e = block_err(bad, ref)
    print("d_table without G chunk 1, in TOL_HEAD_DE:", round(e / TOL_HEAD_DE, 1))
    assert e >= 10 * TOL_HEAD_DE


# ======================================================================================================================
# GPU 1: the training step against the fp64 reference, and stage checks on block 0's own operands
# ======================================================================================================================
def _run_step(case, B, drop, cuda, seed):
    from replay_b200.engine import EncoderConfig, SasRecEngine

    cfg = EncoderConfig(n_items=case.I, d=case.d, n_heads=case.H, n_blocks=2, max_len=case.max_len, dropout=drop,
                        variant=case.variant)
    P = case.params(seed)
    ids, pad, labels, tmask = step_batch(B, case.L, case.I, seed + 1, lengths=C5_LENGTHS)
    eng = SasRecEngine(cfg, B, case.L, cuda, seed=SEED)
    assert not eng.fused_attn_bwd and not eng.fused_pre_attn and not eng.fused_post_attn_bwd
    assert eng.fused_wgrad == (cfg.dp <= 256)
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
    ref = ref_loss_and_grads_chunked(Pe, ids.to(cuda), pad.to(cuda), labels.to(cuda), tmask.to(cuda), case.H,
                                     case.variant, case.lnf_eps, keeps)
    return eng, keeps, loss, x, G, ref, pad.to(cuda)


def _check_step(case, loss, x, G, ref, pad, tag):
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
        if e >= (TOL_GRAD_TABLE if name == "item_emb" and case.I >= 1_000_000 else TOL_GRAD):
            bad.append((name, round(e, 4)))
    assert not bad, bad


def _heads(t, B, L, H, hd):
    """[T, H * hd] token-major -> float64 [B, H, L, hd]"""
    return t.double().view(B, L, H, hd).transpose(1, 2)


def _tokens(t):
    """[B, H, L, hd] -> [T, H * hd]"""
    B, H, L, hd = t.shape
    return t.transpose(1, 2).reshape(B * L, H * hd)


def _stage_checks(eng, keeps, pad, tag):
    """Block 0's backward, stage by stage, in float64 from the bf16 operands the engine saved or produced (the operands
    of each stage are the engine's own, so each stage is one rounding away from its reference)."""
    cfg, s, a, G = eng.cfg, eng.s, eng.act[0], eng.grads
    B, L, T, d, H, hd = eng.B, eng.L, eng.T, cfg.dp, cfg.n_heads, cfg.head_slot
    assert cfg.hd_valid == 0, "the stage checks assume no padded feature slots"
    D = lambda t: t.double()  # noqa: E731
    W = lambda k: D(eng.params16[f"b0.{k}"])  # noqa: E731
    f = lambda k: D(eng.params[f"b0.{k}"])  # noqa: E731
    valid = torch.ones(d, dtype=torch.bool, device=eng.dev)
    drop = cfg.dropout
    ks = 1.0 / (1.0 - float(np.float32(drop))) if drop > 0 else 1.0
    kb = keeps["blocks"][0] if keeps is not None else None

    def ulp(name, got, A, Bm, res=None):
        """got (bf16) against A . Bm (+ res) in fp64, the fp32 accumulation slack allowed"""
        ref = D(A) @ Bm
        atol = HALF_ULP_SLACK * (D(A).abs() @ Bm.abs()) + 1e-30
        if res is not None:
            ref, atol = ref + D(res), atol + HALF_ULP_SLACK * D(res).abs()
        return _note(f"stage {name} ulp{tag}", ulp_err(got, ref, atol))

    # ---- rp_dropout_bwd of the FFN-output site: d_t = dz * keep / (1 - p), bit pattern of the ported mask
    dz = s["dxb"]                      # the upstream gradient of block 0 (block 1's input gradient)
    if kb is not None:
        keep2 = kb["ffn2"].reshape(T, d)
        assert not bool(((s["d_t"] != 0) & (keep2 == 0)).any()), "d_t not zero where site 2 dropped"
        assert _note(f"stage d_t ulp{tag}", ulp_err(s["d_t"], D(dz) * keep2, 1e-30)) < TOL_ULP
        d_t = s["d_t"]
    else:
        d_t = dz
    # ---- FFN backward: du = (d_t . W2) gated by u != 0 at 1/(1-p); dy = du . W1 + dz
    gate = (a["u"] != 0).double() * ks
    ref = (D(d_t) @ W("w2")) * gate
    atol = HALF_ULP_SLACK * (D(d_t).abs() @ W("w2").abs()) * gate + 1e-30
    assert _note(f"stage du ulp{tag}", ulp_err(s["du"], ref, atol)) < TOL_ULP
    assert ulp("dy", s["dy"], s["du"], W("w1"), dz) < TOL_ULP
    # ---- LayerNorm 2 backward from the saved mean / rstd
    dh_ref, dw_ref, db_ref = ln_bwd_ref(D(s["dy"]), D(a["h"]), f("ln2_w"), D(a["mean2"]), D(a["rstd2"]), valid)
    assert _note(f"stage ln2 dh block{tag}", block_err(s["dh"], dh_ref)) < TOL_BWD
    assert _note(f"stage ln2 dln_w{tag}", _rel(G["b0.ln2_w"], dw_ref)) < TOL_LN_GRAD
    assert _note(f"stage ln2 dln_b{tag}", _rel(G["b0.ln2_b"], db_ref)) < TOL_LN_GRAD
    # ---- out-projection: d_o = dh . Wo
    assert ulp("d_o", s["d_o"], s["dh"], W("out_w")) < TOL_ULP

    # ---- attention: Q, K, V, d_o per head; the saved P now holds Pd, dpd holds dS (rp_attn_softmax_bwd works in place)
    Lp = eng.Lp
    Q, K, V = _heads(a["Q"], B, L, H, hd), _heads(a["KV"][:, :d], B, L, H, hd), _heads(a["KV"][:, d:], B, L, H, hd)
    dO = _heads(s["d_o"], B, L, H, hd)
    Pd_k = a["P"].view(B, H, Lp, Lp)[:, :, :L, :L].double()
    dS_k = s["dpd"].view(B, H, Lp, Lp)[:, :, :L, :L].double()
    scale = 1.0 / math.sqrt(cfg.head_dim)
    causal = torch.tril(torch.ones(L, L, dtype=torch.bool, device=eng.dev))
    vis = (causal[None] if cfg.variant == "legacy" else causal[None] & pad[:, None, :])[:, None]
    sc = (Q @ K.transpose(-1, -2) * scale).masked_fill(~vis, float("-inf"))
    P = torch.softmax(sc, -1).nan_to_num(0.0)
    del sc
    keep = kb["attn"] if kb is not None else torch.ones_like(P)
    if kb is not None:
        assert not bool(((Pd_k != 0) & (keep == 0)).any()), "Pd not zero where the attention site dropped"
    Pd = P * keep
    assert _note(f"stage attn Pd block{tag}", block_err(Pd_k.reshape(-1, L), Pd.reshape(-1, L))) < TOL_BWD
    dPk = (dO @ V.transpose(-1, -2)) * keep
    dS = P * (dPk - (P * dPk).sum(-1, keepdim=True)) * scale
    del dPk
    assert _note(f"stage attn dS block{tag}", block_err(dS_k.reshape(-1, L), dS.reshape(-1, L))) < TOL_BWD
    # the three batched GEMMs, from the kernel's own dS / Pd: one rounding each
    for name, got, A, Bm in (("dQ", s["dQ"], dS_k, K), ("dK", s["dKV"][:, :d], dS_k.transpose(-1, -2), Q),
                             ("dV", s["dKV"][:, d:], Pd_k.transpose(-1, -2), dO)):
        ref, atol = _tokens(A @ Bm), _tokens(A.abs() @ Bm.abs()) * HALF_ULP_SLACK + 1e-30
        assert _note(f"stage attn {name} ulp{tag}", ulp_err(got, ref, atol)) < TOL_ULP
    # and from fp64 dS / Pd of Q, KV and d_o
    for name, got, ref in (("dQ", s["dQ"], dS @ K), ("dK", s["dKV"][:, :d], dS.transpose(-1, -2) @ Q),
                           ("dV", s["dKV"][:, d:], Pd.transpose(-1, -2) @ dO)):
        assert _note(f"stage attn {name} block{tag}", block_err(got, _tokens(ref))) < TOL_BWD
    del P, Pd, dS, Pd_k, dS_k

    # ---- Q projection + LayerNorm 1 backward + K | V projection
    x0 = eng.x[0]
    assert ulp("dq_in", s["dq_in"], s["dQ"], W("in_w")[:d], s["dh"]) < TOL_ULP
    t_ref, dw1, db1 = ln_bwd_ref(D(s["dq_in"]), D(x0), f("ln1_w"), D(a["mean1"]), D(a["rstd1"]), valid)
    assert _note(f"stage ln1 dx block{tag}", block_err(s["tmp"], t_ref)) < TOL_BWD
    assert _note(f"stage ln1 dln_w{tag}", _rel(G["b0.ln1_w"], dw1)) < TOL_LN_GRAD
    assert _note(f"stage ln1 dln_b{tag}", _rel(G["b0.ln1_b"], db1)) < TOL_LN_GRAD
    assert ulp("dx", s["dxa"], s["dKV"], W("in_w")[d:], s["tmp"]) < TOL_ULP

    # ---- the five (dY, X) -> dW, db pairs of the block
    g = lambda k: G[f"b0.{k}"]  # noqa: E731
    pairs = [("w2", d_t, a["u"], g("w2"), g("b2")), ("w1", s["du"], a["y"], g("w1"), g("b1")),
             ("out_w", s["dh"], a["O"], g("out_w"), g("out_b")), ("in_w q", s["dQ"], a["q_in"], g("in_w")[:d], g("in_b")[:d]),
             ("in_w kv", s["dKV"], x0, g("in_w")[d:], g("in_b")[d:])]
    for name, dY, X, dW, db in pairs:
        assert _note(f"stage wgrad {name} dW block{tag}", block_err(dW, D(dY).T @ D(X))) < TOL_SPLITK, name
        assert _note(f"stage wgrad {name} db{tag}", _rel(db, D(dY).sum(0))) < TOL_SUM, name


@pytest.mark.gpu
@pytest.mark.parametrize("name,drop", [("c5", 0.0), ("c5", P_DROP), ("c5_legacy", P_DROP), ("d256h2_L512", P_DROP)])
def test_step_matches_fp64_reference(cuda, name, drop):
    """SasRecEngine with two blocks at L = 512, B = 7 left-padded histories (lengths 512, 511, 257, 256, 255, 129, 64),
    I = 3000, the dropout counter ticked once: config 5 (d 512, 8 heads, max_len 512) with and without dropout, the legacy
    model at that shape (row mask, causal-only attention, positions from the front), and d 256 / 2 heads (head_dim 128,
    rp_wgrad_group) with max_len 520.  Loss, x[-1] of the real rows and every parameter gradient against the fp64
    reference under the ported masks; on the new-path d = 512 cases, block 0's stages against fp64 of its own operands."""
    case = _case(name)
    eng, keeps, loss, x, G, ref, pad = _run_step(case, 7, drop, cuda, seed=case.d + case.H + int(drop * 10))
    _check_step(case, loss, x, G, ref, pad, "")
    if case.variant == "new" and case.d == 512:
        _stage_checks(eng, keeps, pad, "")


@pytest.mark.gpu
def test_c5_full_step_matches_fp64_reference(cuda):
    """Config 5 exactly as bench.py trains it: B = 32 (T = 16 384), L = 512, d = 512, 8 heads, I = 1 000 000, dropout
    0.2, max_len 512, lengths 512, 511, 257, 256, 255, 129, 64, 1 repeated; the reference in float64 on the GPU with its
    CE head in 512-row chunks.  Then block 0's stages against fp64 of its own operands."""
    case = _case("c5_full")
    eng, keeps, loss, x, G, ref, pad = _run_step(case, 32, P_DROP, cuda, seed=55)
    _check_step(case, loss, x, G, ref, pad, " full")
    del ref, G
    torch.cuda.empty_cache()
    _stage_checks(eng, keeps, pad, " full")
    del eng
    torch.cuda.empty_cache()


# ======================================================================================================================
# GPU 2: the d = 512 CE head at a million items
# ======================================================================================================================
_HEAD_NV = [16384, 4225, 15001, 4224, 129, 0]   # 4225 right after 16384: the skipped G tiles hold that call's rows


@pytest.mark.gpu
def test_ce_head_wide_million_items(cuda, monkeypatch):
    """ops.CEHeadState with capacity 16 384, I = 1 000 000, d = 512: loss, lse, d_hc and d_table[:I] against fp64 at
    n_valid 16 384, 4225 (a G chunk of the default budget is 4224 rows), 15 001, 4224, 129 and 0; n_valid_hint 0 and
    exact (different dH split counts); the default G budget and one of 128-row chunks.  Every call after the first finds
    G rows of earlier calls in the tiles it skips.  Rows of hc from n_valid to the next 128-row edge are zero (as the
    engine's compaction leaves them), rows past it hold finite junk; the pad row of d_table keeps its sentinel."""
    from replay_b200 import ops

    cap, I, d = 16384, 1_000_000, 512
    gd = torch.Generator(device=cuda).manual_seed(17)
    hc_all = _bf(torch.randn(cap, d, generator=gd, device=cuda) * 0.7)
    table = _bf(torch.randn(I, d, generator=gd, device=cuda) * 0.15)
    labels = torch.randint(0, I, (cap,), generator=gd, device=cuda)
    labels32 = labels.int()
    budgets = {"default": None, "128-row chunks": str(128 * I * 2)}
    states = {}
    for k, b in budgets.items():
        if b is None:
            monkeypatch.delenv("RP_CE_WIDE_G_BYTES", raising=False)
        else:
            monkeypatch.setenv("RP_CE_WIDE_G_BYTES", b)
        states[k] = ops.CEHeadState(cap, I, d, cuda)
    E = table.double()
    d_hc = torch.zeros(cap, d, device=cuda, dtype=torch.bfloat16)
    d_tab = torch.empty(I + 1, d, device=cuda, dtype=torch.float32)
    for nv in _HEAD_NV:
        hc = hc_all.clone()
        hc[nv:_ru(nv, 128)] = 0
        nv_t = torch.tensor([nv], dtype=torch.int32, device=cuda)
        ref = ce_head_chunked(hc[:nv].double(), E, labels[:nv], rows=512) if nv else None
        for k, b in budgets.items():
            if b is None:
                monkeypatch.delenv("RP_CE_WIDE_G_BYTES", raising=False)
            else:
                monkeypatch.setenv("RP_CE_WIDE_G_BYTES", b)
            for hint in sorted({0, nv}):
                tag = f"n_valid {nv}, hint {hint}, {k}"
                d_hc.fill_(SENT)
                d_tab.fill_(SENT)
                out = ops.ce_head_fwd(states[k], hc, table, labels32, nv_t, d_hc=d_hc, n_valid_hint=hint)
                ops.ce_head_bwd(states[k], hc, table, labels32, nv_t, d_hc, d_tab, n_valid_hint=hint)
                torch.cuda.synchronize()
                assert bool((d_tab[I] == SENT).all()), f"{tag}: pad row of d_table written"
                if nv == 0:
                    assert bool((d_tab[:I] == 0).all()), f"{tag}: d_table must be 0 without targets"
                    continue
                loss, lse, dh, dE = ref
                assert _note("head loss rel", abs(float(out[0]) - float(loss)) / float(loss)) < TOL_HEAD_LOSS, tag
                assert _note("head lse abs", (states[k].lse[:nv].double() - lse).abs().max()) < TOL_LSE, tag
                assert _note("head d_hc block", block_err(d_hc[:nv], dh)) < TOL_HEAD_DH, tag
                assert _note("head d_table block", block_err(d_tab[:I], dE)) < TOL_HEAD_DE, tag
        del ref
    del E, states
    torch.cuda.empty_cache()


# ======================================================================================================================
# GPU 3: the eval body
# ======================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["c5", "c5_legacy"])
def test_eval_hidden_states_match_fp64_reference(cuda, name):
    """forward_hidden_all (every position) and forward_last_hidden (the last position, through the last-row path of the
    final block) at the config-5 shape, B = 32 left-padded histories, against the fp64 eval body."""
    from replay_b200.engine import EncoderConfig, SasRecEngine

    case = _case(name)
    B, L = 32, case.L
    cfg = EncoderConfig(n_items=case.I, d=case.d, n_heads=case.H, n_blocks=2, max_len=case.max_len, dropout=P_DROP,
                        variant=case.variant)
    P = case.params(61)
    ids, pad, _, _ = step_batch(B, L, case.I, 62, lengths=C5_LENGTHS)
    eng = SasRecEngine(cfg, B, L, cuda, seed=SEED, with_grad=False)
    eng.load_canonical(P)
    eng.set_batch(ids.to(cuda), pad.to(cuda))
    hid = eng.unpad_features(eng.forward_hidden_all()).view(B, L, case.d).double()
    hq = eng.unpad_features(eng.forward_last_hidden()).double()
    torch.cuda.synchronize()
    with torch.no_grad():
        _, r_hid = sasrec_body_ref(_map(P, lambda k, v: v.to(cuda).double()), ids.to(cuda), pad.to(cuda), case.H,
                                   case.variant, case.lnf_eps)
    assert _note(f"eval hidden block {name}", seq_block_err(hid, r_hid, pad.to(cuda))) < TOL_EVAL
    assert _note(f"eval last hidden row {name}", block_err(hq, r_hid[:, -1], blk=1)) < TOL_EVAL
