"""The packed-row SASRec body (SasRecEngine.packed_body: each sequence's live suffix only, stored back to back) kernel by
kernel against float64 references and against the padded kernels, with the stale rows poisoned.

Entry points: rp_row_plan, rp_embed_fwd_rows / rp_embed_bwd_rows, rp_ln_qkv_fused_rows / rp_pre_attn_bwd_rows,
rp_post_attn_train_rows / rp_post_attn_bwd_rows, rp_wgrad_group_rows and the packed mode of rp_attn_fwd / rp_attn_bwd
(seq_first / seq_off), then the engine's packed training step against the fp64 model.

Conventions of every kernel case:
- rows past the packed count are stale, possibly not finite: every float input row there is NaN, +Inf or -Inf (varied per
  case), index arrays there hold valid but wrong token ids (a kernel that reads them gives wrong numbers, not a fault);
- output rows past the packed count are pre-filled with a sentinel and must stay untouched, accumulated outputs finite;
- outputs that do not depend on summation order (the embedding, LN1 + QKV, the post-attention forward, the per-row
  backward outputs, attention O, m_save, inv_sum, dQ, dK, dV, and rp_wgrad_group at the padded kernel's row count) are
  bitwise equal to the padded kernel's row of the same token;
- the tolerances are those of test_gpu_sasrec_body.py and test_gpu_attention.py.
Run with -s to print the worst error of each family.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

import sampled_reference
import test_gpu_sasrec_body as sasrec_body
from dropout_stream import drop_keep, keep_draws
from fp64_checks import WorstErrors, block_err, ln_bwd_ref, ln_ref, ulp_err
from replay_b200._lib import AttnBwdDesc, AttnDesc, WgradPair, check, lib
from test_gpu_attention import BIG, OFF, SENT, TOL_INV_REL, TOL_M_ABS, TOL_M_REL, TOL_O
from test_gpu_attention import _case, _check_grads, _d_out, _heads, attn_grads_given_o, attn_ref, visibility
from test_gpu_attention import block_err as head_block_err
from test_gpu_packed_body import _windows, expected_plan
from sasrec_fp64 import (CTR, EPS, P_DROP, SEED, _bf, _Case, _ks, _leaves, _map, _site, engine_keeps, ref_loss_and_grads,
                         sasrec_ref, step_batch)
from test_gpu_sasrec_body import (HALF_ULP_SLACK, TOL_BWD, TOL_LN_GRAD, TOL_SPLITK, TOL_SUM, TOL_ULP, _assert_keep_pattern,
                                  _check_stats, _check_step, _ln_fwd_atol, _post_attn_inputs, _vec, _weights, _x_rows,
                                  post_attn_bwd_ref, post_attn_train_ref)

POISON = (float("nan"), float("inf"), float("-inf"))

_worst = WorstErrors()
_note = _worst.note


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    # the step checks of test_gpu_sasrec_body note their errors there, tagged " packed"
    _worst.worst.update({k: v for k, v in sasrec_body._worst.worst.items() if "packed" in k})
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


def _p(t):
    return None if t is None else t.data_ptr()


def _poison(t, n, k):
    """Rows [n:) of ``t`` <- NaN, +Inf or -Inf (``k`` picks which)."""
    t[n:] = POISON[k % 3]
    return t


def _sent(rows, cols, dev, dtype=torch.bfloat16):
    """A [rows + 64, cols] (or [rows + 64]) output pre-filled with the sentinel."""
    return torch.full((rows + 64, cols) if cols else (rows + 64,), SENT, dtype=dtype, device=dev)


def _untouched(buf, n, what):
    assert (buf[n:] == SENT).all(), f"{what} written past the packed row count"


def _ctr(dev):
    return torch.tensor([CTR], dtype=torch.int64, device=dev)


# ----------------------------------------------------------------------------------------------------------------------
# the row plan
# ----------------------------------------------------------------------------------------------------------------------
def plan_batch(B, L, n_items, seed):
    """Masks of five kinds of sequence: 0 left-padded with a valid target on the row before its first real token, 1
    interior holes with a label -1 under a set target mask before the first real token, 2 empty with labels n_items
    under a set target mask, 3 full, 4 left-padded with a label n_items on the row before the first real token."""
    g = _gen(seed)
    kind = torch.randint(0, 5, (B,), generator=g)
    lens = torch.randint(0, L + 1, (B,), generator=g)
    pos = torch.arange(L)
    start = (L - lens)[:, None]
    pad = pos[None] >= start
    holes = torch.rand(B, L, generator=g) < 0.25
    pad = torch.where((kind == 1)[:, None], pad & ~holes, pad)
    pad[kind == 2] = False
    pad[kind == 3] = True
    labels = torch.randint(0, n_items, (B, L), generator=g)
    tmask = pad & (torch.rand(B, L, generator=g) < 0.8)
    before = pos[None] == start - 1                        # the row before the first real token
    tmask |= before & ((kind == 0) | (kind == 4) | (kind == 1))[:, None]
    labels = torch.where(before & (kind == 4)[:, None], torch.full_like(labels, n_items), labels)
    labels = torch.where(before & (kind == 1)[:, None], torch.full_like(labels, -1), labels)
    junk = (kind == 2)[:, None] & (torch.rand(B, L, generator=g) < 0.3)
    tmask |= junk
    labels = torch.where(junk, torch.full_like(labels, n_items), labels)
    return pad, labels, tmask


def device_plan(pad, labels, tmask, n_items, dev, with_valid=True):
    """rp_row_plan on the device -> dict of its outputs (row_tok / valid_rows pre-filled with valid but wrong rows)."""
    B, L = pad.shape
    T = B * L
    sel = (tmask & (labels >= 0) & (labels < n_items)) if tmask is not None else torch.zeros_like(pad)
    valid_idx = sel.reshape(-1).nonzero()[:, 0].to(torch.int32)
    out = {"seq_first": torch.full((B,), L // 2, dtype=torch.int32, device=dev),
           "seq_off": torch.zeros(B, dtype=torch.int32, device=dev),
           "n_rows": torch.full((1,), -1, dtype=torch.int32, device=dev),
           "row_tok": (T - 1 - torch.arange(T, dtype=torch.int32)).to(dev),
           "valid_rows": torch.zeros(max(T, 1), dtype=torch.int32, device=dev)}
    vi = torch.zeros(max(T, 1), dtype=torch.int32)
    vi[: valid_idx.numel()] = valid_idx
    vi, nv = vi.to(dev), torch.tensor([valid_idx.numel()], dtype=torch.int32, device=dev)
    pad_d = pad.to(dev).contiguous()
    lab_d = labels.to(dev).contiguous() if tmask is not None else None
    tm_d = tmask.to(dev).contiguous() if tmask is not None else None
    check(lib().rp_row_plan(pad_d.data_ptr(), _p(lab_d), _p(tm_d), B, L, n_items, vi.data_ptr() if with_valid else None,
                            nv.data_ptr() if with_valid else None, out["seq_first"].data_ptr(), out["seq_off"].data_ptr(),
                            out["n_rows"].data_ptr(), out["row_tok"].data_ptr(),
                            out["valid_rows"].data_ptr() if with_valid else None, _stream()), "rp_row_plan")
    torch.cuda.synchronize()
    out["P"] = int(out["n_rows"][0])
    out["valid_idx"], out["n_valid"] = valid_idx, valid_idx.numel()
    return out


def check_plan(pl, pad, labels, tmask, n_items, with_valid=True):
    B, L = pad.shape
    T = B * L
    first, off, row_tok, P = expected_plan(pad, tmask if tmask is not None else torch.zeros_like(pad),
                                           labels if labels is not None else torch.zeros(B, L, dtype=torch.long), n_items)
    assert pl["P"] == P
    assert torch.equal(pl["seq_first"].cpu().long(), first.long())
    assert torch.equal(pl["seq_off"].cpu().long(), off.long())
    rt = pl["row_tok"].cpu().long()
    assert torch.equal(rt[:P], row_tok.long())
    assert torch.equal(rt[P:], (T - 1 - torch.arange(T))[P:]), "row_tok written past the packed row count"
    if with_valid:
        nv = pl["n_valid"]
        vr = pl["valid_rows"][:nv].cpu().long()
        assert torch.equal(rt[vr], pl["valid_idx"].long()), "a valid target does not map to the packed row of its token"
    return P


_PLAN_B = [1, 1023, 1024, 1025, 3000]
_PLAN_L = [1, 31, 32, 33, 64, 200, 256]


@pytest.mark.gpu
@pytest.mark.parametrize("L", _PLAN_L)
@pytest.mark.parametrize("B", _PLAN_B)
def test_row_plan_matches_host_restatement(cuda, B, L):
    """rp_row_plan at batches around its 1024-sequence scan slab, lengths around the warp's 32 positions: first kept
    position, packed offsets, row count, token of every packed row, packed row of every valid target; labels -1 and
    n_items under a set target mask keep nothing."""
    I = 500
    pad, labels, tmask = plan_batch(B, L, I, seed=B * 7 + L)
    check_plan(device_plan(pad, labels, tmask, I, cuda), pad, labels, tmask, I)


@pytest.mark.gpu
@pytest.mark.parametrize("B,L", [(1, 1), (1025, 33), (3000, 200)])
def test_row_plan_all_empty_all_full_and_null_pointers(cuda, B, L):
    """An all-empty batch (n_rows 0, nothing in row_tok written), an all-full batch (n_rows B * L), no target mask (the
    real tokens alone) and no valid_idx (valid_rows not written)."""
    I = 500
    empty = torch.zeros(B, L, dtype=torch.bool)
    labels = torch.full((B, L), I, dtype=torch.long)
    pl = device_plan(empty, labels, empty | True, I, cuda)   # every target invalid (label n_items)
    assert check_plan(pl, empty, labels, empty | True, I) == 0
    full = torch.ones(B, L, dtype=torch.bool)
    labels = torch.randint(0, I, (B, L), generator=_gen(B))
    assert check_plan(device_plan(full, labels, full, I, cuda), full, labels, full, I) == B * L
    pad, labels, tmask = plan_batch(B, L, I, seed=B + L)
    check_plan(device_plan(pad, None, None, I, cuda), pad, None, None, I)
    pl = device_plan(pad, labels, tmask, I, cuda, with_valid=False)
    check_plan(pl, pad, labels, tmask, I, with_valid=False)
    assert (pl["valid_rows"] == 0).all(), "valid_rows written without valid_idx"


# ----------------------------------------------------------------------------------------------------------------------
# embedding
# ----------------------------------------------------------------------------------------------------------------------
_EMB_LENGTHS = [0, 1, 63, 64, 65, 128, 129, 200, 0, 37, 199]


@pytest.mark.gpu
@pytest.mark.parametrize("drop", [0.0, P_DROP])
@pytest.mark.parametrize("d", [64, 128])
def test_embed_rows(cuda, d, drop):
    """rp_embed_fwd_rows: packed row r is rp_embed_fwd's row row_tok[r] bit for bit, and (E[id] * sqrt(d) + pos) * keep
    of that token element-wise against fp64.  rp_embed_bwd_rows with NaN / Inf dx rows past n_rows: d_table and d_pos
    against fp64 sums over exactly the packed rows (dropout keyed by the token), no gradient to the pad id, none to the
    positions before any sequence's first kept row."""
    L, I, pos0 = 200, 3000, 10
    ids, pad, labels, tmask = _windows(_EMB_LENGTHS, L, I, seed=d + int(drop * 10))
    B, T = pad.shape[0], pad.numel()
    pl = device_plan(pad, labels, tmask, I, cuda)
    P = check_plan(pl, pad, labels, tmask, I)
    g = _gen(d)
    table = _bf(torch.randn(I + 1, d, generator=g) * 0.5).to(cuda)
    pos = (torch.randn(L + pos0, d, generator=g) * 0.5).to(cuda)
    ids32 = ids.reshape(-1).to(torch.int32).to(cuda)
    pad_d = pad.reshape(-1).to(cuda)
    ctr = _ctr(cuda)
    scale = math.sqrt(d)
    x_pad = torch.empty(T, d, dtype=torch.bfloat16, device=cuda)
    check(lib().rp_embed_fwd(table.data_ptr(), pos.data_ptr(), ids32.data_ptr(), pad_d.data_ptr(), T, L, d, pos0, scale, 0, drop,
                             SEED, 0, ctr.data_ptr(), x_pad.data_ptr(), _stream()), "rp_embed_fwd")
    x = _sent(T, d, cuda)
    check(lib().rp_embed_fwd_rows(table.data_ptr(), pos.data_ptr(), ids32.data_ptr(), pad_d.data_ptr(), pl["row_tok"].data_ptr(),
                                  pl["n_rows"].data_ptr(), T, L, d, pos0, scale, 0, drop, SEED, 0, ctr.data_ptr(), x.data_ptr(),
                                  _stream()), "rp_embed_fwd_rows")
    torch.cuda.synchronize()
    _untouched(x, P, "x")
    tok = pl["row_tok"][:P].long()
    assert torch.equal(x[:P], x_pad[tok]), "packed embedding rows differ from the padded kernel's"
    tok_c = tok.cpu()
    ks = _ks(drop) if drop > 0 else 1.0
    keep = keep_draws(SEED + CTR, 0, drop, tok_c.numpy(), d).double().to(cuda) * ks if drop > 0 else 1.0
    e = table.double()[ids32.long()[tok]] * scale
    pp = pos.double()[pos0 + tok % L]
    assert _note("embed fwd ulp", ulp_err(x[:P], (e + pp) * keep, 1.2e-7 * (e.abs() + pp.abs()) * ks + 1e-30)) < TOL_ULP

    # ---- backward: dx rows past n_rows are not finite
    dx = _poison(_bf(torch.randn(T, d, generator=g)).to(cuda), P, d)
    d_table = torch.zeros(I + 1, d, device=cuda)
    d_pos = torch.zeros(L + pos0, d, device=cuda)
    check(lib().rp_embed_bwd_rows(dx.data_ptr(), ids32.data_ptr(), pad_d.data_ptr(), pl["row_tok"].data_ptr(),
                                  pl["n_rows"].data_ptr(), pl["seq_first"].data_ptr(), pl["seq_off"].data_ptr(), B, L, d, I, pos0,
                                  scale, 0, drop, SEED, 0, ctr.data_ptr(), d_table.data_ptr(), d_pos.data_ptr(), _stream()),
          "rp_embed_bwd_rows")
    torch.cuda.synchronize()
    assert torch.isfinite(d_table).all() and torch.isfinite(d_pos).all(), "a stale dx row reached a gradient"
    gx = dx[:P].double() * keep
    idr = ids32.long()[tok]
    on = idr != I
    rt = torch.zeros(I + 1, d, dtype=torch.float64, device=cuda).index_add_(0, idr[on], gx[on] * scale)
    rp = torch.zeros(L + pos0, d, dtype=torch.float64, device=cuda).index_add_(0, pos0 + tok % L, gx)
    assert (d_table[I] == 0).all(), "the pad id got a gradient"
    first_kept = int(pl["seq_first"].min())
    assert (d_pos[: pos0 + first_kept] == 0).all(), "a position before every sequence's first kept row got a gradient"
    assert _note("embed bwd d_table", block_err(d_table, rt)) < TOL_SUM
    assert _note("embed bwd d_pos", block_err(d_pos, rp)) < TOL_SUM


# ----------------------------------------------------------------------------------------------------------------------
# rp_ln_qkv_fused_rows + rp_pre_attn_bwd_rows
# ----------------------------------------------------------------------------------------------------------------------
T_CAP = 300                                  # two whole 128-row tiles and a ragged third
_ROW_COUNTS = [0, 1, 63, 64, 65, 127, 128, 129, T_CAP - 1, T_CAP]
_FEAT = [(128, 0), (128, 32), (64, 50)]      # (d, hd_valid)


@pytest.mark.gpu
@pytest.mark.parametrize("d,hdv", _FEAT)
@pytest.mark.parametrize("n", _ROW_COUNTS)
def test_ln_qkv_rows_and_pre_attn_bwd_rows(cuda, n, d, hdv):
    """rp_ln_qkv_fused_rows over the first n of T rows (the rest NaN / Inf): q_in, Q, KV, mean, rstd bitwise equal to
    rp_ln_qkv_fused over those n rows and element-wise against fp64, nothing written past n.  rp_pre_attn_bwd_rows with
    every input row past n poisoned: dx bitwise equal to rp_pre_attn_bwd's, dln_w / dln_b the fp64 sums over exactly
    the n live rows, accumulated onto preset values."""
    T = T_CAP
    x, v, g = _x_rows(T, d, hdv, 1000 + n + d + hdv, cuda)
    _poison(x, n, n)
    vc = v.cpu()
    v3 = torch.cat([vc] * 3)
    w_in = _weights(3 * d, d, v3, vc, g).to(cuda)
    b_in = _vec(3 * d, v3, g, 0.1).to(cuda)
    lw, lb = _vec(d, vc, g, 0.2, 1.0).to(cuda), _vec(d, vc, g, 0.1).to(cuda)
    n_dev = torch.tensor([n], dtype=torch.int32, device=cuda)
    outs = {"q_in": _sent(T, d, cuda), "Q": _sent(T, d, cuda), "KV": _sent(T, 2 * d, cuda),
            "mean": _sent(T, 0, cuda, torch.float32), "rstd": _sent(T, 0, cuda, torch.float32)}
    check(lib().rp_ln_qkv_fused_rows(x.data_ptr(), lw.data_ptr(), lb.data_ptr(), EPS, w_in.data_ptr(), b_in.data_ptr(), T, d,
                                     *[outs[k].data_ptr() for k in ("q_in", "Q", "KV", "mean", "rstd")], hdv, n_dev.data_ptr(),
                                     _stream()), "rp_ln_qkv_fused_rows")
    torch.cuda.synchronize()
    for k, b in outs.items():
        _untouched(b, n, k)
    if n:
        ref = {"q_in": _sent(n, d, cuda), "Q": _sent(n, d, cuda), "KV": _sent(n, 2 * d, cuda),
               "mean": _sent(n, 0, cuda, torch.float32), "rstd": _sent(n, 0, cuda, torch.float32)}
        check(lib().rp_ln_qkv_fused(x.data_ptr(), lw.data_ptr(), lb.data_ptr(), EPS, w_in.data_ptr(), b_in.data_ptr(), n, d,
                                    *[ref[k].data_ptr() for k in ("q_in", "Q", "KV", "mean", "rstd")], hdv, _stream()),
              "rp_ln_qkv_fused")
        torch.cuda.synchronize()
        for k in outs:
            assert torch.equal(outs[k][:n], ref[k][:n]), f"{k} differs from the padded kernel's"
        X, W, Bv = x[:n].double(), w_in.double(), b_in.double()
        y_ref, m_ref, r_ref = ln_ref(X, lw.double(), lb.double(), EPS, v)
        q_in = outs["q_in"][:n]
        assert _note("ln_qkv q_in ulp", ulp_err(q_in, y_ref, _ln_fwd_atol(X, m_ref, r_ref, lw.double()))) < TOL_ULP
        _check_stats(outs["mean"][:n], outs["rstd"][:n], m_ref, r_ref, x[:n], v)
        q16 = q_in.double()
        Q_ref = q16 @ W[:d].T + Bv[:d]
        assert _note("ln_qkv Q ulp", ulp_err(outs["Q"][:n], Q_ref,
                                             HALF_ULP_SLACK * (q16.abs() @ W[:d].abs().T + Bv[:d].abs()) + 1e-30)) < TOL_ULP
        KV_ref = X @ W[d:].T + Bv[d:]
        assert _note("ln_qkv KV ulp", ulp_err(outs["KV"][:n], KV_ref,
                                              HALF_ULP_SLACK * (X.abs() @ W[d:].abs().T + Bv[d:].abs()) + 1e-30)) < TOL_ULP

    # ---- rp_pre_attn_bwd_rows: the statistics' stale rows are poisoned too
    mean, rstd = _poison(outs["mean"], n, n + 1), _poison(outs["rstd"], n, n + 2)
    gb = _gen(3 * n + d)
    dQ = _poison(_bf(torch.randn(T, d, generator=gb) * 0.3 * vc).to(cuda), n, n + 1)
    dKV = _poison(_bf(torch.randn(T, 2 * d, generator=gb) * 0.3 * torch.cat([vc, vc])).to(cuda), n, n + 2)
    dh = _poison(_bf(torch.randn(T, d, generator=gb) * 0.3 * vc).to(cuda), n, n)
    dw0, db0 = torch.randn(d, generator=gb).to(cuda), torch.randn(d, generator=gb).to(cuda)
    dw, db = dw0.clone(), db0.clone()
    dx = _sent(T, d, cuda)
    args = (dQ.data_ptr(), dKV.data_ptr(), dh.data_ptr(), x.data_ptr(), mean.data_ptr(), rstd.data_ptr(), lw.data_ptr(),
            w_in.data_ptr())
    check(lib().rp_pre_attn_bwd_rows(*args, T, d, dx.data_ptr(), dw.data_ptr(), db.data_ptr(), hdv, n_dev.data_ptr(), _stream()),
          "rp_pre_attn_bwd_rows")
    torch.cuda.synchronize()
    _untouched(dx, n, "dx")
    assert torch.isfinite(dw).all() and torch.isfinite(db).all(), "a stale row reached dln_w / dln_b"
    if n == 0:
        assert torch.equal(dw, dw0) and torch.equal(db, db0)
        return
    dx2 = _sent(n, d, cuda)
    dw2, db2 = dw0.clone(), db0.clone()
    check(lib().rp_pre_attn_bwd(*args, n, d, dx2.data_ptr(), dw2.data_ptr(), db2.data_ptr(), hdv, _stream()), "rp_pre_attn_bwd")
    torch.cuda.synchronize()
    assert torch.equal(dx[:n], dx2[:n]), "dx differs from the padded kernel's"
    X, W = x[:n].double(), w_in.double()
    _, m_ref, r_ref = ln_ref(X, lw.double(), lb.double(), EPS, v)
    dq = dQ[:n].double() @ W[:d] + dh[:n].double()
    t, dw_ref, db_ref = ln_bwd_ref(dq, X, lw.double(), m_ref, r_ref, v)
    assert _note("pre_attn_bwd dx block", block_err(dx[:n], dKV[:n].double() @ W[d:] + t)) < TOL_BWD
    assert _note("pre_attn_bwd dln_w", block_err((dw - dw0).double().view(-1, 1), dw_ref.view(-1, 1))) < TOL_LN_GRAD
    assert _note("pre_attn_bwd dln_b", block_err((db - db0).double().view(-1, 1), db_ref.view(-1, 1))) < TOL_LN_GRAD


# ----------------------------------------------------------------------------------------------------------------------
# rp_post_attn_train_rows + rp_post_attn_bwd_rows
# ----------------------------------------------------------------------------------------------------------------------
def _tokens(T, seed):
    """Row tokens of a packed batch in a token space of 2T + 1: increasing, with gaps, and row_tok[r] > r (a kernel that
    keys its dropout by the packed row never draws the token's mask by accident)."""
    return (torch.randperm(2 * T, generator=_gen(seed))[:T].sort().values + 1).to(torch.int32)


def _scatter(t, tok, Tp):
    out = torch.zeros((Tp,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    out[tok] = t
    return out


_POST = [(128, 0, P_DROP), (64, 50, P_DROP), (128, 32, 0.0)]   # (d, hd_valid, dropout)


@pytest.mark.gpu
@pytest.mark.parametrize("d,hdv,drop", _POST)
@pytest.mark.parametrize("n", _ROW_COUNTS)
def test_post_attn_train_rows_and_bwd_rows(cuda, n, d, hdv, drop):
    """rp_post_attn_train_rows over the first n of T rows, O / q_in rows past n poisoned, dropout keyed by row_tok: h, y,
    u, mean, rstd, out bitwise equal to rp_post_attn_train's rows of the same tokens (the rows scattered into a padded
    layout), element-wise against fp64 under masks drawn for the tokens; an fp64 reference keyed by the packed row r
    instead is > 10x the tolerance away.  rp_post_attn_bwd_rows with dz / u / h / statistics rows past n poisoned: d_t, du,
    dh, d_o bitwise equal to the padded kernel's rows, per 64-row block against fp64 autograd, dln_w / dln_b the sums
    over exactly the n rows."""
    T = T_CAP
    Tp = 2 * T + 1
    O, q_in, Wo, bo, lw, lb, W1, b1, W2, b2, v = _post_attn_inputs(T, d, hdv, 2000 + n + d + hdv, cuda)
    _poison(O, n, n)
    _poison(q_in, n, n + 1)
    tok_all = _tokens(T, n + d)
    tok_all[n:] = tok_all[n:].flip(0)                            # valid, wrong
    row_tok = tok_all.to(cuda)
    tok = row_tok[:n].long()
    n_dev = torch.tensor([n], dtype=torch.int32, device=cuda)
    ctr = _ctr(cuda)
    off1, off2 = _site(1, 1) << 40, _site(1, 2) << 40
    ks = _ks(drop) if drop > 0 else 1.0
    W = (Wo.data_ptr(), bo.data_ptr(), lw.data_ptr(), lb.data_ptr(), EPS, W1.data_ptr(), b1.data_ptr(), W2.data_ptr(), b2.data_ptr())
    names = ("h", "y", "u", "mean", "rstd", "out")
    bufs = {k: _sent(T, 0 if k in ("mean", "rstd") else d, cuda, torch.float32 if k in ("mean", "rstd") else torch.bfloat16)
            for k in names}
    check(lib().rp_post_attn_train_rows(O.data_ptr(), q_in.data_ptr(), *W, T, d, drop, SEED, off1, off2, ctr.data_ptr(),
                                        *[bufs[k].data_ptr() for k in names], hdv, n_dev.data_ptr(), row_tok.data_ptr(),
                                        _stream()), "rp_post_attn_train_rows")
    torch.cuda.synchronize()
    for k, b in bufs.items():
        _untouched(b, n, k)
    if n:
        pad_bufs = {k: torch.zeros(Tp, device=cuda) if b.dim() == 1 else torch.zeros(Tp, d, dtype=b.dtype, device=cuda)
                    for k, b in bufs.items()}
        Os, qs = _scatter(O[:n], tok, Tp), _scatter(q_in[:n], tok, Tp)
        check(lib().rp_post_attn_train(Os.data_ptr(), qs.data_ptr(), *W, None, Tp, d, drop, SEED, off1, off2, ctr.data_ptr(),
                                       *[pad_bufs[k].data_ptr() for k in names], hdv, _stream()), "rp_post_attn_train")
        torch.cuda.synchronize()
        for k in names:
            assert torch.equal(bufs[k][:n], pad_bufs[k][tok]), f"{k} differs from the padded kernel's rows of the same tokens"
        tc = tok.cpu().numpy()
        k1 = keep_draws(SEED + CTR, off1, drop, tc, d).to(cuda) if drop > 0 else torch.ones(n, d, dtype=torch.bool, device=cuda)
        k2 = keep_draws(SEED + CTR, off2, drop, tc, d).to(cuda) if drop > 0 else k1
        rm1 = torch.ones(n, dtype=torch.uint8, device=cuda)
        got = {k: bufs[k][:n] for k in ("h", "y", "u", "out")}
        ins = (O[:n], q_in[:n], Wo, bo, lw, lb, W1, b1, W2, b2, v)
        ref, m_ref, r_ref = post_attn_train_ref(*ins, k1, k2, rm1, ks, got=got)
        assert _note("post_attn h ulp", ulp_err(got["h"], *ref["h"])) < TOL_ULP
        assert _note("post_attn y ulp", ulp_err(got["y"], *ref["y"])) < TOL_ULP
        _check_stats(bufs["mean"][:n], bufs["rstd"][:n], m_ref, r_ref, got["h"], v)
        _assert_keep_pattern(got["u"][:, v], k1[:, v], ref["u_exact"][:, v], ref["u"][1][:, v], "u (site 1)")
        assert _note("post_attn u ulp", ulp_err(got["u"], *ref["u"])) < TOL_ULP
        assert _note("post_attn out ulp", ulp_err(got["out"], *ref["out"])) < TOL_ULP
        if drop > 0:
            # the masks of the packed row index instead of the token: the kernel's u is far outside the tolerance of it
            r_np = np.arange(n)
            kb1 = keep_draws(SEED + CTR, off1, drop, r_np, d).to(cuda)
            kb2 = keep_draws(SEED + CTR, off2, drop, r_np, d).to(cuda)
            bad, _, _ = post_attn_train_ref(*ins, kb1, kb2, rm1, ks, got=got)
            e = ulp_err(got["u"], *bad["u"])
            _note("post_attn u keyed by row (x TOL)", e / TOL_ULP)
            assert e >= 10 * TOL_ULP, "a reference keyed by the packed row is within the tolerance"

    # ---- rp_post_attn_bwd_rows: every input row past n poisoned
    gb = _gen(7 * n + d)
    dz = _bf(torch.randn(T, d, generator=gb) * 0.5 * v.cpu()).to(cuda)
    dz = _poison(torch.where((dz == 0) & v, torch.full_like(dz, 0.25), dz), n, n + 2)
    for i, k in enumerate(("h", "u", "mean", "rstd")):
        _poison(bufs[k], n, n + i)
    dw0, db0 = torch.randn(d, generator=gb).to(cuda), torch.randn(d, generator=gb).to(cuda)
    dw, db = dw0.clone(), db0.clone()
    gnames = ("d_t", "du", "dh", "d_o")
    o = {k: _sent(T, d, cuda) for k in gnames}
    bw = (lw.data_ptr(), W2.data_ptr(), W1.data_ptr(), Wo.data_ptr())
    check(lib().rp_post_attn_bwd_rows(dz.data_ptr(), bufs["u"].data_ptr(), bufs["h"].data_ptr(), bufs["mean"].data_ptr(),
                                      bufs["rstd"].data_ptr(), *bw, T, d, drop, SEED, off2, ctr.data_ptr(),
                                      o["d_t"].data_ptr() if drop > 0 else None, o["du"].data_ptr(), o["dh"].data_ptr(),
                                      o["d_o"].data_ptr(), dw.data_ptr(), db.data_ptr(), hdv, n_dev.data_ptr(), row_tok.data_ptr(),
                                      _stream()), "rp_post_attn_bwd_rows")
    torch.cuda.synchronize()
    for k, b in o.items():
        _untouched(b, n if (drop > 0 or k != "d_t") else 0, k)
    assert torch.isfinite(dw).all() and torch.isfinite(db).all(), "a stale row reached dln_w / dln_b"
    if n == 0:
        assert torch.equal(dw, dw0) and torch.equal(db, db0)
        return
    sc = {k: _scatter(t[:n], tok, Tp) for k, t in (("dz", dz), ("u", bufs["u"]), ("h", bufs["h"]), ("mean", bufs["mean"]),
                                                     ("rstd", bufs["rstd"]))}
    op = {k: torch.zeros(Tp, d, dtype=torch.bfloat16, device=cuda) for k in gnames}
    dwp, dbp = dw0.clone(), db0.clone()
    check(lib().rp_post_attn_bwd(sc["dz"].data_ptr(), sc["u"].data_ptr(), sc["h"].data_ptr(), sc["mean"].data_ptr(),
                                 sc["rstd"].data_ptr(), *bw, None, Tp, d, drop, SEED, off2, ctr.data_ptr(),
                                 op["d_t"].data_ptr() if drop > 0 else None, op["du"].data_ptr(), op["dh"].data_ptr(),
                                 op["d_o"].data_ptr(), dwp.data_ptr(), dbp.data_ptr(), hdv, _stream()), "rp_post_attn_bwd")
    torch.cuda.synchronize()
    for k in gnames:
        if drop > 0 or k != "d_t":
            assert torch.equal(o[k][:n], op[k][tok]), f"{k} differs from the padded kernel's rows of the same tokens"
    k2 = keep_draws(SEED + CTR, off2, drop, tok.cpu().numpy(), d).to(cuda) if drop > 0 else torch.ones(n, d, dtype=torch.bool,
                                                                                                         device=cuda)
    rm1 = torch.ones(n, dtype=torch.uint8, device=cuda)
    r_dt, r_du, r_dh, r_do, r_dw, r_db = post_attn_bwd_ref(dz[:n], bufs["h"][:n], bufs["u"][:n], lw, lb, W1, W2, Wo, b1, b2, v,
                                                           k2, rm1, ks)
    if drop > 0:
        assert _note("post_attn_bwd d_t block", block_err(o["d_t"][:n], r_dt)) < TOL_BWD
    assert _note("post_attn_bwd du block", block_err(o["du"][:n], r_du)) < TOL_BWD
    assert _note("post_attn_bwd dh block", block_err(o["dh"][:n], r_dh)) < TOL_BWD
    assert _note("post_attn_bwd d_o block", block_err(o["d_o"][:n], r_do)) < TOL_BWD
    assert _note("post_attn_bwd dln_w", block_err((dw - dw0).double().view(-1, 1), r_dw.view(-1, 1))) < TOL_LN_GRAD
    assert _note("post_attn_bwd dln_b", block_err((db - db0).double().view(-1, 1), r_db.view(-1, 1))) < TOL_LN_GRAD


# ----------------------------------------------------------------------------------------------------------------------
# rp_wgrad_group_rows
# ----------------------------------------------------------------------------------------------------------------------
W_CAP = 4400
_WG_N = [0, 1, 63, 64, 65, 64 * 65, 64 * 64 + 1, W_CAP]   # 65 chunks: more than the at most 64 token splits


def _wgrad(pairs, T, accumulate, n_dev, dev):
    arr = (WgradPair * len(pairs))()
    for k, (dY, X, dW, db) in enumerate(pairs):
        arr[k].dY, arr[k].dy_ld, arr[k].n_out = dY.data_ptr(), dY.stride(0), dW.shape[0]
        arr[k].X, arr[k].x_ld, arr[k].n_in = X.data_ptr(), X.stride(0), dW.shape[1]
        arr[k].dW, arr[k].dw_ld, arr[k].db = dW.data_ptr(), dW.stride(0), db.data_ptr()
    need = lib().rp_wgrad_group_workspace(arr, len(pairs))
    ws = torch.zeros(need, device=dev, dtype=torch.uint8)
    if n_dev is None:
        check(lib().rp_wgrad_group(arr, len(pairs), T, accumulate, ws.data_ptr(), need, _stream()), "rp_wgrad_group")
    else:
        check(lib().rp_wgrad_group_rows(arr, len(pairs), T, accumulate, n_dev.data_ptr(), ws.data_ptr(), need, _stream()),
              "rp_wgrad_group_rows")
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("accumulate", [1, 0])
@pytest.mark.parametrize("n", _WG_N)
def test_wgrad_group_rows(cuda, n, accumulate):
    """rp_wgrad_group_rows over the first n of T rows with dY and X rows past n poisoned, as the engine's (dQ, q_in) and
    (dKV, x) pairs: dW = dY^T X and db = sum dY over exactly the n rows against fp64, accumulated onto preset values or
    overwriting a NaN-filled destination; bitwise equal to rp_wgrad_group at T = n (the same token chunks) and to a rerun."""
    T, d = W_CAP, 128
    g = _gen(n + 11 * accumulate)
    bf = lambda c, k: _poison(_bf(torch.randn(T, c, generator=g) * 0.5).to(cuda), n, k)  # noqa: E731
    ops_ = [(bf(d, n), bf(d, n + 1)), (bf(2 * d, n + 2), bf(d, n))]
    shapes = [(d, d), (2 * d, d)]
    W0 = [torch.randn(*s, generator=g).to(cuda) if accumulate else torch.full(s, float("nan"), device=cuda) for s in shapes]
    B0 = [torch.randn(s[0], generator=g).to(cuda) if accumulate else torch.full((s[0],), float("nan"), device=cuda)
          for s in shapes]
    n_dev = torch.tensor([n], dtype=torch.int32, device=cuda)

    def run(rows):
        dst = [(w.clone(), b.clone()) for w, b in zip(W0, B0)]
        pairs = [(dY, X, dW, db) for (dY, X), (dW, db) in zip(ops_, dst)]
        _wgrad(pairs, T if rows else n, accumulate, n_dev if rows else None, cuda)
        return dst

    got = run(True)
    for (dY, X), (dW, db), w0, b0 in zip(ops_, got, W0, B0):
        assert torch.isfinite(dW).all() and torch.isfinite(db).all(), "a stale row reached dW / db"
        base_w = w0.double() if accumulate else 0.0
        base_b = b0.double() if accumulate else 0.0
        if n == 0:
            assert torch.equal(dW.double() - base_w, torch.zeros_like(dW, dtype=torch.float64))
            assert torch.equal(db.double() - base_b, torch.zeros_like(db, dtype=torch.float64))
            continue
        ref = dY[:n].double().T @ X[:n].double()
        assert _note("wgrad_rows dW block", block_err(dW.double() - base_w, ref)) < TOL_SPLITK
        rb = dY[:n].double().sum(0)
        assert _note("wgrad_rows db", block_err((db.double() - base_b).view(-1, 1), rb.view(-1, 1))) < TOL_SUM
    again = run(True)
    for (a, b), (c, e) in zip(got, again):
        assert torch.equal(a, c) and torch.equal(b, e), "rp_wgrad_group_rows reruns must be bit-identical"
    if n:
        padded = run(False)
        for (a, b), (c, e) in zip(got, padded):
            assert torch.equal(a, c) and torch.equal(b, e), "packed and padded weight gradients differ"


# ----------------------------------------------------------------------------------------------------------------------
# packed attention
# ----------------------------------------------------------------------------------------------------------------------
def _attn_firsts(L):
    """First kept position of every sequence: a first sequence whose window starts before row 0 (lead 63), two empty
    sequences, then one that follows them with lead 1, then every edge of the 64-aligned shift and the 128 / 192 rows."""
    edges = [0, 1, 63, 64, 65, 127, 128, 129, L - 1, L]
    out = [min(63, L - 1), L, L, 1] + [f for f in edges if 0 <= f <= L]
    return out


def _attn_batch(L, H, seed, dev):
    firsts = _attn_firsts(L)
    B = len(firsts)
    g = _gen(seed)
    pad = torch.zeros(B, L, dtype=torch.bool)
    tmask = torch.zeros(B, L, dtype=torch.bool)
    for b, f in enumerate(firsts):
        if f >= L:
            continue
        tmask[b, f:] = True
        s = f + (b % 2)                                  # odd sequences: position f is the target-only row
        pad[b, s:] = True
        if b % 3 == 0 and s < L:
            pad[b, s + 1:] &= torch.rand(L - s - 1, generator=g) > 0.2    # interior holes (masked keys)
    labels = torch.randint(0, 100, (B, L), generator=g)
    c = _case(pad, H, 64, 1, seed=seed, dev=dev)
    # the rows of every other sequence hold +-BIG in V: a neighbour row leaking into a window is a large error
    d = c.d
    odd = (torch.arange(B) % 2 == 1).repeat_interleave(L)[:, None]
    sign = torch.randint(0, 2, c.kv[:, d:].shape, generator=g).float() * 2 - 1
    c.kv[:, d:] = torch.where(odd, (BIG * sign).to(torch.bfloat16), c.kv[:, d:])
    c.kvd = c.kv.to(dev)
    c.v64 = _heads(c.kv[:, d:], B, L, H, 64)
    return c, labels, tmask


def _desc(desc, c, q, kv, scale_d, drop, ctr, seq=None):
    T, d = c.T, c.d
    desc.q, desc.q_rows, desc.q_cols, desc.ldq, desc.q_c0 = q.data_ptr(), T, d, d, 0
    desc.k, desc.k_rows, desc.k_cols, desc.ldk, desc.k_c0 = kv.data_ptr(), T, 2 * d, 2 * d, 0
    desc.v, desc.v_rows, desc.v_cols, desc.ldv, desc.v_c0 = kv.data_ptr(), T, 2 * d, 2 * d, d
    desc.B, desc.H, desc.L, desc.head_dim = c.B, c.H, c.L, 64
    desc.causal, desc.mask_pad_keys = 1, 1
    desc.scale = scale_d
    desc.pad_mask = c.padd.data_ptr()
    desc.drop_p, desc.seed, desc.drop_off, desc.seed_ptr = drop, SEED, OFF, ctr.data_ptr()
    if seq is not None:
        desc.seq_first, desc.seq_off = seq
    return desc


def _fwd(c, q, kv, drop, ctr, seq=None):
    out = _sent(c.T, c.d + 64, q.device)[: c.T + 64]
    inv = torch.full((c.B * c.H, c.Lp), -1.0, device=q.device)
    m = torch.full((c.B * c.H, c.Lp), -1.0, device=q.device)
    ad = _desc(AttnDesc(), c, q, kv, 0.0, drop, ctr, seq)
    ad.out, ad.ldo = out.data_ptr(), c.d + 64
    ad.p_save, ad.inv_sum, ad.m_save = None, inv.data_ptr(), m.data_ptr()
    check(lib().rp_attn_fwd(ctypes.byref(ad), _stream()), "rp_attn_fwd")
    torch.cuda.synchronize()
    return out, inv, m


def _bwd(c, q, kv, d_o, fwd, drop, ctr, seq=None):
    out, inv, m = fwd
    dq = _sent(c.T, c.d + 64, q.device)
    dkv = _sent(c.T, 2 * c.d + 64, q.device)
    bd = _desc(AttnBwdDesc(), c, q, kv, 0.0, drop, ctr, seq)
    bd.d_out, bd.do_rows, bd.do_cols, bd.ld_do = d_o.data_ptr(), c.T, c.d, c.d
    bd.out, bd.ldo = out.data_ptr(), c.d + 64
    bd.m_save, bd.inv_sum = m.data_ptr(), inv.data_ptr()
    bd.dq, bd.ld_dq, bd.dq_c0 = dq.data_ptr(), c.d + 64, 0
    bd.dk, bd.ld_dk, bd.dk_c0 = dkv.data_ptr(), 2 * c.d + 64, 0
    bd.dv, bd.ld_dv, bd.dv_c0 = dkv.data_ptr(), 2 * c.d + 64, c.d
    check(lib().rp_attn_bwd(ctypes.byref(bd), _stream()), "rp_attn_bwd")
    torch.cuda.synchronize()
    return dq, dkv


def _unpack_rows(x, tok, T):
    """Packed rows -> the padded layout (rows of no packed token 0)."""
    out = torch.zeros((T,) + tuple(x.shape[1:]), dtype=torch.float64)
    out[tok] = x.double()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("drop", [0.0, P_DROP])
@pytest.mark.parametrize("H", [1, 2])
@pytest.mark.parametrize("L", [64, 65, 128, 200, 256])
def test_packed_attention(cuda, L, H, drop):
    """Packed rp_attn_fwd / rp_attn_bwd (head slot 64, causal, pad keys masked) on a real row plan with Q / K / V / dO
    rows past n_rows NaN / Inf and every other sequence's V at +-BIG: O, m_save, inv_sum, dQ, dK, dV bitwise equal to
    the padded kernels' rows of the same tokens, against fp64 (O per 64-query block, the gradients on the kernel's O),
    nothing written past n_rows or past the heads."""
    c, labels, tmask = _attn_batch(L, H, seed=L * 4 + H + int(drop * 10), dev=cuda)
    B, T, d, Lp = c.B, c.T, c.d, c.Lp
    pl = device_plan(c.pad, labels, tmask, 100, cuda)
    P = check_plan(pl, c.pad, labels, tmask, 100)
    tok = pl["row_tok"][:P].long()
    ctr = _ctr(cuda)
    qp = _poison(torch.cat([c.qd[tok], torch.zeros(T - P, d, dtype=torch.bfloat16, device=cuda)]), P, L)
    kvp = _poison(torch.cat([c.kvd[tok], torch.zeros(T - P, 2 * d, dtype=torch.bfloat16, device=cuda)]), P, L + 1)
    seq = (pl["seq_first"].data_ptr(), pl["seq_off"].data_ptr())
    fwd_p = _fwd(c, qp, kvp, drop, ctr, seq)
    fwd_u = _fwd(c, c.qd, c.kvd, drop, ctr)
    out_p, out_u = fwd_p[0], fwd_u[0]
    _untouched(out_p, P, "O")
    assert (out_p[:, d:] == SENT).all(), "columns past the heads were written"
    assert torch.equal(out_p[:P], out_u[tok]), "packed O differs from the padded kernel's rows of the same tokens"
    first = pl["seq_first"].cpu().long()
    for b in range(B):
        f = int(first[b])
        if f == L:
            continue
        shift = f - f % 64
        for k in (1, 2):   # inv_sum, m_save: the packed row of position i at local index i - shift
            got, ref = fwd_p[k].view(B, H, Lp)[b, :, f - shift: L - shift], fwd_u[k].view(B, H, Lp)[b, :, f:L]
            assert torch.equal(got, ref), ("inv_sum", "m_save")[k - 1] + f" of sequence {b} differs"
    keep = drop_keep(SEED + CTR, OFF, drop, B, H, L, Lp) if drop > 0 else None
    o_ref, m_ref, inv_ref, _ = attn_ref(c.q64, c.k64, c.v64, c.pad, 1, 1, 1.0 / 8.0, keep)
    tok_c = tok.cpu()
    o = _heads(_unpack_rows(out_p[:P, :d].cpu(), tok_c, T), B, L, H, 64)
    live = (torch.arange(L)[None, :] >= first[:, None]).view(B, 1, L, 1)
    assert _note("attn fwd O block", head_block_err(o, o_ref * live)) < TOL_O
    inv_u, m_u = fwd_u[1].cpu().double().view(B, H, Lp)[:, :, :L], fwd_u[2].cpu().double().view(B, H, Lp)[:, :, :L]
    lv = live[..., 0].expand(B, H, L)
    _note("attn fwd m_save abs", (m_u[lv] - m_ref[lv]).abs().max())
    torch.testing.assert_close(m_u[lv], m_ref[lv], rtol=TOL_M_REL, atol=TOL_M_ABS)
    torch.testing.assert_close(inv_u[lv], inv_ref[lv], rtol=TOL_INV_REL, atol=0)

    # ---- backward: dO, and the O the kernel reads, poisoned past n_rows
    d_o = _d_out(c, seed=L + 1).to(cuda)
    dop = _poison(torch.cat([d_o[tok], torch.zeros(T - P, d, dtype=torch.bfloat16, device=cuda)]), P, L + 2)
    _poison(out_p[:T], P, L)
    dq_p, dkv_p = _bwd(c, qp, kvp, dop, fwd_p, drop, ctr, seq)
    dq_u, dkv_u = _bwd(c, c.qd, c.kvd, d_o, fwd_u, drop, ctr)
    _untouched(dq_p, P, "dQ")
    _untouched(dkv_p, P, "dK / dV")
    assert (dq_p[:, d:] == SENT).all() and (dkv_p[:, 2 * d:] == SENT).all(), "columns past the heads were written"
    assert torch.equal(dq_p[:P, :d], dq_u[tok, :d]), "packed dQ differs from the padded kernel's rows"
    assert torch.equal(dkv_p[:P, : 2 * d], dkv_u[tok, : 2 * d]), "packed dK / dV differ from the padded kernel's rows"
    got = [_heads(_unpack_rows(t.cpu(), tok_c, T), B, L, H, 64)
           for t in (dq_p[:P, :d], dkv_p[:P, :d], dkv_p[:P, d: 2 * d])]
    d_o64 = _heads(d_o.cpu(), B, L, H, 64)
    o64 = _heads(out_u[:T].cpu(), B, L, H, 64)
    vis = visibility(c.pad, L, 1, 1) & live.view(B, 1, L, 1)   # queries before first are not rows of the packed batch
    ref = attn_grads_given_o(c.q64, c.k64, c.v64, vis, 1.0 / 8.0, keep, d_o64, o64)
    _check_grads(c, 1, 1, got, ref, "packed bwd")


@pytest.mark.gpu
def test_packed_attention_rejections(cuda):
    """The packed descriptor is refused where it is undefined: seq_first without seq_off (or the reverse), a non-causal
    mask, head_dim 128 and L > 256 in the forward; the first two in the backward."""
    c, labels, tmask = _attn_batch(64, 1, seed=5, dev=cuda)
    pl = device_plan(c.pad, labels, tmask, 100, cuda)
    ctr = _ctr(cuda)
    sf, so = pl["seq_first"].data_ptr(), pl["seq_off"].data_ptr()
    out = _sent(c.T, 2 * c.d, cuda)
    m = torch.zeros(c.B, 512, device=cuda)

    def fwd(**kw):
        ad = _desc(AttnDesc(), c, c.qd, c.kvd, 0.0, 0.0, ctr)
        ad.out, ad.ldo, ad.inv_sum, ad.m_save = out.data_ptr(), 2 * c.d, m.data_ptr(), m.data_ptr()
        for k, v in kw.items():
            setattr(ad, k, v)
        return lib().rp_attn_fwd(ctypes.byref(ad), _stream())

    def bwd(**kw):
        bd = _desc(AttnBwdDesc(), c, c.qd, c.kvd, 0.0, 0.0, ctr)
        bd.d_out, bd.do_rows, bd.do_cols, bd.ld_do = c.qd.data_ptr(), c.T, c.d, c.d
        bd.out, bd.ldo, bd.m_save, bd.inv_sum = out.data_ptr(), 2 * c.d, m.data_ptr(), m.data_ptr()
        bd.dq, bd.ld_dq, bd.dk, bd.ld_dk, bd.dv, bd.ld_dv = (out.data_ptr(), 2 * c.d) * 3
        for k, v in kw.items():
            setattr(bd, k, v)
        return lib().rp_attn_bwd(ctypes.byref(bd), _stream())

    EINVAL, ESHAPE = -1, -2
    assert fwd(seq_first=sf) == EINVAL and fwd(seq_off=so) == EINVAL
    assert fwd(seq_first=sf, seq_off=so, causal=0) == EINVAL
    assert fwd(seq_first=sf, seq_off=so, head_dim=128) == ESHAPE
    assert fwd(seq_first=sf, seq_off=so, L=320, B=1) == ESHAPE
    assert bwd(seq_first=sf) == EINVAL and bwd(seq_off=so) == EINVAL
    assert bwd(seq_first=sf, seq_off=so, causal=0) == EINVAL
    torch.cuda.synchronize()
    assert (out == SENT).all(), "a refused call wrote its output"


# ----------------------------------------------------------------------------------------------------------------------
# the engine's packed training step against the fp64 model
# ----------------------------------------------------------------------------------------------------------------------
_STEP_CASES = {"d128h2": ("new", 128, 2), "d64h2": ("new", 64, 2), "d64h1": ("new", 64, 1), "d50h1": ("new", 50, 1)}


def _packed_engine(case, B, drop, cuda, seed):
    from replay_b200.engine import EncoderConfig, SasRecEngine

    cfg = EncoderConfig(n_items=case.I, d=case.d, n_heads=case.H, n_blocks=2, max_len=case.max_len, dropout=drop,
                        variant=case.variant)
    eng = SasRecEngine(cfg, B, case.L, cuda, seed=SEED)
    eng.load_canonical(case.params(seed))
    eng.packed_body = True
    assert eng.packed_eligible()
    return eng, cfg


def _packed_step(eng, batch, ctr, negatives=None):
    eng.set_batch(*batch)
    if negatives is not None:
        eng.set_negatives(negatives)
    eng.rng_counter.fill_(ctr)
    eng.g32.zero_()
    loss = float(eng.forward_train()[0])
    assert eng._packed, "the step did not run packed"
    eng.backward()
    torch.cuda.synchronize()
    return loss


def sampled_ref(P, batch, H, lnf_eps, keeps, negatives):
    """The fp64 model with the CESampled head (perseq negatives) restated by tests/sampled_reference.py on its hidden
    states: (loss, x[-1], hidden, gradients), the head's d_hc carried back through the body by autograd."""
    ids, pad, labels, tmask = batch
    Q = _map(P, lambda k, v: v.detach().double().clone().requires_grad_(True))
    _, x, hid = sasrec_ref(Q, ids, pad, labels, tmask, H, "new", lnf_eps, keeps)
    I, L = Q["item_emb"].shape[0] - 1, ids.shape[1]
    vi = (tmask & (labels >= 0) & (labels < I)).reshape(-1).nonzero()[:, 0]
    hc = hid.reshape(-1, hid.shape[-1])[vi]
    r = sampled_reference.reference(hc.detach(), Q["item_emb"].detach(), labels.reshape(-1)[vi], vi, negatives, vi.numel(),
                                    sampled_reference.CE_SAMPLED, 2, L=L)
    leaves = _leaves(Q)
    grads = torch.autograd.grad(hc, [t for _, t in leaves], grad_outputs=r["d_hc"], allow_unused=True)
    G = {k: (g if g is not None else torch.zeros_like(t)) for (k, t), g in zip(leaves, grads)}
    G["item_emb"] = G["item_emb"] + r["d_table"]
    G["item_emb"][-1] = 0
    return r["loss"], x.detach(), hid.detach(), G


def _run_packed(case, B, drop, cuda, seed, n_neg=0):
    eng, cfg = _packed_engine(case, B, drop, cuda, seed)
    ids, pad, labels, tmask = step_batch(B, case.L, case.I, seed + 1)
    batch = [t.to(cuda) for t in (ids, pad, labels, tmask)]
    ctr = 12345 if drop > 0 else 0
    neg = None
    if n_neg:
        eng.set_loss("ce_sampled", n_neg=n_neg, neg_shape="perseq")
        neg = torch.randint(0, case.I, (B, n_neg), generator=_gen(seed + 2)).to(cuda)
    loss = _packed_step(eng, batch, ctr, neg)
    # x[-1] of the packed rows, scattered back to the padded layout (rows before a sequence's first kept row: 0)
    P = int(eng.n_rows[0])
    tok = eng.row_tok[:P].long()
    x = torch.zeros(B * case.L, cfg.dp, dtype=torch.float64, device=cuda)
    x[tok] = eng.x[-1][:P].double()
    x = eng.unpad_features(x).view(B, case.L, case.d)
    G = {k: v for k, v in _leaves(eng.export_canonical(eng.grads))}
    keeps = engine_keeps(eng.seed + ctr, drop, B, case.L, cfg, dev=cuda) if drop > 0 else None
    P = _map(case.params(seed), lambda k, v: v.to(cuda))
    if n_neg:
        ref = sampled_ref(P, batch, case.H, case.lnf_eps, keeps, neg)
    else:
        ref = ref_loss_and_grads(P, *batch, case.H, case.variant, case.lnf_eps, keeps)
    return loss, x, G, ref, batch[1]


@pytest.mark.gpu
@pytest.mark.parametrize("drop", [0.0, P_DROP])
@pytest.mark.parametrize("L", [200, 256])
@pytest.mark.parametrize("name", list(_STEP_CASES))
def test_packed_step_matches_fp64_reference(cuda, name, L, drop):
    """SasRecEngine with packed_body on (asserted through _packed) at B = 7 left-padded histories, two blocks, I = 2000,
    max_len L + 10: d 128 / 2 heads, d 64 / 2 heads (head features 32 in slot 64), d 64 / 1 head and d 50 / 1 head.
    Loss, x[-1] of the real rows and every parameter gradient against the fp64 model under the ported masks."""
    case = _Case(*_STEP_CASES[name], L=L)
    loss, x, G, ref, pad = _run_packed(case, 7, drop, cuda, seed=case.d + case.H + L)
    _check_step(case, loss, x, G, ref, pad, tag=" packed")


@pytest.mark.gpu
@pytest.mark.parametrize("drop", [0.0, P_DROP])
def test_packed_step_ce_sampled_matches_fp64_reference(cuda, drop):
    """The packed step with CESampled (37 negatives per sequence) at d 128 / 2 heads, L = 200: loss, x[-1] and every
    gradient against the fp64 model whose head is restated from tests/sampled_reference.py."""
    case = _Case("new", 128, 2, L=200)
    loss, x, G, ref, pad = _run_packed(case, 7, drop, cuda, seed=41, n_neg=37)
    _check_step(case, loss, x, G, ref, pad, tag=" packed ce_sampled")


@pytest.mark.gpu
def test_packed_step_across_the_plan_slab(cuda):
    """One packed step at B = 1100, L = 50 (the row plan's prefix carried across its 1024-sequence slab), dropout 0.2."""
    case = _Case("new", 64, 1, L=50)
    loss, x, G, ref, pad = _run_packed(case, 1100, P_DROP, cuda, seed=31)
    _check_step(case, loss, x, G, ref, pad, tag=" packed B1100")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [0, 1, 127, 128, 129, 250])
def test_layernorm_compact_zeroes_the_head_tile_tail(cuda, n):
    """rp_layernorm_fwd_compact (the final norm compacting the valid targets for the loss heads): the n rows element-wise
    against fp64, the rows after them up to the next 128-row edge zeroed whatever they held (the heads read whole 128-row
    tiles, and a NaN there reached every item's gradient through a zero weight), rows past that edge and the statistics
    past n untouched; gather and the device row count are required."""
    T, d = 260, 128
    g = _gen(n)
    x = _bf(torch.randn(T, d, generator=g)).to(cuda)
    gather = torch.randperm(T, generator=g).to(torch.int32).to(cuda)
    w, b = (1 + 0.2 * torch.randn(d, generator=g)).to(cuda), (0.1 * torch.randn(d, generator=g)).to(cuda)
    y = torch.full((T, d), float("nan"), dtype=torch.bfloat16, device=cuda)
    mean, rstd = _sent(T, 0, cuda, torch.float32), _sent(T, 0, cuda, torch.float32)
    n_dev = torch.tensor([n], dtype=torch.int32, device=cuda)
    args = (x.data_ptr(), w.data_ptr(), b.data_ptr(), 1e-5, T, d)
    outs = (y.data_ptr(), mean.data_ptr(), rstd.data_ptr(), 0, _stream())
    assert lib().rp_layernorm_fwd_compact(*args, None, gather.data_ptr(), *outs) == -1
    assert lib().rp_layernorm_fwd_compact(*args, n_dev.data_ptr(), None, *outs) == -1
    check(lib().rp_layernorm_fwd_compact(*args, n_dev.data_ptr(), gather.data_ptr(), *outs), "rp_layernorm_fwd_compact")
    torch.cuda.synchronize()
    edge = min(T, (n + 127) // 128 * 128)
    assert (y[n:edge] == 0).all(), "rows past the count up to the tile edge must be zero"
    assert torch.isnan(y[edge:].float()).all(), "rows past the tile edge were written"
    _untouched(mean, n, "mean")
    _untouched(rstd, n, "rstd")
    if n:
        X = x[gather[:n].long()].double()
        y_ref, m_ref, r_ref = ln_ref(X, w.double(), b.double(), 1e-5, torch.ones(d, dtype=torch.bool))
        assert _note("final norm y ulp", ulp_err(y[:n], y_ref, _ln_fwd_atol(X, m_ref, r_ref, w.double()))) < TOL_ULP


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["d128h2", "d50h1"])
def test_packed_step_ignores_stale_buffers(cuda, name):
    """The same packed step on zeroed buffers and with every T-row activation, statistics and scratch buffer (x[*],
    act[*], s[*], meanf / rstdf, hc) filled with NaN first: finite loss and gradients, bitwise equal except the
    gradients summed by fp32 atomics (the embedding tables, and any tensor whose two clean runs differ), which agree to
    1e-6 norm-relative."""
    case = _Case(*_STEP_CASES[name], L=200)
    eng, _ = _packed_engine(case, 61, P_DROP, cuda, seed=9)
    lengths = [0 if i % 5 == 0 else (i * 37) % 200 + 1 for i in range(61)]
    batch = [t.to(cuda) for t in _windows(lengths, 200, case.I, seed=4)]

    def run():
        loss = _packed_step(eng, batch, 777)
        return loss, {k: v.detach().clone() for k, v in eng.grads.items()}

    loss_a, ga = run()
    loss_b, gb = run()
    bufs = list(eng.x) + [t for a in eng.act for t in a.values()] + list(eng.s.values()) + [eng.meanf, eng.rstdf, eng.hc]
    for t in bufs:
        if t.is_floating_point():
            t.fill_(float("nan"))
    loss_n, gn = run()
    assert math.isfinite(loss_n) and loss_n == loss_a
    for k in ga:
        assert torch.isfinite(gn[k]).all(), f"{k}: a stale row reached the gradient"
        if torch.equal(ga[k], gb[k]) and k not in ("item_emb", "pos_emb"):
            assert torch.equal(gn[k], ga[k]), f"{k} differs from the step on zeroed buffers"
        else:
            den = max(float(ga[k].double().norm()), 1e-30)
            assert _note("stale buffers atomics rel", float((gn[k].double() - ga[k].double()).norm()) / den) < 1e-6, k
