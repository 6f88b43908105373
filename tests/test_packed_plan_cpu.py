"""Host-side pieces of test_gpu_packed_fp64.py: the row-plan restatement against a position-by-position definition, the
coverage of the batch and attention-window generators, and the dropout-keying discrimination of the post-attention
reference."""
import numpy as np
import pytest
import torch

from dropout_stream import keep_draws
from test_gpu_packed_body import expected_plan
from test_gpu_packed_fp64 import T_CAP, _attn_firsts, _tokens, plan_batch
from sasrec_fp64 import CTR, P_DROP, SEED, _bf, _ks, _site
from test_gpu_sasrec_body import TOL_ULP, _post_attn_inputs, post_attn_train_ref
from fp64_checks import ulp_err


def _brute_plan(pad, tmask, labels, n_items):
    B, L = pad.shape
    first, rows = [], []
    for b in range(B):
        f = next((l for l in range(L) if pad[b, l] or (tmask[b, l] and 0 <= labels[b, l] < n_items)), L)
        first.append(f)
        rows += [b * L + l for l in range(f, L)]
    n = [L - f for f in first]
    off = [sum(n[:b]) for b in range(B)]
    return first, off, rows


@pytest.mark.parametrize("B,L", [(1, 1), (37, 1), (37, 33), (50, 200), (3, 256)])
def test_expected_plan_matches_position_by_position_definition(B, L):
    I = 500
    pad, labels, tmask = plan_batch(B, L, I, seed=B + L)
    first, off, row_tok, P = expected_plan(pad, tmask, labels, I)
    f, o, rows = _brute_plan(pad, tmask, labels, I)
    assert first.tolist() == f and off.tolist() == o and row_tok.tolist() == rows and P == len(rows)


def test_plan_batch_covers_every_kind():
    """Empty and full sequences, a valid target-only row before the first real token, and labels -1 / n_items under a
    set target mask that keep nothing."""
    B, L, I = 60, 200, 500
    pad, labels, tmask = plan_batch(B, L, I, seed=1)
    first = expected_plan(pad, tmask, labels, I)[0]
    real_first = torch.where(pad.any(1), pad.int().argmax(1), torch.full((B,), L))
    assert (first == L).any() and (first == 0).any() and (pad.all(1)).any()
    assert (first < real_first).any(), "no sequence keeps a target-only row before its first real token"
    invalid = tmask & ((labels < 0) | (labels >= I))
    assert (invalid & (labels < 0)).any() and (invalid & (labels >= I)).any()
    pos = torch.arange(L)[None]
    assert (invalid & (pos < real_first[:, None])).any(), "no invalid label before a first real token"


@pytest.mark.parametrize("L", [64, 65, 128, 200, 256])
def test_attention_windows_cover_the_edges(L):
    """The packed attention batches: lead 0 and 63, a shift of 0, 64 and 128 (and 192 where L > 192), empty sequences
    followed by a live one, and a first sequence whose window starts before row 0."""
    firsts = _attn_firsts(L)
    leads = {f % 64 for f in firsts if f < L}
    shifts = {f - f % 64 for f in firsts if f < L}
    assert {0, 63} <= leads and 0 in shifts
    assert all(s in shifts for s in (64, 128) if s < L)
    assert firsts[0] % 64 > 0 and firsts[1] == firsts[2] == L and firsts[3] < L
    assert max(L - (f - f % 64) for f in firsts if f < L) == L   # a window over the whole sequence


def test_post_attn_reference_discriminates_row_keyed_dropout():
    """At the kernel test's shape, an fp64 post-attention reference whose dropout masks are drawn for the packed row r
    instead of its token row_tok[r] moves u by >= 10x TOL_ULP."""
    n, d = 129, 128
    O, q_in, Wo, bo, lw, lb, W1, b1, W2, b2, v = _post_attn_inputs(n, d, 0, 5, None)
    tok = _tokens(T_CAP, 3)[:n].numpy()
    off1, off2 = _site(1, 1) << 40, _site(1, 2) << 40
    rm = torch.ones(n, dtype=torch.uint8)
    args = (O, q_in, Wo, bo, lw, lb, W1, b1, W2, b2, v)
    keys = lambda rows: (keep_draws(SEED + CTR, off1, P_DROP, rows, d), keep_draws(SEED + CTR, off2, P_DROP, rows, d))  # noqa: E731
    ref, _, _ = post_attn_train_ref(*args, *keys(tok), rm, _ks(P_DROP))
    bad, _, _ = post_attn_train_ref(*args, *keys(np.arange(n)), rm, _ks(P_DROP))
    e = ulp_err(_bf(bad["u"][0]).double(), ref["u"][0], ref["u"][1])
    assert e >= 10 * TOL_ULP
