"""The block kinds of the fused attention backward (rp_attn_bwd, with the rp_attn_fwd that feeds it) in one launch each:
interior blocks that every query sees (taken without per-element masks), diagonal blocks, block 0 of a window with lead
rows, and a partial last block; dQ from the dS blocks stored by the causal phase 1.  Against the fp64 references and
tolerances of test_gpu_attention.py, with bitwise equal reruns.

- packed rows: windows of 1 to 4 64-row blocks with lead 0, 1 and 63 in one batch, with and without dropout (the checks
  of test_gpu_packed_fp64.test_packed_attention on this mix of windows);
- padded rows: left-padded windows whose first real key falls inside a 64-key block, causal and not.
"""
import pytest
import torch

import test_gpu_packed_fp64 as packed
from dropout_stream import drop_keep
from test_gpu_attention import CTR, MODES, OFF, P_DROP, SEED, _attn_fwd, _case, _check_fwd, _fused_bwd_case

# first kept position of every sequence: lead 0, 1 and 63 at every window length 1 .. 4 blocks of L = 256
_FIRSTS = [0, 1, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255]


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("drop", [0.0, P_DROP])
@pytest.mark.parametrize("L", [200, 256])
def test_packed_windows_of_every_length_and_lead(cuda, monkeypatch, L, drop):
    """L 256: whole last blocks; L 200: every window ends in a partial block."""
    monkeypatch.setattr(packed, "_attn_firsts", lambda L: [f for f in _FIRSTS if f < L])
    packed.test_packed_attention(cuda, L, 2, drop)


@pytest.mark.gpu
@pytest.mark.parametrize("drop", [0.0, P_DROP])
def test_packed_reruns_bitwise_equal(cuda, monkeypatch, drop):
    monkeypatch.setattr(packed, "_attn_firsts", lambda L: _FIRSTS)
    c, labels, tmask = packed._attn_batch(256, 2, seed=17, dev=cuda)
    pl = packed.device_plan(c.pad, labels, tmask, 100, cuda)
    seq = (pl["seq_first"].data_ptr(), pl["seq_off"].data_ptr())
    ctr = packed._ctr(cuda)
    d_o = torch.randn(c.T, c.d, generator=torch.Generator().manual_seed(3)).to(torch.bfloat16).to(cuda)
    runs = []
    for _ in range(2):
        fwd = packed._fwd(c, c.qd, c.kvd, drop, ctr, seq)
        runs.append(fwd + packed._bwd(c, c.qd, c.kvd, d_o, fwd, drop, ctr, seq))
    for name, a, b in zip(("O", "inv_sum", "m_save", "dQ", "dK / dV"), *runs):
        assert torch.equal(a, b), f"{name} differs between two runs"


def _left_padded(L, firsts):
    pad = torch.zeros(len(firsts), L, dtype=torch.bool)
    for b, f in enumerate(firsts):
        pad[b, f:] = True
    return pad


@pytest.mark.gpu
@pytest.mark.parametrize("drop", [0.0, P_DROP])
@pytest.mark.parametrize("mode", ["sasrec", "bert"])
@pytest.mark.parametrize("L", [200, 256])
def test_padded_first_key_inside_a_block(cuda, L, mode, drop):
    """Padded rows, pad keys masked: the first real key at 1, 37, 63 positions into a 64-key block (and at a block
    start), so the key blocks before it are fully masked, the one holding it is masked in part and those after it are
    interior."""
    causal, mpk = MODES[mode]
    c = _case(_left_padded(L, [0, 1, 37, 63, 64, 69, 130, 191, L - 1]), 2, 64, mpk, seed=7 * L + causal, dev=cuda)
    ctr = torch.tensor([CTR], dtype=torch.int64, device=cuda)
    keep = drop_keep(SEED + CTR, OFF, drop, c.B, c.H, L, c.Lp) if drop > 0 else None
    _check_fwd(c, causal, mpk, 0.0, _attn_fwd(c, causal, mpk, 0.0, drop=drop, ctr=ctr), keep=keep)
    _fused_bwd_case(cuda, c, causal, mpk, 0.0, drop)
