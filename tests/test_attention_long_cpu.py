"""Sequence-length bounds of the attention path without a GPU: both engine configurations accept 256 < L <= 512 with
128-wide head slots and still refuse L > 512, and rp_attn_fwd refuses unsupported shapes before any CUDA call."""
import ctypes

import pytest

from replay_b200._lib import AttnDesc, lib

ESHAPE = -2


def _engine_stub(kind, d, H, L):
    """an engine object with only its configuration set (_check_geometry reads nothing else)"""
    if kind == "sasrec":
        from replay_b200.engine import EncoderConfig, SasRecEngine

        e = SasRecEngine.__new__(SasRecEngine)
        e.cfg = EncoderConfig(n_items=100, d=d, n_heads=H, n_blocks=1, max_len=L, variant="new")
    elif kind == "legacy":
        from replay_b200.engine import EncoderConfig, SasRecEngine

        e = SasRecEngine.__new__(SasRecEngine)
        e.cfg = EncoderConfig(n_items=100, d=d, n_heads=H, n_blocks=1, max_len=L, variant="legacy")
    else:
        from replay_b200.engine_bert import Bert4RecEngine, BertConfig

        e = Bert4RecEngine.__new__(Bert4RecEngine)
        e.cfg = BertConfig(n_items=100, d=d, n_heads=H, n_blocks=1, max_len=L)
    return e


@pytest.mark.parametrize("kind", ["sasrec", "legacy", "bert"])
@pytest.mark.parametrize("d,H", [(128, 1), (100, 1), (512, 4), (300, 4)])
def test_geometry_accepts_long_windows_with_128_wide_heads(kind, d, H):
    for L in (257, 512):
        e = _engine_stub(kind, d, H, L)
        assert e.cfg.head_slot == 128
        e._check_geometry(L)
    e = _engine_stub(kind, d, H, 513)
    with pytest.raises(ValueError):
        e._check_geometry(513)


def _desc(L, head_dim):
    a = AttnDesc()
    fake = 1 << 20   # never dereferenced: the shape checks come first
    a.q = a.k = a.v = a.out = a.pad_mask = fake
    H = 2
    a.q_rows = a.k_rows = a.v_rows = 4 * L
    a.q_cols = a.ldq = H * head_dim
    a.k_cols = a.ldk = a.v_cols = a.ldv = 2 * H * head_dim
    a.v_c0 = H * head_dim
    a.B, a.H, a.L, a.head_dim = 4, H, L, head_dim
    a.causal, a.mask_pad_keys = 1, 1
    a.ldo = H * head_dim
    return a


@pytest.mark.parametrize("L,head_dim", [(513, 64), (513, 128), (300, 96), (300, 256), (100, 32), (512, 192)])
def test_attn_fwd_rejects_unsupported_shapes(L, head_dim):
    assert lib().rp_attn_fwd(ctypes.byref(_desc(L, head_dim)), None) == ESHAPE
