"""rp_gemm's argument checks (include/rp_b200.h): every one is decided before a tensor map is made or a kernel launched,
so each return code is checked here, with dummy host buffers, on a machine without a GPU."""
import ctypes

import pytest

from replay_b200._lib import GemmDesc, lib

EINVAL, ESHAPE, EALIGN, EDRIVER = -1, -2, -3, -4

_BUF = ctypes.create_string_buffer(4096 + 64)
_BASE = (ctypes.addressof(_BUF) + 63) // 64 * 64      # 64-byte aligned dummy memory; nothing reads it


def _desc(**kw):
    """A valid bf16 [256, 128] x [128, 128] GEMM on dummy pointers, with the fields of ``kw`` changed."""
    g = GemmDesc()
    g.A, g.a_rows, g.a_cols, g.lda = _BASE, 256, 128, 128
    g.B, g.b_rows, g.b_cols, g.ldb = _BASE, 128, 128, 128
    g.M, g.N, g.K, g.batch, g.inner = 256, 128, 128, 1, 1
    g.C, g.ldc, g.out_mode, g.alpha, g.split_k = _BASE, 128, 0, 1.0, 1
    for k, v in kw.items():
        setattr(g, k, v)
    return g


_P = _BASE + 256     # a second, 16-byte aligned dummy pointer

_CASES = {
    # split_k > 1 runs the epilogue once per split: only alpha and rowmask may be split
    "split_bias": (EINVAL, dict(out_mode=1, split_k=2, bias=_P)),
    "split_act": (EINVAL, dict(out_mode=3, split_k=2, act=1)),
    "split_residual": (EINVAL, dict(out_mode=1, split_k=3, residual=_P)),
    "split_gate": (EINVAL, dict(out_mode=1, split_k=2, gate=_P)),
    "split_c2": (EINVAL, dict(out_mode=3, split_k=2, C2=_P)),
    "split_dropout": (EINVAL, dict(out_mode=1, split_k=2, drop_p=0.1)),
    "split_post_dropout": (EINVAL, dict(out_mode=1, split_k=2, post_drop_p=0.1)),
    "split_out_mode_2": (EINVAL, dict(out_mode=2, split_k=2)),
    "split_out_mode_4": (EINVAL, dict(out_mode=4, split_k=2)),
    # TMA boxes start at 16-byte aligned columns of the stored operands
    "a_c0": (EALIGN, dict(a_c0=6)),
    "a_co": (EALIGN, dict(batch=2, a_co=4)),
    "a_ci": (EALIGN, dict(batch=2, inner=2, a_ci=1)),
    "b_c0": (EALIGN, dict(b_c0=3)),
    "b_co": (EALIGN, dict(batch=2, b_co=12)),
    "b_ci": (EALIGN, dict(batch=2, inner=2, b_ci=2)),
    # act 3 / 4 need the per-row offsets; act 4 takes K-major operands only
    "exp2_without_offsets": (EINVAL, dict(act=3)),
    "sigmoid_a_mn": (EINVAL, dict(act=4, row_exp2_offset=_P, a_mn=1)),
    "sigmoid_b_mn": (EINVAL, dict(act=4, row_exp2_offset=_P, b_mn=1)),
    "sigmoid_split": (EINVAL, dict(act=4, row_exp2_offset=_P, out_mode=1, split_k=2)),
    # out_mode 0 stores 16 bytes at a time
    "bf16_ldc": (EALIGN, dict(ldc=132)),
    "bf16_c_pointer": (EALIGN, dict(C=_BASE + 8)),
    "bf16_c_off0": (EALIGN, dict(c_off0=4)),
    "bf16_c_oo": (EALIGN, dict(batch=2, c_oo=128 * 256 + 4)),
    "bf16_c_oi": (EALIGN, dict(batch=2, inner=2, c_oi=128 * 256 + 2)),
    # the residual is read 16 bytes at a time at C's geometry, whatever C's type
    "residual_pointer": (EALIGN, dict(out_mode=2, residual=_P + 2)),
    "residual_ldc": (EALIGN, dict(out_mode=2, ldc=130, residual=_P)),
    "residual_c_off0": (EALIGN, dict(out_mode=2, c_off0=1, residual=_P)),
    "residual_c_oo": (EALIGN, dict(out_mode=2, batch=2, c_oo=128 * 256 + 4, residual=_P)),
    # C2 is stored in bf16 pairs
    "c2_ldc": (EALIGN, dict(out_mode=2, ldc=129, C2=_P)),
    "c2_c_off0": (EALIGN, dict(out_mode=2, c_off0=3, C2=_P)),
    "c2_c_oi": (EALIGN, dict(out_mode=2, batch=2, inner=2, c_oi=1, C2=_P)),
    "c2_pointer": (EALIGN, dict(out_mode=2, C2=_P + 2)),
}


@pytest.mark.parametrize("case", sorted(_CASES))
def test_rp_gemm_rejects_descriptor(case):
    rc, kw = _CASES[case]
    assert lib().rp_gemm(ctypes.byref(_desc(**kw)), None) == rc


def test_rp_gemm_argument_checks_do_not_reject_their_neighbours():
    """Descriptors one step from the rejected ones pass every argument check.  Their grid is too large to launch
    (2^30 rows x 2^20 columns: 2^36 tiles), so they end at the tensor maps without a driver (RP_EDRIVER) or at the grid-size
    check with one (RP_ESHAPE): no kernel ever runs on the dummy pointers."""
    huge = dict(M=1 << 30, N=1 << 20)
    ok = [dict(out_mode=1, split_k=7, alpha=-2.0, rowmask=_P), dict(out_mode=3, split_k=5, rowmask=_P),
          dict(out_mode=2, ldc=129, c_off0=1), dict(out_mode=4, c_off0=1), dict(out_mode=2, ldc=130, C2=_P, c_off0=2),
          dict(c_off0=8, batch=2, c_oo=128 * 256 + 8, residual=_P), dict(act=4, row_exp2_offset=_P)]
    for kw in ok:
        assert lib().rp_gemm(ctypes.byref(_desc(**kw, **huge)), None) in (EDRIVER, ESHAPE), kw
