"""rp_gemm (csrc/rp_gemm.cu) against its float64 model (tests/gemm_reference.py) at every operand layout, tile edge,
batch geometry, epilogue stage, output mode and dynamic limit.

Operands are views with padded pitches inside buffers filled with finite poison (300.0): an element fetched past a view's
bounds shows up in the result.  Every output buffer starts as a sentinel; elements the kernel must leave alone (rows >= M,
columns >= N, the pitch padding, skipped tiles) must keep its bits.  fp32 outputs must be within the model's tolerance
(about 1e-5 x sum_k |a_k b_k| carried through the epilogue), bf16 outputs within one bf16 rounding on top of it; the
model's exact zeros (dropped elements, empty splits, act 4 at a -inf offset) must be exact.
Run with -s to print the worst error of each family.
"""
import numpy as np
import pytest
import torch

import gemm_reference as gr
from fp64_checks import WorstErrors
from replay_b200 import ops
from replay_b200._lib import check, lib

POISON = 300.0
SENT = -3.25                          # exact in bf16 and fp32
SEED, CTR = 0x5EED1234ABC, 987654321  # dropout stream (seed_ptr holds CTR)

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


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _ru(x, m):
    return (x + m - 1) // m * m


def _view(vals, dev, r0=1, c0=8, extra=16):
    """``vals`` [rows, cols] as a view at (r0, c0) of a poison-filled bf16 buffer with a padded pitch (multiple of 8)."""
    rows, cols = vals.shape
    buf = torch.full((r0 + rows + 2, _ru(c0 + cols, 8) + extra), POISON, dtype=torch.bfloat16)
    buf[r0:r0 + rows, c0:c0 + cols] = vals.to(torch.bfloat16)
    return buf.to(dev)[r0:r0 + rows, c0:c0 + cols]


def _randn(rows, cols, g, scale=1.0):
    return (torch.randn(rows, cols, generator=g) * scale).to(torch.bfloat16)


def _out(rows, ldc, dev, dtype, fill=SENT):
    """A sentinel-filled output buffer of ``rows`` rows with pitch ``ldc`` (plus one spare row)."""
    return torch.full((rows + 1, ldc), fill, dtype=dtype, device=dev)


def _cpu(v):
    return v.cpu() if torch.is_tensor(v) else v


def _run(A, B, C, M, N, K, **kw):
    """rp_gemm through ops.gemm and the model on copies of the same buffers; returns {name: (kernel buffer flat, model)}."""
    model_kw = {}
    for k, v in kw.items():
        if torch.is_tensor(v):
            # copy whole storages so the model sees what surrounds a view (C's neighbours, gate / residual geometry)
            full = gr.flat_from(v).cpu()
            model_kw[k] = torch.as_strided(full, v.shape, v.stride(), 0) if v.dim() else full
        else:
            model_kw[k] = v
    Cc = torch.as_strided(gr.flat_from(C).cpu(), C.shape, C.stride(), 0)
    if kw.get("C2") is not None:
        model_kw["C2"] = torch.as_strided(gr.flat_from(kw["C2"]).cpu(), kw["C2"].shape, kw["C2"].stride(), 0)
    exp = gr.gemm(_cpu(A), _cpu(B), Cc, M, N, K, **model_kw)
    dev_kw = dict(kw)
    if kw.get("seed_ptr") is not None:
        dev_kw["seed_ptr"] = kw["seed_ptr"].data_ptr()
    ops.gemm(A, B, C, M, N, K, **dev_kw)
    torch.cuda.synchronize()
    out = {"C": (gr.flat_from(C), exp["C"])}
    if kw.get("C2") is not None:
        out["C2"] = (gr.flat_from(kw["C2"]), exp["C2"])
    return out


def _check(res, family):
    for name, (got, exp) in res.items():
        bf16 = got.dtype == torch.bfloat16
        n_bad = gr.untouched(got, exp)
        assert n_bad == 0, f"{family} {name}: {n_bad} elements that must be left alone changed"
        e = _note(f"{family} {name}", gr.err(got, exp, bf16))
        if e >= 1.0:
            i = int(gr.worst(got, exp, bf16))
            pytest.fail(f"{family} {name}: error {e:.3g} tolerances at flat element {i}: kernel {float(got[i])!r}, "
                        f"model {float(exp['out'][i])!r} +- {float(exp['atol'][i]):.3g}")


# ----------------------------------------------------------------------------------------------------------------------
# operand layouts x tile edges
# ----------------------------------------------------------------------------------------------------------------------
# N 1 / 8 / 33 / 64 take the BN = 64 tiles, 65 .. 257 the BN = 128 ones; K 128 -> 129 switches the 2-stage ring to the
# 4-stage one and K 1000 wraps it several times
_SHAPES = [(1, 1, 8), (63, 8, 63), (127, 33, 64), (128, 64, 65), (129, 65, 128), (300, 127, 129), (128, 128, 256),
           (63, 129, 257), (300, 257, 1000), (1, 64, 1000), (129, 1, 129)]


@pytest.mark.gpu
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("M,N,K", _SHAPES)
def test_layouts_and_tile_edges(cuda, M, N, K, a_mn, b_mn):
    """Both majors of both operands at every tile edge of M, N and K; bf16 and fp32 outputs alternate over the shapes."""
    g = _gen(M * 7 + N * 3 + K + 11 * a_mn + 13 * b_mn)
    a = _randn(M, K, g)
    b = _randn(N, K, g, 0.1)
    A = _view(a.T.contiguous() if a_mn else a, cuda)
    B = _view(b.T.contiguous() if b_mn else b, cuda, r0=2, c0=16)
    bf16 = _SHAPES.index((M, N, K)) % 2 == 0
    C = _out(M, _ru(N, 8) + 8, cuda, torch.bfloat16 if bf16 else torch.float32)
    res = _run(A, B, C[:M, :N], M, N, K, a_mn=a_mn, b_mn=b_mn, out_mode=0 if bf16 else 2)
    _check(res, "layouts " + ("bf16" if bf16 else "fp32"))


# ----------------------------------------------------------------------------------------------------------------------
# epilogue stages
# ----------------------------------------------------------------------------------------------------------------------
_STAGES = ["plain", "bias", "alpha", "relu", "gelu", "exp2", "sigmoid", "gate0", "gate1", "residual", "rowmask",
           "dropout", "post_dropout", "c2", "all"]


def _stage_kw(stage, M, N, ldc, g, dev):
    ctr = torch.tensor([CTR], dtype=torch.int64, device=dev)
    drop = dict(drop_p=0.2, drop_offset=3 << 40, seed=SEED, seed_ptr=ctr)

    def like_c(scale, zeros=0.0):
        buf = torch.full((M + 1, ldc), POISON, dtype=torch.bfloat16)
        v = torch.randn(M, N, generator=g) * scale
        v = v.masked_fill(torch.rand(M, N, generator=g) < zeros, 0.0)
        buf[:M, :N] = v.to(torch.bfloat16)
        return buf.to(dev)[:M, :N]

    off = torch.empty(M).uniform_(-2.0, 2.0, generator=g)
    off[::7] = float("-inf")
    bias = (torch.randn(N, generator=g) * 0.5).to(dev)
    rowmask = (torch.rand(M, generator=g) > 0.3).to(torch.uint8).to(dev)
    c2 = torch.full((M + 1, ldc), SENT, dtype=torch.bfloat16, device=dev)[:M, :N]
    kw = {"plain": {}, "bias": dict(bias=bias), "alpha": dict(alpha=-0.6875), "relu": dict(act=1, bias=bias),
          "gelu": dict(act=2), "exp2": dict(act=3, row_exp2_offset=off.to(dev)),
          "sigmoid": dict(act=4, row_exp2_offset=off.to(dev), bias=bias),
          "gate0": dict(gate=like_c(1.0, zeros=0.4), gate_scale=1.25),
          "gate1": dict(gate=like_c(1.5, zeros=0.1), gate_mode=1, gate_scale=0.8),
          "residual": dict(residual=like_c(2.0)), "rowmask": dict(rowmask=rowmask), "dropout": drop,
          "post_dropout": dict(residual=like_c(1.0), post_drop_p=0.1, post_drop_offset=4 << 40, seed=SEED, seed_ptr=ctr),
          "c2": dict(C2=c2, bias=bias, act=2),
          "all": dict(drop, bias=bias, alpha=-0.75, act=2, C2=c2, gate=like_c(1.0, zeros=0.3), gate_scale=1.1,
                      residual=like_c(1.0), post_drop_p=0.1, post_drop_offset=4 << 40, rowmask=rowmask)}
    return kw[stage]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("N", [200, 40])
@pytest.mark.parametrize("stage", _STAGES)
def test_epilogue_stage(cuda, stage, N, dtype):
    """Each stage alone, then all of them, at M 300 and K 192 (ragged row tile, three K chunks) with N 200 (BN 128,
    ragged column tile) and N 40 (BN 64): alpha < 0, gates with exact zeros, act 4 at offsets including -inf, dropout
    drawn behind a device seed counter (its zero pattern must match exactly)."""
    if stage == "sigmoid" and N == 40:
        pytest.skip("act 4 always runs 128-column tiles; N 200 covers it")
    M, K = 300, 192
    g = _gen(_STAGES.index(stage) * 1000 + N)
    A = _view(_randn(M, K, g), cuda)
    scale = 0.02 if stage in ("exp2", "sigmoid") else 0.1
    B = _view(_randn(N, K, g, scale), cuda, c0=24)
    ldc = _ru(N, 8) + 8
    C = _out(M, ldc, cuda, dtype)
    kw = _stage_kw(stage, M, N, ldc, g, cuda)
    res = _run(A, B, C[:M, :N], M, N, K, out_mode=0 if dtype == torch.bfloat16 else 2, **kw)
    _check(res, f"epilogue {stage}")


@pytest.mark.gpu
@pytest.mark.parametrize("N", [1, 33, 127, 129, 255])
def test_c2_at_odd_n_leaves_column_n_alone(cuda, N):
    """C2 is stored in bf16 pairs; at odd N the last column is stored alone.  C2's rows have a pitch of N rounded up to 8,
    so column N of every row is pitch padding holding a sentinel that must survive."""
    M, K = 130, 64
    g = _gen(N)
    A, B = _view(_randn(M, K, g), cuda), _view(_randn(N, K, g, 0.1), cuda)
    ldc = _ru(N, 8)
    C = _out(M, ldc, cuda, torch.float32)
    C2 = _out(M, ldc, cuda, torch.bfloat16)
    res = _run(A, B, C[:M, :N], M, N, K, out_mode=2, C2=C2[:M, :N], act=1)
    assert (C2[:M, N:] == SENT).all(), "C2 written at or past column N"
    _check(res, "c2 odd N")


# ----------------------------------------------------------------------------------------------------------------------
# output modes
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("split,K", [(1, 1000), (2, 1000), (3, 1000), (7, 1000), (7, 129), (3, 64)])
def test_atomic_split_k_onto_prefilled_c(cuda, split, K):
    """out_mode 1 adds alpha * sum * rowmask onto C's previous contents with 1 .. 7 K splits, also with more splits than
    K chunks (7 over 3, 3 over 1: empty splits add zeros)."""
    M, N = 200, 96
    g = _gen(split * 100 + K)
    A, B = _view(_randn(M, K, g), cuda), _view(_randn(K, N, g, 0.1), cuda)
    C = torch.randn(M + 1, N + 8, generator=g).to(cuda)
    rowmask = (torch.rand(M, generator=g) > 0.2).to(torch.uint8).to(cuda)
    res = _run(A, B, C[:M, :N], M, N, K, b_mn=True, out_mode=1, split_k=split, alpha=-1.5, rowmask=rowmask)
    _check(res, "out_mode 1 split-K")


def _partials(cuda, split, M, N, K, g, lim=None, klim=None):
    A, B = _view(_randn(K, M, g), cuda), _view(_randn(K, N, g), cuda)
    n = M * N
    ws = torch.full((split * n + 64,), 7.0, device=cuda)
    kw = dict(a_mn=True, b_mn=True, out_mode=3, split_k=split, c_geom=(N, 0, 0, 0), c_split_stride=n)
    if lim is not None:
        kw.update(m_limit=lim, m_limit_base=3)
    if klim is not None:
        kw.update(k_limit=klim, k_limit_base=10)
    return A, B, ws, kw


@pytest.mark.gpu
@pytest.mark.parametrize("accumulate", [0, 1])
@pytest.mark.parametrize("split", [1, 8, 9, 100])
def test_split_partials_and_reduction(cuda, split, accumulate):
    """out_mode 3 stores each split's partial at C + s * c_split_stride (empty splits: exact zeros; nothing past the last
    split), rp_reduce_splits sums them onto a pre-filled or a fresh destination; both are bitwise reproducible."""
    M, N, K = 200, 64, 1000
    n = M * N
    g = _gen(split * 2 + accumulate)
    A, B, ws, kw = _partials(cuda, split, M, N, K, g)
    preset = torch.randn(n + 8, generator=g).to(cuda)

    def run():
        w = ws.clone()
        res = _run(A, B, w, M, N, K, **kw)
        dst = preset.clone()
        exp = gr.reduce_splits(w.cpu(), split, n, n, dst.cpu(), accumulate)
        check(lib().rp_reduce_splits(w.data_ptr(), split, n, n, dst.data_ptr(), accumulate,
                                     torch.cuda.current_stream().cuda_stream), "rp_reduce_splits")
        torch.cuda.synchronize()
        return res, w, dst, exp

    res, w, dst, exp = run()
    _check(res, "out_mode 3 partials")
    assert gr.untouched(dst, exp) == 0
    assert _note("reduce_splits", gr.err(dst, exp, False)) < 1.0
    _, w2, dst2, _ = run()
    assert torch.equal(w, w2) and torch.equal(dst, dst2), "split-K reruns must be bit-identical"


@pytest.mark.gpu
@pytest.mark.parametrize("c_off0", [0, 1])
def test_read_modify_write_aligned_and_scalar(cuda, c_off0):
    """out_mode 4 (C += x): a 16-byte aligned C takes the float4 path, c_off0 = 1 the scalar one."""
    M, N, K = 150, 136, 200
    g = _gen(40 + c_off0)
    A, B = _view(_randn(M, K, g), cuda), _view(_randn(N, K, g, 0.1), cuda)
    ldc = N + 8
    C = torch.randn((M + 1) * ldc, generator=g).to(cuda)
    res = _run(A, B, C, M, N, K, out_mode=4, c_geom=(ldc, c_off0, 0, 0), alpha=0.5)
    _check(res, "out_mode 4")


@pytest.mark.gpu
def test_bf16_store_at_an_offset_with_a_wide_pitch(cuda):
    """out_mode 0 at c_off0 = 16 with ldc = N + 24: only [M, N] from the offset is written."""
    M, N, K = 140, 72, 96
    g = _gen(50)
    A, B = _view(_randn(M, K, g), cuda), _view(_randn(N, K, g, 0.1), cuda)
    ldc = N + 24
    C = torch.full(((M + 2) * ldc,), SENT, dtype=torch.bfloat16, device=cuda)
    res = _run(A, B, C, M, N, K, out_mode=0, c_geom=(ldc, 16, 0, 0), bias=torch.randn(N, generator=g).to(cuda))
    _check(res, "out_mode 0 offset")


# ----------------------------------------------------------------------------------------------------------------------
# batched geometry
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("batch,inner", [(1, 1), (3, 1), (3, 2), (6, 2), (6, 3), (3, 3)])
def test_batched_offsets_and_c_geometry(cuda, batch, inner, a_mn, b_mn):
    """batch = outer x inner with outer stepping the operands' rows and inner their columns (K-major) or K rows
    (MN-major), so that the K tail (K = 100) reads the next batch element; C at an offset per-(outer, inner) geometry,
    rowmask by outer.  Column offsets are multiples of 8 (TMA boxes start 16-byte aligned); row offsets are not."""
    M, N, K = 90, 72, 100
    n_outer = -(-batch // inner)
    g = _gen(batch * 10 + inner + 100 * a_mn + 200 * b_mn)

    def stored(rows_mn, mn):
        """(view, offsets): outer steps the MN rows, inner steps K."""
        if mn:      # stored [K rows, MN cols]: inner along the rows, outer along the columns
            v = _view(_randn(inner * K + 30, n_outer * (_ru(rows_mn, 8) + 8) + 16, g, 0.3), cuda)
            return v, (2, 0, K, 8, _ru(rows_mn, 8) + 8, 0)
        v = _view(_randn(n_outer * (rows_mn + 5) + 4, inner * _ru(K, 8) + 40, g, 0.3), cuda)
        return v, (1, rows_mn + 5, 0, 8, 0, _ru(K, 8))

    A, a_off = stored(M, a_mn)
    B, b_off = stored(N, b_mn)
    ldc = N + 8
    oi, oo = M * ldc, inner * M * ldc + 16
    bf16 = (batch + inner) % 2 == 0
    C = torch.full((n_outer * oo + 8 + 64,), SENT, dtype=torch.bfloat16 if bf16 else torch.float32, device=cuda)
    rowmask = (torch.rand(n_outer * M + 5, generator=g) > 0.3).to(torch.uint8).to(cuda)
    res = _run(A, B, C, M, N, K, a_mn=a_mn, b_mn=b_mn, batch=batch, inner=inner, a_off=a_off, b_off=b_off,
               c_geom=(ldc, 8, oo, oi), rowmask=rowmask, rowmask_oo=M, out_mode=0 if bf16 else 2)
    _check(res, "batched")


def _attn_bwd_buffers(B_, H, L, hd, g, dev):
    """QKV bf16 [T, 3 H hd] (q | k | v), d_o [T, H hd], P / dS [B H Lp, Lp] with zero pad rows and columns, dQKV sentinel."""
    T, Lp = B_ * L, _ru(L, 64)
    QKV = _randn(T, 3 * H * hd, g).to(dev)
    d_o = _randn(T, H * hd, g).to(dev)
    P = torch.zeros(B_ * H, Lp, Lp)
    P[:, :L, :L] = torch.rand(B_ * H, L, L, generator=g) / L
    dS = torch.zeros(B_ * H, Lp, Lp)
    dS[:, :L, :L] = torch.randn(B_ * H, L, L, generator=g) / L
    return (T, Lp, QKV, d_o, P.to(torch.bfloat16).to(dev).view(B_ * H * Lp, Lp),
            dS.to(torch.bfloat16).to(dev).view(B_ * H * Lp, Lp))


@pytest.mark.gpu
@pytest.mark.parametrize("L", [50, 200])
def test_engine_attention_backward_descriptors(cuda, L):
    """The four batched GEMMs of SasRecEngine's un-fused attention backward (engine.py), with their exact descriptors at
    B 3, H 2, head slot 64: dPd = dO V^T into [B H Lp, Lp], dQ = dS K, dK = dS^T Q and dV = Pd^T dO into per-head column
    blocks of [T, 3 H hd].  The K tails run into the next sequence's rows of Q / K / V / dO, against zero pad rows and
    columns of dS / Pd."""
    B_, H, hd = 3, 2, 64
    g = _gen(L)
    T, Lp, QKV, d_o, P, dS = _attn_bwd_buffers(B_, H, L, hd, g, cuda)
    BH = B_ * H
    q, k, v = (QKV, 0), (QKV, H * hd), (QKV, 2 * H * hd)
    dQKV = torch.full((T, 3 * H * hd), SENT, dtype=torch.bfloat16, device=cuda)
    dpd = torch.full((BH * Lp, Lp), SENT, dtype=torch.bfloat16, device=cuda)
    heads = dict(batch=BH, inner=H, a_off=(0, H * Lp, Lp, 0, 0, 0))
    out = lambda t, c0: (t.stride(0), c0, L * t.stride(0), hd)  # noqa: E731
    res = _run(d_o, v[0], dpd, L, L, hd, batch=BH, inner=H, a_off=(0, L, 0, 0, 0, hd), b_off=(0, L, 0, v[1], 0, hd),
               c_geom=(Lp, 0, H * Lp * Lp, Lp * Lp))
    _check(res, "engine dPd")
    res = _run(dS, k[0], dQKV, L, hd, L, b_mn=True, b_off=(0, L, 0, k[1], 0, hd), c_geom=out(dQKV, 0), **heads)
    _check(res, "engine dQ")
    res = _run(dS, q[0], dQKV, L, hd, L, a_mn=True, b_mn=True, b_off=(0, L, 0, q[1], 0, hd), c_geom=out(dQKV, H * hd),
               **heads)
    _check(res, "engine dK")
    res = _run(P, d_o, dQKV, L, hd, L, a_mn=True, b_mn=True, b_off=(0, L, 0, 0, 0, hd), c_geom=out(dQKV, 2 * H * hd),
               **heads)
    _check(res, "engine dV")


@pytest.mark.gpu
@pytest.mark.parametrize("L", [50, 200])
def test_diff_engine_attention_backward_descriptors(cuda, L):
    """The batched GEMMs of DiffSasRecEngine's attention backward (engine_diff.py) at B 3, H 2, v_slot 128: dA = dO_pre
    V^T, dQ1 / dQ2 = dS K and dK1 / dK2 = dS^T Q into 64-wide slots of dQKV, dV = A^T dO_pre."""
    B_, H, slot, vs = 3, 2, 64, 128
    g = _gen(L + 1)
    T, Lp = B_ * L, _ru(L, 64)
    n = H * 2 * slot * 2 + H * vs
    kc, vc = H * 2 * slot, H * 4 * slot
    QKV = _randn(T, n, g).to(cuda)
    dOpre = _randn(T, H * vs, g).to(cuda)
    BH = B_ * H
    pads = []
    for _ in range(3):
        t = torch.zeros(BH, Lp, Lp)
        t[:, :L, :L] = torch.randn(BH, L, L, generator=g) / L
        pads.append(t.to(torch.bfloat16).to(cuda).view(BH * Lp, Lp))
    dS1, dS2, Amat = pads
    dQKV = torch.full((T, n), SENT, dtype=torch.bfloat16, device=cuda)
    dA = torch.full((BH * Lp, Lp), SENT, dtype=torch.bfloat16, device=cuda)
    heads = dict(batch=BH, inner=H, a_off=(0, H * Lp, Lp, 0, 0, 0))
    out = lambda c0, width: (n, c0, L * n, width)  # noqa: E731
    res = _run(dOpre, QKV, dA, L, L, vs, batch=BH, inner=H, a_off=(0, L, 0, 0, 0, vs), b_off=(0, L, 0, vc, 0, vs),
               c_geom=(Lp, 0, H * Lp * Lp, Lp * Lp))
    _check(res, "diff dA")
    for half, dS in ((0, dS1), (slot, dS2)):
        res = _run(dS, QKV, dQKV, L, slot, L, b_mn=True, b_off=(0, L, 0, kc + half, 0, 2 * slot),
                   c_geom=out(half, 2 * slot), **heads)
        _check(res, "diff dQ")
        res = _run(dS, QKV, dQKV, L, slot, L, a_mn=True, b_mn=True, b_off=(0, L, 0, half, 0, 2 * slot),
                   c_geom=out(kc + half, 2 * slot), **heads)
        _check(res, "diff dK")
    res = _run(Amat, dOpre, dQKV, L, vs, L, a_mn=True, b_mn=True, b_off=(0, L, 0, 0, 0, vs), c_geom=out(vc, vs), **heads)
    _check(res, "diff dV")


# ----------------------------------------------------------------------------------------------------------------------
# dynamic limits
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("lim", [0, 1, 127, 128, 129, 300, 400])
def test_m_limit_skips_whole_row_tiles(cuda, lim):
    """Row tiles with m0 + m_limit_base >= *m_limit keep C's sentinel (base 3: limits 0 and 1 skip every tile, 127 and
    128 compute tile 0 only, 129 tiles 0 and 1, 300 and 400 all three)."""
    M, N, K = 300, 136, 128
    g = _gen(lim)
    A, B = _view(_randn(M, K, g), cuda), _view(_randn(N, K, g, 0.1), cuda)
    C = _out(M, N + 8, cuda, torch.bfloat16)
    res = _run(A, B, C[:M, :N], M, N, K, m_limit=torch.tensor([lim], dtype=torch.int32, device=cuda), m_limit_base=3,
               bias=torch.randn(N, generator=g).to(cuda), act=1)
    _check(res, "m_limit")


@pytest.mark.gpu
@pytest.mark.parametrize("lim", [0, 1, 63, 64, 65, 200, 260])
def test_k_limit_trims_the_contraction(cuda, lim):
    """The contraction stops at *k_limit - k_limit_base (base 10), rounded up to whole 64-element chunks of the stored
    operands (the rest of the last chunk is read as stored); 0 gives an empty contraction (the epilogue of zero)."""
    M, N, K = 140, 72, 200
    g = _gen(lim + 7)
    A, B = _view(_randn(K, M, g), cuda), _view(_randn(K, N, g), cuda)
    C = _out(M, N + 8, cuda, torch.float32)
    res = _run(A, B, C[:M, :N], M, N, K, a_mn=True, b_mn=True, out_mode=2,
               k_limit=torch.tensor([lim + 10], dtype=torch.int32, device=cuda), k_limit_base=10,
               bias=torch.randn(N, generator=g).to(cuda))
    _check(res, "k_limit")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [1, 3])
@pytest.mark.parametrize("m_lim,k_lim", [(0, 1000), (131, 1000), (300, 65), (200, 0), (131, 700)])
def test_limits_with_split_k(cuda, mode, m_lim, k_lim):
    """m_limit and k_limit under split-K: skipped tiles keep their sentinel in every split's partial (out_mode 3) or in C
    (out_mode 1); splits past the trimmed contraction store or add zeros."""
    M, N, K, split = 300, 64, 1000, 6
    g = _gen(m_lim * 3 + k_lim + mode)
    lim = torch.tensor([m_lim + 3], dtype=torch.int32, device=cuda)
    klim = torch.tensor([k_lim + 10], dtype=torch.int32, device=cuda)
    A, B, ws, kw = _partials(cuda, split, M, N, K, g, lim, klim)
    if mode == 1:
        kw.update(out_mode=1, c_split_stride=0)
        ws = torch.randn(M * N + 64, generator=g).to(cuda)
    res = _run(A, B, ws, M, N, K, **kw)
    _check(res, f"limits split-K mode {mode}")


# ----------------------------------------------------------------------------------------------------------------------
# determinism
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 2])
def test_stores_are_bitwise_reproducible(cuda, mode):
    """out_mode 0 and 2 give the same bits on a rerun (out_mode 3 + reduce: test_split_partials_and_reduction)."""
    M, N, K = 300, 257, 1000
    g = _gen(60 + mode)
    A, B = _view(_randn(M, K, g), cuda), _view(_randn(N, K, g, 0.1), cuda)
    outs = []
    for _ in range(2):
        C = _out(M, _ru(N, 8) + 8, cuda, torch.bfloat16 if mode == 0 else torch.float32)
        ops.gemm(A, B, C[:M, :N], M, N, K, out_mode=mode, bias=torch.ones(N, device=cuda), act=2)
        torch.cuda.synchronize()
        outs.append(C)
    assert torch.equal(outs[0], outs[1])
