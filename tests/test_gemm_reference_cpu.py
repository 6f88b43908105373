"""The float64 model of rp_gemm (tests/gemm_reference.py) against plain torch, a hand-written batched loop, and the
mistakes its tolerance must reject - no GPU needed."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import gemm_reference as gr
from dropout_stream import keep_draws

SENT = -3.25
SEED, CTR = 0x5EED1234ABC, 987654321


def _bf(x):
    return x.to(torch.bfloat16)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _run(A, B, M, N, K, dtype=torch.float32, **kw):
    C = torch.full((M, N), SENT, dtype=dtype)
    r = gr.gemm(A, B, C, M, N, K, **kw)
    out = r["C"]["out"].view(M, N)
    c2 = r["C2"]["out"].view(M, N) if r["C2"] is not None else None
    return out, c2, r


@pytest.mark.parametrize("stage", ["plain", "alpha", "bias", "relu", "gelu", "exp2", "sigmoid", "gate0", "gate1",
                                   "residual", "rowmask", "dropout", "post_dropout", "c2"])
def test_single_stage_matches_plain_torch(stage):
    """Batch 1, K-major operands, K % 64 == 0: each epilogue stage alone is the torch expression of the header."""
    g = _gen(1)
    M, N, K = 37, 29, 128
    A, W = _bf(torch.randn(M, K, generator=g)), _bf(torch.randn(N, K, generator=g) / 8)
    x = F.linear(A.double(), W.double())
    bias = torch.randn(N, generator=g)
    off = torch.randn(M, generator=g)
    gate = _bf(torch.randn(M, N, generator=g)).masked_fill(torch.rand(M, N, generator=g) < 0.3, 0)
    res = _bf(torch.randn(M, N, generator=g))
    rowmask = (torch.rand(M, generator=g) > 0.4).to(torch.uint8)
    ctr = torch.tensor([CTR])
    keep = keep_draws(SEED + CTR, 5 << 40, 0.25, np.arange(M), N).double() / 0.75
    kw, want = {}, x
    if stage == "alpha":
        kw, want = dict(alpha=-0.75), -0.75 * x
    elif stage == "bias":
        kw, want = dict(bias=bias), F.linear(A.double(), W.double(), bias.double())
    elif stage == "relu":
        kw, want = dict(act=1), torch.relu(x)
    elif stage == "gelu":
        kw, want = dict(act=2), F.gelu(x, approximate="none")
    elif stage == "exp2":
        kw, want = dict(act=3, row_exp2_offset=off), torch.exp2(x * math.log2(math.e) + off.double()[:, None])
    elif stage == "sigmoid":
        kw, want = dict(act=4, row_exp2_offset=off), torch.sigmoid(x) * torch.exp2(off.double()[:, None])
    elif stage == "gate0":
        kw, want = dict(gate=gate, gate_scale=1.5), x * (gate != 0).double() * 1.5
    elif stage == "gate1":
        z = gate.double().requires_grad_(True)
        F.gelu(z, approximate="none").sum().backward()
        kw, want = dict(gate=gate, gate_mode=1, gate_scale=0.5), x * z.grad * 0.5
    elif stage == "residual":
        kw, want = dict(residual=res), x + res.double()
    elif stage == "rowmask":
        kw, want = dict(rowmask=rowmask), x * rowmask.double()[:, None]
    elif stage == "dropout":
        kw, want = dict(drop_p=0.25, drop_offset=5 << 40, seed=SEED, seed_ptr=ctr), x * keep
    elif stage == "post_dropout":
        kw, want = dict(post_drop_p=0.25, post_drop_offset=5 << 40, seed=SEED, seed_ptr=ctr, residual=res), \
            (x + res.double()) * keep
    out, c2, _ = _run(A, W, M, N, K, **kw, **(dict(C2=torch.zeros(M, N, dtype=torch.bfloat16), act=1, bias=bias)
                                              if stage == "c2" else {}))
    if stage == "c2":
        torch.testing.assert_close(c2, F.linear(A.double(), W.double(), bias.double()), rtol=1e-12, atol=1e-12)
        want = torch.relu(F.linear(A.double(), W.double(), bias.double()))
    torch.testing.assert_close(out, want, rtol=1e-12, atol=1e-12)


def test_sigmoid_at_minus_inf_offset_is_exactly_zero():
    g = _gen(2)
    A, W = _bf(torch.randn(8, 64, generator=g) * 10), _bf(torch.randn(8, 64, generator=g))
    off = torch.tensor([0.0, float("-inf")] * 4)
    out, _, _ = _run(A, W, 8, 8, 64, act=4, row_exp2_offset=off)
    assert (out[1::2] == 0).all() and (out[0::2] != 0).all()


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)])
def test_batched_fetch_matches_a_loop_over_outer_and_inner(a_mn, b_mn):
    """batch 6 = outer 2 x inner 3 with row and column offsets on both operands, K = 70 (a 58-element K tail that reads
    the following columns / rows of the stored array, zeros past its end), C at an offset geometry."""
    g = _gen(3)
    M, N, K, batch, inner = 5, 7, 70, 6, 3
    Kc = 128
    a_off, b_off = (2, 3, 1, 1, 40, 11), (0, 13, 4, 3, 29, 7)
    a_rows = (a_off[0] + a_off[1] + 2 * a_off[2] + (Kc if a_mn else M))
    a_cols = (a_off[3] + a_off[4] + 2 * a_off[5] + (M if a_mn else Kc)) - 9     # the last elements' tails run past it
    b_rows = (b_off[0] + b_off[1] + 2 * b_off[2] + (Kc if b_mn else N))
    b_cols = (b_off[3] + b_off[4] + 2 * b_off[5] + (N if b_mn else Kc)) - 5
    A = _bf(torch.randn(a_rows, a_cols, generator=g))
    B = _bf(torch.randn(b_rows, b_cols, generator=g))
    ldc = 11
    C = torch.full((batch * M * ldc + 50,), SENT)
    geom = (ldc, 3, inner * M * ldc, M * ldc)
    r = gr.gemm(A, B, C, M, N, K, a_mn=a_mn, b_mn=b_mn, batch=batch, inner=inner, a_off=a_off, b_off=b_off,
                c_geom=geom, out_mode=2)
    want = C.double().clone()

    def el(X, i, j):
        return float(X[i, j]) if i < X.shape[0] and j < X.shape[1] else 0.0

    for outer in range(2):
        for i in range(inner):
            ar, ac = a_off[0] + outer * a_off[1] + i * a_off[2], a_off[3] + outer * a_off[4] + i * a_off[5]
            br, bc = b_off[0] + outer * b_off[1] + i * b_off[2], b_off[3] + outer * b_off[4] + i * b_off[5]
            for m in range(M):
                for n in range(N):
                    s = 0.0
                    for k in range(Kc):
                        a = el(A, ar + k, ac + m) if a_mn else el(A, ar + m, ac + k)
                        b = el(B, br + k, bc + n) if b_mn else el(B, br + n, bc + k)
                        s += a * b
                    want[geom[1] + outer * geom[2] + i * geom[3] + m * ldc + n] = s
    torch.testing.assert_close(r["C"]["out"], want, rtol=1e-12, atol=1e-12)
    assert int(r["C"]["written"].sum()) == batch * M * N


def test_split_ranges_limits_and_untouched_elements():
    """Split partials cover [kc*s/S, kc*(s+1)/S) chunks (empty splits store zeros), k_limit trims the contraction to
    whole chunks, m_limit skips whole 128-row tiles; skipped rows, columns >= N and the pitch keep their contents."""
    g = _gen(4)
    M, N, K, S = 300, 20, 200, 7
    A, W = _bf(torch.randn(M, K, generator=g)), _bf(torch.randn(N, K, generator=g))
    ws = torch.full((S * M * 24 + 10,), SENT)
    lim = torch.tensor([131], dtype=torch.int32)          # tile 1 (128 + 2 < 131) runs, tile 2 is skipped
    r = gr.gemm(A, W, ws, M, N, K, out_mode=3, split_k=S, c_geom=(24, 0, 0, 0), c_split_stride=M * 24, m_limit=lim,
                m_limit_base=2, k_limit=torch.tensor([70], dtype=torch.int32), k_limit_base=5)
    out = r["C"]["out"][:S * M * 24].view(S, M, 24)
    x = A.double()[:, :128] @ W.double()[:, :128].T        # K_eff = 65 -> two chunks
    chunks = [(2 * s // S, 2 * (s + 1) // S) for s in range(S)]
    for s, (c0, c1) in enumerate(chunks):
        part = A.double()[:, 64 * c0:64 * c1] @ W.double()[:, 64 * c0:64 * c1].T
        torch.testing.assert_close(out[s, :256, :N], part[:256], rtol=1e-12, atol=1e-12)
        assert (out[s, 256:] == SENT).all() and (out[s, :, N:] == SENT).all()
    torch.testing.assert_close(out[:, :256, :N].sum(0), x[:256], rtol=1e-12, atol=1e-9)
    assert (r["C"]["out"][S * M * 24:] == SENT).all()


# ----------------------------------------------------------------------------------------------------------------------
# the tolerance of the GPU tests rejects every plausible mistake of the model
# ----------------------------------------------------------------------------------------------------------------------
def _fwd_case(g):
    """Batched forward with every stage but the gate: batch 6 = 2 x 3, K = 100 with the tail read from the next batch
    element, bias, C2, GELU, dropout, residual, post-residual dropout, rowmask by outer."""
    M, N, K, batch, inner = 70, 40, 100, 6, 3
    A = _bf(torch.randn(M, batch * K + 40, generator=g))
    B = _bf(torch.randn(N, batch * K + 40, generator=g) / 8)
    ldc = N + 8
    C = torch.full((batch * M * ldc,), SENT, dtype=torch.bfloat16)
    C2 = torch.full_like(C, SENT)
    res = _bf(torch.randn(batch * M * ldc, generator=g))
    rowmask = (torch.rand(3 * M, generator=g) > 0.3).to(torch.uint8)
    kw = dict(batch=batch, inner=inner, a_off=(0, 0, 0, 0, inner * K, K), b_off=(0, 0, 0, 0, inner * K, K),
              c_geom=(ldc, 0, inner * M * ldc, M * ldc), bias=torch.randn(N, generator=g), act=2, C2=C2, residual=res,
              drop_p=0.2, drop_offset=3 << 40, post_drop_p=0.1, post_drop_offset=4 << 40, seed=SEED,
              seed_ptr=torch.tensor([CTR]), rowmask=rowmask, rowmask_oo=M, alpha=-0.5)
    return (A, B, C, M, N, K), kw


def _bwd_case(g):
    """gelu' gate (gate_mode 1) after dropout, B MN-major."""
    M, N, K = 90, 72, 128
    A = _bf(torch.randn(M, K, generator=g))
    B = _bf(torch.randn(K, N, generator=g) / 8)
    C = torch.full((M, N), SENT, dtype=torch.bfloat16)
    gate = _bf(torch.randn(M, N, generator=g) * 2)
    kw = dict(b_mn=True, gate=gate, gate_mode=1, gate_scale=1.0, drop_p=0.2, drop_offset=6 << 40, seed=SEED,
              seed_ptr=torch.tensor([CTR]))
    return (A, B, C, M, N, K), kw


def _split_case(g):
    """out_mode 1 onto a pre-filled C with 3 K splits and a bias."""
    M, N, K = 64, 48, 320
    A, B = _bf(torch.randn(M, K, generator=g)), _bf(torch.randn(N, K, generator=g))
    C = torch.randn(M, N, generator=g)
    return (A, B, C, M, N, K), dict(out_mode=1, split_k=3, bias=torch.randn(N, generator=g) * 4)


_MISTAKES = {m: _fwd_case for m in gr.MISTAKES}
_MISTAKES["gelu_tanh_grad"] = _bwd_case
_MISTAKES["bias_per_split"] = _split_case


def _as_output(exp, dtype):
    """The model's expected buffer as the kernel would leave it: rounded to the output type."""
    return exp["out"].to(dtype)


@pytest.mark.parametrize("mistake", [None] + sorted(_MISTAKES))
def test_tolerance_accepts_the_rounded_model_and_rejects_each_mistake(mistake):
    """The correct model rounded to the output dtype is within the GPU tests' tolerance (err < 1, nothing untouched
    changed); each mistaken model - bias or C2 after the act, dropout before the act, the residual before the dropout,
    the post-residual dropout before the residual, tanh GELU or its derivative, dropout column key n + 1, row key m
    instead of bz*M + m, rowmask by inner, the K tail zero-filled, the bias added once per split - misses it by >= 10x."""
    case = _MISTAKES.get(mistake, _fwd_case)
    args, kw = case(_gen(5))
    ref = gr.gemm(*args, **kw)
    C = args[2]
    if mistake is None:
        for key, buf in (("C", C), ("C2", kw.get("C2"))):
            if ref[key] is None:
                continue
            got = _as_output(ref[key], buf.dtype)
            assert gr.err(got, ref[key], buf.dtype == torch.bfloat16) < 1.0
            assert gr.untouched(got, ref[key]) == 0
        return
    bad = gr.gemm(*args, **kw, mistake=mistake)
    key = "C2" if mistake == "c2_after_act" else "C"
    buf = kw["C2"] if key == "C2" else C
    e = gr.err(_as_output(bad[key], buf.dtype), ref[key], buf.dtype == torch.bfloat16)
    print(mistake, "error in tolerances:", round(e, 1))
    assert e >= 10, e
