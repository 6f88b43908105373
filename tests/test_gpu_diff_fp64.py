"""The DiffTransformer kernels (csrc/rp_diff.cu) called directly through the C ABI, each output against the float64
reference of tests/diff_reference.py with its per-element bound: rp_diff_attn_fwd (out, o_pre, O32, O2, e1 / e2, inv1 /
inv2), rp_diff_attn_softmax_bwd on the forward's own saves (dS1, dS2, A, dlam_part), rp_diff_lambda_bwd onto start values,
rp_rmsnorm_fwd / _bwd and rp_swiglu_fwd / _bwd; then block 0's attention stage of a DiffEngine at its largest shape
against the float64 stage on the engine's own QKV and dOn.

Every buffer region the kernels must not read is NaN (rows and columns [L, Lp) of e1 / e2 / dA, inv past L, q / k / v and
d_on / O32 / O2 columns past the heads, x rows outside ``gather``, gl rows past n, the workspace); every region they must
not write is NaN or a start value and is checked bit for bit afterwards.  Regions the kernels' contract requires to be zero
(the q / k slot padding [hd, 64), the v slot padding [2 hd, v_slot), the padded columns of O32, O2 and d_on) hold exact
zeros.  Grid caps come from the device's SM count.  Run with -s to print the worst error of each family."""
import ctypes

import pytest
import torch

import diff_reference as dr
from fp64_checks import WorstErrors, block_err
from replay_b200._lib import DiffAttnDesc, DiffLambda, check, lib
from replay_b200.engine_diff import lambda_init

pytestmark = pytest.mark.gpu

NAN = float("nan")
LAMBDA_INIT = lambda_init(0)   # block 0's

# Tolerances: max |got - ref| / bound over a family, the bounds of tests/diff_reference.py.  Worst values seen over every
# case of this file on one H100 80GB HBM3 at a 700 W power limit (run with -s) are in the comments.
TOL_FWD = 1.0          # out 0.995, o_pre / O32 / O2 0.999 (the bf16 half ulp dominates the bf16 bounds)
TOL_SAVES = 1.0        # e1 / e2 0.999, inv1 / inv2 0.073
TOL_BWD = 1.0          # dS1 1.0, dS2 0.997, A 1.0, dlam_part 0.10
TOL_LAMBDA = 1.0       # the lambda_* gradients 0.992
TOL_RMS = 1.0          # y 1.0, dx 1.0, dw 0.087
TOL_SWIGLU = 1.0       # u 1.0, dg / dl 1.0
# the engine stage, per-sequence 64-row blocks (the gradients of lambda_* and rms_scale: whole), norm-relative
TOL_STAGE = 1e-2       # out 1.8e-3, dQKV 4.0e-3, rms_scale 1.9e-3, lambda_* 7.3e-7

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


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _bits(x):
    return x.contiguous().view(torch.int16 if x.element_size() == 2 else torch.int32)


def _untouched(x, fill=NAN):
    """every element of x still holds the fill value, bit for bit"""
    return torch.equal(_bits(x), _bits(torch.full_like(x, fill)))


def _assert_ratio(family, got, ref, bound, tol, mask=None):
    r = _note(family, dr.ratio(got, ref, bound, mask))
    assert r <= tol, (family, r)


def _lam_struct(P):
    lam = DiffLambda()
    lam.q1, lam.k1, lam.q2, lam.k2 = (t.data_ptr() for t in (P.lq1, P.lk1, P.lq2, P.lk2))
    lam.head_dim, lam.lambda_init = P.hd, P.li
    return lam


# ------------------------------------------------------------------------------------------------ forward
def run_fwd(P, save=True, ldo_extra=8, flag_off_only=False):
    """rp_diff_attn_fwd with the columns past the heads NaN, every output and save NaN-filled.  flag_off_only: every save
    pointer but e1_save (the save switch) is set, so the saves must stay untouched."""
    B, H, L, Lp, VS = P.B, P.H, P.L, P.Lp, P.VS
    T, BH, dev = B * L, B * H, P.qkv.device
    qkv = P.qkv.clone()
    qkv[:, P.n_qkv:] = NAN
    ldo = H * VS + ldo_extra
    bf = dict(dtype=torch.bfloat16, device=dev)
    f = dict(dtype=torch.float32, device=dev)
    o = {"out": torch.full((T, ldo), NAN, **bf), "o_pre": torch.full((T, ldo), NAN, **bf),
         "O32": torch.full((T, ldo), NAN, **f), "O2": torch.full((T, ldo), NAN, **f),
         "e1": torch.full((BH, Lp, Lp), NAN, **bf), "e2": torch.full((BH, Lp, Lp), NAN, **bf),
         "inv1": torch.full((BH, Lp), NAN, **f), "inv2": torch.full((BH, Lp), NAN, **f), "ldo": ldo}
    pad = P.pad.reshape(-1).to(torch.uint8).contiguous()
    d = DiffAttnDesc()
    d.qk, d.ld_qk, d.q_c0, d.k_c0 = qkv.data_ptr(), P.ld, P.q_c0, P.k_c0
    d.v, d.ldv, d.v_c0 = qkv.data_ptr(), P.ld, P.v_c0
    d.pad_mask = pad.data_ptr()
    d.B, d.H, d.L, d.head_dim, d.v_slot = B, H, L, P.hd, VS
    d.scale, d.eps = P.scale, P.eps
    d.lam = _lam_struct(P)
    d.rms_scale = P.rs.data_ptr()
    d.out, d.ldo = o["out"].data_ptr(), ldo
    if save or flag_off_only:
        d.o_pre, d.e2_save = o["o_pre"].data_ptr(), o["e2"].data_ptr()
        d.inv1, d.inv2 = o["inv1"].data_ptr(), o["inv2"].data_ptr()
        d.o32_save, d.o2_save = o["O32"].data_ptr(), o["O2"].data_ptr()
    if save:
        d.e1_save = o["e1"].data_ptr()
    check(lib().rp_diff_attn_fwd(ctypes.byref(d), None), "rp_diff_attn_fwd")
    torch.cuda.synchronize()
    return o


def check_fwd(P, o, save=True):
    B, H, L, VS, hd = P.B, P.H, P.L, P.VS, P.hd
    W = H * VS
    dev = P.qkv.device
    ref = dr.forward(P)
    padcol = (torch.arange(W, device=dev) % VS) >= 2 * hd
    names = ("out", "o_pre", "O32", "O2") if save else ("out",)
    for name in names:
        x = o[name]
        assert _untouched(x[:, W:]), name                        # columns past the heads
        assert bool((x[:, :W][:, padcol] == 0).all()), name      # the padded value columns are exact zeros
        _assert_ratio("fwd " + ("out" if name == "out" else "saves O"), x[:, :W], ref[name], ref[name + "_b"], TOL_FWD)
    if not save:
        for name in ("o_pre", "O32", "O2", "e1", "e2", "inv1", "inv2"):
            assert _untouched(o[name]), name
        return ref
    upper = torch.ones(L, o["e1"].shape[-1], dtype=torch.bool, device=dev).triu(1)
    for m in ("1", "2"):
        e, inv = o["e" + m], o["inv" + m]
        assert _untouched(e[:, L:, :]), "e" + m                  # rows [L, Lp) are never written
        assert bool((e[:, :L, :][:, upper] == 0).all()), "e" + m  # j > i, columns [L, Lp) included, are exact zeros
        _assert_ratio("fwd e", e[:, :L, :L], ref["e" + m], ref["e" + m + "_b"], TOL_SAVES)
        assert _untouched(inv[:, L:]), "inv" + m
        _assert_ratio("fwd inv", inv[:, :L], ref["inv" + m], ref["inv" + m + "_b"], TOL_SAVES)
    return ref


# ------------------------------------------------------------------------------------------------ softmax backward
def run_softmax_bwd(P, o, alias, seed=1):
    """rp_diff_attn_softmax_bwd on the forward's saves o; rows and columns [L, Lp) of e1 / e2 / dA NaN, inv past L NaN,
    random dA (finite above the diagonal, as the dA GEMM leaves it) and d_on (padded columns zero, columns past the heads
    NaN); dS1 / dS2 / A / dlam_part NaN-filled.  Returns the outputs and the inputs the kernel saw."""
    B, H, L, Lp, VS = P.B, P.H, P.L, P.Lp, P.VS
    dev = P.qkv.device
    BH, W = B * H, H * VS
    dA, d_on = dr.bwd_inputs(P, o, seed)
    e1, e2, dA = o["e1"].clone(), o["e2"].clone(), dA.clone()
    for t in (e1, e2, dA):
        t[:, L:, :] = NAN
        t[:, :, L:] = NAN
    d_on[:, W:] = NAN
    ld_o = d_on.shape[1]
    assert o["ldo"] == ld_o
    dA_in = dA.clone()
    bf = dict(dtype=torch.bfloat16, device=dev)
    out = {"dS1": torch.full((BH, Lp, Lp), NAN, **bf), "dS2": torch.full((BH, Lp, Lp), NAN, **bf),
           "dlam": torch.full((BH, Lp), NAN, dtype=torch.float32, device=dev)}
    out["A"] = dA if alias else torch.full((BH, Lp, Lp), NAN, **bf)
    lam = _lam_struct(P)
    check(lib().rp_diff_attn_softmax_bwd(e1.data_ptr(), e2.data_ptr(), o["inv1"].data_ptr(), o["inv2"].data_ptr(),
                                         dA.data_ptr(), out["dS1"].data_ptr(), out["dS2"].data_ptr(), out["A"].data_ptr(),
                                         out["dlam"].data_ptr(), BH, H, L, P.scale, ctypes.byref(lam), d_on.data_ptr(),
                                         o["O32"].data_ptr(), o["O2"].data_ptr(), P.rs.data_ptr(), P.eps, ld_o, VS, None),
          "rp_diff_attn_softmax_bwd")
    torch.cuda.synchronize()
    out["inputs"] = dict(e1=e1, e2=e2, inv1=o["inv1"], inv2=o["inv2"], dA=dA_in, d_on=d_on, o32=o["O32"], o2=o["O2"])
    return out


def check_softmax_bwd(P, out):
    L = P.L
    ref = dr.softmax_bwd(P, **out["inputs"])
    dev = P.qkv.device
    upper = torch.ones(L, L, dtype=torch.bool, device=dev).triu(1)
    for name in ("dS1", "dS2", "A"):
        x = out[name]
        assert _untouched(x[:, L:, :]) and _untouched(x[:, :L, L:]), name   # rows and columns [L, Lp)
        body = x[:, :L, :L]
        assert bool((body[:, upper] == 0).all()), name
        _assert_ratio("bwd " + name, body, ref[name], ref[name + "_b"], TOL_BWD)
    assert _untouched(out["dlam"][:, L:])
    _assert_ratio("bwd dlam_part", out["dlam"][:, :L], ref["dlam"], ref["dlam_b"], TOL_BWD)
    return ref


# ------------------------------------------------------------------------------------------------ lambda backward
def run_lambda_bwd(P, dlam, B, L, seed=2):
    g = torch.Generator().manual_seed(seed)
    starts = [torch.randn(P.H, P.hd, generator=g).to(P.qkv.device) for _ in range(4)]
    grads = [s.clone() for s in starts]
    lam = _lam_struct(P)
    check(lib().rp_diff_lambda_bwd(dlam.data_ptr(), B, P.H, L, ctypes.byref(lam), *(t.data_ptr() for t in grads), None),
          "rp_diff_lambda_bwd")
    torch.cuda.synchronize()
    return grads, starts


def check_lambda_bwd(P, dlam, B, L, grads, starts):
    ref = dr.lambda_bwd(dlam, B, P.H, L, P.lq1, P.lk1, P.lq2, P.lk2, P.li)
    for name, got, start in zip(("q1", "k1", "q2", "k2"), grads, starts):
        bound = dr.accum_bound(ref[f"g_{name}_b"], start, ref["g_" + name])
        _assert_ratio("lambda grads", got.double() - start.double(), ref["g_" + name], bound, TOL_LAMBDA)


def attention_case(P, alias=True):
    o = run_fwd(P)
    check_fwd(P, o)
    b = run_softmax_bwd(P, o, alias)
    check_softmax_bwd(P, b)
    grads, starts = run_lambda_bwd(P, b["dlam"], P.B, P.L)
    check_lambda_bwd(P, b["dlam"], P.B, P.L, grads, starts)


# ------------------------------------------------------------------------------------------------ attention sweeps
LAMS = (-0.5, 0.0, LAMBDA_INIT, 1.3)
HEAD_CASES = [dict(hd=hd, H=H, L=(65, 33, 129, 200)[(i + H) % 4], pad=dr.PAD_KINDS[(i + H) % 5], lam=LAMS[(i + 2 * H) % 4])
              for i, hd in enumerate((8, 25, 32, 33, 48, 63, 64)) for H in (1, 2, 3, 4)]
LEN_CASES = [dict(hd=hd, H=H, L=L, pad=dr.PAD_KINDS[i % 5], lam=LAMS[i % 4])
             for i, L in enumerate((1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256))
             for hd, H in ((33, 2), (64, 4), (25, 1))]
PAD_CASES = [dict(hd=48, H=2, L=L, pad=p, lam=0.3) for p in dr.PAD_KINDS for L in (33, 129)]
LAMBDA_CASES = ([dict(hd=hd, H=H, L=100, pad="holes", lam=lam) for lam in LAMS for hd, H in ((32, 3), (64, 2))]
                + [dict(hd=hd, H=H, L=L, pad="left", lam=0.999, identical=True) for hd, H, L in ((32, 3, 100), (63, 2, 256))]
                + [dict(hd=hd, H=H, L=L, pad="holes", lam=0.3, qk_std=qs) for hd, H, L in ((32, 3, 100), (64, 4, 256))
                   for qs in (3.0, 5.0)])
# the (head width, heads, L, B) grid and the backward shapes the kernels were first tested at, pads and lambdas as then
FIRST_CASES = ([dict(hd=hd, H=H, L=L, B=B, pad=("all", "last", "left")[L % 3], lam=(-0.5, 0.0, 0.2, 1.3)[(L + H) % 4])
                for hd, H in ((32, 1), (48, 2), (64, 4), (32, 4), (64, 1), (48, 1))
                for L, B in ((1, 3), (2, 37), (63, 3), (64, 1), (65, 3), (127, 1), (128, 3), (129, 1), (200, 3), (255, 1),
                             (256, 3))]
               + [dict(hd=hd, H=H, L=L, B=B, pad="left", lam=0.3)
                  for hd, H, L, B in ((32, 2, 50, 3), (48, 4, 129, 2), (64, 2, 200, 2), (64, 1, 256, 1), (32, 1, 1, 5))])


def _cid(c):
    extra = "-same" if c.get("identical") else (f"-z{c['qk_std']}" if "qk_std" in c else "")
    return f"hd{c['hd']}x{c['H']}-L{c['L']}-B{c.get('B', 3)}-{c['pad']}-lam{c['lam']:.3g}{extra}"


def _attn(cuda, c, B=3, seed=0):
    return dr.make_attn(c.get("B", B), c["L"], c["hd"], c["H"], pad=c["pad"], lam_target=c["lam"], li=LAMBDA_INIT,
                        qk_std=c.get("qk_std", 1.0), identical=c.get("identical", False), seed=seed, device=cuda)


@pytest.mark.parametrize("case", HEAD_CASES + LEN_CASES + PAD_CASES + LAMBDA_CASES + FIRST_CASES, ids=_cid)
def test_attention(cuda, case):
    """forward, softmax backward and lambda backward of one input; A aliases dA (the engine's call) on every other case"""
    seed = case["hd"] * 1000 + case["H"] * 300 + case["L"]
    attention_case(_attn(cuda, case, B=4 if case["pad"] == "left" else 3, seed=seed), alias=seed % 2 == 0)


@pytest.mark.parametrize("ldo_extra", [0, 8, 64])
def test_forward_without_saves(cuda, ldo_extra):
    """e1_save switches the saves: with it null the other save buffers stay untouched, and out equals the saving run's"""
    P = _attn(cuda, dict(hd=33, H=3, L=129, pad="holes", lam=0.3), seed=5)
    o = run_fwd(P, save=False, ldo_extra=ldo_extra, flag_off_only=True)
    check_fwd(P, o, save=False)
    o2 = run_fwd(P, save=True, ldo_extra=ldo_extra)
    assert torch.equal(_bits(o["out"]), _bits(o2["out"]))


def _rows_shape(rows):
    """(B, H, L) with B * H * L == rows, L <= 256, preferring several heads and long sequences"""
    for H in (4, 2, 1, 3):
        for L in range(256, 0, -1):
            if rows % (H * L) == 0:
                return rows // (H * L), H, L
    raise AssertionError(rows)


@pytest.mark.parametrize("which", ["cap-1", "cap", "cap+1", "4cap"])
@pytest.mark.parametrize("alias", [True, False])
def test_softmax_bwd_warp_cap(cuda, which, alias):
    """the softmax backward runs at most SMs * 16 blocks of 8 warps; past that cap a warp takes rows cap apart, which
    belong to other sequences and, with several heads, other heads (each with its own lambda)"""
    cap = _sms() * dr.BWD_WARPS_PER_SM
    rows = {"cap-1": cap - 1, "cap": cap, "cap+1": cap + 1, "4cap": 4 * cap}[which]
    B, H, L = _rows_shape(rows)
    P = dr.make_attn(B, L, 33 if H == 1 else 64, H, pad="left", lam_target=0.3, li=LAMBDA_INIT, seed=rows, device=cuda)
    o = run_fwd(P)
    b = run_softmax_bwd(P, o, alias)
    check_softmax_bwd(P, b)
    grads, starts = run_lambda_bwd(P, b["dlam"], B, L)
    check_lambda_bwd(P, b["dlam"], B, L, grads, starts)


@pytest.mark.parametrize("BL", [1, 255, 256, 257, 66 * 256])
@pytest.mark.parametrize("H", [1, 4])
def test_lambda_bwd(cuda, BL, H):
    """the fixed-order per-head sum over B * L partials (a thread takes every 256th), chained onto start values; the
    partials past L are NaN"""
    L = 256 if BL % 256 == 0 else (BL if BL <= 256 else 1)
    B = BL // L
    P = dr.make_attn(1, 1, 48, H, lam_target=0.3, li=LAMBDA_INIT, seed=BL + H, device=cuda)
    Lp = dr.lp_of(L)
    g = torch.Generator().manual_seed(BL)
    dlam = torch.full((B * H, Lp), NAN)
    dlam[:, :L] = torch.randn(B * H, L, generator=g) * 0.1
    dlam = dlam.to(cuda)
    grads, starts = run_lambda_bwd(P, dlam, B, L)
    check_lambda_bwd(P, dlam, B, L, grads, starts)


# ------------------------------------------------------------------------------------------------ RMSNorm
def run_rms(x, w, dy, eps, alpha, n_rows, d, G, n_true, n_rows_dev=None, gather=None, dw_start=None):
    """rp_rmsnorm_fwd and _bwd; y has two NaN sentinel rows past n_rows, dx (the rows of x) is NaN-filled, the workspace
    NaN, dw starts at dw_start"""
    dev = x.device
    y = torch.full((n_rows + 2, d), NAN, dtype=torch.bfloat16, device=dev)
    dx = torch.full_like(x, NAN)
    dw = dw_start.clone()
    ws = torch.full((lib().rp_rmsnorm_bwd_workspace(G),), 0xFF, dtype=torch.uint8, device=dev)
    nrd = None if n_rows_dev is None else torch.tensor([n_rows_dev], dtype=torch.int32, device=dev)
    ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    check(lib().rp_rmsnorm_fwd(x.data_ptr(), w.data_ptr(), eps, alpha, n_rows, d, G, n_true, ptr(nrd), ptr(gather),
                               y.data_ptr(), None), "rp_rmsnorm_fwd")
    check(lib().rp_rmsnorm_bwd(dy.data_ptr(), x.data_ptr(), w.data_ptr(), eps, alpha, n_rows, d, G, n_true, ptr(nrd),
                               ptr(gather), dx.data_ptr(), dw.data_ptr(), ws.data_ptr(), ws.numel(), None), "rp_rmsnorm_bwd")
    torch.cuda.synchronize()
    return y, dx, dw


def rms_case(cuda, G, d, kind, rows, alpha, eps, gathered=False, n_rows_dev=None, seed=0):
    x, w, dy, n_true = dr.make_rms(rows, d, G, kind, seed=seed, zero_row=7)
    g = torch.Generator().manual_seed(seed + 1)
    gather = None
    if gathered:   # output row r reads input row gather[r] of 2 * rows; the rows outside gather are NaN
        gather = torch.randperm(2 * rows, generator=g)[:rows].to(torch.int32)
        xs = torch.full((2 * rows, d), NAN, dtype=torch.bfloat16)
        xs[gather.long()] = x
        x = xs
    n_proc = rows if n_rows_dev is None else min(rows, n_rows_dev)
    dyb = torch.full((rows + 2, d), NAN, dtype=torch.bfloat16)
    dyb[:n_proc] = dy[:n_proc]                          # rows past the processed ones are NaN
    x, w, dyb = x.to(cuda), w.to(cuda), dyb.to(cuda)
    gather = None if gather is None else gather.to(cuda)
    dw0 = torch.randn(G, generator=g).to(cuda)
    y, dx, dw = run_rms(x, w, dyb, eps, alpha, rows, d, G, n_true, n_rows_dev, gather, dw0)
    ry, ry_b, orow = dr.rmsnorm_fwd(x, w, eps, alpha, rows, d, G, n_true, n_rows_dev, gather)
    assert _untouched(y[n_proc:])
    _assert_ratio("rms y", y[:n_proc], ry, ry_b, TOL_RMS)
    rb = dr.rmsnorm_bwd(dyb, x, w, eps, alpha, rows, d, G, n_true, n_rows_dev, gather)
    written = torch.zeros(x.shape[0], dtype=torch.bool, device=cuda)
    written[rb["src"]] = True
    assert _untouched(dx[~written])
    _assert_ratio("rms dx", dx[rb["src"]], rb["dx"], rb["dx_b"], TOL_RMS)
    pad = (w == 0).repeat(d // G)
    assert bool((y[:n_proc][:, pad] == 0).all()) and bool((dx[rb["src"]][:, pad] == 0).all())
    _assert_ratio("rms dw", dw.double() - dw0.double(), rb["dw"], dr.dw_bound(rb, dw0), TOL_RMS)
    return y, dx, dw


GROUP_D = [(G, d) for G in (64, 128, 256, 512) for d in range(G, 513, G)]
ALPHAS = (1.0, 1.0 - LAMBDA_INIT)
EPSS = (1e-5, dr.RMS_EPS)
RMS_CASES = ([dict(G=G, d=d, kind=k, rows=300, alpha=ALPHAS[i % 2], eps=EPSS[(i // 2) % 2])
              for i, ((G, d), k) in enumerate((gd, k) for gd in GROUP_D for k in ("one", "full", "slots"))]
             + [dict(G=G, d=G, kind="slots" if G < 512 else "full", rows=n, alpha=ALPHAS[j % 2], eps=EPSS[j % 2])
                for G in (64, 128, 256, 512) for j, n in enumerate((1, 1023, 1024, 1025, 20000))]
             + [dict(G=G, d=d, kind="slots", rows=600, alpha=ALPHAS[1], eps=1e-5, gathered=ga, n_rows_dev=nr)
                for G, d in ((128, 256), (512, 512)) for ga in (False, True) for nr in (None, 563, 0)]
             + [dict(G=G, d=d, kind=n, rows=300, alpha=0.7, eps=1e-5, gathered=ga)     # the first n_true columns live
                for G, d, n in ((128, 128, 100), (256, 256, 256), (64, 64, 64), (64, 256, 48), (128, 256, 96))
                for ga in (False, True)])


def _rid(c):
    kind = f"n{c['kind']}" if isinstance(c["kind"], int) else c["kind"]
    return (f"G{c['G']}-d{c['d']}-{kind}-rows{c['rows']}-a{c['alpha']:.2f}-eps{c['eps']:.1e}"
            + ("-gather" if c.get("gathered") else "")
            + (f"-nrd{c['n_rows_dev']}" if c.get("n_rows_dev") is not None else ""))


@pytest.mark.parametrize("case", RMS_CASES, ids=_rid)
def test_rmsnorm(cuda, case):
    c = dict(case)
    rms_case(cuda, c.pop("G"), c.pop("d"), c.pop("kind"), c.pop("rows"), c.pop("alpha"), c.pop("eps"), seed=len(_rid(case)),
             **c)


# ------------------------------------------------------------------------------------------------ SwiGLU
def run_swiglu(gl, du, n, F):
    """rp_swiglu_fwd / _bwd over n rows; u and dgl have NaN sentinel rows past n (gl and du: NaN rows past n)"""
    R = gl.shape[0]
    u = torch.full((R, F), NAN, dtype=torch.bfloat16, device=gl.device)
    dgl = torch.full((R, 2 * F), NAN, dtype=torch.bfloat16, device=gl.device)
    check(lib().rp_swiglu_fwd(gl.data_ptr(), n, F, u.data_ptr(), None), "rp_swiglu_fwd")
    check(lib().rp_swiglu_bwd(du.data_ptr(), gl.data_ptr(), n, F, dgl.data_ptr(), None), "rp_swiglu_bwd")
    torch.cuda.synchronize()
    return u, dgl


def swiglu_case(cuda, n, F):
    """both SwiGLU kernels over n rows of width F (gates up to +-100, every bf16 step around the __expf overflow at
    -88.7), NaN rows past n in every buffer"""
    gl, du = dr.make_swiglu(n, F, seed=F + n)
    gl[n:], du[n:] = NAN, NAN
    gl, du = gl.to(cuda), du.to(cuda)
    u, dgl = run_swiglu(gl, du, n, F)
    assert _untouched(u[n:]) and _untouched(dgl[n:])
    ru, ru_b = dr.swiglu_fwd(gl, n, F)
    _assert_ratio("swiglu u", u[:n], ru, ru_b, TOL_SWIGLU)
    rd, rd_b = dr.swiglu_bwd(du, gl, n, F)
    _assert_ratio("swiglu dgl", dgl[:n], rd, rd_b, TOL_SWIGLU)


def test_swiglu(cuda):
    """777 rows of the item tower's width 384"""
    swiglu_case(cuda, 777, 384)


@pytest.mark.parametrize("F,side", [(F, side) for F in (1, 33, 384, 512, 1024) for side in ("small", "below", "above")])
def test_swiglu_widths_and_grid_cap(cuda, F, side):
    """widths 1 to 1024, with n * F on both sides of the grid cap (SMs * 16 blocks of 256 threads), past which the kernels
    run a grid-stride loop"""
    cap = _sms() * dr.GRID_PER_SM
    swiglu_case(cuda, {"small": 7, "below": (cap - 1) // F, "above": cap // F + 1}[side], F)


# ------------------------------------------------------------------------------------------------ bitwise reruns
def test_reruns_are_bitwise_equal(cuda):
    """no kernel of rp_diff.cu uses float atomics: two runs of each are bitwise equal, past the softmax backward's warp
    cap and the RMSNorm backward's 1024 partials"""
    cap = _sms() * dr.BWD_WARPS_PER_SM
    B = -(-2 * cap // (4 * 129))
    P = dr.make_attn(B, 129, 50, 4, pad="holes", lam_target=0.3, li=LAMBDA_INIT, seed=11, device=cuda)
    f1, f2 = run_fwd(P), run_fwd(P)
    for k in ("out", "o_pre", "O32", "O2", "e1", "e2", "inv1", "inv2"):
        assert torch.equal(_bits(f1[k]), _bits(f2[k])), k
    b1, b2 = run_softmax_bwd(P, f1, False), run_softmax_bwd(P, f1, False)
    for k in ("dS1", "dS2", "A", "dlam"):
        assert torch.equal(_bits(b1[k]), _bits(b2[k])), k
    l1, _ = run_lambda_bwd(P, b1["dlam"], B, 129)
    l2, _ = run_lambda_bwd(P, b1["dlam"], B, 129)
    for a, b in zip(l1, l2):
        assert torch.equal(_bits(a), _bits(b))
    r1 = rms_case(cuda, 256, 512, "slots", 3000, ALPHAS[1], 1e-5, seed=3)
    r2 = rms_case(cuda, 256, 512, "slots", 3000, ALPHAS[1], 1e-5, seed=3)
    for a, b in zip(r1, r2):
        assert torch.equal(_bits(a), _bits(b))
    F = 384
    n = _sms() * dr.GRID_PER_SM // F + 5
    gl, du = dr.make_swiglu(n, F, seed=4)
    gl, du = gl.to(cuda), du.to(cuda)
    for a, b in zip(run_swiglu(gl, du, n, F), run_swiglu(gl, du, n, F)):
        assert torch.equal(_bits(a), _bits(b))


# ------------------------------------------------------------------------------------------------ engine stage
@pytest.mark.parametrize("d,H,L,B", [(256, 4, 256, 66), (200, 4, 129, 9), (100, 4, 100, 5)])
def test_engine_attention_stage(cuda, d, H, L, B):
    """One training forward, then block 0's attention backward from a random dOn: the per-head RMSNorm backward, dA and the
    softmax backward, the lambda chain and the batched dQ / dK / dV GEMMs at the Lp pitch.  d 256 / 4 heads / L 256 / B 66
    is the largest supported shape and puts the softmax backward past its warp cap on an H100; d 200 and 100 leave slot
    padding, which the real QKV GEMM must leave exactly zero."""
    from replay_b200.engine_diff import DiffConfig, DiffEngine

    n_items = 500
    cfg = DiffConfig(n_items=n_items, d=d, n_heads=H, n_blocks=1, max_len=L)
    eng = DiffEngine(cfg, B, L, cuda, seed=3)
    g = torch.Generator().manual_seed(d + L)
    with torch.no_grad():   # lambda_* at a few tenths (xavier draws of [H, hd] are larger) and rms_scale around one
        hd = cfg.head_dim
        for k in ("q1", "k1", "q2", "k2"):
            eng.params[f"b0.lambda_{k}"].copy_(torch.randn(H, hd, generator=g) * 0.15)
        eng.import_named("b0.rms_scale", 1 + 0.25 * torch.randn(2 * hd, generator=g))
        eng.refresh_shadow()
    lens = torch.randint(1, L + 1, (B,), generator=g)
    lens[0] = L
    pm = torch.arange(L)[None, :] >= (L - lens)[:, None]
    ids = torch.where(pm, torch.randint(0, n_items, (B, L), generator=g), torch.full((B, L), n_items))
    lab = torch.randint(0, n_items, (B, L), generator=g)
    eng.set_batch(ids.to(cuda), pm.to(cuda), lab.to(cuda), pm.to(cuda))
    eng.forward_train()
    a, s, G = eng.act[0], eng.s, eng.grads
    VS, T, li = cfg.v_slot, B * L, lambda_init(0)
    # the zero contract: the slot padding of Q, K and V after the real QKV GEMM
    QKV = a["QKV"]
    qk = QKV[:, :H * 4 * dr.SLOT].reshape(T, H * 4, dr.SLOT)
    assert bool((qk[..., hd:] == 0).all())
    assert bool((QKV[:, H * 4 * dr.SLOT:].reshape(T, H, VS)[..., 2 * hd:] == 0).all())
    dOn = torch.zeros(T, H, VS)
    dOn[..., :2 * hd] = torch.randn(T, H, 2 * hd, generator=g)
    s["dOn"].copy_(dOn.reshape(T, -1).to(torch.bfloat16))
    eng.g32.zero_()
    eng._rms_bwd(s["dOn"], a["Opre"], eng.params["b0.rms_scale"], 1e-5, s["dOpre"], G["b0.rms_scale"], T, VS, 2 * hd,
                 alpha=1.0 - li)
    eng._attention_backward(0)
    torch.cuda.synchronize()
    lp = [eng.params[f"b0.lambda_{k}"] for k in ("q1", "k1", "q2", "k2")]
    pad = pm.to(cuda)
    ref = dr.attention_stage(QKV, s["dOn"], pad, *lp, eng.params["b0.rms_scale"], li, H, hd)
    for name, got, want in (("On", a["On"], ref["On"]), ("Opre", a["Opre"], ref["Opre"]), ("dQKV", s["dQKV"], ref["dQKV"])):
        err = max(block_err(got[b * L:(b + 1) * L], want[b * L:(b + 1) * L]) for b in range(B))
        assert _note("stage " + ("dQKV" if name == "dQKV" else "out"), err) <= TOL_STAGE, (name, err)
    # the lambda and rms_scale gradients: each kernel against its bound on its own inputs, and the chain norm-relative
    P = dr.Attn(qkv=QKV, q_c0=0, k_c0=H * 2 * dr.SLOT, v_c0=H * 4 * dr.SLOT, pad=pad, lq1=lp[0], lk1=lp[1], lq2=lp[2],
                lk2=lp[3], li=li, rs=eng.params["b0.rms_scale"], eps=1e-5, B=B, H=H, L=L, hd=hd)
    # dlam_part from the forward's saves (dA, overwritten by A, does not enter it)
    rb = dr.softmax_bwd(P, a["e1"], a["e2"], a["inv1"], a["inv2"], s["dA"], s["dOn"], a["O32"], a["O2"])
    assert _untouched(s["dlam"][:, L:], 0.0)          # the engine's zero-initialised partials past L
    _assert_ratio("bwd dlam_part", s["dlam"][:, :L], rb["dlam"], rb["dlam_b"], TOL_BWD)
    rl = dr.lambda_bwd(s["dlam"], B, H, L, *lp, li)
    zero = torch.zeros(H, hd, dtype=torch.float64, device=cuda)
    for k in ("q1", "k1", "q2", "k2"):
        got = G[f"b0.lambda_{k}"]
        _assert_ratio("lambda grads", got, rl["g_" + k], dr.accum_bound(rl[f"g_{k}_b"], zero, rl["g_" + k]), TOL_LAMBDA)
        err = float((got.double() - ref["d_" + k]).norm() / ref["d_" + k].norm())
        assert _note("stage lambda grads", err) <= TOL_STAGE, (k, err)
    rsb = dr.rmsnorm_bwd(s["dOn"], a["Opre"], eng.params["b0.rms_scale"], 1e-5, 1.0 - li, T, H * VS, VS, 2 * hd)
    got = G["b0.rms_scale"]
    _assert_ratio("rms dw", got, rsb["dw"], dr.dw_bound(rsb, torch.zeros(VS, device=cuda)), TOL_RMS)
    err = float((got[:2 * hd].double() - ref["d_rs"]).norm() / ref["d_rs"].norm())
    assert _note("stage rms_scale grad", err) <= TOL_STAGE, err
