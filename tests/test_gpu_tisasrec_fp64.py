"""TiSASRec's time-interval kernels (csrc/rp_tisasrec.cu) called directly through the C ABI, each output against the float64
reference of tests/tisasrec_reference.py with its per-element bound: rp_ti_attn_fwd (A, Ad, hpre), rp_ti_attn_bwd (dS, Ad,
dq_t and the time tables' gradients added onto start values), rp_ti_pos_add (bit for bit against a host emulation) and
rp_ti_pos_bwd; then one config-2 training step's block-0 attention stage against the reference on the engine's own inputs.

Every buffer region the kernels must not read is NaN (S outside j <= i, rows and columns [L, Lp), q / q_in / dO columns past
H * 64, the workspace); every region they must not write is NaN or a start value and is checked bit for bit afterwards.
Sweeps: L across the 32-key lane and 64-key tile edges, head widths 32 / 50 / 64 with 1 to 4 heads, time_span 1 to 320,
int64 / float32 / float64 timestamps at their interval edges, dropout with and without a seed pointer, Ad aliasing A, and the
backward's CTAs that take several sequences (B around G = 256 / H).  Run with -s to print the worst error of each family.
"""
import ctypes

import pytest
import torch

import tisasrec_reference as tr
from fp64_checks import WorstErrors, block_err
from replay_b200._lib import TI_MAX_SPAN, TiAttnDesc, check, lib

pytestmark = pytest.mark.gpu

SEED, COUNTER = 0x5EED, 977
P_DROP = 0.2
NAN16 = float("nan")

# Tolerances: max |got - ref| / bound over the family, the bounds of tests/tisasrec_reference.py.  Worst values seen over
# every case of this file on one H100 80GB HBM3 at a 700 W power limit (run with -s) are in the comments.
TOL_A = 1.0            # A and the forward's Ad; worst seen 0.997 (the bf16 half ulp dominates the bound)
TOL_HPRE = 1.0         # hpre; worst seen 1.0
TOL_DS = 1.0           # dS and the backward's Ad; worst seen 1.0
TOL_DQT = 1.0          # dq_t; worst seen 0.996
TOL_TIME = 1.0         # d_time_k / d_time_v; worst seen 0.97
TOL_POS = 1.0          # d_pos_k / d_pos_v; worst seen 0.293
# the config-2 stage, per-sequence 64-row blocks (time tables: per bucket row), norm-relative
TOL_STAGE_H = 1e-2     # worst seen 2.6e-3
TOL_STAGE_GRAD = 1e-2  # dQ, dK', dV'; worst seen 4.7e-3
TOL_STAGE_TIME = 1e-2  # worst seen 4.0e-3

CTA_CASE = dict(head_dim=64, span=63, p=P_DROP, times="mixed")   # the backward's multi-sequence CTA sweep (also CPU-tested)

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


def _bits(x):
    return x.contiguous().view(torch.int16 if x.element_size() == 2 else torch.int32)


def _problem(dev, B, L, head_dim, H, span, p=0.0, times="mixed", dtype=torch.int64, pad="mixed", use_ptr=True, seed=0):
    seed_eff = SEED + (COUNTER if p > 0 and use_ptr else 0)
    P = tr.make_problem(B, L, head_dim, H, span, p, times, dtype, pad, seed=seed, seed_eff=seed_eff, ld_extra=8)
    P = tr.to(P, dev)
    P.use_ptr = use_ptr
    for t in (P.tk, P.tv):      # table columns past H * 64 are never read
        t[:, P.H * tr.SLOT:] = NAN16
    return P


def _desc(P, q, seed_buf):
    d = TiAttnDesc()
    d.q, d.ldq, d.pad_mask = q.data_ptr(), P.ldq, P.pad_u8.data_ptr()
    d.times, d.times_dtype = P.times_dev.data_ptr(), tr.DTYPE_CODE[P.times.dtype]
    d.time_k, d.time_v, d.ld_t = P.tk.data_ptr(), P.tv.data_ptr(), P.tk.stride(0)
    d.B, d.H, d.L, d.head_dim, d.time_span = P.B, P.H, P.L, P.head_dim, P.span
    d.scale, d.drop_p, d.seed = P.scale, P.p, SEED
    d.seed_ptr = seed_buf.data_ptr() if P.use_ptr else None
    d.att_off, d.tk_off, d.tv_off = P.att_off, P.tk_off, P.tv_off
    return d


def _nan_cols(x, d):
    y = x.clone()
    y[:, d:] = NAN16
    return y


def run_fwd(P, alias=False):
    """rp_ti_attn_fwd on P with every unread region NaN -> dict of the outputs and the inputs the kernel saw"""
    B, H, L, Lp, d = P.B, P.H, P.L, P.Lp, P.H * tr.SLOT
    dev = P.q.device
    P.pad_u8 = P.pad.reshape(-1).to(torch.uint8).contiguous()
    P.times_dev = P.times.reshape(-1).contiguous()
    S = P.S.clone()
    S[:, L:, :] = float("nan")
    S[:, :, L:] = float("nan")
    S[:, :L, :L].masked_fill_(torch.ones(L, L, dtype=torch.bool, device=dev).triu(1), float("nan"))
    q, q_in = _nan_cols(P.q, d), _nan_cols(P.q_in, d)
    a_save = torch.full((B * H, Lp, Lp), NAN16, dtype=torch.bfloat16, device=dev)
    ad = a_save if alias else torch.full_like(a_save, NAN16)
    hpre = torch.full_like(q, NAN16)
    seed_buf = torch.tensor([COUNTER], dtype=torch.int64, device=dev)
    desc = _desc(P, q, seed_buf)
    check(lib().rp_ti_attn_fwd(ctypes.byref(desc), S.data_ptr(), q_in.data_ptr(), a_save.data_ptr(), ad.data_ptr(),
                               hpre.data_ptr(), None), "rp_ti_attn_fwd")
    torch.cuda.synchronize()
    return {"A": a_save, "Ad": ad, "hpre": hpre, "q_in": q_in}


def check_fwd(P, out, alias=False):
    B, H, L, Lp, d = P.B, P.H, P.L, P.Lp, P.H * tr.SLOT
    A, Ad, hpre = out["A"], out["Ad"], out["hpre"]
    ref = tr.forward(P, ad_kernel=A if alias else Ad)
    dev = A.device
    live = P.pad.reshape(B, 1, L).expand(B, H, L).reshape(B * H, L)
    upper = torch.ones(L, Lp, dtype=torch.bool, device=dev).triu(1)
    for name, x in (("A", A), ("Ad", Ad)):
        # rows [L, Lp) untouched; j > i (up to Lp) and dead rows exactly 0
        assert bool(torch.isnan(x[:, L:, :].float()).all()), name
        body = x[:, :L, :].float()
        assert bool((body[:, upper] == 0).all()), name
        assert bool((body[~live] == 0).all()), name
        assert not bool(torch.isnan(body).any()), name
    if not alias:
        r = _note("Ad (fwd)", tr.ratio(Ad[:, :L, :L], ref["Ad"], ref["Ad_b"]))
        assert r <= TOL_A, r
    r = _note("A", tr.ratio(A[:, :L, :L], ref["A"], ref["A_b"]))
    assert r <= TOL_A, r
    # hpre: dead rows are q_in bit for bit; columns past H * 64 untouched
    dead = ~P.pad.reshape(-1)
    assert torch.equal(_bits(hpre[dead, :d]), _bits(out["q_in"][dead, :d]))
    assert bool(torch.isnan(hpre[:, d:].float()).all())
    r = _note("hpre", tr.ratio(hpre[:, :d], ref["hpre"], ref["hpre_b"]))
    assert r <= TOL_HPRE, r
    return ref


def run_bwd(P, A, alias=False, start_seed=1):
    """rp_ti_attn_bwd on the forward's A and P.dpd, table gradients added onto random start values"""
    B, H, L, Lp, d, n_r = P.B, P.H, P.L, P.Lp, P.H * tr.SLOT, P.span + 1
    dev = A.device
    dpd = P.dpd.clone()
    dpd[:, L:, :] = NAN16
    dpd[:, :, L:] = NAN16
    dpd[:, :L, :L].masked_fill_(torch.ones(L, L, dtype=torch.bool, device=dev).triu(1), NAN16)
    ad = A if alias else torch.full_like(A, NAN16)
    d_o, q = _nan_cols(P.d_o, d), _nan_cols(P.q, d)
    dq_t = torch.full_like(q, NAN16)
    n_ws = lib().rp_ti_attn_bwd_workspace(B, H, P.span)
    assert n_ws == tr.bwd_ctas(B, H) * H * 2 * n_r * tr.SLOT * 4
    ws = torch.full((n_ws,), 0xFF, dtype=torch.uint8, device=dev)    # NaN floats: every partial is written first
    g = torch.Generator().manual_seed(start_seed)
    starts = [torch.randn(n_r, P.ldq, generator=g).to(dev) for _ in range(2)]
    for s in starts:
        s[:, d:] = float("nan")
    d_tk, d_tv = starts[0].clone(), starts[1].clone()
    seed_buf = torch.tensor([COUNTER], dtype=torch.int64, device=dev)
    desc = _desc(P, q, seed_buf)
    check(lib().rp_ti_attn_bwd(ctypes.byref(desc), A.data_ptr(), dpd.data_ptr(), ad.data_ptr(), d_o.data_ptr(),
                               dq_t.data_ptr(), ws.data_ptr(), n_ws, d_tk.data_ptr(), d_tv.data_ptr(), None),
          "rp_ti_attn_bwd")
    torch.cuda.synchronize()
    return {"dS": dpd, "Ad": ad, "dq_t": dq_t, "d_time_k": d_tk, "d_time_v": d_tv, "starts": starts}


def check_bwd(P, A, out, alias=False):
    B, H, L, Lp, d = P.B, P.H, P.L, P.Lp, P.H * tr.SLOT
    ref = tr.backward(P, A=A)
    dev = A.device
    live = P.pad.reshape(B, 1, L).expand(B, H, L).reshape(B * H, L)
    upper = torch.ones(L, L, dtype=torch.bool, device=dev).triu(1)
    dS = out["dS"]
    # dS: written at rows and columns < L only (the GEMMs read no more); j > i and dead rows exactly 0
    assert bool(torch.isnan(dS[:, L:, :].float()).all()) and bool(torch.isnan(dS[:, :, L:].float()).all())
    body = dS[:, :L, :L].float()
    assert bool((body[:, upper] == 0).all()) and bool((body[~live] == 0).all())
    r = _note("dS", tr.ratio(body, ref["dS"], ref["dS_b"]))
    assert r <= TOL_DS, r
    if not alias:
        adb = out["Ad"][:, :L, :L].float()
        assert bool((adb[:, upper] == 0).all()) and bool((adb[~live] == 0).all())
        r = _note("Ad (bwd)", tr.ratio(adb, ref["Ad"], ref["Ad_b"]))
        assert r <= TOL_DS, r
    dq = out["dq_t"]
    dead = ~P.pad.reshape(-1)
    assert bool((dq[dead, :d].float() == 0).all())
    assert bool(torch.isnan(dq[:, d:].float()).all())
    r = _note("dq_t", tr.ratio(dq[:, :d], ref["dq_t"], ref["dq_t_b"]))
    assert r <= TOL_DQT, r
    true_cols = (torch.arange(d, device=dev) % tr.SLOT) < P.head_dim
    for name, start in (("d_time_k", out["starts"][0]), ("d_time_v", out["starts"][1])):
        got = out[name]
        # padded columns, buckets no live pair falls in, and columns past H * 64 keep their start value bit for bit
        keep = torch.ones_like(got, dtype=torch.bool)
        keep[:, :d] = ~(true_cols[None, :] & ref["used"])
        assert torch.equal(_bits(got[keep]), _bits(start[keep])), name
        bound = tr.table_bound(ref[name + "_b"], start[:, :d], ref[name])
        r = _note("d_time", tr.ratio(got[:, :d] - start[:, :d].double(), ref[name], bound, true_cols[None, :].expand_as(bound)))
        assert r <= TOL_TIME, (name, r)
    return ref


# ------------------------------------------------------------------------------------------------ forward sweep
FWD_CASES = (
    [dict(L=L, head_dim=64, H=2, span=63, p=p) for L in (1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 200, 255, 256)
     for p in (0.0, P_DROP)]
    + [dict(L=65, head_dim=hd, H=H, span=256, p=p, dtype=dt) for hd, H in ((64, 1), (50, 2), (32, 4), (64, 4))
       for dt in (torch.int64, torch.float32, torch.float64) for p in (0.0, P_DROP)]
    + [dict(L=129, head_dim=32, H=4, span=s, p=p, dtype=torch.float64) for s in (1, 2, 63, 256, TI_MAX_SPAN)
       for p in (0.0, P_DROP)]
)


def _cid(c):
    dt = {torch.int64: "i64", torch.float32: "f32", torch.float64: "f64"}[c.get("dtype", torch.int64)]
    return f"L{c['L']}-hd{c['head_dim']}x{c['H']}-span{c['span']}-p{c['p']}-{dt}"


@pytest.mark.parametrize("case", FWD_CASES, ids=_cid)
def test_forward(cuda, case):
    c = dict(case)
    P = _problem(cuda, 5, c.pop("L"), c.pop("head_dim"), c.pop("H"), c.pop("span"), c.pop("p"), **c)
    check_fwd(P, run_fwd(P))


@pytest.mark.parametrize("p,use_ptr,alias", [(0.0, False, True), (0.0, True, False), (P_DROP, False, False),
                                             (P_DROP, True, False)])
def test_forward_seed_pointer_and_ad_alias(cuda, p, use_ptr, alias):
    P = _problem(cuda, 5, 100, 64, 2, 64, p, use_ptr=use_ptr)
    out = run_fwd(P, alias)
    check_fwd(P, out, alias)
    check_bwd(P, out["A"], run_bwd(P, out["A"], alias), alias)


INTERVAL_CASES = [
    ("edges", torch.int64, 1), ("edges", torch.int64, 2), ("edges", torch.int64, 63), ("edges", torch.int64, 256),
    ("edges", torch.int64, TI_MAX_SPAN), ("decreasing", torch.int64, 63), ("unsorted", torch.int64, 63),
    ("big_int", torch.int64, 63), ("epoch_f32", torch.float32, 256), ("frac", torch.float32, 8), ("frac", torch.float64, 8),
    ("frac", torch.float64, 63), ("epoch_f64", torch.float64, 8), ("edges", torch.float64, 63),
    ("decreasing", torch.float32, 63),
]


@pytest.mark.parametrize("kind,dtype,span", INTERVAL_CASES, ids=lambda v: str(v).replace("torch.", ""))
@pytest.mark.parametrize("p", [0.0, P_DROP])
def test_interval_edges(cuda, kind, dtype, span, p):
    """Adjacent table rows are independent, so a pair put in a neighbouring bucket moves its logit by O(1), far outside A's
    bound; the same timestamps feed the backward's table gradients."""
    P = _problem(cuda, 5, 65, 64, 2, span, p, times=kind, dtype=dtype)
    out = run_fwd(P)
    check_fwd(P, out)
    check_bwd(P, out["A"], run_bwd(P, out["A"]))


# ------------------------------------------------------------------------------------------------ backward sweep
BWD_CASES = (
    [dict(L=L, head_dim=64, H=2, span=63, p=p) for L in (1, 33, 64, 65, 129, 256) for p in (0.0, P_DROP)]
    + [dict(L=77, head_dim=hd, H=H, span=16, p=P_DROP) for hd, H in ((64, 1), (50, 2), (32, 4), (64, 4))]
    + [dict(L=96, head_dim=50, H=1, span=s, p=P_DROP, dtype=dt) for s in (1, TI_MAX_SPAN)
       for dt in (torch.int64, torch.float32, torch.float64)]
)


@pytest.mark.parametrize("case", BWD_CASES, ids=_cid)
def test_backward(cuda, case):
    c = dict(case)
    P = _problem(cuda, 5, c.pop("L"), c.pop("head_dim"), c.pop("H"), c.pop("span"), c.pop("p"), **c)
    out = run_fwd(P, alias=P.p == 0)
    check_bwd(P, out["A"], run_bwd(P, out["A"], alias=P.p == 0), alias=P.p == 0)


@pytest.mark.parametrize("H", [1, 2, 4])
@pytest.mark.parametrize("which", ["1", "G-1", "G", "G+1", "2G+3"])
@pytest.mark.parametrize("L", [9, 65])
def test_backward_ctas_over_several_sequences(cuda, H, which, L):
    """G = 256 / H CTAs per head; CTA g takes sequences g, g + G, ...: B at and around G and 2G puts a second and third
    sequence in some CTAs, whose timestamps are reloaded and whose pairs add into the same shared-memory sums."""
    G = tr.BWD_CTAS // H
    B = {"1": 1, "G-1": G - 1, "G": G, "G+1": G + 1, "2G+3": 2 * G + 3}[which]
    P = _problem(cuda, B, L, CTA_CASE["head_dim"], H, CTA_CASE["span"], CTA_CASE["p"], times=CTA_CASE["times"], seed=B)
    out = run_fwd(P)
    check_bwd(P, out["A"], run_bwd(P, out["A"]))


def test_backward_largest_span_four_heads_several_sequences(cuda):
    """span 320 and H 4: the backward's largest shared-memory footprint, with B = 2 * 64 + 1 sequences over 64 CTAs"""
    P = _problem(cuda, 2 * 64 + 1, 200, 64, 4, TI_MAX_SPAN, P_DROP, times="edges")
    out = run_fwd(P)
    check_fwd(P, out)
    check_bwd(P, out["A"], run_bwd(P, out["A"]))


def test_rerun_is_bitwise_equal_but_the_time_tables(cuda):
    P = _problem(cuda, 70, 65, 50, 4, 63, P_DROP)
    f1, f2 = run_fwd(P), run_fwd(P)
    for k in ("A", "Ad", "hpre"):
        assert torch.equal(_bits(f1[k]), _bits(f2[k])), k
    b1, b2 = run_bwd(P, f1["A"]), run_bwd(P, f1["A"])
    for k in ("dS", "Ad", "dq_t"):
        assert torch.equal(_bits(b1[k]), _bits(b2[k])), k
    ref = tr.backward(P, A=f1["A"])
    d = P.H * tr.SLOT
    for k, s in (("d_time_k", 0), ("d_time_v", 1)):   # fp32 atomics: the order of the shared-memory sums varies
        bound = tr.table_bound(ref[k + "_b"], b1["starts"][s][:, :d], ref[k])
        r = _note("d_time", tr.ratio(b2[k][:, :d], b1[k][:, :d].double(), 2 * bound, torch.isfinite(bound)))
        assert r <= TOL_TIME, (k, r)


# ------------------------------------------------------------------------------------------------ positional terms
@pytest.mark.parametrize("B,L,H,p", [(3, 50, 2, 0.0), (2, 200, 4, 0.5), (5, 7, 1, 0.5), (1, 1, 2, 0.5)])
def test_pos_add_bit_exact(cuda, B, L, H, p):
    """kv += dropout(pos) rounded to bf16 once, keyed by token and column; ld_kv > 2d.  p 0.5: 1 / (1 - p) is a power of two,
    so the kernel's fast-math reciprocal is exact and the emulation can match it bit for bit."""
    d = H * tr.SLOT
    T, ld = B * L, 2 * d + 24
    g = torch.Generator().manual_seed(B * 1000 + L)
    kv = (torch.randn(T, ld, generator=g)).to(torch.bfloat16).to(cuda)
    kv[:, 2 * d:] = NAN16
    pos_k, pos_v = (torch.randn(L, d, generator=g).to(cuda) for _ in range(2))
    seed_buf = torch.tensor([COUNTER], dtype=torch.int64, device=cuda)
    seed_eff = SEED + (COUNTER if p > 0 else 0)
    want = tr.pos_add(kv[:, :2 * d], pos_k, pos_v, L, d, p, seed_eff, tr.SITE_TK, tr.SITE_TV)
    check(lib().rp_ti_pos_add(kv.data_ptr(), ld, pos_k.data_ptr(), pos_v.data_ptr(), T, L, d, p, SEED, seed_buf.data_ptr(),
                              tr.SITE_TK, tr.SITE_TV, None), "rp_ti_pos_add")
    torch.cuda.synchronize()
    assert torch.equal(_bits(kv[:, :2 * d]), _bits(want))
    assert bool(torch.isnan(kv[:, 2 * d:].float()).all())


@pytest.mark.parametrize("B,L,H,hd,p", [(7, 50, 2, 50, P_DROP), (256, 200, 2, 64, P_DROP), (3, 1, 4, 32, 0.0),
                                        (130, 33, 1, 64, 0.0)])
def test_pos_bwd(cuda, B, L, H, hd, p):
    """d_pos += the dropout' of dK' / dV' summed over the sequences, onto preset values; padded columns untouched"""
    d = H * tr.SLOT
    T, ld = B * L, 2 * d + 8
    g = torch.Generator().manual_seed(B + L)
    dkv = torch.randn(T, ld, generator=g).to(torch.bfloat16).to(cuda)
    dkv[:, 2 * d:] = NAN16
    starts = [torch.randn(L, d, generator=g).to(cuda) for _ in range(2)]
    d_pk, d_pv = starts[0].clone(), starts[1].clone()
    seed_buf = torch.tensor([COUNTER], dtype=torch.int64, device=cuda)
    seed_eff = SEED + (COUNTER if p > 0 else 0)
    check(lib().rp_ti_pos_bwd(dkv.data_ptr(), ld, B, L, d, hd, p, SEED, seed_buf.data_ptr(), tr.SITE_TK, tr.SITE_TV,
                              d_pk.data_ptr(), d_pv.data_ptr(), None), "rp_ti_pos_bwd")
    torch.cuda.synchronize()
    rk, bk, rv, bv, true_cols = tr.pos_bwd(dkv[:, :2 * d], B, L, d, hd, p, seed_eff, tr.SITE_TK, tr.SITE_TV)
    for got, start, ref, b in ((d_pk, starts[0], rk, bk), (d_pv, starts[1], rv, bv)):
        assert torch.equal(_bits(got[:, ~true_cols]), _bits(start[:, ~true_cols]))
        bound = tr.table_bound(b, start, ref)
        r = _note("d_pos", tr.ratio(got - start.double(), ref, bound, true_cols[None, :].expand_as(bound)))
        assert r <= TOL_POS, r


# ------------------------------------------------------------------------------------------------ config-2 stage
def _c2_batch(B, L, n_items, span, g):
    """left-padded windows with ties and gaps beyond the span (int64 timestamps)"""
    lens = torch.randint(1, L + 1, (B,), generator=g)
    lens[0] = L
    ids = torch.full((B, L), n_items, dtype=torch.int64)
    pm = torch.zeros(B, L, dtype=torch.bool)
    ts = torch.zeros(B, L, dtype=torch.int64)
    for b in range(B):
        n = int(lens[b])
        ids[b, L - n:] = torch.randint(0, n_items, (n,), generator=g)
        pm[b, L - n:] = True
        ts[b, L - n:] = 10**6 + (torch.randint(0, 3, (n,), generator=g) * torch.randint(0, span, (n,), generator=g)).cumsum(0)
    lab = torch.randint(0, n_items, (B, L), generator=g)
    return ids, pm, ts, lab, pm.clone()


def test_config2_stage_against_reference(cuda):
    """B 256 > G = 128, L 200, d 128, 2 heads, span 256, dropout 0.2: one training step, then block 0's attention backward
    re-run with the time-table gradients zeroed; h, dQ, dK', dV' and every bucket row of both tables' gradients against
    the float64 stage on the engine's own Q, K' | V', q_in and dh."""
    import oracle.tisasrec as oti
    from replay_b200.engine_tisasrec import TiConfig, TiSasRecEngine

    B, L, d, H, n_items, span = 256, 200, 128, 2, 50_000, 256
    cfg = TiConfig(n_items=n_items, d=d, n_heads=H, n_blocks=2, max_len=L, dropout=P_DROP, time_span=span)
    eng = TiSasRecEngine(cfg, B, L, cuda, seed=7)
    eng.load_canonical(oti.random_params(n_items, d, L, 2, span, seed=3))
    ids, pm, ts, lab, tm = _c2_batch(B, L, n_items, span, torch.Generator().manual_seed(2))
    eng.set_batch(ids.to(cuda), pm.to(cuda), lab.to(cuda), tm.to(cuda))
    eng.set_times(ts.to(cuda))
    eng.tick_rng()
    eng.forward_train()
    eng.g32.zero_()
    eng.backward()
    eng.grads["time_k"].zero_()
    eng.grads["time_v"].zero_()
    eng._ti_attention_backward(0, P_DROP)
    torch.cuda.synchronize()
    a, s = eng.act[0], eng.s
    seed_eff = eng.seed + int(eng.rng_counter.item())
    ref = tr.attention_stage(a["Q"], a["KV"], a["q_in"], s["dh"], ts.to(cuda), pm.to(cuda), eng.params16["time_k"],
                             eng.params16["time_v"], H, 64, span, P_DROP, seed_eff, eng._site(0, 0) << 40)
    got = {"h": a["h"], "dQ": s["dQ"], "dK": s["dKV"][:, :d], "dV": s["dKV"][:, d:]}
    for name, tol in (("h", TOL_STAGE_H), ("dQ", TOL_STAGE_GRAD), ("dK", TOL_STAGE_GRAD), ("dV", TOL_STAGE_GRAD)):
        err = max(block_err(got[name][b * L:(b + 1) * L], ref[name][b * L:(b + 1) * L]) for b in range(B))
        fam = "stage h" if name == "h" else "stage grads"
        assert _note(fam, err) <= tol, (name, err)
    for name in ("time_k", "time_v"):
        err = block_err(eng.grads[name].double(), ref["d_" + name], blk=1)
        assert _note("stage time tables", err) <= TOL_STAGE_TIME, (name, err)
