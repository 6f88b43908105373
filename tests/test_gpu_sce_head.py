"""The scalable cross-entropy head (csrc/rp_sce_head.cu: rp_sce_head_fwd / rp_sce_head_bwd) called through the C ABI, each
case against the float64 reference of tests/sce_reference.py computed from the same bf16 inputs and the kernel's own
bucket matrix and selections.

Layout as SasRecEngine._set_sce passes it: hc bf16 [capacity, d] (rows >= n_rows hold finite garbage the head must
ignore), table bf16 [n_items, d], both in the engine's feature layouts - unpadded, or d 50 / 1 head (dp 64), 96 / 1 head
(dp 128), 192 / 4 heads (dp 256), 400 / 4 heads (dp 512) with zero padded columns; labels int64, pad_mask uint8, n_rows
int32 on the device.  The bucket matrix is read back from workspace offset 0, omega (mix_x) from the next 256-byte
aligned region (both pinned by test_sce_reference_cpu.py).

Families: the Philox draw against tests/philox_stream.py and N(0, 1); the bucket matrix and omega; the two top-Ks against
fp64 scores; loss and d_hc with collisions, rows of CE exactly 0, out-of-catalog labels, large logits and duplicated
buckets (exact ties: the cnt > 1 branch of sce_collect_kernel); chunks of buckets forced through RP_SCE_CHUNK_BYTES and one
that chunks at the default budget; the staged forward, determinism and workspace reuse.  Run with -s to print the worst
error of each family.
"""
import ctypes
import math
from dataclasses import dataclass

import numpy as np
import pytest
import torch

import philox_stream as ps
import sce_reference as sr
from fp64_checks import WorstErrors, block_err, feat_mask, ulp_err
from replay_b200._lib import SCE_ALL, SCE_BUCKET_CE, SCE_DRAW, SCE_SELECT_X, SCE_SELECT_Y, SceDesc, check, lib

pytestmark = pytest.mark.gpu

SENT = -3.25                 # sentinel for d_hc memory (exact in bf16)
N_ITEMS = 5000
SEED, COUNTER = 0x5EED5EED1234, 977
LAYOUTS = {64: (50, 50), 128: (96, 96), 256: (192, 48), 512: (400, 100)}   # padded: (d_true, hd_valid)
DEFAULT_CHUNK_BYTES = 256 << 20

# Tolerances: about 3x the worst value seen over every case of this file on one H100 80GB HBM3 (run with -s); the bucket
# tolerances are the rounding bounds themselves.
TOL_DRAW = 0.2               # |draw - port| / (2e-3 + 1e-5 |z|); worst seen 0.059
TOL_BUCKET_ULP = 1.0         # non-mix buckets / omega, bf16 ulps of the fp32 product (one rounding: 0.5); worst seen 0.5
TOL_MIX_ULP = 2.0            # mix buckets, half-ulps of bf16 with 2^-18 sum |omega| |hc| for fp32 accumulation; worst 1.0
TOL_SEL = 1e-7               # fp64 k-th best - picked, relative to the bucket's largest sum |b| |h|; worst seen 3.4e-8
TOL_SCORE_X = 6e-7           # |score_x - fp64 score| / sum |b| |h|; worst seen 1.9e-7
TOL_LOSS_ULPS = 9.0          # |loss - ref| in units of 2^-24 * mean(|lse| + |c| + 1) of the counted rows; worst seen 3.0
TOL_HC_ULP = 3.0             # d_hc, half-ulps of bf16 with sce_reference.SLACK * sum_j |G_j| |Y_j|; worst seen 0.90
TOL_HC_BLOCK = 7e-3          # d_hc per 64-row block, norm-relative; worst seen 2.3e-3

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


def _ru(x, m):
    return (x + m - 1) // m * m


def buckets_per_chunk(d, bsx, bsy, nb, budget=DEFAULT_CHUNK_BYTES):
    """sce_layout's chunk of buckets: the fp32 S [bs_x64, bs_y64] and dX [bs_x64, d] of each fit the budget, >= 1, <= n_b."""
    per = _ru(bsx, 64) * _ru(bsy, 64) * 4 + _ru(bsx, 64) * d * 4
    return min(max(budget // per, 1), nb)


@dataclass
class Case:
    d: int
    padded: bool
    cap: int
    n_rows: int
    nb: int
    bsx: int
    bsy: int
    mix: bool = False
    labels: str = "random"    # "random", "collide" (drawn from the selecting buckets' items), "item" (bs_y 1: the item)
    invalid: bool = False     # real rows with label -100 or n_items
    scale: float = 1.0        # std of the logits
    dup: tuple = ()           # groups of buckets drawn identically (exact ties)
    per_chunk: int = 0        # forced buckets per chunk (RP_SCE_CHUNK_BYTES), 0 = default budget
    n_items: int = N_ITEMS

    @property
    def layout(self):
        return LAYOUTS[self.d] if self.padded else (self.d, 0)

    @property
    def id(self):
        s = f"d{self.d}{'p' if self.padded else ''}-cap{self.cap}-n{self.n_rows}-nb{self.nb}-x{self.bsx}-y{self.bsy}"
        s += "-mix" if self.mix else ""
        s += f"-{self.labels}" if self.labels != "random" else ""
        s += "-inval" if self.invalid else ""
        s += f"-s{self.scale:g}" if self.scale != 1.0 else ""
        s += "-dup" + "_".join(str(len(g)) for g in self.dup) if self.dup else ""
        s += f"-I{self.n_items}" if self.n_items != N_ITEMS else ""
        return s

    def chunks(self):
        per = buckets_per_chunk(self.d, self.bsx, self.bsy, self.nb, self.budget() or DEFAULT_CHUNK_BYTES)
        return -(-self.nb // per)

    def budget(self):
        if not self.per_chunk:
            return 0
        return self.per_chunk * (_ru(self.bsx, 64) * _ru(self.bsy, 64) * 4 + _ru(self.bsx, 64) * self.d * 4)


CASES = [
    Case(64, False, 300, 300, 64, 64, 33),
    Case(64, True, 301, 250, 3, 65, 1024, mix=True, invalid=True),
    Case(64, True, 700, 700, 64, 64, 64, labels="collide"),
    Case(64, False, 300, 200, 1, 63, 1024, invalid=True),
    Case(64, False, 600, 600, 64, 1, 1000, scale=12.0),
    Case(64, True, 500, 500, 8, 63, 33, dup=((0, 1), (4, 5, 6))),
    Case(128, False, 1200, 1200, 64, 256, 256, mix=True),
    Case(128, True, 700, 613, 600, 1, 1, labels="item"),
    Case(128, False, 1100, 900, 3, 1024, 1000),
    Case(128, True, 1000, 1000, 64, 128, 256, scale=12.0, labels="collide"),
    Case(128, False, 800, 800, 16, 64, 64, dup=((2, 3), (7, 8, 9))),
    Case(256, False, 1000, 1000, 64, 63, 1024, labels="collide"),
    Case(256, True, 1200, 1100, 1, 1024, 33, invalid=True),
    Case(256, True, 333, 333, 3, 1, 1, labels="item", invalid=True),
    Case(512, False, 500, 500, 3, 65, 1000, n_items=1000),
    Case(512, True, 900, 777, 64, 64, 1024, mix=True, labels="collide"),
    Case(512, True, 300, 300, 600, 1, 33, dup=((598, 599),)),
]

CHUNK_CASES = [   # (case, expected number of chunks)
    (Case(128, False, 500, 500, 6, 64, 64, dup=((2, 3),), per_chunk=1), 6),
    (Case(64, True, 500, 500, 7, 65, 100, dup=((1, 2), (3, 4, 5)), per_chunk=2), 4),
    (Case(256, False, 600, 600, 9, 64, 128, dup=((7, 8),), per_chunk=8), 2),
    (Case(128, True, 500, 450, 5, 64, 64, mix=True, dup=((1, 2),), per_chunk=2), 3),
    (Case(512, False, 1500, 1500, 43, 1024, 1024, dup=((41, 42),)), 2),   # the default budget: 42 + 1
]


# ----------------------------------------------------------------------------------------------------------------------
# inputs and calls
# ----------------------------------------------------------------------------------------------------------------------
def _feat(c: Case):
    return feat_mask(c.d, c.layout[1]).nonzero()[:, 0]


def make_inputs(c: Case, dev, seed=0):
    g = torch.Generator().manual_seed(seed * 7919 + c.d * 131 + c.cap * 7 + c.nb * 3 + c.bsx + c.bsy)
    d_true, hdv = c.layout
    feat, I = _feat(c), c.n_items
    table = torch.zeros(I, c.d)
    table[:, feat] = torch.randn(I, d_true, generator=g) * (c.scale / math.sqrt(d_true))
    hc = torch.zeros(c.cap, c.d)
    hc[:, feat] = torch.randn(c.cap, d_true, generator=g)
    hc[c.n_rows:] *= 8.0                                              # stale rows: finite garbage
    pad = (torch.rand(c.cap, generator=g) < 0.85).to(torch.uint8)
    labels = torch.randint(0, I, (c.cap,), generator=g)
    if c.invalid:
        t = torch.arange(c.cap)
        labels[t % 11 == 3] = -100
        labels[t % 11 == 7] = I
    x = dict(hc=hc.to(torch.bfloat16).to(dev), table=table.to(torch.bfloat16).to(dev), labels=labels.to(dev),
             pad=pad.to(dev), n_rows=torch.tensor([c.n_rows], dtype=torch.int32, device=dev),
             counter=torch.tensor([COUNTER], dtype=torch.int64, device=dev), draw_given=0, g=g)
    n_draw = c.cap * c.nb if c.mix else c.nb * d_true
    x["draw"] = torch.zeros(n_draw + 1, device=dev)                  # one sentinel element past the draw
    x["draw"][-1] = 12345.0
    if c.dup:
        draw = torch.randn(c.cap, c.nb, generator=g) if c.mix else torch.randn(c.nb, d_true, generator=g)
        for grp in c.dup:
            for b in grp[1:]:
                if c.mix:
                    draw[:, b] = draw[:, grp[0]]
                else:
                    draw[b] = draw[grp[0]]
        x["draw"][:n_draw] = draw.reshape(-1).to(dev)
        x["draw_given"] = 1
    return x


def workspace(c: Case, dev, fill=0):
    n = lib().rp_sce_head_workspace(c.cap, c.n_items, c.d, c.nb, c.bsx, c.bsy, int(c.mix))
    assert n > 0
    return torch.full((n,), fill, dtype=torch.uint8, device=dev)


def _desc(c: Case, x, ws, out, seed=SEED):
    s = SceDesc()
    s.hc, s.table, s.labels, s.pad_mask, s.n_rows = (x[k].data_ptr() for k in ("hc", "table", "labels", "pad", "n_rows"))
    s.capacity, s.n_items, s.d = c.cap, c.n_items, c.d
    s.d_true, s.hd_valid = c.layout
    s.n_buckets, s.bucket_size_x, s.bucket_size_y, s.mix_x = c.nb, c.bsx, c.bsy, int(c.mix)
    s.seed, s.rng_counter, s.draw_given = seed, x["counter"].data_ptr(), x["draw_given"]
    s.draw = x["draw"].data_ptr()
    s.top_x, s.score_x, s.top_y, s.loss_out = (out[k].data_ptr() for k in ("top_x", "score_x", "top_y", "loss"))
    s.workspace, s.workspace_bytes = ws.data_ptr(), ws.numel()
    return s


def new_out(c: Case, dev):
    return dict(top_x=torch.full((c.nb, c.bsx), -7, dtype=torch.int64, device=dev),
                score_x=torch.full((c.nb, c.bsx), 7.0, device=dev),
                top_y=torch.full((c.nb, c.bsy), -7, dtype=torch.int64, device=dev),
                loss=torch.full((2,), 7.0, device=dev),
                d_hc=torch.full((c.cap + 64, c.d), SENT, dtype=torch.bfloat16, device=dev))


def fwd(c: Case, x, ws, out, stages=SCE_ALL, seed=SEED):
    s = _desc(c, x, ws, out, seed)
    check(lib().rp_sce_head_fwd(ctypes.byref(s), stages, torch.cuda.current_stream().cuda_stream), "rp_sce_head_fwd")
    torch.cuda.synchronize()
    return s


def bwd(c: Case, x, ws, out):
    s = _desc(c, x, ws, out)
    check(lib().rp_sce_head_bwd(ctypes.byref(s), out["d_hc"].data_ptr(), torch.cuda.current_stream().cuda_stream),
          "rp_sce_head_bwd")
    torch.cuda.synchronize()


def set_labels(c: Case, x, ws):
    """"collide" / "item": labels from the items of buckets that select the row (selections first, then the labels; the
    row selection depends on the labels only through their validity, which does not change)."""
    if c.labels == "random":
        return
    out = new_out(c, ws.device)
    fwd(c, x, ws, out, SCE_DRAW | SCE_SELECT_X | SCE_SELECT_Y)
    tx, sx, ty = out["top_x"].cpu(), out["score_x"].cpu(), out["top_y"].cpu()
    lab = x["labels"].cpu()
    sel = sr.selectable(lab, x["pad"].cpu(), c.n_rows, c.n_items)
    g = x["g"]
    for b in range(c.nb):
        for i in range(c.bsx):
            t = int(tx[b, i])
            if not (math.isfinite(float(sx[b, i])) and sel[t]):
                continue
            if c.labels == "item":
                lab[t] = ty[b, 0]
            elif float(torch.rand(1, generator=g)) < 0.5:
                lab[t] = ty[b, int(torch.randint(0, c.bsy, (1,), generator=g))]
    x["labels"].copy_(lab)


def run(c: Case, x, ws):
    out = new_out(c, ws.device)
    fwd(c, x, ws, out)
    out["buckets"] = ws[: c.nb * c.d * 2].view(torch.bfloat16).view(c.nb, c.d).clone()
    bwd(c, x, ws, out)
    return out


# ----------------------------------------------------------------------------------------------------------------------
# checks
# ----------------------------------------------------------------------------------------------------------------------
def check_selections(c: Case, x, out, err, bad):
    sel = sr.selectable(x["labels"], x["pad"], c.n_rows, c.n_items)
    n_sel = int(sel.sum())
    sx, sy, ax, ay = sr.selection_scores(out["buckets"], x["hc"], x["table"], sel)
    fin = torch.isfinite(out["score_x"])
    for name, top, s, a, k, f in (("x", out["top_x"], sx, ax, c.bsx, fin),
                                  ("y", out["top_y"], sy, ay, c.bsy, torch.ones_like(out["top_y"], dtype=torch.bool))):
        n_cols = s.shape[1]
        ids = top.clamp(0, n_cols - 1)
        srt = torch.where(top >= 0, top, -torch.arange(1, k + 1, device=top.device)).sort(1).values
        if not bool((srt[:, 1:] != srt[:, :-1]).all()):
            bad.append(f"top_{name}: an id repeats within a bucket")
        if not bool(((top[f] >= 0) & (top[f] < n_cols)).all()):
            bad.append(f"top_{name}: a finite slot holds an id outside [0, {n_cols})")
            continue
        picked = s.gather(1, ids)
        kth = sr.kth_best(s, k)[:, None]
        scale = a.amax(1, keepdim=True).clamp_min(1e-300)
        gap = ((kth - picked) / scale).masked_fill(~f, 0).clamp_min(0)
        err[f"selection {name}"] = float(gap.max())
    n_fin = fin.sum(1)
    if not bool((n_fin == min(c.bsx, n_sel)).all()):
        bad.append(f"finite top_x slots per bucket {sorted(set(n_fin.tolist()))}, expected min(bs_x, {n_sel})")
    if not bool(sel[out["top_x"].clamp(0, c.cap - 1)][fin].all()):
        bad.append("an unselectable row (pad, >= n_rows or label outside the catalog) holds a finite top_x slot")
    if bool(fin.any()):
        ids = out["top_x"].clamp(0, c.cap - 1)
        d = (out["score_x"].double() - sx.gather(1, ids)).abs() / ax.gather(1, ids).clamp_min(1e-300)
        err["score_x"] = float(d[fin].max())
    return n_sel


def check_loss_and_grad(c: Case, x, out, err, bad, r=None):
    if r is None:
        r = sr.reference(x["hc"], x["table"], x["labels"], x["pad"], c.n_rows, out["top_x"], out["score_x"], out["top_y"])
    loss, d_hc = out["loss"], out["d_hc"]
    inv = float(loss[1])
    n_k = round(1.0 / inv) if inv > 0 else 0
    if inv > 0 and inv != float(torch.tensor(1.0) / n_k):
        bad.append(f"loss_out[1] = {inv!r} is not float32(1 / {n_k})")
    nc, na = r["n_counted"], r["n_ambiguous"]
    if not nc <= n_k <= nc + na:
        bad.append(f"the kernel counts {n_k} rows; the reference {nc} surely and {na} ambiguous")
    if n_k == 0:
        if not (math.isnan(float(loss[0])) and inv == 0.0):
            bad.append(f"no counted row: loss_out = {loss.tolist()}, expected [NaN, 0]")
    elif not math.isfinite(float(loss[0])):
        bad.append("loss is not finite")
    else:
        ref_sum = float(r["row_max"][r["counted"]].sum())
        e = max(abs(float(loss[0]) - ref_sum / n_k) - r["ce_sum_ambiguous"] / n_k, 0.0) / r["loss_unit"]
        err["loss (ulps)"] = e
    got = d_hc[: c.cap].double()
    if not bool(torch.isfinite(got).all()):
        bad.append("NaN / Inf in d_hc")
    if bool((d_hc[: c.cap] == SENT).all(1).any()):
        bad.append("a d_hc row was not written")
    if not bool((d_hc[c.cap:] == SENT).all()):
        bad.append("d_hc rows >= capacity were written")
    pad_cols = ~feat_mask(c.d, c.layout[1]).to(got.device)
    if bool(pad_cols.any()) and not bool((got[:, pad_cols] == 0).all()):
        bad.append("padded columns of d_hc are not zero")
    zero_rows = ~(r["counted"] | r["ambiguous"])
    if not bool((got[zero_rows] == 0).all()):
        bad.append("rows that carry no loss (unselected, pad, >= n_rows, CE 0) have a non-zero d_hc")
    if n_k:
        k = r["checked"]
        ref = r["d_hc"] * (nc / n_k)
        slack = sr.SLACK * r["mag_hc"] * (nc / n_k) + 1e-30
        err["d_hc ulp"] = ulp_err(got[k], ref[k], slack[k])
        err["d_hc block"] = block_err(got * k[:, None], ref * k[:, None])
    return r


def assert_within(c, err, bad):
    tol = {"selection x": TOL_SEL, "selection y": TOL_SEL, "score_x": TOL_SCORE_X, "loss (ulps)": TOL_LOSS_ULPS,
           "d_hc ulp": TOL_HC_ULP, "d_hc block": TOL_HC_BLOCK}
    for k, v in err.items():
        _note(k, v)
    over = {k: v for k, v in err.items() if v > tol[k]}
    assert not bad and not over, (c.id, bad, over)


def _full_check(c: Case, x, out):
    err, bad = {}, []
    check_selections(c, x, out, err, bad)
    r = check_loss_and_grad(c, x, out, err, bad)
    return r, err, bad


def _collision_fraction(c, x, out, r):
    live = r["live"]
    lab = x["labels"].clamp(0, c.n_items - 1)[out["top_x"].clamp(0, c.cap - 1)]
    hit = (lab[:, :, None] == out["top_y"][:, None, :]).any(-1) & live
    return float(hit.sum()) / max(int(live.sum()), 1)


def _tied_rows(r):
    return int(((r["winners"] >= 2) & r["counted"]).sum())


# ----------------------------------------------------------------------------------------------------------------------
# the draw and the bucket matrix
# ----------------------------------------------------------------------------------------------------------------------
def _draw_err(got, seed, counter):
    want = torch.from_numpy(ps.sce_normals(seed, counter, got.numel())).to(got.device)
    return float(((got.double() - want).abs() / (2e-3 + 1e-5 * want.abs())).max())


@pytest.mark.parametrize("c", [Case(128, True, 300, 300, 64, 1, 1), Case(64, False, 301, 290, 3, 1, 1, mix=True)],
                         ids=lambda c: c.id)
def test_draw_matches_philox_port(cuda, c):
    """Element-wise against the port; under mix_x capacity x n_b = 903 is odd, so the last pair writes its cosine only."""
    x = make_inputs(c, cuda)
    ws = workspace(c, cuda)
    fwd(c, x, ws, new_out(c, cuda), SCE_DRAW)
    n = x["draw"].numel() - 1
    assert float(x["draw"][n]) == 12345.0, "the draw wrote past its last element"
    assert _note("draw vs port", _draw_err(x["draw"][:n], SEED, COUNTER)) <= TOL_DRAW


def test_draw_distribution(cuda):
    """2^20 draws: N(0, 1) by mean, variance and Kolmogorov-Smirnov; the cosine and sine halves uncorrelated; the next counter
    and another seed give streams uncorrelated with the first."""
    from scipy import stats
    c = Case(64, False, 4096, 4096, 256, 1, 1, mix=True)
    x = make_inputs(c, cuda)
    ws = workspace(c, cuda)
    n = c.cap * c.nb
    streams = []
    for seed, counter in ((SEED, COUNTER), (SEED, COUNTER + 1), (SEED + (1 << 32), COUNTER)):
        x["counter"].fill_(counter)
        fwd(c, x, ws, new_out(c, cuda), SCE_DRAW, seed=seed)
        z = x["draw"][:n].double()
        assert bool(torch.isfinite(z).all())
        _note("draw vs port", _draw_err(z, seed, counter))
        zc = z.cpu().numpy()
        assert abs(zc.mean()) < 5 / math.sqrt(n) and abs(zc.var() - 1) < 5 * math.sqrt(2 / n), (zc.mean(), zc.var())
        assert stats.kstest(zc, "norm").pvalue > 1e-4
        assert abs(np.corrcoef(zc[0::2], zc[1::2])[0, 1]) < 5 / math.sqrt(n / 2)
        streams.append(zc)
    for other in streams[1:]:
        assert abs(np.corrcoef(streams[0], other)[0, 1]) < 5 / math.sqrt(n)
    assert _worst.worst["draw vs port"][0] <= TOL_DRAW


def _bf16_ulp(v):
    return torch.exp2(torch.floor(torch.log2(v.abs().clamp_min(1e-30))) - 7)


@pytest.mark.parametrize("given", [False, True])
@pytest.mark.parametrize("padded", [False, True])
@pytest.mark.parametrize("d", [64, 128, 256, 512])
def test_bucket_matrix(cuda, d, padded, given):
    """Non-mix: buckets = bf16(draw * d_true^-1/4) scattered into the feature slots, padded columns exactly 0; a given draw
    is read as given."""
    c = Case(d, padded, 300, 300, 37, 1, 1)
    x = make_inputs(c, cuda)
    if given:
        x["draw_given"] = 1
        x["draw"][:-1] = torch.linspace(-4, 4, x["draw"].numel() - 1, device=cuda)
    ws = workspace(c, cuda)
    before = x["draw"].clone()
    fwd(c, x, ws, new_out(c, cuda), SCE_DRAW)
    if given:
        assert torch.equal(x["draw"], before), "a given draw was changed"
    d_true, _ = c.layout
    b = ws[: c.nb * c.d * 2].view(torch.bfloat16).view(c.nb, c.d).double()
    want = (x["draw"][:-1].view(c.nb, d_true) * np.float32(d_true ** -0.25)).double()
    feat = _feat(c).to(cuda)
    got = b[:, feat]
    e = float(((got - want).abs() / _bf16_ulp(want)).max())
    assert _note("buckets (bf16 ulps)", e) <= TOL_BUCKET_ULP
    pad_cols = torch.ones(c.d, dtype=torch.bool, device=cuda)
    pad_cols[feat] = False
    assert bool((b[:, pad_cols] == 0).all())


@pytest.mark.parametrize("c", [Case(128, True, 1200, 1000, 64, 1, 1, mix=True), Case(512, False, 301, 77, 3, 1, 1, mix=True),
                               Case(64, True, 4133, 4133, 100, 1, 1, mix=True)], ids=lambda c: c.id)
def test_mix_buckets(cuda, c):
    """mix_x: omega = bf16(draw * d_true^-1/4) over the first n_rows rows (zero beyond, and in the columns past n_b),
    buckets = bf16(omega^T . hc) over those rows only - the stale rows behind them hold large finite garbage."""
    x = make_inputs(c, cuda)
    ws = workspace(c, cuda)
    fwd(c, x, ws, new_out(c, cuda), SCE_DRAW)
    d_true, _ = c.layout
    nbp, cap64 = _ru(c.nb, 64), _ru(c.cap, 64)
    o = _ru(c.nb * c.d * 2, 256)
    om = ws[o: o + cap64 * nbp * 2].view(torch.bfloat16).view(cap64, nbp).double()
    want = (x["draw"][:-1].view(c.cap, c.nb)[: c.n_rows] * np.float32(d_true ** -0.25)).double()
    e = float(((om[: c.n_rows, : c.nb] - want).abs() / _bf16_ulp(want)).max())
    _note("buckets (bf16 ulps)", e)
    assert e <= TOL_BUCKET_ULP
    assert bool((om[c.n_rows:] == 0).all()) and bool((om[:, c.nb:] == 0).all())
    b = ws[: c.nb * c.d * 2].view(torch.bfloat16).view(c.nb, c.d).double()
    h = x["hc"][: c.n_rows].double()
    ref = om[: c.n_rows, : c.nb].T @ h
    slack = 2.0 ** -18 * (om[: c.n_rows, : c.nb].abs().T @ h.abs())
    assert _note("mix buckets (half-ulps)", ulp_err(b, ref, slack + 1e-30)) <= TOL_MIX_ULP


# ----------------------------------------------------------------------------------------------------------------------
# selections, loss and d_hc
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", CASES, ids=lambda c: c.id)
def test_sce_head_matches_fp64(cuda, c):
    x = make_inputs(c, cuda)
    ws = workspace(c, cuda)
    set_labels(c, x, ws)
    out = run(c, x, ws)
    r, err, bad = _full_check(c, x, out)
    if c.labels == "collide":
        f = _note("collision fraction (info)", _collision_fraction(c, x, out, r))
        if f <= 0.1:
            bad.append(f"only {f:.3f} of the slots collide with their row's label")
    if c.labels == "item" and not bool(((r["row_max"] == 0) & r["selectable"]).any()):
        bad.append("no selected row has CE exactly 0")
    if c.dup and _tied_rows(r) == 0:
        bad.append("duplicated buckets produced no exactly tied row")
    if c.scale > 1 and float(r["row_max"].max()) < 20:
        bad.append(f"large logits reach a CE of only {float(r['row_max'].max()):.1f}")
    _note("ambiguous rows (info)", r["n_ambiguous"])
    _note("near-tie rows (info)", r["near_tie"])
    # a second call on the same workspace: bit for bit
    out2 = run(c, x, ws)
    for k in ("loss", "top_x", "score_x", "top_y", "d_hc", "buckets"):
        if not torch.equal(out[k], out2[k]) and not (k == "loss" and torch.equal(out[k].isnan(), out2[k].isnan())
                                                     and torch.equal(out[k].nan_to_num(), out2[k].nan_to_num())):
            bad.append(f"a second identical call gave a different {k}")
    assert_within(c, err, bad)


@pytest.mark.parametrize("c,n_chunks", CHUNK_CASES, ids=lambda v: v.id if isinstance(v, Case) else f"{v}chunks")
def test_chunk_boundaries(cuda, monkeypatch, c, n_chunks):
    """The bucket-chunk loops of the forward and backward and sce_collect_kernel's per-chunk winner lookup, with exactly tied
    buckets on both sides of a chunk boundary; one case chunks at the default 256 MiB budget."""
    if c.per_chunk:
        monkeypatch.setenv("RP_SCE_CHUNK_BYTES", str(c.budget()))
    else:
        monkeypatch.delenv("RP_SCE_CHUNK_BYTES", raising=False)
    assert c.chunks() == n_chunks
    per = buckets_per_chunk(c.d, c.bsx, c.bsy, c.nb, c.budget() or DEFAULT_CHUNK_BYTES)
    assert any(b // per != grp[0] // per for grp in c.dup for b in grp), "no tied group straddles a chunk boundary"
    print(f"\n{c.id}: {per} buckets per chunk, {n_chunks} chunks")
    x = make_inputs(c, cuda)
    ws = workspace(c, cuda)
    out = run(c, x, ws)
    r, err, bad = _full_check(c, x, out)
    if _tied_rows(r) == 0:
        bad.append("no exactly tied row")
    _note("tied rows (info)", _tied_rows(r))
    assert_within(c, err, bad)
    if c.per_chunk:   # the same head in one chunk: selections and loss bit for bit, d_hc to the tolerance
        monkeypatch.delenv("RP_SCE_CHUNK_BYTES")
        one = run(c, x, workspace(c, cuda))
        for k in ("loss", "top_x", "score_x", "top_y"):
            assert torch.equal(one[k], out[k]), k
        assert torch.equal(one["d_hc"], out["d_hc"])


def test_no_counted_row(cuda):
    """One item, every label equal to it: every bucket CE is exactly 0 - loss NaN, loss_out[1] 0, d_hc exactly 0."""
    c = Case(64, False, 100, 100, 3, 8, 1, n_items=1)
    x = make_inputs(c, cuda)
    x["labels"].zero_()
    x["pad"].fill_(1)
    out = run(c, x, workspace(c, cuda))
    assert math.isnan(float(out["loss"][0])) and float(out["loss"][1]) == 0.0
    assert bool((out["d_hc"][: c.cap] == 0).all()) and bool((out["d_hc"][c.cap:] == SENT).all())
    err, bad = {}, []
    check_loss_and_grad(c, x, out, err, bad)
    assert not bad, bad


# ----------------------------------------------------------------------------------------------------------------------
# contracts
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mix", [False, True])
def test_stages_equal_one_call(cuda, mix):
    """DRAW, SELECT_X, SELECT_Y and BUCKET_CE as four calls equal one RP_SCE_ALL call bit for bit, and so do the gradients."""
    c = Case(128, True, 700, 650, 16, 100, 200, mix=mix)
    x = make_inputs(c, cuda)
    ws = workspace(c, cuda)
    a = run(c, x, ws)
    draw_a = x["draw"].clone()
    b = new_out(c, cuda)
    x["draw"].zero_()
    for st in (SCE_DRAW, SCE_SELECT_X, SCE_SELECT_Y, SCE_BUCKET_CE):
        fwd(c, x, ws, b, st)
    bwd(c, x, ws, b)
    assert torch.equal(x["draw"][:-1], draw_a[:-1])
    for k in ("loss", "top_x", "score_x", "top_y", "d_hc"):
        assert torch.equal(a[k], b[k]), k


def test_workspace_reuse_with_a_smaller_batch(cuda):
    """A full batch, then one with fewer rows and other labels on the same workspace, equals the second batch on a fresh
    workspace (maxkey / cnt / win, dacc and the loss ticket are reset by every call)."""
    c = Case(128, False, 900, 900, 32, 128, 128, dup=((3, 4),))
    x = make_inputs(c, cuda)
    ws = workspace(c, cuda)
    run(c, x, ws)
    small = Case(128, False, 900, 500, 32, 128, 128, dup=((3, 4),))
    x["n_rows"].fill_(500)
    x["labels"].copy_(torch.randint(0, N_ITEMS, (c.cap,), generator=torch.Generator().manual_seed(1)).to(cuda))
    reused = run(small, x, ws)
    fresh = run(small, x, workspace(small, cuda))
    for k in ("loss", "top_x", "score_x", "top_y", "d_hc"):
        assert torch.equal(reused[k], fresh[k]), k
    r, err, bad = _full_check(small, x, reused)
    assert_within(small, err, bad)
