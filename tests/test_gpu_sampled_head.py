"""The sampled training heads (csrc/rp_sampled_head.cu: rp_sampled_head_fwd / rp_sampled_head_bwd) called through the C ABI,
each case against the float64 reference of tests/sampled_reference.py computed from the same bf16 inputs.

Layout as SasRecEngine._sampled_desc passes it: hc bf16 [capacity, d] holds the compacted valid targets in its first
n_valid rows (the rows after them hold finite garbage, which the head must ignore), table bf16 [n_items + 1, d] (the pad
row last), labels int32 [capacity], valid_idx int32 = ascending flat b * L + l positions, negatives int64 [N] (shared),
[B * L, N] (per position) or [B, N] (per sequence).  d_hc has 64 sentinel rows past capacity, and d_table starts from a
non-zero pattern: the head accumulates into it.

Case matrix: the four loss kinds x three negative layouts at d = 128; CE and BCE at d = 64, 256 and 512 in every layout; a
legacy case at d = 512.  capacity 300 (not a multiple of 64), 1200 (config 2: B 6 x L 200) and 4133; n_valid 0, 1, 127,
128, 129, capacity - 10 and capacity.  Shared N 1 ... 2048 crosses the forward's N tiles, the 64-wide K chunks of dH and
the 128-row M tiles of dE_neg; per-row N 1, 31, 33, 100 crosses the 32-lane loops.  Negative lists hold collisions with
the positive (in some rows only), duplicates, the ignore index (an item id, or the pad id n_items) and, for legacy CE,
rows where all but one negative is rejected.  BCE cases with log_eps 1e-3 / clamp 5.5 and logits of about +-20 make both
clamps fire.  Run with -s to print the worst error of each family.
"""
import ctypes
import math
from dataclasses import dataclass

import pytest
import torch

import sampled_reference as sr
from fp64_checks import WorstErrors, block_err, ulp_err
from replay_b200._lib import SampledDesc, check, lib

pytestmark = pytest.mark.gpu

SENT = -3.25                 # sentinel for d_hc memory the head must not write (exact in bf16)
N_ITEMS = 5000
KINDS = {"ce": sr.CE_SAMPLED, "bce": sr.BCE_SAMPLED, "lce": sr.LEGACY_CE, "lbce": sr.LEGACY_BCE}
MODES = {"shared": 0, "perpos": 1, "perseq": 2}

# d_hc is compared element-wise in half-ulp units of bf16 (ulp_err; rounding to nearest alone gives 1) with an absolute
# slack of SLACK x sum_j |dz_j| |E_j|: per-row negatives accumulate in fp32 (SLACK_ROW), shared negatives pass dz through
# bf16 into the tensor cores and round the GEMM's output to bf16 before the positive's term is added (SLACK_SHARED).
# d_table is compared element-wise as |got - preset - ref| / (sum_t |dz_t| |h_t| + |preset|): fp32 atomics onto the preset,
# and in shared mode the bf16 dz of the dE_neg GEMM.
# Tolerances: about 3x the worst error observed over every case of this file on one H100 80GB HBM3 (700 W power limit).
SLACK_ROW = 2.0 ** -16
SLACK_SHARED = 2.0 ** -8
TOL_LOSS = 2e-6              # relative loss error (floor 1e-3); worst seen 6.3e-7
TOL_HC_ULP_ROW = 3.0         # d_hc, per-row negatives, half-ulp units; worst seen 1.0
TOL_HC_ULP_SHARED = 4.0      # d_hc, shared negatives, half-ulp units with the bf16-dz slack; worst seen 1.3
TOL_HC_BLOCK_ROW = 5e-3      # d_hc per 64-row block norm-relative, per-row negatives; worst seen 1.7e-3
TOL_HC_BLOCK_SHARED = 8.5e-3 # d_hc per 64-row block norm-relative, shared negatives; worst seen 2.8e-3
TOL_TABLE_ROW = 7.5e-4       # d_table element-wise relative to its magnitude, per-row negatives; worst seen 2.5e-4 (BCE:
                             #   fp32 1 - sigmoid(z) of a large positive logit)
TOL_TABLE_SHARED = 9e-3      # d_table element-wise relative to its magnitude, shared negatives; worst seen 3.0e-3

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


@dataclass
class Case:
    kind: str
    mode: str
    d: int
    cap: int
    nv: int
    N: int
    L: int = 200
    ignore: str = "item"      # "item": an ordinary id, "pad": n_items, "none": -100
    scale: float = 2.0        # std of the logits
    log_eps: float = 1e-6
    clamp: float = 100.0
    vocab: int = N_ITEMS      # legacy CE's vocab_size
    reject_all: bool = True   # legacy CE: one row where all negatives but one are rejected

    @property
    def id(self):
        s = f"{self.kind}-{self.mode}-d{self.d}-cap{self.cap}-nv{self.nv}-N{self.N}"
        if self.mode == "perseq" or self.mode == "perpos":
            s += f"-L{self.L}"
        s += f"-{self.ignore}"
        if self.clamp != 100.0:
            s += "-clamp"
        if self.vocab != N_ITEMS:
            s += f"-V{self.vocab}"
        return s


CASES = [
    # the four kinds x three layouts at d = 128
    Case("ce", "shared", 128, 1200, 1200, 1000),
    Case("ce", "perpos", 128, 1200, 1190, 100, ignore="pad"),
    Case("ce", "perseq", 128, 1200, 129, 33, L=50),
    Case("bce", "shared", 128, 1200, 127, 257),
    Case("bce", "perpos", 128, 1200, 128, 31, ignore="none"),
    Case("bce", "perseq", 128, 1200, 1200, 100, ignore="pad"),
    Case("lce", "shared", 128, 1200, 1, 65),
    Case("lce", "perpos", 128, 1200, 1200, 100, ignore="none"),
    Case("lce", "perseq", 128, 1200, 1190, 31, L=50),
    Case("lbce", "shared", 128, 1200, 1190, 2048, ignore="none"),
    Case("lbce", "perpos", 128, 1200, 129, 1),
    Case("lbce", "perseq", 128, 1200, 1200, 33, L=50, ignore="none"),
    # CE and BCE at d = 64, 256, 512 in every layout
    Case("ce", "shared", 64, 300, 290, 7),
    Case("ce", "perpos", 64, 300, 300, 33, L=50),
    Case("ce", "perseq", 64, 4133, 4133, 100, ignore="pad"),
    Case("bce", "shared", 64, 4133, 4123, 8, ignore="pad"),
    Case("bce", "perpos", 64, 300, 1, 100, L=50, ignore="none"),
    Case("bce", "perseq", 64, 300, 129, 31, L=50),
    Case("ce", "shared", 256, 4133, 4133, 129),
    Case("ce", "perpos", 256, 1200, 128, 31, ignore="none"),
    Case("ce", "perseq", 256, 300, 290, 1, L=50, ignore="none"),
    Case("bce", "shared", 256, 300, 129, 64, ignore="none"),
    Case("bce", "perpos", 256, 4133, 4123, 100, L=50, ignore="pad"),
    Case("bce", "perseq", 256, 1200, 127, 33),
    Case("ce", "shared", 512, 1200, 1200, 2048, ignore="pad"),
    Case("ce", "perpos", 512, 4133, 4133, 100, L=50),
    Case("ce", "perseq", 512, 300, 300, 33, L=50, ignore="none"),
    Case("bce", "shared", 512, 4133, 129, 1000),
    Case("bce", "perpos", 512, 300, 290, 31, L=50),
    Case("bce", "perseq", 512, 4133, 4123, 100, ignore="pad"),
    Case("lce", "perpos", 512, 1200, 1190, 100),
    # edges: no valid row, one shared negative, more negatives than legacy CE's vocabulary
    Case("ce", "shared", 128, 300, 0, 65),
    Case("bce", "perpos", 128, 300, 0, 31, L=50),
    Case("ce", "shared", 64, 1200, 1200, 1),
    Case("lce", "perpos", 128, 1200, 1200, 100, vocab=60, reject_all=False),
    # BCE clamps: both the positive and the negative terms leave (-5.5, 5.5)
    Case("bce", "shared", 128, 1200, 1200, 257, scale=8.0, log_eps=1e-3, clamp=5.5),
    Case("bce", "perpos", 128, 1200, 1190, 100, scale=8.0, log_eps=1e-3, clamp=5.5),
    Case("lbce", "perpos", 64, 300, 300, 33, L=50, scale=8.0, log_eps=1e-3, clamp=5.5),
]


# ----------------------------------------------------------------------------------------------------------------------
# inputs and calls
# ----------------------------------------------------------------------------------------------------------------------
def make_inputs(c: Case, dev, seed=0):
    g = torch.Generator().manual_seed(seed * 7919 + c.d * 131 + c.cap + c.nv * 3 + c.N)
    d, cap, nv, N, L, I = c.d, c.cap, c.nv, c.N, c.L, N_ITEMS
    B = -(-cap // L)
    table = torch.randn(I + 1, d, generator=g) * (c.scale / math.sqrt(d))
    hc = torch.randn(cap, d, generator=g)
    hc[nv:] *= 8.0                                    # rows past n_valid: finite garbage the head must ignore
    labels = torch.randint(0, I, (cap,), generator=g)
    valid_idx = torch.zeros(cap, dtype=torch.int64)
    valid_idx[:nv] = torch.randperm(B * L, generator=g)[:nv].sort().values
    rows = {"shared": 1, "perpos": B * L, "perseq": B}[c.mode]
    neg = torch.randint(0, I, (rows, N), generator=g)
    ign = {"item": 17, "pad": I, "none": -100}[c.ignore]
    t = torch.arange(nv)
    if N >= 2:
        neg[:, 1] = neg[:, 0]                         # duplicates: their gradient counts twice
    if c.mode == "shared":
        c0 = int(neg[0, N // 2])
        labels[t[t % 3 == 1]] = c0                    # collisions with the positive in a third of the rows
        if ign >= 0 and N >= 3:
            neg[0, N - 1] = ign
    else:
        r = valid_idx[:nv] if c.mode == "perpos" else valid_idx[:nv] // L
        sel = t % 5 == 0
        neg[r[sel], t[sel] % N] = labels[:nv][sel]    # collisions at every column, the last one included
        if ign >= 0:
            sel = t % 7 == 3
            neg[r[sel], (N - 1 - t[sel]) % N] = ign
        if c.kind == "lce" and c.reject_all and nv > 2 and N >= 2:
            neg[r[2]] = labels[2]                     # all but one negative rejected
            neg[r[2], N // 2] = (labels[2] + 1) % I
    if c.clamp != 100.0 and c.mode == "perpos" and nv >= 2:
        # two rows whose every term is clamped: z_pos = -10, z_neg = +10 -> their d_hc rows are exactly zero
        table[1], table[2] = -0.5, 0.5
        for tt in (0, nv - 1):
            hc[tt] = 20.0 / d
            labels[tt] = 1
            neg[valid_idx[tt]] = 2
    if c.kind in ("lce", "lbce") and c.ignore == "pad":
        raise ValueError("the legacy kinds do not mask: a pad-id negative would score row 0")
    return dict(hc=hc.to(torch.bfloat16).to(dev), table=table.to(torch.bfloat16).to(dev),
                labels=labels.to(torch.int32).to(dev), valid_idx=valid_idx.to(torch.int32).to(dev),
                neg=neg.reshape(-1).contiguous().to(dev) if c.mode == "shared" else neg.to(dev),
                nv=torch.tensor([nv], dtype=torch.int32, device=dev), ignore_index=ign)


def workspace(c: Case, dev, fill=0):
    n = lib().rp_sampled_head_workspace(c.cap, c.d, c.N, MODES[c.mode])
    assert n > 0
    return torch.full((n,), fill, dtype=torch.uint8, device=dev)


def preset_table(c: Case, dev):
    """Non-zero fp32 pattern (exact, positive, ~1e-6) that d_table accumulates onto."""
    k = torch.arange((N_ITEMS + 1) * c.d, device=dev).reshape(N_ITEMS + 1, c.d)
    return ((k % 7) + 1).float() * 2.0 ** -20


def run(c: Case, x, ws, nv=None):
    """fwd + bwd -> (loss_out [2], d_hc [cap + 64, d] with sentinel rows, d_table [n_items + 1, d], preset)."""
    dev = ws.device
    if nv is not None:
        x["nv"].fill_(nv)
    sd = SampledDesc()
    sd.hc, sd.table, sd.labels = x["hc"].data_ptr(), x["table"].data_ptr(), x["labels"].data_ptr()
    sd.valid_idx, sd.negatives, sd.n_valid = x["valid_idx"].data_ptr(), x["neg"].data_ptr(), x["nv"].data_ptr()
    sd.capacity, sd.n_items, sd.d, sd.n_neg, sd.neg_mode, sd.seq_len = c.cap, N_ITEMS, c.d, c.N, MODES[c.mode], c.L
    sd.kind, sd.ignore_index, sd.vocab_size = KINDS[c.kind], x["ignore_index"], c.vocab
    sd.log_eps, sd.clamp = c.log_eps, c.clamp
    loss = torch.full((2,), float("nan"), dtype=torch.float32, device=dev)
    sd.loss_out = loss.data_ptr()
    sd.workspace, sd.workspace_bytes = ws.data_ptr(), ws.numel()
    d_hc = torch.full((c.cap + 64, c.d), SENT, dtype=torch.bfloat16, device=dev)
    preset = preset_table(c, dev)
    d_table = preset.clone()
    st = torch.cuda.current_stream().cuda_stream
    L = lib()
    check(L.rp_sampled_head_fwd(ctypes.byref(sd), st), "rp_sampled_head_fwd")
    check(L.rp_sampled_head_bwd(ctypes.byref(sd), d_hc.data_ptr(), d_table.data_ptr(), st), "rp_sampled_head_bwd")
    torch.cuda.synchronize()
    return loss, d_hc, d_table, preset


def reference(c: Case, x):
    return sr.reference(x["hc"], x["table"], x["labels"], x["valid_idx"], x["neg"], int(x["nv"][0]), KINDS[c.kind],
                        MODES[c.mode], L=c.L, ignore_index=x["ignore_index"], vocab_size=c.vocab, log_eps=c.log_eps,
                        clamp=c.clamp)


# ----------------------------------------------------------------------------------------------------------------------
# checks
# ----------------------------------------------------------------------------------------------------------------------
def errors(c: Case, nv, out, ref):
    """Every measured error of one call, and the list of exact properties that failed."""
    loss, d_hc, d_table, preset = out
    shared = c.mode == "shared"
    fam = "shared" if shared else "row"
    bad = []
    err = {}
    if not (torch.isfinite(loss).all() and torch.isfinite(d_hc.float()).all() and torch.isfinite(d_table).all()):
        bad.append("NaN / Inf in loss_out, d_hc or d_table")
    inv = torch.tensor(1.0, dtype=torch.float32) / nv if nv else torch.tensor(0.0)
    if float(loss[1]) != float(inv):
        bad.append(f"loss_out[1] = {float(loss[1])!r}, expected float32(1 / n_valid) = {float(inv)!r}")
    if nv == 0 and float(loss[0]) != 0.0:
        bad.append(f"loss_out[0] = {float(loss[0])} with no valid row")
    err["loss"] = abs(float(loss[0]) - float(ref["loss"])) / max(abs(float(ref["loss"])), 1e-3)
    # d_hc: rows < n_valid against the reference; the rest of the buffer as documented in include/rp_b200.h
    tail = d_hc[nv:].float()
    if shared:
        z_end = min(_ru(nv, 128), c.cap)
        if not (tail[: z_end - nv] == 0).all():
            bad.append(f"shared: d_hc rows [{nv}, {z_end}) are not zero")
        if not (tail[z_end - nv:] == SENT).all():
            bad.append(f"shared: d_hc rows >= {z_end} were written")
    elif not (tail == SENT).all():
        bad.append(f"d_hc rows >= n_valid = {nv} were written")
    if nv:
        got = d_hc[:nv].double()
        slack = (SLACK_SHARED if shared else SLACK_ROW) * ref["mag_hc"] + ref["edge_hc"] + 1e-30
        err[f"d_hc ulp ({fam})"] = ulp_err(got, ref["d_hc"], slack)
        gap = got - ref["d_hc"]
        gap = gap.sign() * (gap.abs() - ref["edge_hc"]).clamp_min(0)    # less what the BCE clamp's edge allows
        err[f"d_hc block ({fam})"] = block_err(ref["d_hc"] + gap, ref["d_hc"])
    # d_table: preset + gradient; rows nobody references (and the pad row) bit for bit the preset
    untouched = ~ref["referenced"]
    if not torch.equal(d_table[untouched], preset[untouched]):
        n = int((d_table[untouched] != preset[untouched]).any(1).sum())
        bad.append(f"{n} table rows that no positive or live negative references were changed")
    if not torch.equal(d_table[-1], preset[-1]):
        bad.append("the pad row of d_table was changed")
    diff = ((d_table.double() - preset.double() - ref["d_table"]).abs() - ref["edge_table"]).clamp_min(0)
    err[f"d_table ({fam})"] = float((diff / (ref["mag_table"] + preset.double())).max())
    return err, bad


def assert_within(c: Case, err, bad):
    shared = c.mode == "shared"
    tol = {"loss": TOL_LOSS,
           "d_hc ulp (row)": TOL_HC_ULP_ROW, "d_hc ulp (shared)": TOL_HC_ULP_SHARED,
           "d_hc block (row)": TOL_HC_BLOCK_ROW, "d_hc block (shared)": TOL_HC_BLOCK_SHARED,
           "d_table (row)": TOL_TABLE_ROW, "d_table (shared)": TOL_TABLE_SHARED}
    over = {k: v for k, v in err.items() if v > tol[k]}
    assert not bad and not over, (c.id, "shared" if shared else "per-row", bad, over)


# ----------------------------------------------------------------------------------------------------------------------
# tests
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", CASES, ids=lambda c: c.id)
def test_sampled_head_matches_fp64(cuda, c):
    x = make_inputs(c, cuda)
    ws = workspace(c, cuda)
    out = run(c, x, ws)
    ref = reference(c, x)
    err, bad = errors(c, c.nv, out, ref)
    for k, v in err.items():
        _note(k, v)
    # a second identical call on the same workspace: loss and d_hc bit for bit; d_table (fp32 atomics) to tolerance
    out2 = run(c, x, ws)
    if not (torch.equal(out2[0], out[0]) and torch.equal(out2[1], out[1])):
        bad.append("a second identical call gave a different loss or d_hc")
    t_gap = float(((out2[2].double() - out[2].double()).abs() / (ref["mag_table"] + out[3].double())).max())
    _note("d_table run-to-run", t_gap)
    if t_gap > (TOL_TABLE_SHARED if c.mode == "shared" else TOL_TABLE_ROW):
        bad.append(f"d_table differs between two identical calls by {t_gap:.3g}")
    if c.clamp != 100.0 and c.mode == "perpos" and c.nv >= 2:
        # rows whose every term is clamped: the clamp's gradient is exactly zero
        for tt in (0, c.nv - 1):
            if not (out[1][tt].float() == 0).all():
                bad.append(f"d_hc row {tt}, all of whose terms are clamped, is not zero")
    assert_within(c, err, bad)


@pytest.mark.parametrize("nv", [290, 300])
def test_shared_negatives_ignore_stale_workspace(cuda, nv):
    """The workspace starts as 0xFF bytes (NaN in fp32 and bf16): whatever the head reads must be written first.  capacity
    300 is not a multiple of 64, so the dE_neg GEMM's last 64-row K chunk reaches past the capacity into the bf16 dz rows."""
    c = Case("ce", "shared", 128, 300, nv, 65)
    x = make_inputs(c, cuda)
    out = run(c, x, workspace(c, cuda, fill=0xFF))
    err, bad = errors(c, nv, out, reference(c, x))
    for k, v in err.items():
        _note(k, v)
    assert_within(c, err, bad)
    fresh = run(c, x, workspace(c, cuda))
    assert torch.equal(out[0], fresh[0]) and torch.equal(out[1], fresh[1])


@pytest.mark.parametrize("mode", ["shared", "perpos"])
def test_workspace_reuse_after_larger_call(cuda, mode):
    """A call with many valid rows, then one with few on the same workspace, must equal the small call on a fresh one."""
    c = Case("bce", mode, 128, 1200, 129, 100)
    x = make_inputs(c, cuda)
    ws = workspace(c, cuda)
    run(c, x, ws, nv=1200)
    small = run(c, x, ws, nv=129)
    fresh = run(c, x, workspace(c, cuda), nv=129)
    assert torch.equal(small[0], fresh[0]) and torch.equal(small[1], fresh[1])
    err, bad = errors(c, 129, small, reference(c, x))
    assert_within(c, err, bad)
