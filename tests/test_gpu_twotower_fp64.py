"""TwoTower's own device code against float64 (tests/twotower_reference.py):

1. rp_tower_compact through the C ABI, exactly, against the host restatement: catalogs around the 4096-item scan tile up
   to 1 052 673 items (258 tiles, where a thread of tile_assign_kernel first sums two earlier tiles), candidates on every
   tile's first and last item, on 16-item thread boundaries, with empty tiles between populated ones and one tile fully
   flagged; the three negative layouts, ignore_index in and out of the catalog, ids outside it, duplicates, negatives equal
   to positives; every entry the kernels must not read holds an id that would open a new slot; the gathered rows bit for
   bit, the rows from n_slots to cap zero, the row buffer untouched without rows; a reused workspace.  Then the engine's
   own compaction (TwoTowerEngine._compact) at the config-2 and config-5 sampled setups.
2. rp_tower_scatter_rows, exactly: identity and slot-mapped modes, NaN rows past n_slots, a device n_slots past n_rows.
3. The item tower stage by stage, per element, on the engine's own bf16 inputs to each stage (GL, U, z, the norm output;
   dz, dU, dGL, dx; dW by 64-row block, db, d norm), at 1 .. 50 000 rows and d 50 .. 512; the rule that rows past the
   slots are skipped by the forward and add exactly zero in the backward, with large finite garbage in those rows; the
   inference table in several passes.
4. TwoTowerEngine's training step against float64 autograd of the restatement on the engine's parameters: every loss kind
   at the config-2 shape, the full batch, dropout, and a config-5 sampled step.

Tolerances, as max |got - ref| / bound (per-element families) or the largest 64-row block's norm-relative error (block
families).  The worst values seen over every case of this file on one H100 80GB HBM3 at a 700 W power limit (run with -s)
are in the comments; each tolerance is about 3x its worst value, or 1.0 for the per-element bounds.  On that card the whole
file runs in about 35 s with a peak of 35 GiB allocated (the config-5 step and its float64 reference).

Not covered here: the side-feature item tower (tests/test_gpu_twotower_side_features.py).  The bias gradients are reduced
with fp32 atomics (rp_colsum_multi), so two runs agree on them to rounding only; every other tower gradient is bitwise
reproducible and is checked so."""
import math

import numpy as np
import pytest
import torch

import diff_reference as dr
import sampled_ext_reference as sx
import sampled_reference as sr
import twotower_reference as tr
from fp64_checks import WorstErrors, block_err
from sasrec_fp64 import P_DROP, SEED, _bf, _map, engine_keeps, engine_view, sasrec_body_ref, step_batch

pytestmark = pytest.mark.gpu

NAN = float("nan")

TOL_STAGE = 1.0        # per-element stage bounds: GL 0.999, z 0.998, dU 0.995, dx 0.998 (GEMM); U 1.0, dGL 1.0 (SwiGLU);
                       # out 1.0, dz 1.0, d norm 0.012 (RMSNorm)
TOL_WGRAD = 6e-5       # dW by 64-row block 2.0e-5, db 5.6e-7: fp32 split-K / column sums of bf16 products
TOL_CHAIN = 2e-2       # the whole tower from fp64 parameters, gradients by 64-row block: 6.6e-3
TOL_OUT = 17.0         # the tower's output against the fp64 chain, in (half bf16 ulp + 2^-8 row RMS) units: 5.7
TOL_LOSS = 1.2e-3      # step loss, relative: 4.0e-4
TOL_HID = 1.7e-2       # step: compacted hidden rows by 64-row block: 5.7e-3
TOL_GRAD = 0.55        # step: every parameter gradient by 64-row block: 0.18 (item_emb, bce_sampled shared), 0.14
                       # (item_emb, bce); body parameters 0.06 or less at config 2
TOL_BIAS_RERUN = 1e-5  # rerun difference of the [bg; b1] / b2 gradients, relative to their largest entry: 3.1e-7
TOL_GRAD_C5 = 0.7      # the config-5 step, as above: 0.23 (b0.ln1_w); cf. test_gpu_config5_fp64.py's 0.25 for SASRec

_worst = WorstErrors()
_note = _worst.note


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    _worst.report()
    if torch.cuda.is_available():
        print(f"  peak device memory allocated: {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda")


def _bits(x):
    return x.contiguous().view(torch.int16 if x.element_size() == 2 else torch.int32 if x.element_size() == 4 else
                               torch.int64)


def _lib():
    from replay_b200._lib import lib

    return lib()


def _check(rc, name):
    from replay_b200._lib import check

    check(rc, name)


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ================================================================================================ 1. compaction
def _edge_items(n, rng):
    """first and last item of every tile, a 16-item thread boundary in each, every third tile empty (not the last), one
    tile fully flagged (the second, or the only one), item 0 and n - 1"""
    tiles = -(-n // tr.TILE)
    S = {0, n - 1}
    for t in range(tiles):
        if t % 3 == 2 and t != tiles - 1:
            continue
        a, b = t * tr.TILE, min(n, (t + 1) * tr.TILE) - 1
        S |= {a, b}
        k = a + tr.PER_THREAD * int(rng.integers(1, tr.TILE // tr.PER_THREAD))
        if k < n:
            S |= {k - 1, k}
    full = 1 if tiles > 2 else 0
    S |= set(range(full * tr.TILE, min(n, (full + 1) * tr.TILE)))
    return np.array(sorted(S), dtype=np.int64)


def make_case(n_items, S, mode, n_neg, nv_kind, ignore, seed, L=8):
    """Compaction inputs that put the items S (as far as the read entries hold them), ignored ids, ids outside the
    catalog, duplicates and positives among the negatives into the entries the kernels read, and an id that would open a
    new slot into every entry they must not read (labels past n_valid, per-position rows of positions that are not
    valid).  nv_kind: "zero", "one", "part" (labels past n_valid exist) or "all"."""
    rng = np.random.default_rng(seed)
    S = rng.permutation(np.unique(np.asarray(S, np.int64)))
    K = S.size
    special = np.array([ignore if ignore >= 0 else 7, -1, n_items, 1 << 40], dtype=np.int64)
    if mode == 1:
        nv = {"zero": 0, "one": 1}.get(nv_kind, max(1, -(-K // (n_neg // 2 + 1))))
    else:
        rows = max(1, -(-K // 2 // n_neg)) if mode == 2 else 1
        read_neg = rows * n_neg
        nv = {"zero": 0, "one": 1}.get(nv_kind, max(1, K - read_neg + special.size + 2))
    T = nv if nv_kind == "all" else nv + 7
    T = max(T, 1)
    n_rows = {0: 1, 1: T, 2: rows if mode == 2 else 1}[mode]
    # poison: items outside S other than 0 and the ignore id (each would open a new slot)
    comp = np.setdiff1d(np.arange(n_items, dtype=np.int64), np.concatenate([S, [0, 7]]))
    poison = rng.choice(comp, size=min(comp.size, 4096), replace=False) if comp.size else np.array([0], np.int64)
    labels = rng.choice(poison, size=T).astype(np.int64)
    negatives = rng.choice(poison, size=(n_rows, n_neg)).astype(np.int64)
    perm = np.arange(T)
    if mode == 1:
        perm = rng.permutation(T)
    valid_idx = np.concatenate([np.sort(perm[:nv]), perm[nv:]]).astype(np.int64)
    _, idx = tr.read_entries(nv, T, negatives, n_neg, mode, valid_idx, n_rows)
    lab_vals = S[:nv] if nv <= K else np.concatenate([S, rng.choice(S, nv - K)]) if K else np.zeros(nv, np.int64)
    labels[:nv] = lab_vals[:nv] if lab_vals.size >= nv else np.resize(lab_vals, nv)
    rest = S[nv:]
    extra = [special]
    if nv:
        extra.append(labels[:1])                      # a negative equal to a positive
    if rest.size:
        extra.append(rest[:1])                        # a duplicate
    vals = np.concatenate([rest[:max(0, idx.size - sum(e.size for e in extra))]] + extra) if idx.size else rest[:0]
    if idx.size:
        if vals.size < idx.size:
            vals = np.concatenate([vals, rng.choice(S if K else np.array([1], np.int64), idx.size - vals.size)])
        flat = negatives.reshape(-1)
        flat[idx] = rng.permutation(vals[:idx.size])
    cap = min(n_items, T + {0: n_neg, 1: T * n_neg, 2: n_rows * n_neg}[mode])
    return dict(n_items=n_items, labels=labels, n_valid=nv, negatives=negatives, n_neg=n_neg, mode=mode,
                valid_idx=valid_idx, L=L, ignore=ignore, cap=cap, n_rows=n_rows)


def _alloc_out(cuda, c, d, rows=True):
    i32 = dict(dtype=torch.int32, device=cuda)
    return dict(ns=torch.full((1,), -7, **i32), ios=torch.full((c["cap"],), -7, **i32),
                lab=torch.full((len(c["labels"]),), -7, **i32),
                neg=torch.full(c["negatives"].shape, -7, dtype=torch.int64, device=cuda),
                rows=torch.full((c["cap"], d), 3.0, dtype=torch.bfloat16, device=cuda),
                ws=torch.full((_lib().rp_tower_compact_workspace(c["n_items"]),), 0x5A, dtype=torch.uint8, device=cuda),
                with_rows=rows)


def run_compact(cuda, c, table, out):
    L_ = _lib()
    lab = torch.as_tensor(c["labels"], dtype=torch.int32).to(cuda)
    nv = torch.tensor([c["n_valid"]], dtype=torch.int32, device=cuda)
    neg = torch.as_tensor(c["negatives"]).to(cuda)
    vi = torch.as_tensor(c["valid_idx"], dtype=torch.int32).to(cuda)
    _check(L_.rp_tower_compact(lab.data_ptr(), nv.data_ptr(), lab.numel(), neg.data_ptr(), c["n_neg"], c["mode"],
                               c["n_rows"], vi.data_ptr(), c["L"], c["ignore"], c["n_items"], table.data_ptr(),
                               table.shape[1], c["cap"], out["ns"].data_ptr(), out["ios"].data_ptr(), out["lab"].data_ptr(),
                               out["neg"].data_ptr(), out["rows"].data_ptr() if out["with_rows"] else None,
                               out["ws"].data_ptr(), out["ws"].numel(), _stream()), "rp_tower_compact")
    torch.cuda.synchronize()


def check_compact(c, table, out):
    ref = tr.compact_ref(c["n_items"], c["labels"], c["n_valid"], len(c["labels"]), c["negatives"], c["n_neg"], c["mode"],
                         c["valid_idx"], c["ignore"], c["cap"], c["n_rows"])
    ns = int(out["ns"])
    assert ns == ref["n_slots"], (ns, ref["n_slots"])
    ios = out["ios"].cpu().long().numpy()
    assert np.array_equal(ios, ref["item_of_slot"])                 # -1 from n_slots on
    lab = out["lab"].cpu().long().numpy()
    nv = ref["nv"]
    assert np.array_equal(lab[:nv], ref["labels_out"]) and (lab[nv:] == -7).all()
    neg = out["neg"].cpu().numpy().reshape(-1)
    written = np.zeros(neg.size, dtype=bool)
    written[ref["neg_idx"]] = True
    assert np.array_equal(neg[ref["neg_idx"]], ref["neg_out"]) and (neg[~written] == -7).all()
    rows = out["rows"]
    if out["with_rows"]:
        if ns:
            want = table[torch.from_numpy(ref["item_of_slot"][:ns]).to(rows.device)]
            assert torch.equal(_bits(rows[:ns]), _bits(want))
        assert not bool(_bits(rows[ns:]).any())
    else:
        assert torch.equal(_bits(rows), _bits(torch.full_like(rows, 3.0)))
    return ref


SIZES = (4095, 4096, 4097, 8192, 12289, 50000, 1000000, 1052673)
EDGE_CASES = [dict(n=n, mode=i % 3, n_neg=(1, 33, 256)[(i + 1) % 3], ignore=(7, -100)[i % 2], d=(64, 128, 256, 512)[i % 4])
              for i, n in enumerate(SIZES)]
EDGE_CASES += [dict(n=n, mode=(i + 1) % 3, n_neg=(33, 256, 1)[i % 3], ignore=(-100, 7)[i % 2], d=(512, 256, 128, 64)[i % 4])
               for i, n in enumerate(SIZES)]


@pytest.mark.parametrize("c", EDGE_CASES, ids=lambda c: f"n{c['n']}-mode{c['mode']}-neg{c['n_neg']}-ign{c['ignore']}-d{c['d']}")
def test_compaction_tile_edges(cuda, c):
    n = c["n"]
    if n == 1052673:
        assert -(-n // tr.TILE) == 258
    rng = np.random.default_rng(n + c["mode"])
    case = make_case(n, _edge_items(n, rng), c["mode"], c["n_neg"], "part", c["ignore"], seed=n + c["n_neg"])
    table = torch.randn(n + 1, c["d"], device=cuda).to(torch.bfloat16)
    out = _alloc_out(cuda, case, c["d"])
    run_compact(cuda, case, table, out)
    ref = check_compact(case, table, out)
    assert ref["n_slots"] > 0


NV_CASES = [dict(n=n, mode=m, n_neg=nn, nv=k, ignore=ig) for n, ig in ((12289, 7), (50000, -100)) for m in (0, 1, 2)
            for k, nn in (("zero", 33), ("one", 1), ("all", 256))]


@pytest.mark.parametrize("c", NV_CASES, ids=lambda c: f"n{c['n']}-mode{c['mode']}-neg{c['n_neg']}-nv_{c['nv']}-ign{c['ignore']}")
def test_compaction_valid_counts(cuda, c):
    """n_valid 0, 1 and capacity, candidates spread over every tile"""
    rng = np.random.default_rng(c["n"] + c["mode"])
    S = rng.choice(c["n"], size=300, replace=False)
    case = make_case(c["n"], S, c["mode"], c["n_neg"], c["nv"], c["ignore"], seed=c["mode"] * 7 + c["n_neg"])
    table = torch.randn(c["n"] + 1, 128, device=cuda).to(torch.bfloat16)
    out = _alloc_out(cuda, case, 128)
    run_compact(cuda, case, table, out)
    check_compact(case, table, out)


@pytest.mark.parametrize("which", ["every_item", "far_below_cap"])
def test_compaction_slot_count_edges(cuda, which):
    """n_slots equal to cap (every item of the catalog referenced, cap the whole catalog) and far below it (a few items
    repeated over many entries)"""
    if which == "every_item":
        n = 8193
        S = np.arange(n)
        case = make_case(n, S, 0, 256, "all", -100, seed=1)
        assert case["cap"] == n
    else:
        n = 50000
        S = np.array([5, 4095, 4096, 40000])
        case = make_case(n, np.resize(S, 4000), 1, 33, "part", 7, seed=2)
    table = torch.randn(n + 1, 64, device=cuda).to(torch.bfloat16)
    out = _alloc_out(cuda, case, 64)
    run_compact(cuda, case, table, out)
    ref = check_compact(case, table, out)
    if which == "every_item":
        assert ref["n_slots"] == case["cap"]
    else:
        assert ref["n_slots"] <= 8 and 30 * ref["n_slots"] < case["cap"]


def test_compaction_without_rows_and_reuse(cuda):
    """rows_out = None leaves the row buffer alone; one workspace and one set of outputs reused for a second call with
    fewer candidates keeps no stale slot or row; a rerun is bitwise equal"""
    n = 50000
    rng = np.random.default_rng(3)
    big = make_case(n, _edge_items(n, rng), 2, 33, "part", 7, seed=4)
    table = torch.randn(n + 1, 128, device=cuda).to(torch.bfloat16)
    out = _alloc_out(cuda, big, 128, rows=False)
    run_compact(cuda, big, table, out)
    check_compact(big, table, out)
    out["with_rows"] = True
    run_compact(cuda, big, table, out)
    check_compact(big, table, out)
    small = dict(big)
    small["negatives"] = big["negatives"].copy()
    small["negatives"][:] = 12
    small["n_valid"] = 3
    out["lab"].fill_(-7)
    out["neg"].fill_(-7)
    run_compact(cuda, small, table, out)
    ref = check_compact(small, table, out)
    assert ref["n_slots"] <= 4
    first = {k: v.clone() for k, v in out.items() if torch.is_tensor(v) and k != "ws"}
    run_compact(cuda, small, table, out)
    for k, v in first.items():
        assert torch.equal(_bits(v), _bits(out[k])), k


# ================================================================================================ 2. scatter
def run_scatter(dx, ios, ns_dev, n_rows, d, table):
    _check(_lib().rp_tower_scatter_rows(dx.data_ptr(), None if ios is None else ios.data_ptr(),
                                        None if ns_dev is None else ns_dev.data_ptr(), n_rows, d, table.data_ptr(),
                                        _stream()), "rp_tower_scatter_rows")
    torch.cuda.synchronize()


def _pattern(R, d, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    return (torch.randn(R, d, device=dev, generator=g) * 3).float()


@pytest.mark.parametrize("n_rows", [1, 50000, 1000000])
@pytest.mark.parametrize("d", [128, 512])
def test_scatter_identity(cuda, n_rows, d):
    """d_table[i] += dx[i] for i < n_rows: each element one fp32 add; the rows past n_rows unchanged"""
    table = _pattern(n_rows + 3, d, cuda, n_rows + d)
    g = torch.Generator(device=cuda).manual_seed(d)
    dx = torch.randn(n_rows + 3, d, device=cuda, generator=g).to(torch.bfloat16)
    dx[n_rows:] = NAN
    want = tr.scatter_ref(table, dx, None, None, n_rows)
    got = table.clone()
    run_scatter(dx, None, None, n_rows, d, got)
    assert torch.equal(_bits(got), _bits(want))


@pytest.mark.parametrize("which", ["below", "clamped"])
@pytest.mark.parametrize("d", [128, 512])
def test_scatter_slots(cuda, which, d):
    """slot-mapped: below - n_slots < n_rows with NaN dx rows past n_slots; clamped - a device n_slots past n_rows (the
    kernel reads n_rows slots); rows of items outside item_of_slot[:n] are bitwise unchanged"""
    n_items, n_rows = 50000, 20000
    g = torch.Generator().manual_seed(d)
    items = torch.randperm(n_items, generator=g)[:n_rows + 100].sort().values
    table = _pattern(n_items + 1, d, cuda, d)
    dx = torch.randn(n_rows + 100, d, generator=g).to(torch.bfloat16).to(cuda)
    ios = items.to(torch.int32).to(cuda)
    if which == "below":
        ns = 12345
        dx[ns:] = NAN
        ios[ns:n_rows] = -1
    else:
        ns = n_rows + 50
        dx[n_rows:] = NAN
    ns_dev = torch.tensor([ns], dtype=torch.int32, device=cuda)
    want = tr.scatter_ref(table, dx, ios, ns, n_rows)
    got = table.clone()
    run_scatter(dx, ios, ns_dev, n_rows, d, got)
    assert torch.equal(_bits(got), _bits(want))
    n = min(ns, n_rows)
    untouched = torch.ones(n_items + 1, dtype=torch.bool, device=cuda)
    untouched[ios[:n].long()] = False
    assert torch.equal(_bits(got[untouched]), _bits(table[untouched]))


# ================================================================================================ 3. the item tower
_HEADS = {50: 1, 64: 1, 128: 2, 256: 4, 320: 4, 512: 8}


def _tower_engine(cuda, n_items, d, seed, with_grad=True):
    from replay_b200.engine_twotower import TOWER_LAYERS, TwoTowerConfig, TwoTowerEngine

    cfg = TwoTowerConfig(n_items=n_items, d=d, n_heads=_HEADS[d], n_blocks=1, max_len=8)
    eng = TwoTowerEngine(cfg, 1, 8, cuda, seed=seed, with_grad=with_grad)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        eng.import_named("item_emb", tr.tower_input(n_items + 1, d, g))
        for p in TOWER_LAYERS:
            for k, s in (("wg", (2 * d, d)), ("w1", (2 * d, d)), ("w2", (d, 2 * d))):
                eng.import_named(p + k, torch.randn(s, generator=g) * math.sqrt(2.0 / (3 * d)))
            eng.import_named(p + "norm", 1 + 0.1 * torch.randn(d, generator=g))
            for k, s in (("bg", 2 * d), ("b1", 2 * d), ("b2", d)):
                scale = 1e-3 if (p, k) == ("tw0.", "b2") else 0.1
                eng.import_named(p + k, scale * torch.randn(s, generator=g))
    eng.refresh_shadow()
    eng.tower_valid = False
    return eng


def _layer_params(eng, p):
    F = eng.cfg.ffn_p
    return dict(WGW1=eng._span(eng.params16, p + "wg", p + "w1", 2 * F), bgb1=eng._span(eng.params, p + "bg", p + "b1", 1)[0],
                W2=eng.params16[p + "w2"], b2=eng.params[p + "b2"], norm=eng.params[p + "norm"])


def _fp64_params(eng, padded=True):
    """the tower's parameters as twotower_reference.tower takes them (float64 leaves), in the padded layout"""
    P = {}
    for p in ("tw0.", "tw1."):
        lp = _layer_params(eng, p)
        P.update({p + "wgw1": lp["WGW1"], p + "bgb1": lp["bgb1"], p + "w2": lp["W2"], p + "b2": lp["b2"],
                  p + "norm": lp["norm"]})
    return {k: v.detach().double().clone().requires_grad_(True) for k, v in P.items()}


def _masks(eng):
    """bool [dp] true model columns, bool [2F] true hidden entries of [G; L]"""
    cfg, dev = eng.cfg, eng.dev
    col = torch.zeros(cfg.dp, dtype=torch.bool, device=dev)
    col[cfg.feat_index(dev)] = True
    F = cfg.ffn_p
    hid = (torch.arange(2 * F, device=dev) % F) < 2 * cfg.d
    return col, hid


def _stage(family, got, ref_bound, mask=None):
    ref, bound = ref_bound
    r = _note(family, dr.ratio(got, ref, bound, mask))
    assert r <= TOL_STAGE, (family, r)


def check_fwd_stages(eng, p, x, lay, out, rows):
    lp = _layer_params(eng, p)
    F, dt = eng.cfg.ffn_p, eng.cfg.d
    ref = tr.block_fwd_stages(x, lp["WGW1"], lp["bgb1"], lp["W2"], lp["b2"], lay["GL"], lay["U"], lay["z"], lp["norm"], F,
                              dt, rows)
    col, hid = _masks(eng)
    _stage("fwd GL", lay["GL"][:rows], ref["GL"])
    _stage("fwd U", lay["U"][:rows], ref["U"])
    _stage("fwd z", lay["z"][:rows], ref["z"])
    _stage("fwd out", out[:rows], ref["out"])
    for t, m in ((lay["GL"], ~hid), (lay["U"], ~hid[:F]), (lay["z"], ~col), (out, ~col)):
        assert bool((t[:rows][:, m] == 0).all()), p   # padded columns exactly zero (either sign)


def check_bwd_stages(eng, p, dout, x, lay, dxbuf, rows):
    tw, G, F, dt = eng.tw, eng.grads, eng.cfg.ffn_p, eng.cfg.d
    lp = _layer_params(eng, p)
    ref = tr.block_bwd_stages(dout, x, lp["WGW1"], lp["W2"], lay["GL"], lay["U"], lay["z"], lp["norm"], tw["dz"], tw["dU"],
                              tw["dGL"], F, dt, rows)
    col, hid = _masks(eng)
    _stage("bwd dz", tw["dz"][:rows], ref["dz"])
    _stage("bwd dU", tw["dU"][:rows], ref["dU"])
    _stage("bwd dGL", tw["dGL"][:rows], ref["dGL"])
    _stage("bwd dx", dxbuf[:rows], ref["dx"])
    for t, m in ((tw["dz"], ~col), (tw["dU"], ~hid[:F]), (tw["dGL"], ~hid), (dxbuf, ~col)):
        assert bool((t[:rows][:, m] == 0).all()), p
    for fam, got, want in (("wgrad dW", G[p + "w2"], ref["dW2"]), ("wgrad dW", eng._span(G, p + "wg", p + "w1", 2 * F), ref["dWGW1"]),
                           ("wgrad db", G[p + "b2"].view(-1, 1), ref["db2"].view(-1, 1)),
                           ("wgrad db", eng._span(G, p + "bg", p + "b1", 1)[0].view(-1, 1), ref["dbgb1"].view(-1, 1))):
        e = _note(fam, block_err(got, want) if rows else float(got.abs().max()))
        assert e <= TOL_WGRAD, (p, fam, e)
    rb = ref["rms"]
    zero = torch.zeros_like(G[p + "norm"])
    _stage("bwd d norm", G[p + "norm"], (rb["dw"], dr.dw_bound(rb, zero)))


def _dY(eng, rows, seed):
    col, _ = _masks(eng)
    g = torch.Generator(device=eng.dev).manual_seed(seed)
    return torch.randn(rows, eng.cfg.dp, device=eng.dev, generator=g) * col


@pytest.mark.parametrize("rows", [1, 127, 128, 129, 4097, 50000])
@pytest.mark.parametrize("d", [50, 128, 256, 320, 512])
def test_item_tower_stages(cuda, rows, d):
    """each stage of both sub-blocks against fp64 on the engine's own bf16 inputs; d 50 pads 14 model and 28 hidden
    columns, 256 is the widest [bg; b1] colsum in one pair, 320 and 512 split it, 512 runs the group-512 RMSNorm"""
    eng = _tower_engine(cuda, rows, d, seed=rows + d)
    tw = eng._alloc_tower()
    (l0, l1), F = tw["layers"], eng.cfg.ffn_p
    x0 = eng.params16["item_emb"]
    out = tw["cache"]
    eng.tower_forward(x0, rows, out)
    torch.cuda.synchronize()
    check_fwd_stages(eng, "tw0.", x0, l0, tw["x1"], rows)
    check_fwd_stages(eng, "tw1.", tw["x1"], l1, out, rows)
    eng.g32.zero_()
    tw["dY"][:rows].copy_(_dY(eng, rows, d).to(torch.bfloat16))
    eng._swiglu_block_bwd("tw1.", tw["dY"], tw["x1"], l1["GL"], l1["U"], l1["z"], tw["dz"], tw["dU"], tw["dGL"], tw["dxa"],
                          rows, F)
    torch.cuda.synchronize()
    check_bwd_stages(eng, "tw1.", tw["dY"], tw["x1"], l1, tw["dxa"], rows)
    eng._swiglu_block_bwd("tw0.", tw["dxa"], x0[:rows], l0["GL"], l0["U"], l0["z"], tw["dz"], tw["dU"], tw["dGL"], tw["dxb"],
                          rows, F)
    torch.cuda.synchronize()
    check_bwd_stages(eng, "tw0.", tw["dxa"], x0, l0, tw["dxb"], rows)


def _out_err(got, ref):
    """max |got - ref| in units of half a bf16 ulp of ref plus 2^-8 of the row's RMS"""
    rms = ref.pow(2).mean(-1, keepdim=True).sqrt()
    return float(((got.double() - ref).abs() / (dr.bf16_bound(ref, 0 * ref) + 2.0 ** -8 * rms)).max()) if ref.numel() else 0.0


def _chain(eng, x0, rows, dY=None):
    """the fp64 tower on the engine's bf16 x0 rows and parameters: (out, {name: grad}, d x0)"""
    P = _fp64_params(eng)
    x = x0[:rows].double().clone().requires_grad_(True)
    y = tr.tower(x, P, eng.cfg.ffn_p, eng.cfg.d)
    if dY is None:
        return y.detach(), None, None
    y.backward(dY)
    return y.detach(), {k: v.grad for k, v in P.items()}, x.grad


def _engine_tower_grads(eng):
    G, F = eng.grads, eng.cfg.ffn_p
    out = {}
    for p in ("tw0.", "tw1."):
        out.update({p + "wgw1": eng._span(G, p + "wg", p + "w1", 2 * F), p + "bgb1": eng._span(G, p + "bg", p + "b1", 1)[0],
                    p + "w2": G[p + "w2"], p + "b2": G[p + "b2"], p + "norm": G[p + "norm"]})
    return out


@pytest.mark.parametrize("d,ns", [(128, 300), (128, 1), (320, 700), (512, 129)])
def test_rows_past_the_slots(cuda, d, ns):
    """tower_forward with n_rows_dev = n_slots < rows: x0 rows past n_slots are zero (as the gather leaves them), GL / U /
    z / x1 / out rows past them hold large finite garbage.  Output rows below n_slots equal a run over exactly n_slots
    rows bit for bit; the backward over every row with d(out) zero past n_slots leaves dx exactly zero there; the
    parameter gradients match the fp64 tower on the slots alone and do not change when the garbage does: bit for bit, but
    for the bias gradients, whose column sums (rp_colsum_multi) add per-CTA partials with fp32 atomics and so may differ in
    the last bits from run to run; a garbage row leaking into them would move them by orders of magnitude more"""
    R = 1000
    eng = _tower_engine(cuda, R, d, seed=d + ns)
    tw = eng._alloc_tower()
    (l0, l1), dp = tw["layers"], eng.cfg.dp
    x0 = torch.zeros(R, dp, dtype=torch.bfloat16, device=cuda)
    x0[:ns] = eng.params16["item_emb"][:ns]
    exact = torch.full((R, dp), NAN, dtype=torch.bfloat16, device=cuda)
    eng.tower_forward(x0, ns, exact)
    nsd = torch.tensor([ns], dtype=torch.int32, device=cuda)
    out = torch.empty(R, dp, dtype=torch.bfloat16, device=cuda)

    def poison(seed):
        g = torch.Generator(device=cuda).manual_seed(seed)
        for t in (l0["GL"], l0["U"], l0["z"], l1["GL"], l1["U"], l1["z"], tw["x1"], out):
            w = t[ns:]
            w.copy_((torch.rand(w.shape, device=cuda, generator=g) * 2 - 1) * 3000.0)

    dY = _dY(eng, R, ns)
    dY[ns:] = 0
    runs = []
    for seed in (1, 2):
        poison(seed)
        eng.tower_forward(x0, R, out, nsd)
        torch.cuda.synchronize()
        assert torch.equal(_bits(out[:ns]), _bits(exact[:ns]))
        tw["dY32"].copy_(dY)
        eng.g32.zero_()
        eng.tower_backward(x0, R)
        torch.cuda.synchronize()
        assert bool((tw["dxb"][ns:] == 0).all())
        runs.append(({k: v.clone() for k, v in _engine_tower_grads(eng).items()}, tw["dxb"][:ns].clone()))
    for k, a in runs[0][0].items():
        b = runs[1][0][k]
        if k.endswith(("bgb1", "b2")):   # rp_colsum_multi adds its per-CTA partials with fp32 atomics
            e = _note("rerun bias grads", float((a - b).abs().max() / a.abs().max()))
            assert e <= TOL_BIAS_RERUN, (k, e)
        else:
            assert torch.equal(a, b), k
    assert torch.equal(_bits(runs[0][1]), _bits(runs[1][1]))
    y, G, dx = _chain(eng, x0, ns, dY[:ns].to(torch.bfloat16).double())
    assert _note("chain out", _out_err(out[:ns], y)) <= TOL_OUT
    for k, g in _engine_tower_grads(eng).items():
        e = _note("chain grads", block_err(g.reshape(g.shape[0], -1), G[k].reshape(g.shape[0], -1)))
        assert e <= TOL_CHAIN, (k, e)
    assert _note("chain grads", block_err(tw["dxb"][:ns], dx)) <= TOL_CHAIN


def test_inference_table(cuda):
    """tower_table() of an engine without gradients over 150 000 items: three passes of INFER_ROWS, the last short, each
    element against the fp64 tower"""
    n, d = 150000, 128
    eng = _tower_engine(cuda, n, d, seed=9, with_grad=False)
    assert eng.INFER_ROWS < n < 3 * eng.INFER_ROWS and n % eng.INFER_ROWS
    tab = eng.tower_table()
    torch.cuda.synchronize()
    y, _, _ = _chain(eng, eng.params16["item_emb"], n)
    assert _note("infer out", _out_err(tab, y)) <= TOL_OUT
    col, _ = _masks(eng)
    assert bool((tab[:, ~col] == 0).all())


# ================================================================================================ 4. the training step
def _tower_true(d, seed):
    """the tower's parameters at their true shapes, matrices bf16-exact"""
    g = torch.Generator().manual_seed(seed)
    P = {}
    for p in ("tw0.", "tw1."):
        for k, s in (("wg", (2 * d, d)), ("w1", (2 * d, d)), ("w2", (d, 2 * d))):
            P[p + k] = _bf(torch.randn(s, generator=g) * math.sqrt(2.0 / (3 * d))).float()
        P[p + "bg"], P[p + "b1"] = 0.1 * torch.randn(2 * d, generator=g), 0.1 * torch.randn(2 * d, generator=g)
        P[p + "b2"], P[p + "norm"] = 0.05 * torch.randn(d, generator=g), 1 + 0.1 * torch.randn(d, generator=g)
    return P


def _true_tower(Tw):
    """the true-shape parameters in twotower_reference.tower's form (F = 2d)"""
    out = {}
    for p in ("tw0.", "tw1."):
        out[p + "wgw1"] = torch.cat([Tw[p + "wg"], Tw[p + "w1"]])
        out[p + "bgb1"] = torch.cat([Tw[p + "bg"], Tw[p + "b1"]])
        out[p + "w2"], out[p + "b2"], out[p + "norm"] = Tw[p + "w2"], Tw[p + "b2"], Tw[p + "norm"]
    return out


def _negatives(kind_layout, B, L, labels, ignore, I, g):
    layout, N = kind_layout
    shape = {"shared": (N,), "perseq": (B, N), "perpos": (B, L, N)}[layout]
    neg = torch.randint(0, I, shape, generator=g)
    if layout == "shared":
        neg[:3] = ignore
        neg[3] = neg[4]
        neg[5] = labels[0, -1]
    elif layout == "perseq":
        neg[:, 0] = ignore
        neg[:, 1] = neg[:, 2]
        neg[:, 3] = labels[:, -1]
    else:
        neg[..., 0] = ignore
        neg[..., 1] = neg[..., 2]
        neg[..., 3] = labels
    return neg


def _step(cuda, kind, layout=None, B=64, L=200, I=50000, d=128, H=2, drop=0.0, seed=0, ignore=7):
    from replay_b200.engine_twotower import TwoTowerConfig, TwoTowerEngine

    cfg = TwoTowerConfig(n_items=I, d=d, n_heads=H, n_blocks=2, max_len=L, dropout=drop)
    eng = TwoTowerEngine(cfg, B, L, cuda, seed=SEED)
    from oracle import sasrec as osr

    Pq = engine_view(osr.random_params(I, d, L, 2, seed=seed, bias_scale=0.1))
    Tw = _tower_true(d, seed + 1)
    with torch.no_grad():
        for name in eng.layout:
            if name.startswith("tw"):
                eng.import_named(name, Tw[name])
            else:
                blk, _, leaf = name.partition(".")
                eng.import_named(name, Pq["blocks"][int(blk[1:])][leaf] if leaf else Pq[name])
    eng.refresh_shadow()
    g = torch.Generator().manual_seed(seed + 2)
    ids, pad, labels, tmask = step_batch(B, L, I, seed + 3)
    sampled = kind.endswith(("sampled", "sampled_weighted"))
    neg = _negatives(layout, B, L, labels, ignore, I, g) if sampled else None
    if sampled:
        eng.set_loss(kind, n_neg=layout[1], neg_shape=layout[0], ignore_index=ignore)
    else:
        eng.set_loss(kind)
    w = (0.25 + torch.rand(B, L, generator=g)) if kind in ("ce_weighted", "ce_sampled_weighted") else None
    if drop > 0:
        eng.tick_rng()
    ctr = int(eng.rng_counter.item())
    eng.set_batch(ids.to(cuda), pad.to(cuda), labels.to(cuda), tmask.to(cuda))
    if sampled:
        eng.set_negatives(neg.to(cuda))
    if w is not None:
        eng.set_row_weights(w.to(cuda))
    loss = float(eng.forward_train()[0])
    eng.g32.zero_()
    eng.backward()
    torch.cuda.synchronize()

    # ---- float64 reference on the device
    ids, pad, labels, tmask = (t.to(cuda) for t in (ids, pad, labels, tmask))
    Q = _map(_map(Pq, lambda k, v: v.to(cuda)), lambda k, v: v.detach().double().clone().requires_grad_(True))
    T64 = {k: v.to(cuda).double().clone().requires_grad_(True) for k, v in Tw.items()}
    keeps = engine_keeps(eng.seed + ctr, drop, B, L, cfg, dev=cuda) if drop > 0 else None
    _, hid = sasrec_body_ref(Q, ids, pad, H, "new", cfg.lnf_eps, keeps)
    sel = tmask & (labels >= 0) & (labels < I)
    h = hid[sel]
    y = labels[sel]
    flat = torch.nonzero(sel.reshape(-1))[:, 0]
    PT = _true_tower(T64)
    nv = int(eng.n_valid.item())
    assert nv == h.shape[0]
    res = dict(eng=eng, loss=loss, nv=nv)
    if not sampled:
        Y = tr.tower(Q["item_emb"][:I], PT, 2 * d, d)
        wc = w.to(cuda).double()[sel] if w is not None else None
        rl, d_h, d_Y = tr.full_head_chunked(kind, h.detach(), Y.detach(), y, wc)
        torch.autograd.backward([h, Y], [d_h, d_Y])
        res.update(tower_got=eng.unpad_features(eng.tw["cache"][:I]), tower_ref=Y.detach(), referenced=None)
    else:
        mode = {"shared": 0, "perpos": 1, "perseq": 2}[layout[0]]
        sp = eng.sampled
        cref = tr.compact_ref(I, eng.labels_c[:nv].cpu().numpy(), nv, eng.T, neg.reshape(-1).numpy(), layout[1], mode,
                              eng.valid_idx.cpu().numpy(), ignore, sp["cap"], neg.reshape(-1, layout[1]).shape[0])
        ns = cref["n_slots"]
        tw = eng.tw
        assert int(tw["n_slots"]) == ns
        assert np.array_equal(tw["item_of_slot"].cpu().long().numpy(), cref["item_of_slot"])
        assert np.array_equal(sp["labels_r"][:nv].cpu().long().numpy(), cref["labels_out"])
        assert np.array_equal(sp["neg_r"].reshape(-1)[torch.from_numpy(cref["neg_idx"]).to(cuda)].cpu().numpy(),
                              cref["neg_out"])
        items = torch.from_numpy(cref["item_of_slot"][:ns]).to(cuda)
        Yc = tr.tower(Q["item_emb"][items], PT, 2 * d, d)
        slot_of = torch.full((I,), -1, dtype=torch.int64, device=cuda)
        slot_of[items] = torch.arange(ns, device=cuda)
        negd = neg.to(cuda)
        neg_s = torch.where(negd == ignore, torch.full_like(negd, ns), slot_of[negd.clamp(0, I - 1)])
        table = torch.cat([Yc.detach(), torch.zeros(1, d, dtype=torch.float64, device=cuda)])
        neg_s = neg_s.reshape(-1, layout[1]) if mode == 1 else neg_s
        kid = {"ce_sampled": 0, "bce_sampled": 1, "login_ce_sampled": 4, "ce_sampled_weighted": 5}[kind]
        common = dict(hc=h.detach(), table=table, labels=slot_of[y], valid_idx=flat, negatives=neg_s, n_valid=nv, kind=kid,
                      neg_mode=mode, L=L, ignore_index=ns)
        if kid in (0, 1):
            r = sr.reference(**common)
        else:
            r = sx.reference(**common, row_weight=w.to(cuda).double()[sel] if w is not None else None)
        rl = r["loss"]
        torch.autograd.backward([h, Yc], [r["d_hc"], r["d_table"][:ns]])
        res.update(tower_got=eng.unpad_features(tw["out"][:ns]), tower_ref=Yc.detach(), referenced=items)
    res.update(ref_loss=float(rl), hc_got=eng.unpad_features(eng.hc[:nv]), hc_ref=h.detach())
    G = {}
    for name in eng.layout:
        if name.startswith("tw"):
            G[name] = T64[name].grad
        else:
            blk, _, leaf = name.partition(".")
            t = Q["blocks"][int(blk[1:])][leaf] if leaf else Q[name]
            G[name] = t.grad if t.grad is not None else torch.zeros_like(t)
    G["item_emb"][I] = 0
    res.update(G=G, ids=ids, pad=pad)
    return res


def _check_step(res, tag, tol_grad=TOL_GRAD):
    eng, I = res["eng"], res["eng"].cfg.n_items
    assert _note(f"step loss rel{tag}", abs(res["loss"] - res["ref_loss"]) / abs(res["ref_loss"])) <= TOL_LOSS
    assert _note(f"step hidden{tag}", block_err(res["hc_got"], res["hc_ref"])) <= TOL_HID
    assert _note(f"step tower out{tag}", _out_err(res["tower_got"], res["tower_ref"])) <= TOL_OUT
    bad = []
    for name, ref in res["G"].items():
        got = eng.export_named(name, eng.grads).to(ref.device).double()
        if name == "item_emb":
            assert not bool(got[I].any())     # the padding row
            used = torch.zeros(I + 1, dtype=torch.bool, device=ref.device)
            used[res["ids"][res["pad"]]] = True
            used[res["referenced"] if res["referenced"] is not None else slice(0, I)] = True
            assert not bool(got[~used].any())   # rows referenced by neither the batch nor a candidate
        if name.endswith("in_b"):
            d = eng.cfg.d
            got, ref = torch.cat([got[:d], got[2 * d:]]), torch.cat([ref[:d], ref[2 * d:]])
        g2, r2 = got.reshape(got.shape[0], -1), ref.reshape(ref.shape[0], -1)
        e = _note(f"step grad{tag}", block_err(g2, r2))
        if e > tol_grad:
            bad.append((name, round(e, 4)))
    assert not bad, bad


FULL = ("ce", "ce_weighted", "login_ce", "bce")
SAMPLED = ("ce_sampled", "bce_sampled", "login_ce_sampled", "ce_sampled_weighted")
LAYOUTS = (("shared", 256), ("perseq", 64), ("perpos", 8))


@pytest.mark.parametrize("kind", FULL)
def test_step_full_catalog(cuda, kind):
    """config-2 shape (L 200, d 128, 2 heads, 2 blocks, 50 000 items), B 64, dropout 0"""
    res = _step(cuda, kind, seed=11)
    _check_step(res, "")


@pytest.mark.parametrize("layout", LAYOUTS, ids=lambda x: x[0])
@pytest.mark.parametrize("kind", SAMPLED)
def test_step_sampled(cuda, kind, layout):
    """config-2 shape, B 64, ignore_index 7 among the negatives with duplicates and negatives equal to the positive"""
    res = _step(cuda, kind, layout, seed=13)
    _check_step(res, " sampled")


def test_step_full_batch_ce(cuda):
    res = _step(cuda, "ce", B=512, seed=17)
    _check_step(res, " B512")


def test_step_dropout_ce(cuda):
    """the query tower's dropout sites are SasRecEngine's (the item tower has none): engine_keeps ports them"""
    res = _step(cuda, "ce", drop=P_DROP, seed=19)
    _check_step(res, " dropout")


def test_step_config5_sampled(cuda):
    """config 5: 1 000 000 items (245 scan tiles), d 512, 8 heads, L 512, B 32, 256 shared negatives: the compaction and
    the split [bg; b1] colsum inside a real step"""
    assert -(-1000000 // tr.TILE) == 245
    res = _step(cuda, "ce_sampled", ("shared", 256), B=32, L=512, I=1000000, d=512, H=8, seed=23)
    _check_step(res, " c5", TOL_GRAD_C5)
