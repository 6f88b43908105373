"""The side-feature input kernels (csrc/rp_features.cu) called directly through the C ABI, every output against the float64
reference of tests/features_reference.py with its per-element bound: rp_feature_embed_fwd / _bwd and their packed-row
twins (x, d_s, v_rows and every d_table), the BERT form, rp_concat_embed_fwd and rp_concat_scatter.

Sweeps: d 64 / 128 / 256 / 512 (float2 atomics at VEC 2, float4 from VEC 4) with hd_valid 0, 50, 48 and 75 in the
engine's padded layout; T 1, 7, 255, 256, 257 and one T past two full waves of the grid (8 blocks of 8 warps per SM, read
from the device); packed row counts 0, 1, T - 1 and T over a shuffled subset of the tokens; dropout 0, 0.1 and 0.5 with a
seed counter and a non-zero site offset; bags of widths 1, 5 and 33 with repeated, padding, negative and out-of-range
ids and all-padding mean bags; padding values 0, cardinality and -1; a one-row table; numerical widths 1, 31, 32 and 33
and 64 columns in all; 16 features of every kind; one hot id shared by every token of the large case.
Every backward runs once in accumulate mode onto a non-zero d_table.  Output rows past *n_rows start as a sentinel and
must keep it bit for bit; the packed dx rows past the count are NaN and +-Inf, and d_table must stay finite.  Run with -s
to print the worst bound ratio of each family."""
import ctypes

import pytest
import torch

import features_reference as fr
from fp64_checks import WorstErrors
from replay_b200._lib import RpFeature, check, lib

pytestmark = pytest.mark.gpu

# Tolerance: max |got - ref| / bound over each family, with the bounds of tests/features_reference.py.  Worst values seen
# over every case of this file on one H100 80GB HBM3 at a 700 W power limit (run with -s): x 0.997, d_s 0.999, d_table
# 0.221, BERT x 1.0, concat x 1.0 (the bf16 half ulp dominates every bound but the tables').
TOL = 1.0
SENT = -3.0     # sentinel of every row a kernel must not write
V_LD = fr.FEAT_MAX_NUM_COLS

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


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _bits(x):
    return x.contiguous().view(torch.int16 if x.element_size() == 2 else torch.int32).cpu()


def _big_T(L):
    """B L tokens with B L > two full waves of the feature kernels' grid (sm count x 8 blocks x 8 warps, one row each)"""
    wave = torch.cuda.get_device_properties(0).multi_processor_count * 64
    T = (-(-2 * wave // L) + 1) * L
    assert T > 2 * wave
    return T


def _poison(x, n):
    """rows n.. of x: NaN, +Inf, -Inf in turn"""
    vals = torch.tensor([float("nan"), float("inf"), float("-inf")], dtype=x.dtype)
    if n < x.shape[0]:
        x[n:] = vals[torch.arange(x.shape[0] - n) % 3][:, None]
    return x


def _descs(c, dev, grads=None):
    """(rp_feature array, device buffers to keep alive) of c's features; grads: feature index -> device d_table"""
    arr = (RpFeature * len(c["feats"]))()
    keep = []
    for k, f in enumerate(c["feats"]):
        a = arr[k]
        a.kind, a.width = f["kind"], f["width"]
        v = f["values"].contiguous().to(dev)
        keep.append(v)
        a.values = v.data_ptr()
        if f["kind"] in fr.CAT_KINDS:
            a.n_rows, a.padding_value = f["n_rows"], f["padding_value"]
            t = f["table"].to(dev)
            keep.append(t)
            a.table = t.data_ptr()
            a.d_table = grads[k].data_ptr() if grads is not None else None
        elif f["kind"] == fr.NUM:
            W, b = f["table"].to(dev), f["bias"].to(dev)
            keep += [W, b]
            a.table, a.bias, a.val_col = W.data_ptr(), b.data_ptr(), f["val_col"]
    return arr, keep


def _starts(c, seed, width=None):
    """feature index -> fp32 start value of its d_table: random true columns (padding rows included), padded columns 0"""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k, f in enumerate(c["feats"]):
        if f["kind"] in fr.CAT_KINDS:
            if width is None:
                out[k] = fr.padded(g, f["n_rows"], c["d"], c["hd_valid"], 0.5)
            else:
                out[k] = torch.randn(f["n_rows"], f["dim"], generator=g) * 0.5
    return out


def _check_tables(c, grads, starts, ref_tables, pad_cols=True):
    real = fr.true_cols(c["d"], c["hd_valid"]) >= 0
    for k, start in starts.items():
        f = c["feats"][k]
        got = grads[k].cpu()
        assert torch.isfinite(got).all(), k
        con, ab, cnt = ref_tables[k]
        assert _note("d_table", fr.ratio(got, start.double() + con, fr.table_bound(start, ab, cnt))) <= TOL, k
        if pad_cols:
            assert not got[:, ~real].any(), k
        pv = f["padding_value"]
        if 0 <= pv < f["n_rows"]:
            assert torch.equal(_bits(got[pv]), _bits(start[pv])), k
        untouched = cnt == 0
        assert torch.equal(_bits(got[untouched]), _bits(start[untouched])), k


# ------------------------------------------------------------------------------------------------ SASRec sum form
def _sum_fwd(c, arr, out, rows=None):
    item, pos, ids = c["dev_item"], c["dev_pos"], c["dev_ids"]
    a = (c["T"], c["L"], c["d"], c["hd_valid"], c["pos0"], c["scale"], c["p"], fr.SEED, fr.DROP_OFF, c["seed_ptr"],
         out.data_ptr(), _stream())
    if rows is None:
        return lib().rp_feature_embed_fwd(item.data_ptr(), pos.data_ptr(), ids.data_ptr(), arr, len(arr), *a)
    rt, nr = rows
    return lib().rp_feature_embed_fwd_rows(item.data_ptr(), pos.data_ptr(), ids.data_ptr(), arr, len(arr), rt.data_ptr(),
                                           nr.data_ptr(), *a)


def _sum_bwd(c, arr, dx, d_s, v_rows, rows=None):
    a = (c["T"], c["d"], c["hd_valid"], c["scale"], c["p"], fr.SEED, fr.DROP_OFF, c["seed_ptr"], d_s.data_ptr(),
         v_rows.data_ptr(), V_LD, _stream())
    if rows is None:
        return lib().rp_feature_embed_bwd(dx.data_ptr(), arr, len(arr), *a)
    rt, nr = rows
    return lib().rp_feature_embed_bwd_rows(dx.data_ptr(), arr, len(arr), rt.data_ptr(), nr.data_ptr(), *a)


def _to_dev(c, dev):
    c["dev_item"], c["dev_pos"], c["dev_ids"] = c["item"].to(dev), c["pos"].to(dev), c["ids"].to(dev)
    c["ctr"] = torch.tensor([fr.COUNTER], device=dev, dtype=torch.int64)
    c["seed_ptr"] = c["ctr"].data_ptr() if c["use_ptr"] else None
    return c


def _run_sum(dev, c, n_rows=None, seed=0):
    """forward and backward of case c, dense (n_rows None) or on packed rows, every output against its bound"""
    _to_dev(c, dev)
    T, d = c["T"], c["d"]
    real = fr.true_cols(d, c["hd_valid"]) >= 0
    starts = _starts(c, seed + 1)
    grads = {k: s.to(dev) for k, s in starts.items()}
    arr, keep = _descs(c, dev, grads)
    out = torch.full((T, d), SENT, device=dev, dtype=torch.bfloat16)
    if n_rows is None:
        n, toks, rows = T, torch.arange(T), None
        check(_sum_fwd(c, arr, out), "rp_feature_embed_fwd")
    else:
        rt = fr.row_plan(T, n_rows, seed)
        n, toks = n_rows, rt[:n_rows].long()
        rows = (rt.to(dev), torch.tensor([n_rows], device=dev, dtype=torch.int32))
        check(_sum_fwd(c, arr, out, rows), "rp_feature_embed_fwd_rows")
        dense = torch.full((T, d), SENT, device=dev, dtype=torch.bfloat16)
        check(_sum_fwd(c, arr, dense), "rp_feature_embed_fwd")
        # the same fp32 order and the same dropout key: packed row r is the dense row of its token, bit for bit
        assert torch.equal(_bits(out[:n]), _bits(dense[toks.to(dev)]))
        assert torch.equal(_bits(out[n:]), _bits(torch.full((T - n, d), SENT, dtype=torch.bfloat16)))
    got = out[:n].cpu()
    x, xb = fr.forward(c, None if n_rows is None else toks)
    assert _note("x", fr.ratio(got, x, xb)) <= TOL
    assert not got[:, ~real].any()
    # backward, accumulating onto the start values
    g = torch.Generator().manual_seed(seed + 2)
    dx = fr.padded(g, T, d, c["hd_valid"], 0.1).to(torch.bfloat16)
    _poison(dx, n)
    d_s = torch.full((T, d), SENT, device=dev, dtype=torch.bfloat16)
    v_rows = torch.full((T, V_LD), SENT, device=dev, dtype=torch.bfloat16)
    check(_sum_bwd(c, arr, dx.to(dev), d_s, v_rows, rows), "rp_feature_embed_bwd")
    torch.cuda.synchronize()
    ref = fr.backward(c, dx[:n].float(), None if n_rows is None else toks)
    got = d_s[:n].cpu()
    assert _note("d_s", fr.ratio(got, ref["d_s"], ref["d_s_b"])) <= TOL
    assert not got[:, ~real].any()
    assert torch.equal(_bits(v_rows[:n]), _bits(fr.v_rows_ref(c, toks, V_LD)))
    sent = lambda w: _bits(torch.full((T - n, w), SENT, dtype=torch.bfloat16))  # noqa: E731
    assert torch.equal(_bits(d_s[n:]), sent(d)) and torch.equal(_bits(v_rows[n:]), sent(V_LD))
    _check_tables(c, grads, starts, ref["tables"])
    return ref


SUM_CASES = [
    # every hidden size (VEC 2 / 4 / 8 / 16) and head-slot layout: one 64 slot of 50, two 64 slots of 48, 128 slots of 75
    (64, 0, 257, 13, 0.1, "mixed"), (128, 0, 257, 13, 0.1, "mixed"), (256, 0, 257, 13, 0.1, "mixed"),
    (512, 0, 257, 13, 0.1, "mixed"), (64, 50, 257, 13, 0.1, "mixed"), (128, 48, 257, 13, 0.1, "mixed"),
    (256, 50, 257, 13, 0.1, "mixed"), (512, 75, 257, 13, 0.1, "mixed"),
    # row counts around the 8-warp block and one past 256
    (128, 48, 1, 1, 0.5, "mixed"), (128, 48, 7, 7, 0.5, "mixed"), (128, 48, 255, 13, 0.5, "mixed"),
    (128, 48, 256, 16, 0.5, "mixed"),
    # dropout off and at one half
    (64, 50, 255, 17, 0.0, "mixed"), (256, 0, 255, 17, 0.5, "mixed"),
    # 64 numerical columns exactly; 16 features of every kind
    (256, 0, 257, 13, 0.1, "num64"), (64, 50, 257, 13, 0.0, "num64"), (512, 75, 257, 13, 0.1, "max16"),
    (64, 0, 257, 13, 0.0, "max16"),
]


@pytest.mark.parametrize("d,hd_valid,T,L,p,feats", SUM_CASES,
                         ids=[f"d{d}-hd{h}-T{T}-p{p}-{f}" for d, h, T, L, p, f in SUM_CASES])
def test_sum_form(cuda, d, hd_valid, T, L, p, feats):
    _run_sum(cuda, fr.make_case(d, hd_valid, T, L, p, feats, seed=T))


def test_sum_form_without_seed_pointer(cuda):
    _run_sum(cuda, fr.make_case(128, 0, 257, 13, 0.1, use_ptr=False, seed=5))


@pytest.mark.parametrize("n_rows", ["0", "1", "T-1", "T"])
def test_sum_form_packed_rows(cuda, n_rows):
    T = fr.SUM_CASE["T"]
    n = {"0": 0, "1": 1, "T-1": T - 1, "T": T}[n_rows]
    _run_sum(cuda, fr.make_case(**fr.SUM_CASE, p=0.1, seed=9), n_rows=n, seed=n)


@pytest.mark.parametrize("d", [64, 256])
def test_sum_form_large_T_one_hot_id(cuda, d):
    """every token shares id 3 of the first categorical feature and of the width-33 mean bag, and row 0 of the one-row
    table: tens of thousands of atomics into one row, against the order-free fp64 sum"""
    L = 200
    T = _big_T(L)
    c = fr.make_case(d, 0, T, L, 0.1, "mixed", seed=1, hot=3)
    ref = _run_sum(cuda, c)
    assert ref["tables"][0][2][3] == T            # the hot row took one atomic per token
    assert ref["tables"][1][2][0] > T // 2        # the one-row table: every live id


def test_sum_form_rejects_17_features_and_65_numerical_columns(cuda):
    c = _to_dev(fr.make_case(64, 0, 7, 7, 0.0, "max16"), cuda)
    c["feats"].append(dict(c["feats"][0]))
    grads = {k: torch.zeros(f["n_rows"], 64, device=cuda) for k, f in enumerate(c["feats"]) if f["kind"] in fr.CAT_KINDS}
    arr, keep = _descs(c, cuda, grads)
    out = torch.zeros(7, 64, device=cuda, dtype=torch.bfloat16)
    d_s, v_rows = torch.zeros_like(out), torch.zeros(7, V_LD, device=cuda, dtype=torch.bfloat16)
    rows = (torch.arange(7, device=cuda, dtype=torch.int32), torch.tensor([7], device=cuda, dtype=torch.int32))
    assert _sum_fwd(c, arr, out) == -2
    assert _sum_fwd(c, arr, out, rows) == -2
    assert _sum_bwd(c, arr, out, d_s, v_rows) == -2
    assert _sum_bwd(c, arr, out, d_s, v_rows, rows) == -2
    c = _to_dev(fr.make_case(64, 0, 7, 7, 0.0, "num64"), cuda)
    last = c["feats"][-1]
    last["width"], last["values"] = 2, torch.randn(7, 2)   # 32 + 31 + 2 = 65 columns
    grads = {0: torch.zeros(c["feats"][0]["n_rows"], 64, device=cuda)}
    arr, keep = _descs(c, cuda, grads)
    assert _sum_fwd(c, arr, out) == -2
    assert _sum_bwd(c, arr, out, d_s, v_rows) == -2
    last["width"], last["values"] = 1, torch.randn(7, 1)   # 64: accepted
    arr, keep = _descs(c, cuda, grads)
    assert _sum_fwd(c, arr, out) == 0


# ------------------------------------------------------------------------------------------------ BERT form
@pytest.mark.parametrize("d,hd_valid", [(64, 0), (512, 75)])
def test_bert_form_large_T_one_hot_id(cuda, d, hd_valid):
    """padding_value -1 (id 0 a live row, the hot id of every real token), the one-row table, an identity feature;
    row 5 appears at masked and pad tokens only, so it must get no gradient"""
    L = 200
    T = _big_T(L)
    c = _to_dev(fr.make_case(d, hd_valid, T, L, 0.1, "bert", seed=2), cuda)
    g = torch.Generator().manual_seed(4)
    B = T // L
    lens = torch.randint(1, L + 1, (B,), generator=g)
    pad = (torch.arange(L)[None, :] >= (L - lens)[:, None]).reshape(-1)
    tok = (torch.rand(T, generator=g) > 0.2) & pad
    ok = pad & tok
    v = c["feats"][0]["values"][:, 0]
    v[ok & (torch.rand(T, generator=g) < 0.6)] = 0
    v[ok & (v == 5)] = 4
    v[~ok & (torch.rand(T, generator=g) < 0.5)] = 5
    mask_emb = fr.padded(g, 1, d, hd_valid, 0.3)[0].to(torch.bfloat16)
    starts = _starts(c, 6)
    grads = {k: s.to(cuda) for k, s in starts.items()}
    arr, keep = _descs(c, cuda, grads)
    tok8, pad8 = tok.to(torch.uint8).to(cuda), pad.to(torch.uint8).to(cuda)
    real = fr.true_cols(d, hd_valid) >= 0
    for with_pos in (True, False):
        out = torch.full((T, d), SENT, device=cuda, dtype=torch.bfloat16)
        check(lib().rp_bert_feature_embed_fwd(c["dev_item"].data_ptr(), mask_emb.to(cuda).data_ptr(),
                                              c["dev_pos"].data_ptr() if with_pos else None, c["dev_ids"].data_ptr(),
                                              tok8.data_ptr(), arr, len(arr), T, L, d, hd_valid, c["p"], fr.SEED, fr.DROP_OFF,
                                              c["seed_ptr"], out.data_ptr(), _stream()), "rp_bert_feature_embed_fwd")
        x, xb = fr.bert_forward(c, tok, mask_emb, with_pos)
        got = out.cpu()
        assert _note("bert x", fr.ratio(got, x, xb)) <= TOL
        assert not got[:, ~real].any()
    dx = fr.padded(g, T, d, hd_valid, 0.1)
    dx[~ok] = float("nan")     # the masked and pad tokens' rows are never read
    dx = dx.to(torch.bfloat16)
    check(lib().rp_bert_feature_embed_bwd(dx.to(cuda).data_ptr(), pad8.data_ptr(), tok8.data_ptr(), arr, len(arr), T, d,
                                          hd_valid, c["p"], fr.SEED, fr.DROP_OFF, c["seed_ptr"], _stream()),
          "rp_bert_feature_embed_bwd")
    torch.cuda.synchronize()
    ref = fr.bert_backward(c, dx.float(), pad, tok)
    _check_tables(c, grads, starts, ref["tables"])
    assert ref["tables"][0][2][5] == 0 and ref["tables"][0][2][0] > T // 8
    assert torch.equal(_bits(grads[0][5]), _bits(starts[0][5]))


# ------------------------------------------------------------------------------------------------ ConcatAggregator
def _concat_descs(c, dev, grads=None):
    arr, keep = _descs(c, dev, grads)
    n = len(c["feats"])
    cols = (ctypes.c_int * n)(*[f["col"] for f in c["feats"]])
    dims = (ctypes.c_int * n)(*[f["dim"] for f in c["feats"]])
    return arr, cols, dims, keep


def _run_concat(dev, c, n_rows=None, seed=0):
    _to_dev(c, dev)
    T, d, kp = c["T"], c["d"], c["kp"]
    real = fr.true_cols(d, c["hd_valid"]) >= 0
    g = torch.Generator().manual_seed(seed + 3)
    if n_rows is None:
        n, toks, rt, nr = T, torch.arange(T), None, None
    else:
        rt_h = fr.row_plan(T, n_rows, seed)
        n, toks = n_rows, rt_h[:n_rows].long()
        rt, nr = rt_h.to(dev), torch.tensor([n_rows], device=dev, dtype=torch.int32)
    ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    # rp_concat_embed_fwd: y rows are output rows; the packed rows past the count are NaN and never read
    y_dense = fr.padded(g, T, d, c["hd_valid"], 0.5)
    y = y_dense
    if n_rows is not None:
        y = torch.full((T, d), float("nan"))
        y[:n] = y_dense[toks]
    out = torch.full((T, d), SENT, device=dev, dtype=torch.bfloat16)
    check(lib().rp_concat_embed_fwd(y.to(dev).data_ptr(), c["dev_pos"].data_ptr(), ptr(rt), ptr(nr), T, c["L"], d, c["pos0"],
                                    c["scale"], c["p"], fr.SEED, fr.DROP_OFF, c["seed_ptr"], out.data_ptr(), _stream()),
          "rp_concat_embed_fwd")
    x, xb = fr.concat_embed_fwd(c, y[:n], toks)
    got = out[:n].cpu()
    assert _note("concat x", fr.ratio(got, x, xb)) <= TOL
    assert not got[:, ~real].any()
    if n_rows is not None:
        dense = torch.full((T, d), SENT, device=dev, dtype=torch.bfloat16)
        check(lib().rp_concat_embed_fwd(y_dense.to(dev).data_ptr(), c["dev_pos"].data_ptr(), None, None, T, c["L"], d,
                                        c["pos0"], c["scale"], c["p"], fr.SEED, fr.DROP_OFF, c["seed_ptr"], dense.data_ptr(),
                                        _stream()), "rp_concat_embed_fwd")
        assert torch.equal(_bits(out[:n]), _bits(dense[toks.to(dev)]))
        assert torch.equal(_bits(out[n:]), _bits(torch.full((T - n, d), SENT, dtype=torch.bfloat16)))
    # rp_concat_scatter: dX's columns past the segments and its packed rows past the count are NaN / Inf, never read
    starts = _starts(c, seed + 4, width=True)
    grads = {k: s.to(dev) for k, s in starts.items()}
    item_start = fr.padded(g, c["n_items"] + 1, d, c["hd_valid"], 0.5)
    d_item = item_start.to(dev)
    arr, cols, dims, keep = _concat_descs(c, dev, grads)
    dx = torch.randn(T, kp, generator=g) * 0.1
    dx[:, c["width"]:] = float("nan")
    dx = _poison(dx, n).to(torch.bfloat16)
    v_rows = torch.full((T, V_LD), SENT, device=dev, dtype=torch.bfloat16)
    check(lib().rp_concat_scatter(dx.to(dev).data_ptr(), c["dev_ids"].data_ptr(), d_item.data_ptr(), c["pad_id"], arr, cols,
                                  dims, len(arr), c["item_col"], ptr(rt), ptr(nr), T, d, c["hd_valid"], kp, v_rows.data_ptr(),
                                  V_LD, _stream()), "rp_concat_scatter")
    torch.cuda.synchronize()
    ref = fr.concat_scatter(c, dx[:n].float(), toks)
    _check_tables(c, grads, starts, ref["tables"], pad_cols=False)
    _check_tables(dict(c, feats=[dict(n_rows=c["n_items"] + 1, padding_value=c["pad_id"])]), {0: d_item}, {0: item_start},
                  {0: ref["item"]})
    assert torch.equal(_bits(v_rows[:n]), _bits(fr.v_rows_ref(c, toks, V_LD)))
    assert torch.equal(_bits(v_rows[n:]), _bits(torch.full((T - n, V_LD), SENT, dtype=torch.bfloat16)))


CONCAT_CASES = [(64, 0, 0.1), (64, 50, 0.5), (128, 48, 0.0), (256, 0, 0.1), (512, 75, 0.1)]


@pytest.mark.parametrize("d,hd_valid,p", CONCAT_CASES, ids=[f"d{d}-hd{h}-p{p}" for d, h, p in CONCAT_CASES])
def test_concat(cuda, d, hd_valid, p):
    _run_concat(cuda, fr.make_concat_case(d, hd_valid, 257, 13, p, seed=1))


@pytest.mark.parametrize("n_rows", ["0", "1", "T-1", "T"])
def test_concat_packed_rows(cuda, n_rows):
    T = 257
    n = {"0": 0, "1": 1, "T-1": T - 1, "T": T}[n_rows]
    _run_concat(cuda, fr.make_concat_case(512, 75, T, 13, 0.1, seed=2), n_rows=n, seed=n)
