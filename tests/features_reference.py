"""float64 restatement of the side-feature input kernels (csrc/rp_features.cu) with a per-element error bound for every
output, and the inputs the kernel tests draw.  The restatement follows the contract at the top of rp_features.cu and in
include/rp_b200.h, from the same bf16 tables and fp32 values the kernels read:

  SASRec sum form (rp_feature_embed_fwd / _rows), token t of output row r (t = r, or row_tok[r] on packed rows):
    s_t = E_item[id_t] + sum_cat E_f[id] + sum_bag (sum, or mean over the live ids) + sum_num (v W^T + b) + sum_ident v
    x_r = keep(t) ks (s_t scale + P[pos0 + t % L])
  an id is live iff id != padding_value and 0 <= id < n_rows; a mean bag divides by its live count (an all-padding bag
  gives zero); an identity value lands at padded column c from true feature feat_true_col(c) (padded columns get nothing).
  Backward (rp_feature_embed_bwd / _rows): dS_r = scale ks keep(t) dx_r; d_s = bf16(dS); every live id of token t adds
  w dS_r into its d_table row, w = 1 or 1 / live count; v_rows = bf16 of the numerical values at their val_col, zero past.
  BERT form: s_t as above over CAT and IDENT features, replaced by mask_emb where tok_mask is 0, plus P[t % L] (optional),
  no scale; its backward adds dropout'(dx) at tokens with pad_mask and tok_mask only.
  rp_concat_embed_fwd: x_r = keep(t) ks (Y_r scale + P[pos0 + t % L]).  rp_concat_scatter: dX's item segment into
  d_item[id_t] at the padded columns feat_pad_col(j) (pad_id frozen), each categorical segment into its d_table rows with
  weight w as above.
keep(t) is the 0 / 1 draw of tests/dropout_stream.py keyed by the TOKEN t (site drop_off, seed + *seed_ptr);
ks = 1 / (1 - p).

Error bounds (u = 2^-24, gamma_n = n u / (1 - n u)).  The kernels build with fast math, so 1 / cnt and 1 / (1 - p) are
approximate reciprocals within two fp32 ulps (4 u); ks = 1 / (1 - p) carries the rounding of 1 - p too: KS_REL = 5 u.
  Forward.  The fp32 accumulator of one output element sums n terms: the item row, every live bag row (times w), every
  bias and every v_j W[c, j] product (FMAs, or a product rounding each: one more term's worth), every identity value.
  Whatever the order and nesting (a bag is summed on its own first), that is within gamma_{n+1} sum |terms| = gamma_{n+1} A.
  A mean bag's 1 / cnt and its product add RCP + u of that bag's |terms| (A_mean):
      e_s = gamma_{n+1} A + (RCP + u) A_mean
  then y = s scale + p (at most two roundings) and x = y ks keep (ks and the product):
      e_y = scale e_s + u (|s| scale + |y|),   e_x = keep (ks e_y + (KS_REL + u) |x|)
  and one bf16 rounding of the fp32 value:  bound = hulp(|x| + E) + E,  E = SAFETY e_x,  hulp = half a bf16 ulp.
  The BERT form is the same with the position row as one more term and no scale.
  d_s.  dx scale ks keep: scale ks is one fp32 product (KS_REL + u), times dx one more:  e = (KS_REL + 2 u) |dS|,
  bound = hulp(|dS| + E) + E.
  Table gradients.  Row k of a d_table receives n_c atomics, term w dS (fp32 products: dS's KS_REL + 2 u, w's RCP, the
  product u: TERM_REL = 12 u of |term|), added in any order onto the start value:
      bound = SAFETY (gamma_{n_c+2} (|start| + A) + TERM_REL A),  A = sum |w dS| over the row's terms.
  rp_concat_embed_fwd is the forward with e_s = 0 and Y for s; rp_concat_scatter's terms are bf16(dX) (times w).
SAFETY = 2; every bound gets FLOOR = 1e-30 on top, so an exact zero compares against an exact zero.
Exact, bit for bit: v_rows; padding rows, padded columns and rows past *n_rows; packed forward row r against the dense row
row_tok[r] (the same fp32 order and the same dropout key).

Each function takes ``bug=`` to restate one plausible kernel mistake (BUGS); tests/test_features_reference_cpu.py checks
that each breaks its bound by at least ten times on the GPU cases' inputs."""
import math

import numpy as np
import torch

from dropout_stream import keep_draws

U = 2.0 ** -24
FLOOR = 1e-30
SAFETY = 2.0
RCP = 4 * U           # fast-math reciprocal: within two fp32 ulps
KS_REL = RCP + U      # ks = 1 / (1 - p): the subtraction and the reciprocal
TERM_REL = 12 * U     # one table-gradient term w dS: dS (KS_REL + 2 u), w (RCP), their product (u)
CAT, BAG_SUM, BAG_MEAN, NUM, IDENT = range(5)   # rp_feature.kind
CAT_KINDS = (CAT, BAG_SUM, BAG_MEAN)
FEAT_MAX, FEAT_MAX_NUM_COLS = 16, 64
SEED, COUNTER, DROP_OFF = 0x5EED1234ABC, 977, (7 << 40) + 5
SUM_CASE = dict(d=128, hd_valid=48, T=257, L=13)   # two 64-wide head slots of 48 features, one token past 256

BUGS = {
    "mean_by_width": "a mean bag divided by its width instead of its live count",
    "count_padding": "padding ids counted in a mean bag's count",
    "dedup": "duplicate ids of one bag counted once",
    "scale_pos": "scale applied to the position row too",
    "ident_padded_col": "an identity value read at padded column c instead of feat_true_col(c)",
    "no_bias": "the numerical bias omitted",
    "w_transposed": "W indexed [j, c] instead of [c, j]",
    "pos_no_pos0": "the position row t % L without pos0",
    "drop_key_row": "dropout keyed by the packed row instead of the token",
    "bwd_mean_twice": "the mean weight applied twice in the backward",
    "concat_item_col_j": "the concat item segment scattered to column j instead of feat_pad_col(j)",
}


# ------------------------------------------------------------------------------------------------ measures
def gamma(n):
    return n * U / (1.0 - n * U)


def hulp(x):
    """half a bf16 ulp of |x| (x float64)"""
    return torch.exp2(torch.floor(torch.log2(x.abs().clamp_min(1e-300))) - 8)


def bf16_bound(ref, e):
    return hulp(ref.abs() + e) + e + FLOOR


def ratio(got, ref, bound):
    """max |got - ref| / bound (inf where got is not finite); 0 for an empty selection"""
    if ref.numel() == 0:
        return 0.0
    r = (got.double() - ref).abs() / bound
    r = torch.where(torch.isfinite(got.double()), r, torch.full_like(r, math.inf))
    return float(r.max())


def table_bound(start, absum, cnt):
    """bound on |d_table - start - contribution| of a table row that took cnt[row] fp32 atomics of sum |terms| absum"""
    return SAFETY * (gamma(cnt.double() + 2)[:, None] * (start.double().abs() + absum) + TERM_REL * absum) + FLOOR


def f32(x):
    return float(np.float32(x))


def ks_of(p):
    return 1.0 / (1.0 - f32(p)) if p > 0 else 1.0


def keep(seed_eff, off, p, keys, d):
    """float64 [len(keys), d] 0 / 1: the dropout draws of the embedding site keyed by ``keys``"""
    keys = torch.as_tensor(keys).long()
    if p == 0:
        return torch.ones(len(keys), d, dtype=torch.float64)
    return keep_draws(seed_eff, off, p, keys.numpy().astype(np.uint64), d).double()


# ------------------------------------------------------------------------------------------------ padded head slots
def slot_of(hd_valid):
    return 64 if hd_valid <= 64 else 128


def d_true_of(d, hd_valid):
    return d if hd_valid == 0 else d // slot_of(hd_valid) * hd_valid


def true_cols(d, hd_valid):
    """feat_true_col of every padded column: the true feature, -1 for a padded column"""
    c = torch.arange(d)
    if hd_valid == 0:
        return c
    slot = slot_of(hd_valid)
    j = c % slot
    return torch.where(j < hd_valid, (c // slot) * hd_valid + j, torch.full_like(c, -1))


def pad_cols(d_true, hd_valid):
    """feat_pad_col of every true feature"""
    j = torch.arange(d_true)
    return j if hd_valid == 0 else (j // hd_valid) * slot_of(hd_valid) + j % hd_valid


# ------------------------------------------------------------------------------------------------ categorical weights
def live(f, v):
    return (v != f["padding_value"]) & (v >= 0) & (v < f["n_rows"])


def entry_weights(f, v, bug=None):
    """float64 [n, K]: the weight of every entry of a categorical feature's ids v [n, K] (0 for a dead id)"""
    lv = live(f, v)
    if bug == "dedup":   # a later entry repeating a live id of the same bag is dropped
        K = v.shape[1]
        earlier = torch.tril(torch.ones(K, K, dtype=torch.bool), -1)          # [j, j'] j' < j
        rep = ((v[:, :, None] == v[:, None, :]) & lv[:, None, :] & earlier).any(-1)
        lv = lv & ~rep
    w = lv.double()
    if f["kind"] == BAG_MEAN:
        cnt = w.sum(1, keepdim=True)
        if bug == "mean_by_width":
            cnt = torch.full_like(cnt, v.shape[1])
        elif bug == "count_padding":
            cnt = ((v >= 0) & (v < f["n_rows"])).double().sum(1, keepdim=True)
        w = w / cnt.clamp_min(1)
    return w


# ------------------------------------------------------------------------------------------------ SASRec sum form
def sum_input(c, toks, bug=None):
    """(s, A, n, A_mean) of tokens ``toks``: the summed input s float64 [n, d], the sum of |terms| A, the term count n [n, 1]
    and the |terms| of mean bags A_mean, for case ``c`` (make_case's dict)"""
    d, hd = c["d"], c["hd_valid"]
    tc = true_cols(d, hd)
    real = tc >= 0
    s = c["item"].double()[c["ids"].long()[toks]]
    a = s.abs()
    am = torch.zeros_like(s)
    nt = torch.ones(len(toks), 1, dtype=torch.float64)
    for f in c["feats"]:
        if f["kind"] in CAT_KINDS:
            v = f["values"].long()[toks]
            w = entry_weights(f, v, bug)
            tab = f["table"].double()
            for j in range(v.shape[1]):
                rows = tab[v[:, j].clamp(0, f["n_rows"] - 1)] * w[:, j:j + 1]
                s += rows
                a += rows.abs()
                if f["kind"] == BAG_MEAN:
                    am += rows.abs()
            nt += (w > 0).double().sum(1, keepdim=True)
        elif f["kind"] == NUM:
            v = f["values"].double()[toks]
            W = f["table"].double()
            if bug == "w_transposed":   # the flat [d, K] buffer read at j * d + c
                W = W.reshape(-1).reshape(W.shape[1], W.shape[0]).T
            b = f["bias"].double()
            if bug != "no_bias":
                s += b
                a += b.abs()
            s += v @ W.T
            a += v.abs() @ W.abs().T
            nt += 1 + v.shape[1]
        else:
            K = f["values"].shape[1]
            vals = torch.zeros_like(s)
            if bug == "ident_padded_col":   # the flat [T, K] values read at t * K + c
                flat = f["values"].double().reshape(-1)
                idx = (toks.long()[:, None] * K + torch.arange(d)[None, real]).clamp_max(flat.numel() - 1)
                vals[:, real] = flat[idx]
            else:
                vals[:, real] = f["values"].double()[toks][:, tc[real]]
            s += vals
            a += vals.abs()
            nt += 1
    return s, a, nt, am


def _finish(y, e_y, keys, c):
    """x = keep ks y and its bound, from y float64 [n, d] and its fp32 error e_y"""
    p = c["p"]
    kp = keep(c["seed_eff"], c["drop_off"], p, keys, y.shape[1])
    ks = ks_of(p)
    x = y * ks * kp
    e_x = kp * (ks * e_y + (KS_REL + U) * x.abs()) if p > 0 else e_y
    return x, bf16_bound(x, SAFETY * e_x)


def forward(c, rows=None, bug=None):
    """(x, bound) float64 [n, d] of rp_feature_embed_fwd (rows None) or _rows (rows = row_tok[:n])"""
    toks = torch.arange(c["T"]) if rows is None else torch.as_tensor(rows).long()
    s, a, nt, am = sum_input(c, toks, bug)
    pos = c["pos"].double()[(0 if bug == "pos_no_pos0" else c["pos0"]) + toks % c["L"]]
    sc = c["scale"]
    y = (s + pos) * sc if bug == "scale_pos" else s * sc + pos
    e_s = gamma(nt + 1) * a + (RCP + U) * am
    e_y = sc * e_s + U * (s.abs() * sc + y.abs())
    return _finish(y, e_y, torch.arange(len(toks)) if bug == "drop_key_row" else toks, c)


def backward(c, dx, rows=None, bug=None, tok_ok=None):
    """rp_feature_embed_bwd (rows None) or _rows (rows = row_tok[:n]) from dx [n, d] (row r = token toks[r]):
    {"d_s": float64 [n, d], "d_s_b": its bound, "tables": {feature index: (contribution, sum |terms|, terms per row)}}.
    tok_ok: bool [T], the tokens whose gradient reaches the tables (the BERT form), None for all."""
    toks = torch.arange(c["T"]) if rows is None else torch.as_tensor(rows).long()
    kp = keep(c["seed_eff"], c["drop_off"], c["p"], toks, c["d"])
    g = dx.double() * (c["scale"] * ks_of(c["p"])) * kp
    out = {"d_s": g, "d_s_b": bf16_bound(g, SAFETY * (KS_REL + 2 * U) * g.abs()), "tables": {}}
    ok = torch.ones(len(toks), dtype=torch.bool) if tok_ok is None else tok_ok[toks]
    for k, f in enumerate(c["feats"]):
        if f["kind"] not in CAT_KINDS:
            continue
        v = f["values"].long()[toks]
        w = entry_weights(f, v, None if bug == "bwd_mean_twice" else bug)
        if bug == "bwd_mean_twice" and f["kind"] == BAG_MEAN:
            w = w * w
        w = w * ok.double()[:, None]
        out["tables"][k] = _scatter(f["n_rows"], g, v, w)
    return out


def _scatter(n_rows, g, v, w):
    """(contribution, sum |terms|, terms per row) of adding w[:, j] g into rows v[:, j] for every live entry"""
    con = torch.zeros(n_rows, g.shape[1], dtype=torch.float64)
    ab = torch.zeros_like(con)
    cnt = torch.zeros(n_rows, dtype=torch.float64)
    for j in range(v.shape[1]):
        m = w[:, j] > 0
        terms = g[m] * w[m, j:j + 1]
        con.index_add_(0, v[m, j], terms)
        ab.index_add_(0, v[m, j], terms.abs())
        cnt.index_add_(0, v[m, j], torch.ones(int(m.sum()), dtype=torch.float64))
    return con, ab, cnt


def v_rows_ref(c, toks, v_ld):
    """bf16 [n, v_ld]: the numerical values at their val_col, zero past them"""
    out = torch.zeros(len(toks), v_ld, dtype=torch.bfloat16)
    for f in c["feats"]:
        if f["kind"] == NUM:
            out[:, f["val_col"]:f["val_col"] + f["width"]] = f["values"][toks].to(torch.bfloat16)
    return out


# ------------------------------------------------------------------------------------------------ BERT form
def bert_forward(c, tok_mask, mask_emb, with_pos):
    """(x, bound) of rp_bert_feature_embed_fwd: tok_mask bool [T], mask_emb bf16 [d]"""
    toks = torch.arange(c["T"])
    s, a, nt, _ = sum_input(c, toks)
    m = ~tok_mask
    s[m] = mask_emb.double()
    a[m] = mask_emb.double().abs()
    nt[m] = 1
    if with_pos:
        pos = c["pos"].double()[toks % c["L"]]
        s = s + pos
        a = a + pos.abs()
        nt = nt + 1
    return _finish(s, gamma(nt + 1) * a, toks, c)


def bert_backward(c, dx, pad_mask, tok_mask):
    return backward({**c, "scale": 1.0}, dx, tok_ok=pad_mask & tok_mask)


# ------------------------------------------------------------------------------------------------ ConcatAggregator
def concat_x(c):
    """float64 X [T, width] of rp_concat_gather: the item's true features at item_col, each feature's segment at its col"""
    T, d_true = c["T"], d_true_of(c["d"], c["hd_valid"])
    X = torch.zeros(T, c["width"], dtype=torch.float64)
    X[:, c["item_col"]:c["item_col"] + d_true] = c["item"].double()[c["ids"].long()][:, pad_cols(d_true, c["hd_valid"])]
    for f in c["feats"]:
        seg = slice(f["col"], f["col"] + f["dim"])
        if f["kind"] in CAT_KINDS:
            v = f["values"].long()
            w = entry_weights(f, v)
            tab = f["table"].double()
            X[:, seg] = sum(tab[v[:, j].clamp(0, f["n_rows"] - 1)] * w[:, j:j + 1] for j in range(v.shape[1]))
        elif f["kind"] == NUM:
            X[:, seg] = f["values"].double() @ f["table"].double().T + f["bias"].double()
        else:
            X[:, seg] = f["values"].double()
    return X


def concat_embed_fwd(c, y, rows=None, bug=None):
    """(x, bound) of rp_concat_embed_fwd from the projection y fp32 [n, d] (row r = token toks[r])"""
    toks = torch.arange(c["T"]) if rows is None else torch.as_tensor(rows).long()
    y = y.double()
    pos = c["pos"].double()[(0 if bug == "pos_no_pos0" else c["pos0"]) + toks % c["L"]]
    sc = c["scale"]
    z = (y + pos) * sc if bug == "scale_pos" else y * sc + pos
    e_z = U * (y.abs() * sc + z.abs())
    return _finish(z, e_z, torch.arange(len(toks)) if bug == "drop_key_row" else toks, c)


def concat_scatter(c, dx, rows=None, bug=None):
    """rp_concat_scatter from dx bf16 [n, kp] (row r = token toks[r]): {"item": (contribution [n_items + 1, d], sum |terms|,
    terms per row), "tables": {feature index: (contribution [n_rows, dim], ...)}}"""
    toks = torch.arange(c["T"]) if rows is None else torch.as_tensor(rows).long()
    g = dx.double()
    d_true = d_true_of(c["d"], c["hd_valid"])
    ids = c["ids"].long()[toks]
    m = ids != c["pad_id"]
    cols = torch.arange(d_true) if bug == "concat_item_col_j" else pad_cols(d_true, c["hd_valid"])
    seg = torch.zeros(len(toks), c["d"], dtype=torch.float64)
    seg[:, cols] = g[:, c["item_col"]:c["item_col"] + d_true]
    out = {"item": _scatter(c["n_items"] + 1, seg, ids[:, None], m.double()[:, None]), "tables": {}}
    for k, f in enumerate(c["feats"]):
        if f["kind"] not in CAT_KINDS:
            continue
        v = f["values"].long()[toks]
        w = entry_weights(f, v)
        if bug == "bwd_mean_twice" and f["kind"] == BAG_MEAN:
            w = w * w
        out["tables"][k] = _scatter(f["n_rows"], g[:, f["col"]:f["col"] + f["dim"]], v, w)
    return out


# ------------------------------------------------------------------------------------------------ inputs
def padded(g, rows, d, hd_valid, std):
    """fp32 [rows, d]: random true features, zero padded columns"""
    t = torch.zeros(rows, d)
    real = true_cols(d, hd_valid) >= 0
    t[:, real] = torch.randn(rows, int(real.sum()), generator=g) * std
    return t


def _ids(g, T, K, n_rows, padding_value, p_pad=0.2, p_bad=0.05, dup=True):
    """int32 [T, K] ids of a categorical feature: live ids, padding ids (p_pad), ids outside [0, n_rows) (p_bad: -1, -7,
    n_rows, n_rows + 1000) and, with dup, repeats of a bag's first id"""
    v = torch.randint(0, n_rows, (T, K), generator=g)
    r = torch.rand(T, K, generator=g)
    v = torch.where(r < p_pad, torch.full_like(v, padding_value), v)
    bad = torch.tensor([-1, -7, n_rows, n_rows + 1000])[torch.randint(0, 4, (T, K), generator=g)]
    v = torch.where((r >= p_pad) & (r < p_pad + p_bad), bad, v)
    if dup and K > 1:
        rep = torch.rand(T, generator=g) < 0.3
        v[rep, 1] = v[rep, 0]
    return v.to(torch.int32)


def _cat(g, kind, T, K, card, padding_value, d, hd_valid, **kw):
    """a categorical feature of ``card`` live rows (+1 zero padding row when padding_value is a row), engine layout"""
    n_rows = card + 1 if 0 <= padding_value <= card else card
    tab = padded(g, n_rows, d, hd_valid, 0.1)
    if 0 <= padding_value < n_rows:
        tab[padding_value] = 0
    return dict(kind=kind, width=K, n_rows=n_rows, padding_value=padding_value, table=tab.to(torch.bfloat16),
                values=_ids(g, T, K, n_rows, padding_value, **kw))


def _num(g, T, K, d, hd_valid):
    W = torch.zeros(d, K)
    real = true_cols(d, hd_valid) >= 0
    W[real] = torch.randn(int(real.sum()), K, generator=g) * (0.3 / math.sqrt(K))
    return dict(kind=NUM, width=K, n_rows=0, padding_value=0, table=W, bias=padded(g, 1, d, hd_valid, 0.1)[0],
                values=torch.randn(T, K, generator=g))


def feature_set(name, g, T, d, hd_valid, hot=None):
    """The side features of a case.  "mixed": categorical (padding = cardinality), a one-row table (padding -1), a sum bag
    of width 5 (padding 0), mean bags of widths 33 and 1, numerical widths 1 and 33, an identity feature.  "num64":
    numerical widths 32 + 31 + 1 = 64 columns.  "max16": 16 features of every kind.  "bert": the BERT form's kinds with
    padding -1, id 0 live.  hot: every token's first categorical id and first mean-bag id are ``hot``."""
    dt = d_true_of(d, hd_valid)
    ident = lambda: dict(kind=IDENT, width=dt, n_rows=0, padding_value=0, values=torch.randn(T, dt, generator=g))  # noqa: E731
    if name == "mixed":
        fs = [_cat(g, CAT, T, 1, 7, 7, d, hd_valid), _cat(g, CAT, T, 1, 1, -1, d, hd_valid),
              _cat(g, BAG_SUM, T, 5, 11, 0, d, hd_valid), _cat(g, BAG_MEAN, T, 33, 9, 9, d, hd_valid, p_pad=0.5),
              _cat(g, BAG_MEAN, T, 1, 4, 4, d, hd_valid), _num(g, T, 1, d, hd_valid), _num(g, T, 33, d, hd_valid), ident()]
        fs[3]["values"][: max(1, T // 10)] = 9            # all-padding mean bags
    elif name == "num64":
        fs = [_cat(g, BAG_MEAN, T, 3, 5, 5, d, hd_valid), _num(g, T, 32, d, hd_valid), _num(g, T, 31, d, hd_valid),
              _num(g, T, 1, d, hd_valid)]
    elif name == "max16":
        fs = [_cat(g, CAT, T, 1, 3 + i, 3 + i, d, hd_valid) for i in range(4)]
        fs += [_cat(g, BAG_SUM, T, 2 + i, 6, 0, d, hd_valid) for i in range(3)]
        fs += [_cat(g, BAG_MEAN, T, 3 + 2 * i, 5, 5, d, hd_valid) for i in range(3)]
        fs += [_num(g, T, 16, d, hd_valid) for _ in range(4)] + [ident(), ident()]
    elif name == "bert":
        fs = [_cat(g, CAT, T, 1, 7, -1, d, hd_valid, p_pad=0.0), _cat(g, CAT, T, 1, 1, -1, d, hd_valid, p_pad=0.0), ident()]
    else:
        raise ValueError(name)
    if hot is not None:
        cats = [f for f in fs if f["kind"] == CAT]
        means = [f for f in fs if f["kind"] == BAG_MEAN]
        for f in cats[:1] + means[:1]:
            f["values"][:, 0] = hot
    col = 0
    for f in fs:
        if f["kind"] == NUM:
            f["val_col"] = col
            col += f["width"]
        else:
            f["val_col"] = 0
    return fs


def make_case(d, hd_valid, T, L, p=0.0, feats="mixed", seed=0, hot=None, use_ptr=True):
    """One sum-form (or BERT-form) problem in the engine's padded layout: T tokens of L positions, pos0 = 3, scale =
    sqrt(true d) as an fp32, the item table's last row the zero padding row."""
    g = torch.Generator().manual_seed(seed * 1000 + d + hd_valid)
    n_items = 500
    item = padded(g, n_items + 1, d, hd_valid, 0.1)
    item[n_items] = 0
    ids = torch.randint(0, n_items + 1, (T,), generator=g).to(torch.int32)
    pos0 = 3
    return dict(d=d, hd_valid=hd_valid, T=T, L=L, p=p, pos0=pos0, scale=f32(math.sqrt(d_true_of(d, hd_valid))),
                seed_eff=SEED + (COUNTER if p > 0 and use_ptr else 0), drop_off=DROP_OFF, use_ptr=use_ptr,
                n_items=n_items, item=item.to(torch.bfloat16), pos=padded(g, pos0 + L, d, hd_valid, 0.1), ids=ids,
                feats=feature_set(feats, g, T, d, hd_valid, hot))


def make_concat_case(d, hd_valid, T, L, p=0.0, seed=0):
    """A ConcatAggregator problem: segments of widths 11 (categorical), 13 (mean bag), the item's true features, 33 (sum
    bag), 64 (numerical) and 65 (identity), in that host order; kp as the engine pads it."""
    g = torch.Generator().manual_seed(seed * 1000 + d + hd_valid + 7)
    d_true = d_true_of(d, hd_valid)
    n_items = 400

    def unpadded(f, dim):   # the feature's table at its own width
        f["table"] = (torch.randn(f["n_rows"], dim, generator=g) * 0.1)
        if 0 <= f["padding_value"] < f["n_rows"]:
            f["table"][f["padding_value"]] = 0
        f["table"] = f["table"].to(torch.bfloat16)
        f["dim"] = dim
        return f

    fs = [unpadded(_cat(g, CAT, T, 1, 7, 7, 64, 0), 11), unpadded(_cat(g, BAG_MEAN, T, 5, 9, 0, 64, 0, p_pad=0.4), 13),
          unpadded(_cat(g, BAG_SUM, T, 3, 6, 6, 64, 0), 33)]
    fs[1]["values"][: max(1, T // 10)] = 0   # all-padding mean bags
    nf = _num(g, T, 7, 64, 0)
    nf.update(dim=64, val_col=0)
    fs.append(nf)
    fs.append(dict(kind=IDENT, width=65, dim=65, n_rows=0, padding_value=0, values=torch.randn(T, 65, generator=g)))
    for f in fs:
        f.setdefault("val_col", 0)
    col, item_col = 0, 0
    for k, f in enumerate(fs):
        if k == 2:
            item_col, col = col, col + d_true
        f["col"] = col
        col += f["dim"]
    width = col
    kp = 64 if width <= 64 else -(-width // 128) * 128
    item = padded(g, n_items + 1, d, hd_valid, 0.1)
    item[n_items] = 0
    ids = torch.randint(0, n_items + 1, (T,), generator=g).to(torch.int32)
    pos0 = 2
    return dict(d=d, hd_valid=hd_valid, T=T, L=L, p=p, pos0=pos0, scale=f32(math.sqrt(d_true)), seed_eff=SEED + COUNTER,
                drop_off=DROP_OFF, use_ptr=True, n_items=n_items, pad_id=n_items, item=item.to(torch.bfloat16),
                pos=padded(g, pos0 + L, d, hd_valid, 0.1), ids=ids, feats=fs, item_col=item_col, width=width, kp=kp)


def row_plan(T, n, seed=0):
    """int32 [T] row_tok: n distinct tokens in shuffled order, then valid but wrong tokens (repeats) past the count"""
    g = torch.Generator().manual_seed(seed + 17 * T + n)
    rt = torch.randperm(T, generator=g)
    tail = torch.randint(0, T, (T - n,), generator=g)
    return torch.cat([rt[:n], tail]).to(torch.int32)
