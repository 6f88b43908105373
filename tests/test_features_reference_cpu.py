"""tests/features_reference.py without a GPU: its restatement of the side-feature input stage against the oracle
(oracle/side_features.embed_sum, oracle/concat_features.embed_concat, tied to the real reference's goldens by the other CPU
tests) forward and, through autograd, backward on the golden specs with sum and mean bags; and its bounds' power to tell a
subtly wrong kernel from a right one: each mistake of features_reference.BUGS breaks a bound by at least ten times on the
inputs the GPU tests draw (tests/test_gpu_features_fp64.py, the same make_case shapes)."""
import os

import numpy as np
import pytest
import torch

import features_reference as fr
from oracle import concat_features as ocf
from oracle import sasrec as osr
from oracle import side_features as osf

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DISCRIMINATES = 10.0


def _layout(d, H):
    """(padded width, hd_valid) of d true features over H heads, as the engine lays them out"""
    hd = d // H
    slot = 64 if hd <= 64 else 128
    return H * slot, 0 if hd == slot else hd


def _pad(t, dp, hv):
    out = torch.zeros(t.shape[0], dp, dtype=t.dtype)
    out[:, fr.pad_cols(t.shape[1], hv)] = t
    return out


def _feats_of(z, specs):
    return {f["name"]: torch.from_numpy(z["feat::" + f["name"]]) for f in specs}


def _case_of(z, specs, P, feats, concat):
    """a features_reference case from a golden file's batch and weights (fp32 tables, p 0, scale 1, no positions)"""
    d, H = int(z["d"]), int(z["H"])
    dp, hv = _layout(d, H)
    ids = torch.from_numpy(z["ids"])
    T = ids.numel()
    method = str(z["method"])
    fs = []
    for f in specs:
        v = feats[f["name"]].reshape(T, -1)
        w = f["dim"] if concat else None
        if f["kind"] in ("cat", "bag"):
            kind = fr.CAT if f["kind"] == "cat" else fr.BAG_MEAN if method == "mean" else fr.BAG_SUM
            tab = P["side"][f["name"]]
            fs.append(dict(kind=kind, width=v.shape[1], n_rows=f["cardinality"] + 1, padding_value=f["padding_value"],
                           table=tab if concat else _pad(tab, dp, hv), values=v.to(torch.int32)))
        elif f["kind"] == "num":
            W, b = P["side"][f["name"] + ".w"], P["side"][f["name"] + ".b"]
            if not concat:
                W, b = _pad(W.T, dp, hv).T.contiguous(), _pad(b[None], dp, hv)[0]
            fs.append(dict(kind=fr.NUM, width=v.shape[1], table=W, bias=b, values=v.float()))
        else:
            fs.append(dict(kind=fr.IDENT, width=v.shape[1], values=v.float()))
        if concat:
            fs[-1]["dim"] = w
    n_items = int(z["n_items"])
    return dict(d=dp, hd_valid=hv, T=T, L=ids.shape[1], p=0.0, pos0=0, scale=1.0, seed_eff=0, drop_off=0, n_items=n_items,
                pad_id=n_items, item=_pad(P["item_emb"], dp, hv), pos=torch.zeros(ids.shape[1], dp),
                ids=ids.reshape(-1).to(torch.int32), feats=fs)


def _leaves(P):
    Pg = {k: v for k, v in P.items() if k != "blocks"}
    Pg["item_emb"] = P["item_emb"].double().requires_grad_(True)
    Pg["side"] = {k: v.double().requires_grad_(True) for k, v in P["side"].items()}
    for k in ("proj_w", "proj_b"):
        if k in P:
            Pg[k] = P[k].double()
    return Pg


def _oracle_feats(feats):
    return {k: (v if v.dtype in (torch.int32, torch.int64) else v.double()) for k, v in feats.items()}


@pytest.mark.parametrize("tag", ["d64h2_sum", "d50h1_mean"])
def test_sum_form_matches_the_oracle(tag):
    z = np.load(os.path.join(GOLDEN, f"sasrec_side_{tag}.npz"))
    specs = osf.golden_specs(z)
    sd = osf.golden_state_dict(z)
    P = osr.params_from_new_state_dict(sd)
    P["side"] = osf.side_from_state_dict(sd, specs)
    feats = _feats_of(z, specs)
    c = _case_of(z, specs, P, feats, concat=False)
    d, T = int(z["d"]), c["T"]
    fi = fr.pad_cols(d, c["hd_valid"])
    ids = torch.from_numpy(z["ids"])
    # forward: s (no scale, no positions, no dropout) against embed_sum, padded columns exactly zero
    s, _ = fr.forward(c)
    Pg = _leaves(P)
    want = osf.embed_sum(Pg, specs, ids, _oracle_feats(feats), str(z["method"]))
    assert torch.allclose(s[:, fi], want.detach().reshape(T, d), rtol=1e-12, atol=1e-12)
    pad = torch.ones(c["d"], dtype=torch.bool)
    pad[fi] = False
    assert not s[:, pad].any()
    # backward: the table contributions of dS against autograd through embed_sum (padding rows get nothing)
    dS = torch.randn(T, d, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    (want * dS.view(want.shape)).sum().backward()
    out = fr.backward(c, _pad(dS, c["d"], c["hd_valid"]))
    assert torch.equal(out["d_s"][:, fi], dS)
    n_cat = 0
    for k, f in enumerate(specs):
        if f["kind"] in ("cat", "bag"):
            con = out["tables"][k][0]
            assert torch.allclose(con[:, fi], Pg["side"][f["name"]].grad, rtol=1e-12, atol=1e-12), f["name"]
            assert not con[f["padding_value"]].any() and not con[:, pad].any()
            n_cat += 1
    assert n_cat == len(out["tables"]) > 0


@pytest.mark.parametrize("tag", ["d64h2", "d50h1_mean"])
def test_concat_form_matches_the_oracle(tag):
    z = np.load(os.path.join(GOLDEN, f"sasrec_concat_{tag}.npz"))
    specs = ocf.golden_specs(z)
    sd = osf.golden_state_dict(z)
    P = ocf.params_from_state_dict(sd, specs)
    feats = _feats_of(z, specs)
    c = _case_of(z, specs, P, feats, concat=True)
    d, T, item_name = int(z["d"]), c["T"], str(z["item_name"])
    dims = {f["name"]: f["dim"] for f in specs}
    dims[item_name] = d
    col = 0
    for name in sorted(dims):   # the reference concatenates in ascending name order
        if name == item_name:
            c["item_col"] = col
        else:
            next(f for f, s in zip(c["feats"], specs) if s["name"] == name)["col"] = col
        col += dims[name]
    c["width"] = col
    ids = torch.from_numpy(z["ids"])
    Pg = _leaves(P)
    want = ocf.embed_concat(Pg, specs, ids, _oracle_feats(feats), item_name, str(z["method"]))
    X = fr.concat_x(c)
    W, b = P["proj_w"].double(), P["proj_b"].double()
    assert torch.allclose(X @ W.T + b, want.detach().reshape(T, d), rtol=1e-12, atol=1e-12)
    # backward: dX = dY . W scattered into the item and side tables against autograd through embed_concat
    dY = torch.randn(T, d, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    (want * dY.view(want.shape)).sum().backward()
    out = fr.concat_scatter(c, dY @ W)
    fi = fr.pad_cols(d, c["hd_valid"])
    n_items = c["n_items"]
    con = out["item"][0]
    assert torch.allclose(con[:n_items][:, fi], Pg["item_emb"].grad[:n_items], rtol=1e-12, atol=1e-12)
    assert not con[n_items].any()
    for k, f in enumerate(specs):
        if f["kind"] in ("cat", "bag"):
            assert torch.allclose(out["tables"][k][0], Pg["side"][f["name"]].grad, rtol=1e-12, atol=1e-12), f["name"]


def test_dropout_is_keyed_by_the_token():
    c = fr.make_case(**fr.SUM_CASE, p=0.5)
    rows = fr.row_plan(c["T"], c["T"] - 1)[:c["T"] - 1]
    dense, _ = fr.forward(c)
    packed, _ = fr.forward(c, rows)
    assert torch.equal(packed, dense[rows.long()])
    real = fr.true_cols(c["d"], c["hd_valid"]) >= 0
    assert 0.4 < float((dense[:, real] == 0).double().mean()) < 0.6
    assert not dense[:, ~real].any()


# ------------------------------------------------------------------------------------------------ the bounds discriminate
FWD_BUGS = ["mean_by_width", "count_padding", "dedup", "scale_pos", "ident_padded_col", "no_bias", "w_transposed",
            "pos_no_pos0"]


def _worst(bad, ref, bound):
    return fr.ratio(bad.to(torch.bfloat16), ref, bound)


@pytest.mark.parametrize("bug", FWD_BUGS)
def test_forward_bound_catches(bug):
    c = fr.make_case(**fr.SUM_CASE, p=0.1)
    x, b = fr.forward(c)
    assert fr.ratio(x.to(torch.bfloat16), x, b) <= 1.0
    bad, _ = fr.forward(c, bug=bug)
    assert _worst(bad, x, b) >= DISCRIMINATES, bug


def test_forward_bound_catches_dropout_keyed_by_the_row():
    c = fr.make_case(**fr.SUM_CASE, p=0.1)
    rows = fr.row_plan(c["T"], c["T"] - 1)[:c["T"] - 1]
    x, b = fr.forward(c, rows)
    bad, _ = fr.forward(c, rows, bug="drop_key_row")
    assert _worst(bad, x, b) >= DISCRIMINATES
    y = torch.randn(c["T"] - 1, c["d"], generator=torch.Generator().manual_seed(2))
    x, b = fr.concat_embed_fwd(c, y, rows)
    bad, _ = fr.concat_embed_fwd(c, y, rows, bug="drop_key_row")
    assert _worst(bad, x, b) >= DISCRIMINATES


def _table_worst(ref, bad, start):
    con, ab, cnt = ref
    return fr.ratio(start + bad[0], start.double() + con, fr.table_bound(start, ab, cnt))


def test_table_bound_catches_the_mean_weight_applied_twice():
    c = fr.make_case(**fr.SUM_CASE, p=0.1)
    dx = torch.randn(c["T"], c["d"], generator=torch.Generator().manual_seed(5)).to(torch.bfloat16)
    ref = fr.backward(c, dx)
    bad = fr.backward(c, dx, bug="bwd_mean_twice")
    worst = 0.0
    for k, f in enumerate(c["feats"]):
        if f["kind"] == fr.BAG_MEAN:
            start = torch.randn(f["n_rows"], c["d"], generator=torch.Generator().manual_seed(k))
            worst = max(worst, _table_worst(ref["tables"][k], bad["tables"][k], start))
    assert worst >= DISCRIMINATES
    c = fr.make_concat_case(128, 0, 257, 13)
    dx = torch.randn(c["T"], c["kp"], generator=torch.Generator().manual_seed(5)).to(torch.bfloat16)
    ref = fr.concat_scatter(c, dx)
    bad = fr.concat_scatter(c, dx, bug="bwd_mean_twice")
    k = next(k for k, f in enumerate(c["feats"]) if f["kind"] == fr.BAG_MEAN)
    start = torch.randn(c["feats"][k]["n_rows"], c["feats"][k]["dim"], generator=torch.Generator().manual_seed(1))
    assert _table_worst(ref["tables"][k], bad["tables"][k], start) >= DISCRIMINATES


def test_table_bound_catches_the_item_segment_at_the_true_column():
    c = fr.make_concat_case(512, 75, 257, 13)
    dx = torch.randn(c["T"], c["kp"], generator=torch.Generator().manual_seed(5)).to(torch.bfloat16)
    ref = fr.concat_scatter(c, dx)
    bad = fr.concat_scatter(c, dx, bug="concat_item_col_j")
    start = torch.randn(c["n_items"] + 1, c["d"], generator=torch.Generator().manual_seed(1))
    assert _table_worst(ref["item"], bad["item"], start) >= DISCRIMINATES


def test_every_bug_is_exercised():
    named = set(FWD_BUGS) | {"drop_key_row", "bwd_mean_twice", "concat_item_col_j"}
    assert named == set(fr.BUGS)


def test_honest_fp32_sum_stays_inside_the_bound():
    """the forward summed in fp32 in another order (feature by feature, as torch does it) and rounded to bf16: inside
    the bound, so the bound leaves room for any summation order"""
    c = fr.make_case(**fr.SUM_CASE, p=0.1)
    x, b = fr.forward(c)
    toks = torch.arange(c["T"])
    s = c["item"].float()[c["ids"].long()]
    for f in reversed(c["feats"]):
        if f["kind"] in fr.CAT_KINDS:
            v = f["values"].long()
            w = fr.entry_weights(f, v).float()
            s = s + sum(f["table"].float()[v[:, j].clamp(0, f["n_rows"] - 1)] * w[:, j:j + 1] for j in range(v.shape[1]))
        elif f["kind"] == fr.NUM:
            s = s + (f["values"] @ f["table"].T + f["bias"])
        else:
            tc = fr.true_cols(c["d"], c["hd_valid"])
            vals = torch.zeros_like(s)
            vals[:, tc >= 0] = f["values"][:, tc[tc >= 0]]
            s = s + vals
    keep = fr.keep(c["seed_eff"], c["drop_off"], c["p"], toks, c["d"]).float()
    ks = np.float32(1.0) / (np.float32(1.0) - np.float32(c["p"]))
    y = (s * np.float32(c["scale"]) + c["pos"][c["pos0"] + toks % c["L"]]) * keep * float(ks)
    assert fr.ratio(y.to(torch.bfloat16), x, b) <= 1.0
