"""GPU tests of the full-catalog CE head and its per-row variants (rp_ce_head_fwd_w / rp_ce_head_bwd in csrc/rp_ce_head.cu:
LogOutCEWeighted and CEWeighted through row weights, LogInCE through loss_kind 1) against the float64 reference of
tests/ce_reference.py, element by element within its derived bounds.

Every path of the head runs every row kind: the fused pass with one column split (its direct completion) and with several
(ce_fused_finalize_kernel), the fused pass behind the two-pass forward (the logit bound failed), the un-fused head (two-pass
forward, MODE 0 dH pass) and the d = 512 head (materialised G, one chunk or 128-row chunks).  Each case asserts the path it is
named for.  Inputs are poisoned: hc rows past n_valid hold finite garbage, row weights past n_valid are NaN, d_hc rows past
n_valid and row / entry n_items of d_table / d_bias hold a sentinel that must survive.  Labels are in range everywhere."""
import os

import numpy as np
import pytest
import torch

import ce_reference as cr

pytestmark = pytest.mark.gpu

SENTINEL = 3.0
KINDS = sorted(cr.KINDS)
WORST = {}   # (path, kind) -> largest worst seen, printed at the end of the module


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from replay_b200 import ops as _ops

    yield _ops
    for key in sorted(WORST):
        print(f"worst {key[0]:>10} {key[1]:>9}: {WORST[key]:.3f}")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _run(ops, c, cap, n_valid, d, *, fused, hint, st=None, row_weight="case"):
    """one forward + backward on poisoned buffers -> CPU outputs and whether the fused pass ran"""
    dev = torch.device("cuda")
    I = c["W"].shape[0]
    h, W, lab = c["h"].to(dev), c["W"].to(dev), c["labels"].to(dev, torch.int32)
    b = None
    if c["b"] is not None:
        b = torch.full((cr.cdiv(I, 128) * 128,), 7.0)   # entries past n_items are never an item's bias
        b[:I] = c["b"]
        b = b.to(dev)
    rw = c["row_weight"] if row_weight == "case" else row_weight
    rw = rw.to(dev) if rw is not None else None
    nv = torch.tensor([n_valid], dtype=torch.int32, device=dev)
    st = st or ops.CEHeadState(cap, I, d, dev)
    d_hc = torch.full((cap, d), SENTINEL, device=dev, dtype=torch.bfloat16)
    d_tab = torch.full((I + 1, d), SENTINEL, device=dev)
    d_b = torch.full((I + 1,), SENTINEL, device=dev) if b is not None else None
    loss = ops.ce_head_fwd(st, h, W, lab, nv, bias=b, d_hc=d_hc if fused else None, n_valid_hint=hint, row_weight=rw,
                           loss_kind=c["loss_kind"], log_eps=c["log_eps"], clamp=c["clamp"]).clone()
    taken = ops.ce_head_fused_taken(st) if fused and d <= 256 else None
    ops.ce_head_bwd(st, h, W, lab, nv, d_hc, d_tab, bias=b, d_bias=d_b, n_valid_hint=hint)
    torch.cuda.synchronize()
    return dict(loss=loss.cpu(), d_hc=d_hc.cpu(), d_table=d_tab.cpu(), d_bias=d_b.cpu() if d_b is not None else None,
                taken=taken)


def _check(got, ref, n_valid, key):
    I = ref["d_W"].shape[0]
    loss, inv = got["loss"][0].double(), got["loss"][1].double()
    assert abs(float(loss - ref["loss"])) <= float(ref["bound_loss"]), (float(loss), float(ref["loss"]))
    # 1 / T_v through the fast-math reciprocal: within 2 ulp
    assert abs(float(inv) - (1.0 / n_valid if n_valid else 0.0)) <= 2.0 ** -22 * (1.0 / max(n_valid, 1)), float(inv)
    w = [cr.worst(got["d_hc"][:n_valid], ref["d_h"], ref["bound_h"]),
         cr.worst(got["d_table"][:I], ref["d_W"], ref["bound_W"])]
    if got["d_bias"] is not None:
        w.append(cr.worst(got["d_bias"][:I], ref["d_b"], ref["bound_b"]))
        assert float(got["d_bias"][I]) == SENTINEL, "d_bias[n_items] was written"
    WORST[key] = max(WORST.get(key, 0.0), *w)
    assert max(w) <= 1.0, w
    assert (got["d_hc"][n_valid:] == SENTINEL).all(), "d_hc rows past n_valid were written"
    assert (got["d_table"][I] == SENTINEL).all(), "d_table row n_items was written"


def _path_shape(path, d, sms):
    """(capacity, n_valid, n_items, hint, fused, scale_h, scale_e) of a path"""
    ns = cr.NSTAGE[d]
    if path in ("P1", "behind_P1"):
        cap, nv, I, hint = cr.layout(ns + 1, d, "P1", sms)
    elif path in ("Pn", "behind_Pn"):
        cap, nv, I, hint = 128, 123, 20001, 123
    else:
        cap, nv, I, hint = cr.layout(ns + 1, d, "twopass", sms)
    scale = (2.0, 1.0) if path.startswith("behind") else (0.5, 0.3)
    return cap, nv, I, hint, path != "unfused", *scale


def _assert_path(path, got, cap, hint, I, sms):
    if path == "unfused":
        return
    assert got["taken"] == (not path.startswith("behind")), "the logit bound should " + ("fail" if "behind" in path else "hold")
    P = cr.fused_splits(cap, hint, I, sms)
    assert (P == 1) == path.endswith("P1"), P


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("d", [64, 128, 256])
@pytest.mark.parametrize("path", ["P1", "Pn", "behind_P1", "behind_Pn", "unfused"])
def test_every_path_and_row_kind(ops, path, d, bias, kind):
    """NSTAGE + 1 column tiles per CTA (P == 1, un-fused) or a 20 001-item catalog over 8 splits (P > 1); then a rerun
    must give the same loss and d_hc bit for bit"""
    sms = _sms()
    cap, nv, I, hint, fused, sh, se = _path_shape(path, d, sms)
    c = cr.make_case(cap, nv, I, d, bias=bias, kind=kind, scale_h=sh, scale_e=se)
    got = _run(ops, c, cap, nv, d, fused=fused, hint=hint)
    _assert_path(path, got, cap, hint, I, sms)
    _check(got, cr.case_reference(c, nv), nv, (path, kind))
    again = _run(ops, c, cap, nv, d, fused=fused, hint=hint)
    assert torch.equal(again["loss"], got["loss"]) and torch.equal(again["d_hc"], got["d_hc"])


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("chunks", ["one", "several"])
def test_wide_head_row_kinds(ops, chunks, bias, kind, monkeypatch):
    """d = 512: G materialised per token chunk with the row weight in its exponent offset, the weighted one-hot term in
    ce_dh_reduce_kernel and the label scatter"""
    if chunks == "several":
        monkeypatch.setenv("RP_CE_WIDE_G_BYTES", "1")   # the smallest budget: 128-row chunks
    cap, nv, I = 384, 300, 5003
    c = cr.make_case(cap, nv, I, 512, bias=bias, kind=kind)
    got = _run(ops, c, cap, nv, 512, fused=True, hint=nv)
    _check(got, cr.case_reference(c, nv), nv, ("d512", kind))


@pytest.mark.parametrize("kind", ["weighted", "login_w"])
@pytest.mark.parametrize("split", ["P1", "Pn", "twopass"])
@pytest.mark.parametrize("d,n_ct", [(d, n) for d in (64, 128, 256) for n in (1, cr.NSTAGE[d], cr.NSTAGE[d] + 1)])
def test_column_tiles_per_cta_with_row_weights(ops, d, n_ct, split, kind):
    """1, NSTAGE and NSTAGE + 1 column tiles per CTA, ragged last tiles, biased"""
    cap, nv, I, hint = cr.layout(n_ct, d, split, _sms())
    c = cr.make_case(cap, nv, I, d, bias=True, kind=kind, seed=1)
    got = _run(ops, c, cap, nv, d, fused=split != "twopass", hint=hint)
    if split != "twopass":
        assert got["taken"]
    _check(got, cr.case_reference(c, nv), nv, ("tiles", kind))


@pytest.mark.parametrize("kind", ["weighted", "login_lo"])
@pytest.mark.parametrize("d", [64, 128, 256, 512])
@pytest.mark.parametrize("cap,n_valid", [(384, n) for n in (0, 1, 127, 128, 129, 384)] + [(300, n) for n in (1, 129, 299, 300)])
def test_valid_row_counts(ops, cap, n_valid, d, kind):
    """T_v around the 128-row tiles, 0 and the whole capacity, also on a capacity off the 128-row grid (300)"""
    c = cr.make_case(cap, n_valid, 1031, d, bias=True, kind=kind, seed=2)
    got = _run(ops, c, cap, n_valid, d, fused=True, hint=n_valid)
    _check(got, cr.case_reference(c, n_valid), n_valid, ("n_valid", kind))
    if n_valid == 0:
        assert not got["d_table"][:1031].any() and not got["d_bias"][:1031].any()


@pytest.mark.parametrize("kind", ["plain", "weighted", "login_hi"])
@pytest.mark.parametrize("d", [64, 128, 256, 512])
@pytest.mark.parametrize("n_items", [1, 63, 65, 129, 20001])
def test_catalog_sizes(ops, n_items, d, kind):
    """a single item, catalogs around the 64-column split grid and the 128-column tiles, and 20 001 items"""
    cap, nv = 256, 200
    c = cr.make_case(cap, nv, n_items, d, bias=True, kind=kind, seed=3)
    got = _run(ops, c, cap, nv, d, fused=True, hint=nv)
    _check(got, cr.case_reference(c, nv), nv, ("n_items", kind))


@pytest.mark.parametrize("kind", ["plain", "weighted"])
@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("d", [64, 128, 256, 512])
def test_bias_trap(ops, d, fused, kind):
    """the item with the largest raw score of any row has bias -60: the dE pass exponentiates the raw score against lse (which
    holds the bias) and folds e^{b_i} into the item's row after its loop"""
    cap, nv, I = 512, 400, 3001
    c = cr.make_case(cap, nv, I, d, bias=True, kind=kind, seed=4, bias_trap=True)
    got = _run(ops, c, cap, nv, d, fused=fused, hint=nv)
    _check(got, cr.case_reference(c, nv), nv, ("bias_trap", kind))


@pytest.mark.parametrize("kind", ["weighted", "login_w"])
@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("d", [64, 128, 256, 512])
def test_bitwise_repeatable_with_distinct_labels(ops, d, fused, kind):
    """distinct labels: every item row takes at most one one-hot atomic, so d_table and d_bias repeat bit for bit too"""
    cap, nv, I = 640, 600, 5003
    c = cr.make_case(cap, nv, I, d, bias=True, kind=kind, seed=5, distinct_labels=True)
    a = _run(ops, c, cap, nv, d, fused=fused, hint=nv)
    b = _run(ops, c, cap, nv, d, fused=fused, hint=nv)
    for k in ("loss", "d_hc", "d_table", "d_bias"):
        assert torch.equal(a[k], b[k]), k
    _check(a, cr.case_reference(c, nv), nv, ("distinct", kind))


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("d", [64, 128, 256, 512])
def test_no_stale_row_weight(ops, d, fused):
    """a weighted forward, then a plain forward on the same state, then the backward: the backward reads the row weights
    from the workspace, so it must see the plain forward's, and equal a plain run on a fresh state"""
    cap, nv, I = 640, 600, 5003
    c = cr.make_case(cap, nv, I, d, bias=True, kind="weighted", seed=6, distinct_labels=True)
    plain = dict(c, row_weight=None)
    st = ops.CEHeadState(cap, I, d, "cuda")
    _run(ops, c, cap, nv, d, fused=fused, hint=nv, st=st)
    dev = torch.device("cuda")
    h, W, lab = c["h"].to(dev), c["W"].to(dev), c["labels"].to(dev, torch.int32)
    b = torch.full((cr.cdiv(I, 128) * 128,), 7.0)
    b[:I] = c["b"]
    b = b.to(dev)
    nv_d = torch.tensor([nv], dtype=torch.int32, device=dev)
    d_hc = torch.full((cap, d), SENTINEL, device=dev, dtype=torch.bfloat16)
    d_tab = torch.full((I + 1, d), SENTINEL, device=dev)
    d_b = torch.full((I + 1,), SENTINEL, device=dev)
    loss = ops.ce_head_fwd(st, h, W, lab, nv_d, bias=b, d_hc=d_hc if fused else None, n_valid_hint=nv).clone()
    ops.ce_head_bwd(st, h, W, lab, nv_d, d_hc, d_tab, bias=b, d_bias=d_b, n_valid_hint=nv)
    torch.cuda.synchronize()
    ref = _run(ops, plain, cap, nv, d, fused=fused, hint=nv)
    assert torch.equal(loss.cpu(), ref["loss"])
    assert torch.equal(d_hc.cpu(), ref["d_hc"])
    assert torch.equal(d_tab.cpu(), ref["d_table"]) and torch.equal(d_b.cpu(), ref["d_bias"])
    _check(ref, cr.case_reference(plain, nv), nv, ("stale", "plain"))


@pytest.mark.parametrize("loss", ["LogOutCEWeighted", "CEWeighted", "LogInCE"])
def test_engine_stages_row_weights(golden_dir, loss):
    """new-path SasRec, one forward at a batch whose valid targets are not contiguous: the head's compacted weights are the
    staged ones gathered at valid_idx (CEWeighted: the reference's broadcast mean), and the loss is the fp64 head's on the
    engine's gathered hidden rows and the table before the step"""
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from replay_b200.nn import loss as L
    from replay_b200.nn.sequential import SasRec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    z = np.load(os.path.join(golden_dir, "sasrec_new_tiny.npz"))
    sd = {k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd::")}
    n_items, d, Lmax = int(z["n_items"]), int(z["d"]), z["ids"].shape[1]
    model = SasRec.from_params(TensorSchema(TensorFeatureInfo("item_id", n_items, n_items, d)), embedding_dim=d,
                               num_heads=int(z["H"]), num_blocks=int(z["n_blocks"]), max_sequence_length=Lmax, dropout=0.0,
                               device="cuda")
    model.load_state_dict(sd)
    spec = {"LogOutCEWeighted": lambda: L.LogOutCEWeighted(cardinality=n_items, feature_name="w"),
            "CEWeighted": lambda: L.CEWeighted(feature_name="w"),
            "LogInCE": lambda: L.LogInCE(cardinality=n_items)}[loss]()
    model.loss = spec
    model.train()
    ids, pm = torch.from_numpy(z["ids"]).cuda(), torch.from_numpy(z["pad_mask"]).cuda()
    lab, tm = torch.from_numpy(z["labels"]).cuda(), torch.from_numpy(z["target_mask"]).cuda().clone()
    tm[:, 1::3] = False   # gaps inside every sequence: the valid targets are not contiguous
    g = torch.Generator().manual_seed(11)
    w = torch.rand(*tm.shape, 1, generator=g) * 3
    w[:, ::4] = 0.0
    w = w.cuda()
    out = model(feature_tensors={"item_id": ids, "w": w}, padding_mask=pm, positive_labels=lab.unsqueeze(-1),
                target_padding_mask=tm.unsqueeze(-1))
    torch.cuda.synchronize()
    eng = model.core.engine
    n = int(eng.n_valid.item())
    vi = eng.valid_idx[:n].long()
    assert n == int(tm.sum()) and not torch.equal(vi.cpu(), torch.arange(n))
    roww = None
    if loss != "LogInCE":
        roww = eng.roww_c[:n].cpu()
        want = spec.row_weights({"w": w}, tm).reshape(-1).to(torch.float32)[vi].cpu()
        assert torch.equal(roww, want)
    kind = 1 if loss == "LogInCE" else 0
    ref = cr.reference(eng.hc.cpu(), eng.params16["item_emb"][:n_items].cpu(), None, eng.labels_c.cpu(), n, roww, kind)
    assert abs(float(out["loss"]) - float(ref["loss"])) <= float(ref["bound_loss"]), (float(out["loss"]), float(ref["loss"]))
