"""Multi-positive targets on the H100 ([B, L, P] labels and target mask; P slots per position):
(a) the sampled head (rp_sampled_head_fwd / _bwd with num_positives > 1) against an fp64 restatement on compacted rows, at
    d 64 / 128 / 256, every negative layout, live-row counts on and off the 128-row tile edge, over a NaN-filled workspace;
(b) the engine's training step against the real reference's losses and gradients (tests/golden/multi_positive_losses.npz);
(c) [B, L, 1] against [B, L] bitwise, packed rows against padded rows, LightningModule's graph-replayed fused steps against
    eager steps, the DiffTransformer body;
(d) a config-2-shape step (L 200, d 128, 50 000 items) with P = 4, its head against fp64 on sampled rows."""
import ctypes
import os

import numpy as np
import pytest
import torch

from replay_b200._lib import SampledDesc, check, lib

pytestmark = pytest.mark.gpu
KIND = {"ce_sampled": 0, "bce_sampled": 1, "ce_sampled_weighted": 5}


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda")


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ----------------------------------------------------------------------------------------------------------------------
# (a) the head
# ----------------------------------------------------------------------------------------------------------------------
def _head_inputs(d, nv, cap, P, mode, N, n_items, dev, seed):
    g = torch.Generator().manual_seed(seed)
    L = 16
    hc = (torch.randn(cap, d, generator=g) * 0.5).to(torch.bfloat16)
    table = (torch.randn(n_items, d, generator=g) * 0.5).to(torch.bfloat16)
    lab = torch.randint(0, n_items, (cap, P), generator=g)
    slot = torch.rand(cap, P, generator=g) < 0.6
    slot[torch.arange(cap), torch.randint(0, P, (cap,), generator=g)] = True   # every live row has a set slot
    if P > 2:
        lab[3, 2] = lab[3, 0]                                                    # a duplicated id
    vi = torch.sort(torch.randperm(cap * 2, generator=g)[:cap]).values.to(torch.int32)   # flat b * L + l of each row
    rows = {0: 1, 1: cap * 2, 2: cap * 2 // L + 1}[mode]
    neg = torch.randint(0, n_items, (rows, N), generator=g)
    # collisions with a set non-first slot, a masked-out slot, and the ignore index
    if mode == 0:
        neg[0, 0], neg[0, 1], neg[0, 2] = lab[0, -1], lab[1, -1], 7
    else:
        r = vi.long() if mode == 1 else vi.long() // L
        neg[r, 0] = lab[:, P // 2]
        neg[r, 1] = lab[:, P - 1]
        neg[r[:5], 2] = 7
    w = torch.rand(cap, P, generator=g) * 2 - 0.5
    x = dict(hc=hc, table=table, lab=lab.to(torch.int32), slot=slot.to(torch.uint8), vi=vi, neg=neg, w=w, L=L)
    out = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in x.items()}
    out["n_pairs"] = torch.tensor([int(slot[:nv].sum())], dtype=torch.int32, device=dev)
    out["nv"] = torch.tensor([nv], dtype=torch.int32, device=dev)
    return out


def _run_head(x, kind, mode, N, n_items, P, stale=True):
    cap, d = x["hc"].shape
    ws_bytes = lib().rp_sampled_head_workspace_multi(cap, d, N, mode, P)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x["hc"].device)
    if stale:
        ws.view(torch.float32)[: ws_bytes // 4].fill_(float("nan"))
    loss = torch.zeros(2, dtype=torch.float32, device=x["hc"].device)
    sd = SampledDesc()
    sd.hc, sd.table, sd.labels, sd.valid_idx = x["hc"].data_ptr(), x["table"].data_ptr(), x["lab"].data_ptr(), x["vi"].data_ptr()
    sd.negatives, sd.n_valid = x["neg"].data_ptr(), x["nv"].data_ptr()
    sd.capacity, sd.n_items, sd.d, sd.n_neg, sd.neg_mode, sd.seq_len = cap, n_items, d, N, mode, x["L"]
    sd.kind, sd.ignore_index, sd.vocab_size, sd.log_eps, sd.clamp = KIND[kind], 7, n_items, 1e-6, 100.0
    sd.loss_out, sd.workspace, sd.workspace_bytes = loss.data_ptr(), ws.data_ptr(), ws_bytes
    sd.row_weight = x["w"].data_ptr()
    sd.num_positives, sd.slot_mask, sd.n_pairs = P, x["slot"].data_ptr(), x["n_pairs"].data_ptr()
    check(lib().rp_sampled_head_fwd(ctypes.byref(sd), _stream()), "rp_sampled_head_fwd")
    d_hc = torch.full((cap, d), float("nan"), dtype=torch.bfloat16, device=x["hc"].device)
    d_tab = torch.zeros(n_items, d, dtype=torch.float32, device=x["hc"].device)
    check(lib().rp_sampled_head_bwd(ctypes.byref(sd), d_hc.data_ptr(), d_tab.data_ptr(), _stream()), "rp_sampled_head_bwd")
    torch.cuda.synchronize()
    return loss.cpu(), d_hc.cpu(), d_tab.cpu()


def _ref_head(x, kind, mode, nv):
    """fp64 restatement over the compacted rows: every set slot is a pair scored against its row's negatives, which are
    masked against the row's whole label row and the ignore index."""
    hc = x["hc"][:nv].cpu().double().requires_grad_(True)
    tab = x["table"].cpu().double().requires_grad_(True)
    lab, slot = x["lab"][:nv].cpu().long(), x["slot"][:nv].cpu().bool()
    neg = x["neg"].cpu()
    vi = x["vi"][:nv].cpu().long()
    negr = neg[0].expand(nv, -1) if mode == 0 else (neg[vi] if mode == 1 else neg[vi // x["L"]])
    P = lab.shape[1]
    rr, kk = slot.nonzero(as_tuple=True)
    h = hc[rr]
    zp = (h * tab[lab[rr, kk]]).sum(-1)
    zn = torch.einsum("md,mnd->mn", h, tab[negr[rr]])
    hit = (lab[rr].unsqueeze(-1) == negr[rr].unsqueeze(-2)).any(-2) | (negr[rr] == 7)
    zn = zn.masked_fill(hit, -1e9)
    if kind == "bce_sampled":
        loss = -(torch.clamp(torch.log(torch.sigmoid(zp) + 1e-6), -100, 100).sum()
                 + torch.clamp(torch.log(1 - torch.sigmoid(zn) + 1e-6), -100, 100).sum()) / len(zp)
    else:
        ce = torch.logsumexp(torch.cat((zp.unsqueeze(-1), zn), -1), -1) - zp
        if kind == "ce_sampled_weighted":
            ce = ce * x["w"][:nv].cpu().double()[rr, kk]
        loss = ce.mean()
    loss.backward()
    return float(loss.detach()), hc.grad, tab.grad


@pytest.mark.parametrize("nv", [127, 128, 129, 300])
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("d", [64, 128, 256])
@pytest.mark.parametrize("kind", ["ce_sampled", "bce_sampled", "ce_sampled_weighted"])
def test_head_matches_fp64(cuda, kind, d, mode, nv):
    n_items, N, P, cap = 1500, 70, 5, 300
    x = _head_inputs(d, nv, cap, P, mode, N, n_items, cuda, seed=d + mode + nv)
    loss, d_hc, d_tab = _run_head(x, kind, mode, N, n_items, P)
    ref, g_hc, g_tab = _ref_head(x, kind, mode, nv)
    assert abs(float(loss[0]) - ref) <= 2e-3 * abs(ref) + 1e-5, (float(loss[0]), ref)
    assert abs(float(loss[1]) * int(x["n_pairs"]) - 1) < 1e-6
    scale = g_hc.abs().max()
    assert torch.isfinite(d_hc[:nv].float()).all()
    assert (d_hc[:nv].double() - g_hc).abs().max() <= 1e-2 * scale, float((d_hc[:nv].double() - g_hc).abs().max() / scale)
    tscale = g_tab.abs().max()
    assert (d_tab.double() - g_tab).abs().max() <= 1e-2 * tscale


def test_single_slot_desc_fields_are_the_plain_head(cuda):
    """num_positives 1 with a slot mask runs the single-positive kernels: bitwise the same as num_positives 0."""
    n_items, N, cap, d = 900, 40, 200, 64
    x = _head_inputs(d, 150, cap, 1, 0, N, n_items, cuda, seed=3)
    a = _run_head(x, "ce_sampled", 0, N, n_items, 1, stale=False)
    b = _run_head(x, "ce_sampled", 0, N, n_items, 0, stale=False)
    for u, v in zip(a, b):
        assert torch.equal(u.view(torch.uint8) if u.dtype == torch.bfloat16 else u, v.view(torch.uint8) if v.dtype == torch.bfloat16 else v)


# ----------------------------------------------------------------------------------------------------------------------
# (b) engine vs the reference's goldens
# ----------------------------------------------------------------------------------------------------------------------
CASES = [("bce", "none"), *[(k, s) for k in ("ce_sampled", "bce_sampled", "ce_sampled_weighted")
                            for s in ("shared", "perseq", "perpos")]]


def _load(golden_dir):
    z = np.load(os.path.join(golden_dir, "sasrec_new_tiny.npz"))
    sd = {k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd::")}
    return z, sd, np.load(os.path.join(golden_dir, "multi_positive_losses.npz"))


def _tiny_engine(z, sd, dev, packed=False):
    from oracle import sasrec as osr
    from replay_b200.engine import EncoderConfig, SasRecEngine
    B, L = z["ids"].shape
    cfg = EncoderConfig(n_items=int(z["n_items"]), d=int(z["d"]), n_heads=int(z["H"]), n_blocks=int(z["n_blocks"]), max_len=L,
                        dropout=0.0, variant="new")
    eng = SasRecEngine(cfg, B, L, dev)
    eng.load_canonical(osr.params_from_new_state_dict(sd))
    eng.packed_body = packed
    return eng


def _step(eng, z, lab, m, kind, neg=None, w=None, ign=5):
    if kind == "bce":
        eng.set_loss("bce")
    else:
        eng.set_loss(kind, n_neg=neg.shape[-1], neg_shape={1: "shared", 2: "perseq", 3: "perpos"}[neg.dim()], ignore_index=ign)
    eng.set_batch(torch.from_numpy(z["ids"]).cuda(), torch.from_numpy(z["pad_mask"]).cuda(), lab.cuda(), m.cuda())
    if neg is not None:
        eng.set_negatives(neg.cuda())
    if w is not None:
        eng.set_row_weights(w.cuda())
    loss = eng.forward_train()
    eng.g32.zero_()
    if kind != "bce":
        eng.grads["item_emb"].fill_(3.0)   # a sampled head owns (overwrites) the table gradient
    eng.backward()
    torch.cuda.synchronize()
    return float(loss[0]), eng.export_canonical(eng.grads)


def _cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def _golden_case(zm, kind, shape):
    neg = torch.from_numpy(zm["neg_" + shape]) if kind != "bce" else None
    w = torch.from_numpy(zm["weights"]) if kind == "ce_sampled_weighted" else None
    return torch.from_numpy(zm["labels"]), torch.from_numpy(zm["target_mask"]), neg, w


@pytest.mark.parametrize("kind,shape", CASES)
def test_engine_matches_reference_goldens(golden_dir, cuda, kind, shape):
    z, sd, zm = _load(golden_dir)
    eng = _tiny_engine(z, sd, cuda)
    lab, m, neg, w = _golden_case(zm, kind, shape)
    l, G = _step(eng, z, lab, m, kind, neg, w, int(zm["ignore_index"]))
    ref = float(zm[f"{kind}_{shape}_loss"])
    assert abs(l - ref) < 5e-3 * abs(ref), (l, ref)
    gE, gW = torch.from_numpy(zm[f"{kind}_{shape}_gE"]), torch.from_numpy(zm[f"{kind}_{shape}_gW"])
    for nm, a, b in (("item_emb", G["item_emb"].cpu(), gE), ("in_w", G["blocks"][0]["in_w"].cpu(), gW)):
        c, r = _cos(a, b), float(a.double().norm() / b.double().norm())
        assert c > 0.995 and abs(r - 1) < 0.03, (nm, c, r)


@pytest.mark.parametrize("kind,shape", [("bce", "none"), ("ce_sampled", "perpos"), ("ce_sampled_weighted", "shared")])
def test_packed_rows_match_padded(golden_dir, cuda, kind, shape):
    z, sd, zm = _load(golden_dir)
    lab, m, neg, w = _golden_case(zm, kind, shape)
    out = [_step(_tiny_engine(z, sd, cuda, packed=p), z, lab, m, kind, neg, w, int(zm["ignore_index"])) for p in (False, True)]
    assert abs(out[0][0] - out[1][0]) <= 1e-6 * abs(out[0][0])
    for nm in ("item_emb", "pos_emb", "lnf_w"):
        torch.testing.assert_close(out[1][1][nm], out[0][1][nm], rtol=1e-4, atol=1e-6)
    torch.testing.assert_close(out[1][1]["blocks"][0]["in_w"], out[0][1]["blocks"][0]["in_w"], rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("kind", ["bce", "ce_sampled", "bce_sampled", "ce_sampled_weighted"])
def test_single_slot_is_bitwise_the_plain_batch(golden_dir, cuda, kind):
    """[B, L, 1] runs the [B, L] code: bitwise equal where the engine reduces in a fixed order - the loss, the head's
    d(loss)/d(hidden) and the blocks' weight-matrix gradients (rp_wgrad_group) - and within rounding where fp32 atomics
    accumulate in arrival order (the item and positional tables' scatter, LayerNorm dw / db, bias column sums)."""
    z, sd, zm = _load(golden_dir)
    lab, tm = torch.from_numpy(z["labels"]), torch.from_numpy(z["target_mask"])
    neg = torch.from_numpy(zm["neg_perseq"]) if kind != "bce" else None
    w = torch.from_numpy(zm["weights"])[..., :1] if kind == "ce_sampled_weighted" else None
    eng = _tiny_engine(z, sd, cuda)
    out = []
    for L_, m_, w_ in ((lab.unsqueeze(-1), tm.unsqueeze(-1), w), (lab, tm, None if w is None else w[..., 0])):
        loss, G = _step(eng, z, L_, m_, kind, neg, w_)
        out.append((loss, G, eng.s["dhc"][: int(eng.n_valid)].clone()))
    (la, Ga, ha), (lb, Gb, hb) = out
    assert la == lb
    assert torch.equal(ha.view(torch.int16), hb.view(torch.int16))
    for blk_a, blk_b in zip(Ga["blocks"], Gb["blocks"]):
        for k in blk_a:
            if k in ("in_w", "out_w", "w1", "w2"):
                assert torch.equal(blk_a[k], blk_b[k]), k
            else:   # LayerNorm dw / db and bias column sums: fp32 atomics
                torch.testing.assert_close(blk_a[k], blk_b[k], rtol=1e-5, atol=1e-7)
    for nm in ("item_emb", "pos_emb", "lnf_w", "lnf_b"):
        torch.testing.assert_close(Ga[nm], Gb[nm], rtol=1e-5, atol=1e-7)


def test_far_apart_positives_stay_finite(cuda):
    """One positive of a position ~110 nats above another: every CE pair keeps its own log-sum-exp, so the low pair's
    softmax sum cannot flush to zero."""
    n_items, N, P, cap, d, nv = 600, 32, 2, 128, 64, 100
    x = _head_inputs(d, nv, cap, P, 0, N, n_items, cuda, seed=21)
    g = torch.Generator().manual_seed(21)
    hc = torch.zeros(cap, d)
    hc[:, 0] = 10.0
    tab = torch.randn(n_items, d, generator=g) * 0.01
    tab[:, 0] = 0.0
    tab[1, 0], tab[2, 0] = 10.0, -1.0            # z = 100 and z = -10
    x["hc"] = hc.to(cuda, torch.bfloat16)
    x["table"] = tab.to(cuda, torch.bfloat16)
    x["lab"] = torch.tensor([1, 2], dtype=torch.int32).repeat(cap, 1).to(cuda)
    x["slot"] = torch.ones(cap, P, dtype=torch.uint8, device=cuda)
    x["n_pairs"] = torch.tensor([nv * P], dtype=torch.int32, device=cuda)
    x["neg"] = torch.randint(10, n_items, (1, N), generator=g).to(cuda)
    for kind in ("ce_sampled", "ce_sampled_weighted"):
        loss, d_hc, d_tab = _run_head(x, kind, 0, N, n_items, P)
        ref, g_hc, g_tab = _ref_head(x, kind, 0, nv)
        assert np.isfinite(float(loss[0])) and torch.isfinite(d_hc[:nv].float()).all() and torch.isfinite(d_tab).all()
        assert abs(float(loss[0]) - ref) <= 2e-3 * abs(ref), (float(loss[0]), ref)
        assert (d_hc[:nv].double() - g_hc).abs().max() <= 1e-2 * g_hc.abs().max()
        assert (d_tab.double() - g_tab).abs().max() <= 1e-2 * g_tab.abs().max()


# ----------------------------------------------------------------------------------------------------------------------
# full-catalog BCE with positive sets: rp_bce_head_* on the first positive, rp_bce_head_multi_* on the rest
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d,fused", [(64, True), (128, True), (128, False), (256, True), (512, False)])
def test_bce_positive_sets_match_fp64(cuda, d, fused):
    from replay_b200 import ops

    cap, nv, n_items, P = 300, 257, 3000, 4
    g = torch.Generator().manual_seed(d + fused)
    h = (torch.randn(cap, d, generator=g) * 0.5).to(cuda, torch.bfloat16)
    W = (torch.randn(n_items, d, generator=g) * 0.3).to(cuda, torch.bfloat16)
    lab_p = torch.randint(0, n_items, (cap, P), generator=g)
    lab_p[::5, 2] = lab_p[::5, 1]                 # duplicated ids count once
    lab_p[::7, 3] = n_items + 4                   # ids outside the catalog are skipped
    lab_p[::11, 1] = -1
    lab0 = lab_p[:, 0].clone()                    # the row's positive scored by rp_bce_head_*
    lab_p, lab0 = lab_p.to(torch.int32).to(cuda), lab0.to(torch.int32).to(cuda)
    nvt = torch.tensor([nv], dtype=torch.int32, device=cuda)
    st = ops.CEHeadState(cap, n_items, d, cuda)
    d_hc = torch.full((cap, d), 3.0, device=cuda, dtype=torch.bfloat16)
    d_W = torch.full((n_items, d), 9.0, device=cuda)
    row_sum = torch.full((cap,), float("nan"), device=cuda)
    loss = ops.bce_head_fwd(st, h, W, lab0, nvt, d_hc=d_hc if fused else None)
    check(lib().rp_bce_head_multi_fwd(h.data_ptr(), W.data_ptr(), lab0.data_ptr(), lab_p.data_ptr(), nvt.data_ptr(), cap, P,
                                      n_items, d, loss.data_ptr(), row_sum.data_ptr(), _stream()), "rp_bce_head_multi_fwd")
    ops.bce_head_bwd(st, h, W, lab0, nvt, d_hc, d_W)
    check(lib().rp_bce_head_multi_bwd(h.data_ptr(), W.data_ptr(), lab0.data_ptr(), lab_p.data_ptr(), nvt.data_ptr(), cap, P,
                                      n_items, d, loss.data_ptr(), d_hc.data_ptr(), d_W.data_ptr(), _stream()),
          "rp_bce_head_multi_bwd")
    torch.cuda.synchronize()
    hr = h[:nv].double().cpu().requires_grad_(True)
    Wr = W.double().cpu().requires_grad_(True)
    tgt = torch.zeros(nv, n_items, dtype=torch.float64)
    lp = lab_p[:nv].long().cpu()
    ok = (lp >= 0) & (lp < n_items)
    tgt[torch.arange(nv).unsqueeze(-1).expand_as(lp)[ok], lp[ok]] = 1.0
    ref = torch.nn.functional.binary_cross_entropy_with_logits(hr @ Wr.T, tgt, reduction="sum") / nv
    ref.backward()
    assert abs(float(loss[0]) - float(ref)) <= 1e-4 * abs(float(ref)), (float(loss[0]), float(ref))
    assert (d_hc[:nv].double().cpu() - hr.grad).abs().max() <= 1e-2 * hr.grad.abs().max()
    assert (d_hc[nv:] == 3.0).all()
    assert (d_W.double().cpu() - Wr.grad).abs().max() <= 1e-2 * Wr.grad.abs().max()


# ----------------------------------------------------------------------------------------------------------------------
# (c) the public model
# ----------------------------------------------------------------------------------------------------------------------
def _spec(kind, ign):
    from replay_b200.nn.loss import BCE, BCESampled, CESampled, CESampledWeighted
    return {"bce": lambda: BCE(), "ce_sampled": lambda: CESampled(negative_labels_ignore_index=ign),
            "bce_sampled": lambda: BCESampled(negative_labels_ignore_index=ign),
            "ce_sampled_weighted": lambda: CESampledWeighted("w", negative_labels_ignore_index=ign)}[kind]()


def _model(z, sd):
    from replay_b200.nn.sequential import SasRec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema
    n_items, d, H, L = int(z["n_items"]), int(z["d"]), int(z["H"]), int(z["L"])
    m = SasRec.from_params(TensorSchema(TensorFeatureInfo("item_id", n_items, n_items, d)), embedding_dim=d, num_heads=H,
                           num_blocks=int(z["n_blocks"]), max_sequence_length=L, dropout=0.0)
    m.load_state_dict(sd)
    return m


@pytest.mark.parametrize("kind", ["bce", "ce_sampled", "ce_sampled_weighted"])
def test_lightning_steps_train_on_every_positive(golden_dir, cuda, kind):
    from oracle import sasrec as osr
    from replay_b200.nn.lightning import LightningModule, OptimizerFactory

    z, sd, zm = _load(golden_dir)
    ign = int(zm["ignore_index"])
    lab, m, _, _ = _golden_case(zm, kind, "perseq")
    neg = torch.from_numpy(zm["neg_perseq"]).cuda()
    w = torch.from_numpy(zm["weights"]).cuda()
    ids, pm = torch.from_numpy(z["ids"]).cuda(), torch.from_numpy(z["pad_mask"]).cuda()
    g = torch.Generator().manual_seed(9)
    lab2 = lab.clone()
    lab2[..., 1:] = torch.randint(0, int(z["n_items"]), lab[..., 1:].shape, generator=g)
    batches = [{"feature_tensors": {"item_id": ids, "w": w}, "padding_mask": pm, "positive_labels": L_.cuda(),
                "target_padding_mask": m.cuda(), "negative_labels": neg} for L_ in (lab, lab2)]
    model = _model(z, sd)
    model.loss = _spec(kind, ign)
    model.train()
    ref_eng = _tiny_engine(z, sd, cuda)

    def eager(b):
        return _step(ref_eng, z, b["positive_labels"].cpu(), b["target_padding_mask"].cpu(), kind,
                     None if kind == "bce" else b["negative_labels"].cpu(),
                     w.cpu() if kind == "ce_sampled_weighted" else None, ign)[0]

    # autograd forward against the eager engine; the first slot alone gives another loss
    out = float(model(**batches[0])["loss"])
    assert abs(out - eager(batches[0])) <= 1e-6 * abs(out)
    first = dict(batches[0], positive_labels=batches[0]["positive_labels"][..., :1],
                 target_padding_mask=batches[0]["target_padding_mask"][..., :1],
                 feature_tensors={"item_id": ids, "w": w[..., :1]})
    assert abs(float(model(**first)["loss"]) - out) > 1e-4 * abs(out)
    # fused steps: two eager, then captured and replayed, batches alternating; each against an eager engine step
    lm = LightningModule(model, optimizer_factory=OptimizerFactory(learning_rate=3e-3))
    losses = []
    for i in range(6):
        b = batches[i % 2]
        ref_eng.load_canonical(osr.params_from_new_state_dict(model.state_dict()))
        ref = eager(b)
        got = float(lm.training_step(b, i))
        assert abs(got - ref) <= 2e-5 * abs(ref), (i, got, ref)
        losses.append(got)
    assert losses[4] < losses[0] and losses[5] < losses[1], losses
    # back to one positive per position: the captured multi-positive step is not replayed
    ref_eng.load_canonical(osr.params_from_new_state_dict(model.state_dict()))
    ref = _step(ref_eng, z, lab[..., :1], m[..., :1], kind, None if kind == "bce" else neg.cpu(),
                w[..., :1].cpu() if kind == "ce_sampled_weighted" else None, ign)[0]
    got = float(lm.training_step(first, 6))
    assert abs(got - ref) <= 2e-5 * abs(ref), (got, ref)


def test_diff_body_takes_multi_positive_targets(cuda):
    from replay_b200.nn.loss import CESampled
    from test_gpu_diff_sasrec import _batch, _model as _diff_model

    n_items, d, H, L, B = 400, 64, 2, 50, 8
    ids, pm, labels, tm = (t.to(cuda) for t in _batch(B, L, n_items, seed=4))
    g = torch.Generator().manual_seed(2)
    lab = torch.stack([labels.cpu(), torch.randint(0, n_items, (B, L), generator=g)], -1).to(cuda)
    m2 = torch.stack([tm.cpu(), tm.cpu() & (torch.rand(B, L, generator=g) < 0.5)], -1).to(cuda)
    neg = torch.randint(0, n_items, (B, 32), generator=g).to(cuda)
    mdl = _diff_model(n_items, d, H, L, 2, "layernorm", seed=3)
    mdl.loss = CESampled()
    mdl.train()
    one = float(mdl(feature_tensors={"item_id": ids}, padding_mask=pm, positive_labels=lab[..., :1],
                    negative_labels=neg, target_padding_mask=m2[..., :1])["loss"])
    two = float(mdl(feature_tensors={"item_id": ids}, padding_mask=pm, positive_labels=lab, negative_labels=neg,
                    target_padding_mask=m2)["loss"])
    assert np.isfinite(two) and abs(two - one) > 1e-4 * abs(one)
    losses = [float(mdl.core.fused_step(ids, pm, lab, m2, all_reduce=None, lr=1e-2, negatives=neg)) for _ in range(6)]
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses


# ----------------------------------------------------------------------------------------------------------------------
# (d) config-2 shape
# ----------------------------------------------------------------------------------------------------------------------
def test_config2_shape_step_with_four_positives(cuda):
    """L 200, d 128, 2 heads, 50 000 items, P = 4, CESampled with 256 shared negatives: the head's loss from the engine's
    own final hidden states against fp64, and dH on 64 sampled rows."""
    from replay_b200.engine import EncoderConfig, SasRecEngine

    B, L, n_items, P, N = 64, 200, 50_000, 4, 256
    cfg = EncoderConfig(n_items=n_items, d=128, n_heads=2, n_blocks=2, max_len=L, dropout=0.2, variant="new")
    eng = SasRecEngine(cfg, B, L, cuda)
    g = torch.Generator().manual_seed(11)
    lens = torch.randint(1, L + 1, (B,), generator=g)
    pm = torch.arange(L).unsqueeze(0) >= (L - lens).unsqueeze(1)
    ids = torch.where(pm, torch.randint(0, n_items, (B, L), generator=g), torch.full((B, L), n_items))
    lab = torch.randint(0, n_items, (B, L, P), generator=g)
    m = pm.unsqueeze(-1) & (torch.rand(B, L, P, generator=g) < 0.5)
    m[..., 0] |= pm
    neg = torch.randint(0, n_items, (N,), generator=g)
    eng.set_loss("ce_sampled", n_neg=N, neg_shape="shared")
    eng.set_batch(ids.cuda(), pm.cuda(), lab.cuda(), m.cuda())
    eng.set_negatives(neg.cuda())
    loss = float(eng.forward_train()[0])
    eng.g32.zero_()
    eng._head_backward()   # d(loss)/d(hc) stays in s["dhc"]
    torch.cuda.synchronize()
    nv = int(eng.n_valid)
    assert nv == int(pm.sum()) and int(eng.mp["n_pairs"]) == int(m.sum())
    hc = eng.hc[:nv, : cfg.d].double().cpu()
    tab = eng.params16["item_emb"][:n_items, : cfg.d].double().cpu()
    lab_c = eng.mp["labels_p"][:nv].long().cpu()
    slot = eng.mp["slot"][:nv].bool().cpu()
    hcr = hc.clone().requires_grad_(True)
    rr, kk = slot.nonzero(as_tuple=True)
    zp = (hcr[rr] * tab[lab_c[rr, kk]]).sum(-1)
    zn = (hcr @ tab[neg].T)[rr]
    zn = zn.masked_fill((lab_c[rr].unsqueeze(-1) == neg.view(1, 1, -1)).any(-2), -1e9)
    ref = (torch.logsumexp(torch.cat((zp.unsqueeze(-1), zn), -1), -1) - zp).mean()
    ref.backward()
    assert abs(loss - float(ref)) <= 2e-3 * abs(float(ref)), (loss, float(ref))
    pick = torch.randperm(nv, generator=g)[:64]
    got = eng.s["dhc"][:nv, : cfg.d].double().cpu()[pick]
    want = hcr.grad[pick]
    assert (got - want).abs().max() <= 2e-2 * want.abs().max(), float((got - want).abs().max() / want.abs().max())
