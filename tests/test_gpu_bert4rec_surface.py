"""GPU tests of BERT4Rec's repeated block passes, the model without positional embedding, catalog growth and the
inference-only forward / get_logits: against the reference's goldens (tolerances of test_gpu_bert4rec.py), against a
float64 restatement with the engine's dropout masks (tolerances of test_gpu_bert_body.py), and against the mirror itself
(graph-captured vs eager steps, checkpoint round trips)."""
import math
import os

import numpy as np
import pytest
import torch

from dropout_stream import drop_keep, keep_draws
from fp64_checks import block_err, seq_block_err

pytestmark = pytest.mark.gpu

CASES = ["bert4rec_p2_d64h2.npz", "bert4rec_nopos_tied.npz", "bert4rec_p3_nopos_d96h2.npz"]
_BLK = ("ln1_w", "ln1_b", "in_w", "in_b", "out_w", "out_b", "ln2_w", "ln2_b", "w1", "b1", "w2", "b2")
SEED, P_DROP = 0x5EED1234ABC, 0.1
TOL_LOSS, TOL_HID, TOL_GRAD = 2e-4, 1.6e-2, 5e-2   # test_gpu_bert_body.py's step tolerances


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda")


def _cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def _flat(P):
    out = [(k, P[k]) for k in ("item_emb", "mask_emb", "pos_emb") if k in P]
    for i, b in enumerate(P["blocks"]):
        out += [(f"b{i}.{k}", b[k]) for k in _BLK]
    if "head_w" in P:
        out.append(("head_w", P["head_w"]))
    out.append(("head_b", P["head_b"]))
    return out


def _map(P, f):
    Q = {k: f(k, v) for k, v in P.items() if k != "blocks"}
    Q["blocks"] = [{k: f(f"b{i}.{k}", v) for k, v in blk.items()} for i, blk in enumerate(P["blocks"])]
    return Q


def _golden(golden_dir, name):
    from oracle import bert4rec_passes as op

    z = np.load(os.path.join(golden_dir, name))
    P = op.params_from_state_dict(op.golden_state_dict(z))
    return z, P


def _schema(n_items, d):
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    return TensorSchema(TensorFeatureInfo("item_id", n_items, 0, d))


def _cfg(z, **kw):
    from replay_b200.engine_bert import BertConfig

    L = int(z["L"])
    return BertConfig(n_items=int(z["n_items"]), d=int(z["d"]), n_heads=int(z["H"]), n_blocks=int(z["n_blocks"]), max_len=L,
                      tying=bool(int(z["tying"])), passes=int(z["passes"]), positional=bool(int(z["positional"])), **kw)


# ----------------------------------------------------------------------------------------------------------------------
# golden parity
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_train_step_and_predict_match_reference(golden_dir, cuda, name):
    """Hidden states, loss, every gradient (a repeated block's is the sum over its passes) and predict's logits."""
    from oracle import bert4rec_passes as op
    from replay_b200.engine_bert import Bert4RecEngine
    from replay_b200.models.nn.sequential import Bert4Rec

    z, P = _golden(golden_dir, name)
    B, L = z["ids"].shape
    cfg = _cfg(z, dropout=0.0)
    eng = Bert4RecEngine(cfg, B, L, cuda)
    assert len(eng.act) == cfg.n_blocks * cfg.passes and len(eng.x) == len(eng.act) + 1
    eng.load_canonical(P)
    ids, pm, tok, labels = (torch.from_numpy(z[k]).cuda() for k in ("ids", "pad_mask", "token_mask", "labels"))
    eng.set_batch(ids, pm, tok, labels)
    hid = eng.unpad_features(eng.forward_hidden_all()).float().cpu().view(B, L, -1)
    real = torch.from_numpy(z["pad_mask"])
    # bf16 activations through up to 4 block applications: per-row norm-relative (pad query rows are never consumed)
    ref_h = torch.from_numpy(z["train_hidden"])[real]
    assert float(((hid[real] - ref_h).norm(dim=-1) / ref_h.norm(dim=-1)).max()) < 1.5e-2
    loss = eng.forward_train()
    torch.cuda.synchronize()
    ref_loss = float(z["train_loss"])
    assert abs(loss[0].item() - ref_loss) < 5e-3 * ref_loss, (loss[0].item(), ref_loss)
    eng.g32.zero_()
    eng.backward()
    torch.cuda.synchronize()
    Gref = op.params_from_state_dict({k[6:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("grad::")})
    G = eng.export_canonical(eng.grads)
    assert [n for n, _ in _flat(G)] == [n for n, _ in _flat(Gref)]
    bad = []
    for (nm, a), (_, b) in zip(_flat(G), _flat(Gref)):
        if b.norm() < 1e-12:
            assert a.norm() < 1e-6, nm
            continue
        c, r = _cos(a, b), float(a.double().norm() / b.double().norm())
        if c < 0.995 or abs(r - 1) > 0.03:
            bad.append((nm, round(c, 5), round(r, 4)))
    assert not bad, bad

    # predict through the Lightning mirror (reference checkpoint keys), against the reference's predict()
    m = Bert4Rec(_schema(cfg.n_items, cfg.d), block_count=cfg.n_blocks, head_count=cfg.n_heads, hidden_size=cfg.d,
                 max_seq_len=L, dropout_rate=0.0, pass_per_transformer_block_count=cfg.passes,
                 enable_positional_embedding=cfg.positional, enable_embedding_tying=cfg.tying)
    sd = {"_model." + k: v for k, v in op.golden_state_dict(z).items()}
    m.load_state_dict(sd)
    assert set(m.state_dict()) == set(sd)
    scores = m({"item_id": ids}, pm, tok)
    ref = torch.from_numpy(z["eval_logits"])
    assert (scores.cpu() - ref).abs().max() < 0.1 * max(1.0, float(ref.abs().max()))


# ----------------------------------------------------------------------------------------------------------------------
# dropout: every application draws its own masks
# ----------------------------------------------------------------------------------------------------------------------
def _site(app, k):
    return 1 + app * 8 + k


def _ru(x, m):
    return (x + m - 1) // m * m


def _keeps(seed_eff, p, B, L, d, H, n_apps, site_of=lambda a: a):
    """Keep masks (0 or 1/(1-p), float64) of every dropout site of the training body; application a draws at site numbers
    _site(site_of(a), k).  site_of = block index instead of application index is the mistake of sharing masks."""
    T, Lp, ks = B * L, _ru(L, 64), 1.0 / (1.0 - float(np.float32(p)))
    rows = np.arange(T)

    def tok(off, n):
        return (keep_draws(seed_eff, off, p, rows, n).double() * ks).view(B, L, n).cuda()

    out = {"emb": tok(0, d), "apps": []}
    for a in range(n_apps):
        s = lambda k: _site(site_of(a), k) << 40  # noqa: E731
        out["apps"].append({"attn": drop_keep(seed_eff, s(0), p, B, H, L, Lp).cuda(), "out": tok(s(1), d),
                            "gelu": tok(s(2), 4 * d), "ffn": tok(s(3), d), "blk": tok(s(4), d)})
    return out


def _ln64(x, w, b, eps=1e-5):
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + eps) * w + b


def _ref(P, ids, pad, tok, labels, H, passes, keeps):
    """float64 BERT4Rec training loss with every dropout site, blocks applied ``passes`` times -> (loss, hidden)."""
    B, L = ids.shape
    d = P["item_emb"].shape[1]
    hd = d // H
    x = torch.where(tok[..., None], P["item_emb"][ids], P["mask_emb"].expand(B, L, d))
    if "pos_emb" in P:
        x = x + P["pos_emb"][:L]
    x = x * keeps["emb"]
    vis = pad[:, None, None, :]
    for a in range(len(P["blocks"]) * passes):
        blk, kb = P["blocks"][a // passes], keeps["apps"][a]
        xn = _ln64(x, blk["ln1_w"], blk["ln1_b"])
        qkv = xn @ blk["in_w"].T + blk["in_b"]
        q, k, v = (qkv[..., j * d:(j + 1) * d].reshape(B, L, H, hd).transpose(1, 2) for j in range(3))
        s = ((q @ k.transpose(-1, -2)) / math.sqrt(hd)).masked_fill(~vis, float("-inf"))
        pr = torch.softmax(s, -1) * kb["attn"]
        o = (pr @ v).transpose(1, 2).reshape(B, L, d)
        y = x + (o @ blk["out_w"].T + blk["out_b"]) * kb["out"]
        pre = _ln64(y, blk["ln2_w"], blk["ln2_b"]) @ blk["w1"].T + blk["b1"]
        u = 0.5 * pre * (1.0 + torch.erf(pre / math.sqrt(2.0))) * kb["gelu"]
        x = (y + (u @ blk["w2"].T + blk["b2"]) * kb["ffn"]) * kb["blk"]
    w = P["head_w"] if "head_w" in P else P["item_emb"]
    sel = pad & ~tok
    logits = x[sel] @ w.T + P["head_b"]
    y = labels[sel]
    return (torch.logsumexp(logits, -1) - logits.gather(1, y[:, None])[:, 0]).mean(), x


def _ref_grads(P, ids, pad, tok, labels, H, passes, keeps):
    Q = _map(P, lambda k, v: v.detach().double().cuda().clone().requires_grad_(True))
    loss, h = _ref(Q, ids, pad, tok, labels, H, passes, keeps)
    leaves = _flat(Q)
    grads = torch.autograd.grad(loss, [t for _, t in leaves])
    return float(loss), h.detach(), {k: g for (k, _), g in zip(leaves, grads)}


def _random_params(I, d, L, n_blocks, tied, positional, seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    P = {"item_emb": r(I, d) * 0.5, "mask_emb": r(1, d) * 0.5, "blocks": []}
    if positional:
        P["pos_emb"] = r(L, d) * 0.3
    for _ in range(n_blocks):
        P["blocks"].append({"ln1_w": 1 + 0.1 * r(d), "ln1_b": 0.1 * r(d), "in_w": r(3 * d, d) / math.sqrt(d),
                            "in_b": 0.05 * r(3 * d), "out_w": r(d, d) / math.sqrt(d), "out_b": 0.05 * r(d),
                            "ln2_w": 1 + 0.1 * r(d), "ln2_b": 0.1 * r(d), "w1": r(4 * d, d) / math.sqrt(d),
                            "b1": 0.05 * r(4 * d), "w2": r(d, 4 * d) / math.sqrt(4 * d), "b2": 0.05 * r(d)})
    if not tied:
        P["head_w"] = r(I, d) / math.sqrt(d)
    P["head_b"] = 0.5 * r(I)
    return P


_BF16 = ("item_emb", "mask_emb", "head_w", "in_w", "out_w", "w1", "w2")


def _engine_view(P):
    """the parameters as the engine computes with them: the bf16-consumed ones rounded"""
    return _map(P, lambda k, v: v.to(torch.bfloat16).float() if k.split(".")[-1] in _BF16 else v.float())


def _batch(B, L, I, seed):
    from replay_b200.models.nn.sequential.bert4rec import uniform_masker

    g = torch.Generator().manual_seed(seed)
    lengths = [L, L, 150, 57, 13, 1, 120][:B]
    pad = torch.zeros(B, L, dtype=torch.bool)
    for b, n in enumerate(lengths):
        pad[b, L - min(n, L):] = True
    items = torch.randint(0, I, (B, L), generator=g)
    tok = uniform_masker(pad, 0.2, g)
    tok[B // 2:, -1] = False
    ids = torch.where(pad, items, torch.zeros_like(items))
    labels = torch.where(pad & ~tok, items, torch.zeros_like(items))
    return ids, pad, tok, labels


@pytest.mark.parametrize("positional", [True, False])
def test_two_passes_with_dropout_match_fp64(cuda, positional):
    """d 128, 2 heads (fused attention backward), L 200, 2 blocks x 2 passes, dropout 0.1: the engine against the float64
    restatement with the ported keep masks at the application-indexed sites.  The same restatement with the masks of a
    block shared by its passes is far outside the tolerances, so each application draws its own masks."""
    from replay_b200.engine_bert import Bert4RecEngine, BertConfig

    B, L, I, nb, d, H, p = 7, 200, 2000, 2, 128, 2, 2
    P = _random_params(I, d, L, nb, False, positional, seed=5)
    ids, pad, tok, labels = _batch(B, L, I, seed=6)
    cfg = BertConfig(n_items=I, d=d, n_heads=H, n_blocks=nb, max_len=L, dropout=P_DROP, passes=p, positional=positional)
    eng = Bert4RecEngine(cfg, B, L, cuda, seed=SEED)
    eng.load_canonical(P)
    eng.tick_rng()
    ctr = int(eng.rng_counter.item())
    eng.set_batch(ids.cuda(), pad.cuda(), tok.cuda(), labels.cuda())
    loss = eng.forward_train()
    hid = eng.x[-1].view(B, L, d).double()
    eng.g32.zero_()
    eng.backward()
    torch.cuda.synchronize()
    G = eng.export_canonical(eng.grads)

    Pe = _engine_view(P)
    args = (ids.cuda(), pad.cuda(), tok.cuda(), labels.cuda(), H, p)
    r_loss, r_h, r_G = _ref_grads(Pe, *args, _keeps(eng.seed + ctr, P_DROP, B, L, d, H, nb * p))
    assert abs(loss[0].item() - r_loss) / r_loss < TOL_LOSS
    assert seq_block_err(hid, r_h, pad.cuda()) < TOL_HID
    bad = []
    for name, g in _flat(G):
        g, r = g.cuda().double(), r_G[name]
        if name.endswith("in_b"):   # a key bias cannot change a softmax: compare the query and value thirds
            g, r = torch.cat([g[:d], g[2 * d:]]), torch.cat([r[:d], r[2 * d:]])
        e = block_err(g.reshape(g.shape[0], -1) if g.dim() > 1 else g.view(-1, 1),
                      r.reshape(r.shape[0], -1) if r.dim() > 1 else r.view(-1, 1))
        if e >= TOL_GRAD:
            bad.append((name, round(e, 4)))
    assert not bad, bad

    shared = _keeps(eng.seed + ctr, P_DROP, B, L, d, H, nb * p, site_of=lambda a: a // p)
    with torch.no_grad():
        _, s_h = _ref(_map(Pe, lambda k, v: v.double().cuda()), *args, shared)
    assert seq_block_err(hid, s_h, pad.cuda()) > 10 * TOL_HID


# ----------------------------------------------------------------------------------------------------------------------
# the mirror: captured steps, convergence, forward / get_logits
# ----------------------------------------------------------------------------------------------------------------------
def _mirror(n_items, d, H, L, passes=2, positional=True, tying=False, dropout=0.1, loss_type="CE"):
    from replay_b200.models.nn.sequential import Bert4Rec

    return Bert4Rec(_schema(n_items, d), block_count=2, head_count=H, hidden_size=d, max_seq_len=L, dropout_rate=dropout,
                    pass_per_transformer_block_count=passes, enable_positional_embedding=positional,
                    enable_embedding_tying=tying, loss_type=loss_type)


def _train_batch(B, L, n_items, seed, lo=0, hi=None):
    from replay_b200.models.nn.sequential.bert4rec import uniform_masker

    g = torch.Generator().manual_seed(seed)
    hi = n_items if hi is None else hi
    lens = torch.randint(L // 4, L + 1, (B,), generator=g)
    pad = torch.arange(L)[None, :] >= (L - lens)[:, None]
    items = torch.randint(lo, hi, (B, L), generator=g)
    tok = uniform_masker(pad, 0.2, g)
    ids = torch.where(pad, items, torch.zeros_like(items))
    labels = torch.where(pad & ~tok, items, torch.zeros_like(items))
    return {"query_id": torch.arange(B), "inputs": {"item_id": ids.cuda()}, "pad_mask": pad.cuda(), "token_mask": tok.cuda(),
            "positive_labels": labels.cuda()}


def test_captured_step_equals_eager_step_at_two_passes(cuda):
    """Three fused steps with dropout replayed from the captured graphs against the same steps launched eagerly."""
    ms = [_mirror(500, 64, 2, 32) for _ in range(2)]
    ms[1].load_state_dict(ms[0].state_dict())
    batches = [_train_batch(16, 32, 500, seed=s) for s in range(3)]
    args = lambda b: (b["inputs"]["item_id"], b["pad_mask"], b["token_mask"], b["positive_labels"])  # noqa: E731
    l_eager = [float(ms[0]._model.core.fused_step(*args(b), all_reduce=None)) for b in batches]
    l_graph = [float(ms[1]._model.core.fused_step(*args(b))) for b in batches]
    assert ms[1]._model.core._trainer.use_graph
    # the embedding, LayerNorm and bias gradients accumulate with fp32 atomics, so the runs agree to rounding, not bitwise
    np.testing.assert_allclose(l_eager, l_graph, rtol=1e-4)
    s0, s1 = ms[0].state_dict(), ms[1].state_dict()
    for k in s0:
        diff = (s0[k] - s1[k]).abs()
        assert float(diff.max()) <= 3 * 1e-3 + 1e-6, k           # three Adam steps move an element by at most 3 lr
        assert float((diff > 1e-4).double().mean()) < 0.01, k    # and almost every element agrees closely
    init = _mirror(500, 64, 2, 32).state_dict()
    assert not torch.equal(s0["_model.transformer_blocks.1.attention.in_proj_weight"],
                           init["_model.transformer_blocks.1.attention.in_proj_weight"])


@pytest.mark.parametrize("positional", [True, False])
@pytest.mark.parametrize("tying", [False, True])
def test_dummy_bert_converges(cuda, positional, tying):
    """test_dummy_bert_converges' four (positional, tying) combinations, at two passes through the fused step: one fixed
    batch, the loss falls well below its start."""
    torch.manual_seed(0)
    m = _mirror(60, 64, 2, 16, passes=2, positional=positional, tying=tying, dropout=0.0)
    m._lr = 1e-2
    batch = _train_batch(32, 16, 60, seed=1)
    losses = [float(m.training_step(batch, i)) for i in range(60)]
    assert losses[-1] < 0.3 * losses[0], losses[::10]


@pytest.mark.parametrize("name", CASES)
def test_forward_and_get_logits_match_oracle(golden_dir, cuda, name):
    from oracle import bert4rec_passes as op
    from replay_b200.models.nn.sequential.bert4rec import Bert4RecModel

    z, P = _golden(golden_dir, name)
    cfg = _cfg(z)
    B, L = z["ids"].shape
    mdl = Bert4RecModel(_schema(cfg.n_items, cfg.d), max_len=L, hidden_size=cfg.d, num_blocks=cfg.n_blocks,
                        num_heads=cfg.n_heads, num_passes_over_block=cfg.passes, dropout=0.0,
                        enable_positional_embedding=cfg.positional, enable_embedding_tying=cfg.tying)
    mdl.load_state_dict(op.golden_state_dict(z))
    ids, pm, tok = (torch.from_numpy(z[k]) for k in ("ids", "pad_mask", "token_mask"))
    inputs = {"item_id": ids.cuda()}
    h = mdl.forward_step(inputs, pm.cuda(), tok.cuda())
    assert h.shape == (B, L, cfg.d) and h.dtype == torch.float32
    Pd = _map(P, lambda k, v: v.double())
    r_h = op.body(Pd, ids, pm, tok, cfg.n_heads, cfg.passes)
    real = pm
    assert float(((h.cpu().double()[real] - r_h[real]).norm(dim=-1) / r_h[real].norm(dim=-1)).max()) < 1.5e-2
    # the head on the model's own hidden states against the oracle's head on the same (bf16-exact) rows, over all items and
    # over candidates
    cands = torch.arange(3, cfg.n_items, 7)
    for item_ids in (None, cands):
        lg = mdl.get_logits(h, None if item_ids is None else item_ids.cuda())
        ref = op.logits(Pd, h.cpu().double(), item_ids)
        assert lg.shape == ref.shape
        assert (lg.cpu().double() - ref).abs().max() < 2e-2 * max(1.0, float(ref.abs().max()))
    full = mdl(inputs, pm.cuda(), tok.cuda())
    assert full.shape == (B, L, cfg.n_items)
    torch.testing.assert_close(full, mdl.get_logits(h))
    # the last position of forward equals predict
    torch.testing.assert_close(full[:, -1], mdl.predict(inputs, pm.cuda(), tok.cuda()), atol=1e-4, rtol=1e-4)


# ----------------------------------------------------------------------------------------------------------------------
# catalog growth
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tying", [False, True])
@pytest.mark.parametrize("op", ["by_size", "by_tensor", "append"])
def test_catalog_growth(golden_dir, cuda, tying, op):
    from replay_b200.models.nn.sequential import Bert4Rec

    n_items, d, L = 40, 64, 16
    m = _mirror(n_items, d, 2, L, passes=2, positional=True, tying=tying, dropout=0.1)
    m.candidates_to_score = torch.arange(5).cuda()
    m._lr = 5e-3
    for s in range(3):
        m.training_step(_train_batch(32, L, n_items, seed=s), s)
    core0 = m._model.core
    old = {k[len("_model."):]: v.cpu() for k, v in m.state_dict().items()}
    emb_key = "item_embedder.cat_embeddings.item_id.weight"
    new_rows = None
    if op == "by_size":
        m.set_item_embeddings_by_size(47)
    elif op == "by_tensor":
        t = torch.rand(45, d)
        m.set_item_embeddings_by_tensor(t)
        new_rows = t
    else:
        t = torch.rand(3, d)
        m.append_item_embeddings(t)
        new_rows = torch.cat([old[emb_key], t])
    n_new = {"by_size": 47, "by_tensor": 45, "append": 43}[op]
    assert m._vocab_size == n_new and m._model.item_count == n_new
    assert m._schema.item_id_features.item().cardinality == n_new
    core = m._model.core
    assert core is not core0 and core.cfg.n_items == n_new
    assert torch.equal(m.candidates_to_score, torch.arange(5).cuda())
    assert (core.cfg.passes, core.cfg.positional, core.loss_kind, core.adam_betas) == (2, True, "ce", core0.adam_betas)
    assert not core.engine.with_grad or not core.engine.adam_m.any()
    sd = {k[len("_model."):]: v.cpu() for k, v in m.state_dict().items()}
    # shapes equal the reference's after the same call
    z = np.load(os.path.join(golden_dir, "bert4rec_resize_shapes.npz"))
    tag = f"{'tied' if tying else 'untied'}_{op}::_model."
    ref_shapes = {k[len(tag):]: tuple(int(x) for x in z[k]) for k in z.files if k.startswith(tag)}
    assert {k: tuple(v.shape) for k, v in sd.items()} == ref_shapes
    # kept rows bitwise, provided rows bitwise
    E = sd[emb_key]
    if new_rows is not None:
        assert torch.equal(E, new_rows.float())
    else:
        assert torch.equal(E[:n_items], old[emb_key])
    for k, v in old.items():
        if k.startswith("_head.") and k in sd and "_item_embedder" not in k:
            assert torch.equal(sd[k][:n_items], v), k
        elif k != emb_key and "_item_embedder" not in k:
            assert torch.equal(sd[k], v), k
    assert torch.equal(m.get_all_embeddings()["item_embedding"].cpu(), E)
    assert torch.equal(m.get_all_embeddings()["positional_embedding"].cpu(), sd["item_embedder.position.pe.weight"])

    # training continues on batches labelled with new items, and the loss falls
    batch = _train_batch(32, L, n_new, seed=11, lo=n_items, hi=n_new)
    first = float(m.training_step(batch, 0))
    for i in range(1, 40):
        last = float(m.training_step(batch, i))
    assert last < 0.7 * first, (first, last)
    # predict_topk can return new items
    pb = {"query_id": batch["query_id"], "inputs": batch["inputs"], "pad_mask": batch["pad_mask"],
          "token_mask": batch["pad_mask"]}
    top, _ = m.predict_topk(pb, 5, candidates_to_score=torch.arange(n_new).cuda())
    assert (top >= n_items).any()
    # a fresh model on the grown schema that loads the checkpoint gives identical logits
    m2 = Bert4Rec(_schema(n_new, d), block_count=2, head_count=2, hidden_size=d, max_seq_len=L, dropout_rate=0.1,
                  pass_per_transformer_block_count=2, enable_embedding_tying=tying)
    m2.load_state_dict(m.state_dict())
    torch.testing.assert_close(m2.predict(pb, torch.arange(n_new).cuda()), m.predict(pb, torch.arange(n_new).cuda()),
                               atol=0, rtol=0)
