"""New-path SASRec training on packed rows against the padded rows, same engine and batch.

With the packed body (SasRecEngine.packed_eligible) every block runs on each sequence's live suffix only, stored back to back.
The rows it drops are exactly dead, so one training step must give the padded step's loss and gradients up to summation
order.  Covered: the config-2 shape on bench.py's seeded generator, all-padding and full-length sequences, live suffixes
around the 64- and 128-row tile edges, masks with interior holes, a batch that does not fill the engine, and a captured step
replayed on a batch with another packed row count.  The device row plan is checked against a host restatement.
"""
import pytest
import torch

from replay_b200.engine import EncoderConfig, SasRecEngine
from replay_b200.synthetic import make_sequences

pytestmark = pytest.mark.gpu

TOL = 1e-5   # norm-relative difference per tensor


def expected_plan(pad, tmask, labels, n_items):
    """Host restatement of rp_row_plan: first kept position of every sequence (its first real token or valid target; L if
    none), packed offsets, the token of every packed row and the packed row count."""
    B, L = pad.shape
    keep = pad | (tmask & (labels >= 0) & (labels < n_items))
    first = torch.where(keep.any(1), keep.int().argmax(1), torch.full((B,), L))
    n = L - first
    off = torch.cumsum(n, 0) - n
    row_tok = torch.cat([b * L + torch.arange(int(first[b]), L) for b in range(B)]) if int(n.sum()) else torch.zeros(0, dtype=torch.long)
    return first, off, row_tok, int(n.sum())


def _engine(B, L, n_items=2000, d=128, H=2, dropout=0.2, seed=3):
    cfg = EncoderConfig(n_items=n_items, d=d, n_heads=H, n_blocks=2, max_len=L, dropout=dropout)
    eng = SasRecEngine(cfg, max_batch=B, seq_len=L, device="cuda", seed=seed)
    with torch.no_grad():   # non-trivial LayerNorm parameters and biases
        g = torch.Generator(device="cpu").manual_seed(seed + 1)
        for k, t in eng.params.items():
            if t.dim() == 1:
                t.add_(0.1 * torch.randn(t.shape, generator=g).to(t.device))
    eng.refresh_shadow()
    eng.packed_body = True
    assert eng.packed_eligible()
    return eng


def _step(eng, batch, packed, rng=12345):
    eng.packed_body = packed
    eng.set_batch(*[t.cuda() for t in batch])
    eng.rng_counter.fill_(rng)
    eng.g32.zero_()
    loss = eng.forward_train()
    eng.backward()
    torch.cuda.synchronize()
    assert eng._packed == packed
    return float(loss[0]), {k: v.detach().clone() for k, v in eng.grads.items()}


def _rel(a, b):
    den = float(b.double().norm())
    return float((a.double() - b.double()).norm()) / max(den, 1e-30)


def _compare(eng, batch):
    loss_p, gp = _step(eng, batch, True)
    loss_u, gu = _step(eng, batch, False)
    assert abs(loss_p - loss_u) <= TOL * abs(loss_u), (loss_p, loss_u)
    worst = {k: _rel(gp[k], gu[k]) for k in gu}
    bad = {k: v for k, v in worst.items() if not v <= TOL}
    assert not bad, f"norm-relative gradient differences above {TOL}: {bad}"
    print(f"packed vs padded: loss {loss_p!r} / {loss_u!r}, largest norm-relative gradient difference {max(worst.values()):.3g}")
    return worst


def _check_plan(eng, batch, n_items):
    ids, pad, labels, tmask = batch
    eng.packed_body = True
    eng.set_batch(*[t.cuda() for t in batch])
    eng._prepare(True)
    torch.cuda.synchronize()
    first, off, row_tok, P = expected_plan(pad, tmask, labels, n_items)
    B = pad.shape[0]
    assert int(eng.n_rows[0]) == P
    assert torch.equal(eng.seq_first[:B].cpu().long(), first.long())
    assert torch.equal(eng.seq_off[:B].cpu().long(), off.long())
    assert torch.equal(eng.row_tok[:P].cpu().long(), row_tok.long())
    # every valid target maps to the packed row of its token
    nv = int(eng.n_valid[0])
    tok = eng.row_tok[eng.valid_rows[:nv].long()]
    assert torch.equal(tok.cpu(), eng.valid_idx[:nv].cpu())


def _windows(lengths, L, n_items, seed=0):
    """Left-padded windows whose live suffix (the real tokens and the target-only row before them) is n_b = lengths[b] rows."""
    g = torch.Generator().manual_seed(seed)
    B = len(lengths)
    ids = torch.full((B, L), n_items, dtype=torch.long)
    pad = torch.zeros(B, L, dtype=torch.bool)
    labels = torch.full((B, L), n_items, dtype=torch.long)
    tmask = torch.zeros(B, L, dtype=torch.bool)
    for b, n in enumerate(lengths):
        if n == 0:
            continue
        win = torch.randint(0, n_items, (n,), generator=g)
        k = n - 1 if n < L else n   # real tokens; n == L also covers a window without a target-only row
        if k:
            ids[b, L - k:] = win[n - k:] if k == n else win[:k]
            pad[b, L - k:] = True
        labels[b, L - n:] = win
        tmask[b, L - n:] = True
    return ids, pad, labels, tmask


def test_config2_seeded():
    B, L, I = 512, 200, 50_000
    eng = _engine(B, L, n_items=I)
    batch = make_sequences(B, I, L, seed=1234)
    _check_plan(eng, batch, I)
    _compare(eng, batch)


EDGE = [0, 1, 63, 64, 65, 127, 128, 129, 200, 0, 200, 2, 130, 199, 37]


def test_edge_lengths():
    L, I = 200, 3000
    eng = _engine(len(EDGE), L, n_items=I)
    batch = _windows(EDGE, L, I, seed=1)
    _check_plan(eng, batch, I)
    _compare(eng, batch)


def test_all_padding_batch_rows_and_partial_batch():
    # a batch smaller than the engine (rows past it are padding), with all-padding sequences among the live ones; the row
    # count is not a multiple of the 128-row tile
    L, I = 200, 3000
    eng = _engine(67, L, n_items=I)
    lengths = [0 if i % 5 == 0 else (i * 37) % L + 1 for i in range(61)]
    batch = _windows(lengths, L, I, seed=2)
    _check_plan(eng, batch, I)
    _compare(eng, batch)


def test_holes_and_other_length():
    # masks that are not left-padded: interior holes in the pad mask and targets, sequences starting with a hole
    L, I, B = 150, 3000, 45
    g = torch.Generator().manual_seed(5)
    ids = torch.randint(0, I, (B, L), generator=g)
    pad = torch.rand(B, L, generator=g) < 0.6
    pad[:5] = False
    pad[5:10] = True
    ids[~pad] = I
    labels = torch.randint(0, I, (B, L), generator=g)
    tmask = torch.rand(B, L, generator=g) < 0.5
    tmask[:3] = False
    eng = _engine(B, L, n_items=I)
    batch = (ids, pad, labels, tmask)
    _check_plan(eng, batch, I)
    _compare(eng, batch)


def test_graph_replay_other_row_count():
    L, I, B = 200, 3000, 96
    eng = _engine(B, L, n_items=I)
    a = make_sequences(B, I, L, seed=7)
    b = _windows([(i * 53) % (L + 1) for i in range(B)], L, I, seed=8)
    first_a = expected_plan(a[1], a[3], a[2], I)[3]
    first_b = expected_plan(b[1], b[3], b[2], I)[3]
    assert first_a != first_b
    eng.packed_body = True
    eng.rng_counter.fill_(999)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    eng.set_batch(*[t.cuda() for t in a])
    with torch.cuda.stream(s):
        for _ in range(2):
            eng.g32.zero_()
            eng.forward_train()
            eng.backward()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        eng.g32.zero_()
        loss = eng.forward_train()
        eng.backward()
    eng.set_batch(*[t.cuda() for t in b])
    graph.replay()
    torch.cuda.synchronize()
    loss_g = float(loss[0])
    grads_g = {k: v.detach().clone() for k, v in eng.grads.items()}
    assert int(eng.n_rows[0]) == first_b
    loss_e, grads_e = _step(eng, b, True, rng=999)
    assert loss_g == loss_e
    for k in grads_e:
        assert torch.equal(grads_g[k], grads_e[k]) or _rel(grads_g[k], grads_e[k]) <= TOL, k
