"""GPU tests of the scalable cross-entropy head (rp_sce_head_*, legacy SasRec loss_type="SCE"): against the REAL reference
(tests/golden/sce_losses.npz, its captured draw replayed), against an fp64 restatement (oracle/sce.py) at the config-2 model
shape and at d = 512, determinism and CUDA-graph replay, and the public module."""
import os

import numpy as np
import pytest
import torch

from fp64_checks import block_err

pytestmark = pytest.mark.gpu

CASES = ["nomix", "mix", "bigx", "overlap", "fullcollide", "r111", "r221"]


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda")


def _cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def _engine(cfg_kw, B, L, cuda, P, sce, seed=0):
    from replay_b200.engine import EncoderConfig, SasRecEngine
    eng = SasRecEngine(EncoderConfig(max_len=L, dropout=0.0, variant="legacy", **cfg_kw), B, L, cuda, seed=seed)
    eng.load_canonical(P)
    n_b, bsx, bsy, mix = sce
    eng.set_loss("sce", n_buckets=n_b, bucket_size_x=bsx, bucket_size_y=bsy, mix_x=bool(mix))
    return eng


def _step(eng, ids, pm, lab):
    eng.set_batch(ids.cuda(), pm.cuda(), lab.cuda(), pm.cuda())
    loss = eng.forward_train()
    eng.g32.zero_()
    eng.grads["item_emb"].fill_(3.0)   # the SCE branch owns the table gradient: it must be zeroed, not accumulated into
    eng.backward()
    torch.cuda.synchronize()
    return loss.clone()


def _real_sets(top, pm):
    return [sorted(int(t) for t in row if 0 <= int(t) < pm.numel() and pm[int(t)]) for row in top.cpu()]


@pytest.mark.parametrize("case", CASES)
def test_matches_reference_golden(golden_dir, cuda, case):
    """The reference's captured draw replayed: same selections, loss within 5e-3, gradients as the sampled heads' tests."""
    from oracle import sasrec as osr
    z = np.load(os.path.join(golden_dir, "sasrec_legacy_tiny.npz"))
    sd = {k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd::")}
    zs = np.load(os.path.join(golden_dir, "sce_losses.npz"))
    p = tuple(int(v) for v in zs[f"{case}_params"])
    B, L = z["ids"].shape
    eng = _engine(dict(n_items=int(z["n_items"]), d=int(z["d"]), n_heads=int(z["H"]), n_blocks=int(z["n_blocks"])), B, L, cuda,
                  osr.params_from_legacy_state_dict(sd), p)
    ids, pm = torch.from_numpy(z["ids"]), torch.from_numpy(z["pad_mask"])
    eng.set_sce_draw(torch.from_numpy(zs[f"{case}_draw"]).cuda())
    loss = _step(eng, ids, pm, torch.from_numpy(zs[f"{case}_labels"]))
    pmf = pm.reshape(-1)
    sc = eng.sce
    assert _real_sets(sc["top_x"], pmf) == _real_sets(torch.from_numpy(zs[f"{case}_top_x"]), pmf)
    assert [sorted(r) for r in sc["top_y"].tolist()] == [sorted(r) for r in zs[f"{case}_top_y"].tolist()]
    ref = float(zs[f"{case}_loss"])
    # with one item per bucket the loss is a mean of a few softplus(s - c) terms, which move by ~1 % with the bf16 hidden rows
    tol = 5e-3 if p[2] > 1 else 2e-2
    assert abs(float(loss[0]) - ref) < tol * abs(ref), (float(loss[0]), ref)
    G = eng.export_canonical(eng.grads)
    gE, gW = torch.from_numpy(zs[f"{case}_gE"]), torch.from_numpy(zs[f"{case}_gW"])
    for nm, a, b in (("item_emb", G["item_emb"].cpu(), gE), ("in_w", G["blocks"][0]["in_w"].cpu(), gW)):
        c, r = _cos(a, b), float(a.double().norm() / b.double().norm())
        assert c > 0.995 and abs(r - 1) < 0.03, (nm, c, r)
    # the head sends nothing to the table: only rows that are an input item (and not the pad row) move
    inputs = torch.zeros(gE.shape[0], dtype=torch.bool)
    inputs[ids[pm].unique()] = True
    assert (G["item_emb"].cpu()[~inputs] == 0).all()


def _fp64_case(cuda, B, L, d, H, I, sce, seed, n_blocks=2):
    from oracle import sasrec as osr
    from oracle import sce as osce
    from replay_b200.synthetic import make_sequences
    P = osr.random_params(I, d, L, n_blocks, seed=seed)
    ids, pm, lab, _ = make_sequences(B, I, L, seed=seed + 1)
    lab = lab.clamp(max=I - 1)
    eng = _engine(dict(n_items=I, d=d, n_heads=H, n_blocks=n_blocks), B, L, cuda, P, sce, seed=seed)
    loss = _step(eng, ids, pm, lab)
    sc = eng.sce
    draw, top_x, top_y = sc["draw"].cpu(), sc["top_x"].cpu(), sc["top_y"].cpu()
    n_b, bsx, bsy, mix = sce
    pmf = pm.reshape(-1)
    assert bool(torch.isfinite(sc["score_x"]).all()), "bucket_size_x must stay below the real rows here"
    # selections: fp64 top-k of the engine's own bf16 inputs; a swap is allowed only across an fp64 gap below EPS_SEL
    hc = eng.unpad_features(eng.hc[: B * L]).double().cpu()
    tab = eng.unpad_features(eng.params16["item_emb"][:I]).double().cpu()
    scale = d ** -0.25
    if mix:
        om = (draw[: B * L] * scale).to(torch.bfloat16).double()
        buckets = (om.T @ hc).to(torch.bfloat16).double()
    else:
        buckets = (draw * scale).to(torch.bfloat16).double()
    for top, s, k in ((top_x, (buckets @ hc.T).masked_fill(~pmf.view(1, -1), float("-inf")), bsx), (top_y, buckets @ tab.T, bsy)):
        kth = s.topk(k, dim=1).values[:, -1:]
        picked = s.gather(1, top)
        eps = EPS_SEL_MIX if mix else EPS_SEL
        tol = eps * s.masked_fill(~torch.isfinite(s), 0).abs().amax(1, keepdim=True)
        assert bool((picked >= kth - tol).all()), float((kth - picked).max())
        assert all(len(set(r)) == k for r in top.tolist())
    # loss and gradients with the engine's selections against fp64 autograd
    P64 = osr.params_to(P, torch.float64)
    ref, Gref, _, _ = osce.loss_and_grads(P64, ids, pm, lab, H, draw.double()[: B * L] if mix else draw.double(), bsx, bsy,
                                          bool(mix), top_x=top_x, top_y=top_y)
    assert abs(float(loss[0]) - float(ref)) < TOL_LOSS * abs(float(ref)), (float(loss[0]), float(ref))
    G = eng.export_canonical(eng.grads)
    # the table gradient is the input gather's alone: per item it sums a few tokens whose gradient crossed the whole bf16 body
    # backward, so it is checked as a whole; every other parameter per 64-row block
    a, b = G["item_emb"].cpu(), Gref["item_emb"]
    c, r = _cos(a, b), float(a.double().norm() / b.double().norm())
    print("item_emb cos", c, "norm ratio", r)
    assert c > 0.99 and abs(r - 1) < 0.03, (c, r)
    worst = []
    for k, (a, b) in enumerate(zip(osr.flat_param_list(G)[1:], osr.flat_param_list(Gref)[1:])):
        if b.norm() < 1e-12:
            assert float(a.abs().max()) < 1e-6, k
            continue
        worst.append((block_err(a.cpu(), b), k + 1))
    print("worst block error", max(worst))
    assert max(worst)[0] < TOL_GRAD, max(worst)


EPS_SEL = 1e-5          # fp32 accumulation of exact bf16 products against fp64: relative to the bucket's largest |score|
EPS_SEL_MIX = 2e-2      # mix_x: the fp32 omega^T . hc may round to a different bf16 bucket entry than the fp64 product
TOL_LOSS = 1e-2         # bf16 body + bf16 bucket GEMMs against fp64
TOL_GRAD = 0.15         # per 64-row block, norm-relative; worst seen 7.3e-2 (H100 80GB HBM3, 400 W), about the body's own step error


@pytest.mark.parametrize("mix", [False, True])
def test_fp64_restatement_config2_shape(cuda, mix):
    """Config 2 model shape: L = 200, d = 128, H = 2, |I| = 50K, B = 8 (801 real rows); 64 buckets of 256 rows and 256 items."""
    _fp64_case(cuda, B=8, L=200, d=128, H=2, I=50_000, sce=(64, 256, 256, int(mix)), seed=5)


def test_fp64_restatement_d512(cuda):
    """d = 512: L = 512, H = 8, |I| = 100K, B = 4 (445 real rows); 32 buckets of 256 rows and 1024 items (the fused top-K's
    limit)."""
    _fp64_case(cuda, B=4, L=512, d=512, H=8, I=100_000, sce=(32, 256, 1024, 0), seed=7)


@pytest.mark.parametrize("mix", [False, True])
def test_deterministic_and_graph_replay(cuda, mix):
    """Same seed and counter: bitwise-equal draw, selections, loss and head gradient d_hc (the body's own backward sums some
    weight gradients with float atomics, so g32 is compared to a tolerance); a captured forward + backward replays to the
    eager result; the next counter draws different buckets."""
    from oracle import sasrec as osr
    from replay_b200.synthetic import make_sequences
    B, L, d, H, I = 4, 200, 128, 2, 20_000
    P = osr.random_params(I, d, L, 2, seed=3)
    ids, pm, lab, _ = make_sequences(B, I, L, seed=4)
    sce = (32, 128, 256, int(mix))
    out = []
    for _ in range(2):
        eng = _engine(dict(n_items=I, d=d, n_heads=H, n_blocks=2), B, L, cuda, P, sce, seed=11)
        eng.rng_counter.fill_(12345)
        loss = _step(eng, ids, pm, lab)
        out.append((loss, eng.s["dhc"].clone(), eng.sce["draw"].clone(), eng.sce["top_x"].clone(), eng.sce["top_y"].clone(),
                    eng.g32.clone()))
    for a, b in zip(out[0][:-1], out[1][:-1]):
        assert torch.equal(a, b)
    assert torch.allclose(out[0][-1], out[1][-1], rtol=1e-3, atol=1e-6 * float(out[0][-1].abs().max()))
    # graph: capture forward + backward on the second engine, replay at the same counter
    eng.rng_counter.fill_(12345)
    _step(eng, ids, pm, lab)
    _step(eng, ids, pm, lab)
    g = torch.cuda.CUDAGraph()
    eng.rng_counter.fill_(12345)
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        eng.forward_train()
        eng.g32.zero_()
        eng.backward()
    eng.s["dhc"].fill_(7.0)
    eng.ce.loss.fill_(0.0)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(eng.ce.loss, out[0][0]) and torch.equal(eng.s["dhc"], out[0][1])
    draw0 = eng.sce["draw"].clone()
    eng.tick_rng()
    g.replay()
    torch.cuda.synchronize()
    assert not torch.equal(eng.sce["draw"], draw0)


def test_no_counted_row_gives_nan_and_zero_gradient(cuda):
    """One item, every label equal to it: every bucket CE is exactly 0, so no row is counted - NaN loss, zero gradient."""
    from oracle import sasrec as osr
    B, L, d, I = 2, 16, 64, 1
    P = osr.random_params(I, d, L, 1, seed=1)
    eng = _engine(dict(n_items=I, d=d, n_heads=1, n_blocks=1), B, L, cuda, P, (3, 8, 1, 0))
    ids = torch.zeros(B, L, dtype=torch.long)
    pm = torch.ones(B, L, dtype=torch.bool)
    loss = _step(eng, ids, pm, torch.zeros(B, L, dtype=torch.long))
    assert torch.isnan(loss[0]) and float(loss[1]) == 0.0
    assert bool((eng.g32 == 0).all())


def test_public_module_trains(golden_dir, cuda):
    """SasRec(loss_type="SCE"): the fused step lowers the loss with and without mix_x; the autograd step gives a finite
    flat.grad."""
    from replay_b200.models.nn.loss import SCEParams
    from replay_b200.models.nn.sequential import SasRec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema
    z = np.load(os.path.join(golden_dir, "sasrec_legacy_tiny.npz"))
    n_items, d, L = int(z["n_items"]), int(z["d"]), int(z["L"])
    ids, pm = torch.from_numpy(z["ids"]).cuda(), torch.from_numpy(z["pad_mask"]).cuda()
    lab, tm = torch.from_numpy(z["labels"]).clamp(max=n_items - 1).cuda(), torch.from_numpy(z["target_mask"]).cuda()
    b = {"feature_tensor": {"item_id": ids}, "padding_mask": pm, "positive_labels": lab, "target_padding_mask": tm}
    for mix in (False, True):
        torch.manual_seed(0)
        m = SasRec(TensorSchema(TensorFeatureInfo("item_id", n_items, 0, d)), block_count=1, head_count=1, hidden_size=d,
                   max_seq_len=L, dropout_rate=0.0, loss_type="SCE", sce_params=SCEParams(8, 24, 64, mix))
        losses = [float(m.training_step(b, i)) for i in range(40)]
        assert all(np.isfinite(losses)) and np.mean(losses[-5:]) < np.mean(losses[:5]) - 0.3, (mix, losses[:5], losses[-5:])
    m = SasRec(TensorSchema(TensorFeatureInfo("item_id", n_items, 0, d)), block_count=1, head_count=1, hidden_size=d,
               max_seq_len=L, dropout_rate=0.0, loss_type="SCE", sce_params=SCEParams(4, 16, 32), fused_optimizer=False)
    loss = m.training_step(b, 0)
    loss.backward()
    assert torch.isfinite(loss) and m._model.core.flat.grad is not None and torch.isfinite(m._model.core.flat.grad).all()
