"""The fused optimizer step (``rp_optimizer_step``): Adam with L2 weight decay and SGD with momentum, against a float64
restatement of torch.optim with per-element bounds; then through the engine-backed modules against torch.optim on the
same flat parameter (``fused_optimizer=False``) and on the oracle's fp32 autograd, graph capture, and checkpoint resume.

Bounds of the kernel test (u = 2^-24, every quantity taken at the kernel's own fp32 inputs, scalars rounded to fp32):

- the gradient ``gk = fma(wd, p, g * s)``: ``g * s`` is exact for s in {1, 1/2}; one rounding, ``e_g <= u |gk|``;
- SGD: ``buf' = rn(rn(mu buf) + gk)``, ``e_buf <= u (mu |buf| + |buf'|) + e_g``; ``p' = p - lr buf'`` (one or two
  roundings), ``e_p <= 2u (|p'| + lr |buf'|) + lr e_buf``;
- Adam: ``m'`` and ``v'`` are one FMA over a rounded product each, ``e_m <= 2u (b1 |m| + (1-b1) |gk|) + (1-b1) e_g``,
  ``e_v <= 3u (b2 v + (1-b2) gk^2) + 2 (1-b2) |gk| e_g``.  The update ``lr / bc1 * m' / (sqrt(v') / sqrt(bc2) + eps)``
  runs under fast math: powf as ex2(t log2 b) (relative error <= 8u (1 + t |log2 b|) in b^t, amplified by
  b^t / (1 - b^t) in 1 - b^t), MUFU rsqrt / sqrt and the approximate division (<= 2u each, 16u in all), plus the
  propagated ``e_m`` and ``e_v`` (halved through the square root); then one rounding in ``p - upd``.
Every bound is doubled before the check.
"""
import copy
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
ADAM, SGD = 0, 1


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda")


def f32(x):
    return float(np.float32(x))


def _call(kind, p, g, s0, s1, p16, lr, step, b1=0.9, b2=0.98, eps=1e-8, wd=0.0, mu=0.0, scale=1.0):
    from replay_b200._lib import check, lib

    ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    check(lib().rp_optimizer_step(kind, p.data_ptr(), g.data_ptr(), ptr(s0), ptr(s1), p16.data_ptr(), p.numel(),
                                  lr.data_ptr(), step.data_ptr(), b1, b2, eps, wd, mu, scale, None, 1,
                                  torch.cuda.current_stream().cuda_stream), "rp_optimizer_step")


def _ref_adam(p, g, m, v, t, lr, b1, b2, eps, wd, scale):
    """float64 torch.optim.Adam step and per-element bounds on (p', m', v')"""
    lr, b1, b2, eps, wd = f32(lr), f32(b1), f32(b2), f32(eps), f32(wd)
    gk = g * scale + wd * p
    e_g = U * gk.abs() if wd else torch.zeros_like(gk)
    m1 = b1 * m + (1 - b1) * gk
    v1 = b2 * v + (1 - b2) * gk * gk
    bc1, bc2 = 1 - b1 ** t, 1 - b2 ** t
    denom = v1.sqrt() / math.sqrt(bc2) + eps
    upd = lr / bc1 * m1 / denom
    p1 = p - upd
    e_m = 2 * U * (b1 * m.abs() + (1 - b1) * gk.abs()) + (1 - b1) * e_g
    e_v = 3 * U * (b2 * v + (1 - b2) * gk * gk) + 2 * (1 - b2) * gk.abs() * e_g
    pw = lambda b: 8 * U * (1 + t * abs(math.log2(b))) * b ** t / (1 - b ** t)  # noqa: E731
    rel = 16 * U + pw(b1) + 0.5 * pw(b2)
    sq = v1.sqrt()
    e_upd = upd.abs() * rel + lr / bc1 * (e_m / denom + m1.abs() * (e_v / (2 * sq.clamp_min(1e-300))) / math.sqrt(bc2)
                                          / denom ** 2 * (sq > 0))
    e_p = U * (p1.abs() + upd.abs()) + e_upd
    return (p1, m1, v1), (2 * e_p, 2 * e_m, 2 * e_v)


def _ref_sgd(p, g, buf, lr, mu, wd, scale):
    lr, mu, wd = f32(lr), f32(mu), f32(wd)
    gk = g * scale + wd * p
    e_g = U * gk.abs() if wd else torch.zeros_like(gk)
    b1 = mu * buf + gk if mu else gk
    e_b = U * (mu * buf.abs() + b1.abs()) + e_g if mu else e_g
    p1 = p - lr * b1
    e_p = 2 * U * (p1.abs() + lr * b1.abs()) + lr * e_b
    return (p1, b1), (2 * e_p, 2 * e_b)


def _check(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = err > bound
    assert not bad.any(), (what, int(bad.sum()), float((err / bound.clamp_min(1e-300)).max()))


@pytest.mark.parametrize("n", [4, 1_004, 2_500_004])
@pytest.mark.parametrize("scale", [1.0, 0.5])
@pytest.mark.parametrize("opt", [("adam", 0.0, 0.0), ("adam", 1e-2, 0.0), ("sgd", 0.0, 0.0), ("sgd", 1e-4, 0.0),
                                 ("sgd", 0.0, 0.9), ("sgd", 1e-4, 0.9)])
def test_kernel_against_fp64(cuda, n, scale, opt):
    kind, wd, mu = opt
    gen = torch.Generator().manual_seed(n + int(wd * 1e4) + int(mu * 10) + (7 if kind == "sgd" else 0))
    p = torch.randn(n, generator=gen)
    lr = torch.full((1,), 3e-3, device=cuda)
    step = torch.zeros(1, device=cuda, dtype=torch.int32)
    p16 = torch.empty(n, device=cuda, dtype=torch.bfloat16)
    if kind == "adam":
        m, v = torch.zeros(n), torch.zeros(n)
        if n > 4:   # a later step from a random state (step 7)
            m, v = torch.randn(n, generator=gen) * 1e-2, torch.rand(n, generator=gen) * 1e-4
            step.fill_(6)
        s0, s1 = m.to(cuda), v.to(cuda)
    else:
        # a restored, non-zero buffer before this kernel's first step; a fresh one (zero) at n == 4
        buf = torch.randn(n, generator=gen) * 1e-2 if n > 4 and mu else torch.zeros(n)
        s0, s1 = (buf.to(cuda) if mu else None), None
    pd = p.to(cuda)
    for it in range(2):   # the step from the state above, then a later one
        g = torch.randn(n, generator=gen) * (10.0 ** float(torch.randint(-4, 1, (1,), generator=gen)))
        gd = (g / scale).to(cuda)   # the rank sum that grad_scale averages
        p64 = pd.double().cpu()
        t = int(step.item()) + 1
        if kind == "adam":
            (pr, mr, vr), (bp, bm, bv) = _ref_adam(p64, g.double(), s0.double().cpu(), s1.double().cpu(), t, 3e-3, 0.9,
                                                   0.98, 1e-8, wd, 1.0)
            _call(ADAM, pd, gd, s0, s1, p16, lr, step, wd=wd, scale=scale)
            _check(s0.cpu(), mr, bm, "exp_avg")
            _check(s1.cpu(), vr, bv, "exp_avg_sq")
        else:
            buf64 = s0.double().cpu() if mu else torch.zeros(n, dtype=torch.float64)
            (pr, br), (bp, bb) = _ref_sgd(p64, g.double(), buf64, 3e-3, mu, wd, 1.0)
            _call(SGD, pd, gd, s0, None, p16, lr, step, wd=wd, mu=mu, scale=scale)
            if mu:
                _check(s0.cpu(), br, bb, "momentum_buffer")
        torch.cuda.synchronize()
        _check(pd.cpu(), pr, bp, "param")
        assert torch.equal(p16, pd.to(torch.bfloat16)), "the bf16 shadow is bf16(p)"
        assert float(gd.abs().max()) == 0.0 and not torch.signbit(gd).any(), "the gradient is zeroed"
        assert int(step.item()) == t


def test_adam_without_decay_matches_rp_adam_step_bitwise(cuda):
    """``rp_adam_step`` keeps its contract as a caller of ``rp_optimizer_step`` (Adam, weight decay 0): same bits, same
    step counter.  It does not compare against the previous kernel: that ``optimizer_kernel<Adam, false>`` keeps its
    arithmetic is a property of the compiled code (the same SASS instructions and floating-point operations; only the
    constant-bank offsets of its parameters moved), and the existing Adam tests against torch.optim check its results."""
    from replay_b200._lib import check, lib

    n = 1_081_348
    gen = torch.Generator().manual_seed(3)
    p, g, m, v = (torch.randn(n, generator=gen).to(cuda) for _ in range(4))
    v = v.abs() * 1e-3
    a = [t.clone() for t in (p, g, m, v)]
    b = [t.clone() for t in (p, g, m, v)]
    lr = torch.full((1,), 1e-3, device=cuda)
    sa, sb = torch.full((1,), 4, device=cuda, dtype=torch.int32), torch.full((1,), 4, device=cuda, dtype=torch.int32)
    ha, hb = (torch.empty(n, device=cuda, dtype=torch.bfloat16) for _ in range(2))
    st = torch.cuda.current_stream().cuda_stream
    check(lib().rp_adam_step(a[0].data_ptr(), a[1].data_ptr(), a[2].data_ptr(), a[3].data_ptr(), ha.data_ptr(), n,
                             lr.data_ptr(), sa.data_ptr(), 0.9, 0.98, 1e-8, 0.5, None, 1, st), "rp_adam_step")
    _call(ADAM, b[0], b[1], b[2], b[3], hb, lr, sb, scale=0.5)
    torch.cuda.synchronize()
    for x, y in zip(a + [ha, sa], b + [hb, sb]):
        assert torch.equal(x.view(torch.int8) if x.is_floating_point() else x,
                           y.view(torch.int8) if y.is_floating_point() else y)


# ----------------------------------------------------------------------------------------------------------------------
# the modules: fused step against torch.optim on the same flat parameter, and against the oracle
# ----------------------------------------------------------------------------------------------------------------------
OPTS = {"adam_wd": dict(optimizer="adam", weight_decay=1e-2), "sgd": dict(optimizer="sgd", learning_rate=1e-2),
        "sgd_mom_wd": dict(optimizer="sgd", learning_rate=1e-2, sgd_momentum=0.9, weight_decay=1e-4)}
MODULES = ["sasrec", "diff", "twotower", "legacy_sasrec", "tisasrec", "bert4rec"]
N_ITEMS, D, L, B = 300, 64, 16, 8


def _schema(ts=False):
    from replay_b200.schema import TensorFeatureInfo, TensorSchema

    return TensorSchema(TensorFeatureInfo("item_id", N_ITEMS, N_ITEMS, D), timestamp_feature_name="timestamp" if ts else None)


class _Reader:
    """the item-feature reader of an item-id-only catalog"""

    def __getitem__(self, k):
        return torch.arange(N_ITEMS)

    @property
    def feature_names(self):
        return ["item_id"]


def _module(kind, factory, fused=True, seed=2):
    """(Lightning module, its core)"""
    if kind in ("sasrec", "diff", "twotower"):
        from replay_b200.nn.lightning import LightningModule
        from replay_b200.nn.sequential import SasRec

        if kind == "twotower":
            from replay_b200.nn.sequential.twotower import TwoTower

            model = TwoTower.from_params(_schema(), _Reader(), embedding_dim=D, num_heads=1, num_blocks=1,
                                         max_sequence_length=L, dropout=0.0, seed=seed)
        elif kind == "diff":
            from replay_b200.nn.agg import SumAggregator
            from replay_b200.nn.embedding import SequenceEmbedding
            from replay_b200.nn.loss import CE
            from replay_b200.nn.mask import DefaultAttentionMask
            from replay_b200.nn.sequential import DiffTransformerLayer, PositionAwareAggregator, SasRecBody

            body = SasRecBody(embedder=SequenceEmbedding(_schema()),
                              embedding_aggregator=PositionAwareAggregator(SumAggregator(D), max_sequence_length=L, dropout=0.0),
                              attn_mask_builder=DefaultAttentionMask("item_id", 1), encoder=DiffTransformerLayer(D, 1, 1),
                              output_normalization=torch.nn.LayerNorm(D))
            model = SasRec(body, loss=CE(ignore_index=N_ITEMS), seed=seed)
        else:
            model = SasRec.from_params(_schema(), embedding_dim=D, num_heads=1, num_blocks=1, max_sequence_length=L,
                                       dropout=0.0, seed=seed)
        model.train()
        return LightningModule(model, optimizer_factory=factory, fused_optimizer=fused), model.core
    if kind in ("legacy_sasrec", "tisasrec"):
        from replay_b200.models.nn.sequential import SasRec

        m = SasRec(_schema(ts=kind == "tisasrec"), block_count=1, head_count=1, hidden_size=D, max_seq_len=L,
                   dropout_rate=0.0, ti_modification=kind == "tisasrec", optimizer_factory=factory,
                   fused_optimizer=fused)
        return m, m._model.core
    from replay_b200.models.nn.sequential import Bert4Rec

    m = Bert4Rec(_schema(), block_count=1, head_count=1, hidden_size=D, max_seq_len=L, dropout_rate=0.0,
                 optimizer_factory=factory, fused_optimizer=fused)
    return m, m._model.core


def _batch(kind, seed):
    """one batch of ``kind``'s training_step"""
    from replay_b200.synthetic import make_sequences

    ids, pm, lab, tm = (t.cuda() for t in make_sequences(B, N_ITEMS, L, seed=seed))
    if kind in ("sasrec", "diff", "twotower"):
        return {"feature_tensors": {"item_id": ids}, "padding_mask": pm, "positive_labels": lab.unsqueeze(-1),
                "target_padding_mask": tm.unsqueeze(-1)}
    if kind in ("legacy_sasrec", "tisasrec"):
        ft = {"item_id": ids}
        if kind == "tisasrec":
            ft["timestamp"] = (torch.arange(L, device=ids.device) * 7 + 1000).expand(B, L).to(torch.int64) * pm
        return {"feature_tensor": ft, "padding_mask": pm, "positive_labels": lab, "target_padding_mask": tm}
    from replay_b200.models.nn.sequential.bert4rec import uniform_masker

    g = torch.Generator().manual_seed(seed)
    tok = uniform_masker(pm.cpu(), 0.2, g).cuda()
    return {"query_id": torch.arange(B), "inputs": {"item_id": torch.where(pm, ids, torch.zeros_like(ids))},
            "pad_mask": pm, "token_mask": tok, "positive_labels": torch.where(pm & ~tok, ids, torch.zeros_like(ids))}


def _build(kind, opt, fused):
    from replay_b200.nn.lightning import OptimizerFactory

    torch.manual_seed(0)
    return _module(kind, OptimizerFactory(**OPTS[opt]), fused=fused)


class _Bound:
    """Per-element bound on |fused - torch| after lock-step updates from the same gradients.  Each step adds, per element,
    the rounding of the parameter itself (2u |p|), the update's relative error (Adam under fast math: the powf bias
    corrections at t = 1 dominate with about 300u = 1.8e-5, taken as 5e-5; SGD: the decay FMA and the buffer's two
    roundings accumulated over 1 / (1 - momentum) steps, 32u) and, for Adam, an absolute term for a first
    moment that cancels (lr / bc1 x 2u x |m_prev| / denom <= 256u lr).  The check doubles the sum.  Dropping the decay
    moves a zero-gradient element by more than ten times this bound at the tested settings."""

    def __init__(self, opt, lr, p0):
        adam = OPTS[opt].get("optimizer", "adam") == "adam"
        self.rel, self.abs = (5e-5, 256 * U * lr) if adam else (32 * U, 0.0)
        self.b = torch.zeros_like(p0, dtype=torch.float64)

    def step(self, p_before, p_after):
        self.b += 2 * U * p_before.double().abs() + self.rel * (p_after - p_before).double().abs() + self.abs

    def check(self, got, ref, what):
        _check(got, ref.double(), 2 * self.b, what)


class _WithoutDecay:
    """The factory's torch optimizer with weight_decay 0, stepped on a copy of the parameters with the same gradients: where
    its result lies outside the bound, the check would catch a step that ignored the decay."""

    def __init__(self, opt, p0):
        from replay_b200.nn.lightning import OptimizerFactory

        self.p = p0.detach().clone().requires_grad_()
        self.opt = OptimizerFactory(**dict(OPTS[opt], weight_decay=0.0)).create([self.p])

    def step(self, g):
        self.p.grad = g.detach().clone()
        with torch.no_grad():
            self.opt.step()

    def share_seen(self, ref, bound):
        return float(((self.p.detach().double() - ref.double()).abs() > 2 * bound.b).double().mean())


@pytest.mark.parametrize("opt", list(OPTS))
@pytest.mark.parametrize("kind", MODULES)
def test_fused_step_matches_torch_optimizer(cuda, kind, opt):
    """Five lock-step updates: the module with ``fused_optimizer=False`` computes loss.backward() and steps the factory's
    torch optimizer on ``core.flat``; the fused module's engine takes the same gradient into its own step with the
    configuration its factory gave it.  Every element, padding rows and zero-gradient rows included, agrees to the
    rounding of the update; the saved optimizer state is torch's, to rounding."""
    (mf, cf), (mt, ct) = _build(kind, opt, True), _build(kind, opt, False)
    mt.load_state_dict(mf.state_dict())
    eng = cf.ensure_engine(B, L, with_grad=True)
    lr = OPTS[opt].get("learning_rate", 1e-3)
    eng.lr.fill_(lr)
    topt = mt.configure_optimizers()
    p0 = ct.flat.detach().clone()
    assert torch.equal(eng.p32, p0)
    bound, grad_seen, nodecay = _Bound(opt, lr, p0), torch.zeros_like(p0, dtype=torch.bool), _WithoutDecay(opt, p0)
    for s in range(5):
        before = ct.flat.detach().clone()
        topt.zero_grad()
        mt.training_step(_batch(kind, s), s).backward()
        g = ct.flat.grad.detach()
        grad_seen |= g != 0
        eng.g32.copy_(g)
        nodecay.step(g)
        eng.optimizer_step(opt=cf.optimizer)
        topt.step()
        bound.step(before, ct.flat.detach())
    torch.cuda.synchronize()
    bound.check(eng.p32, ct.flat.detach(), "parameters")
    assert torch.equal(eng.p16, eng.p32.to(torch.bfloat16))
    if OPTS[opt].get("weight_decay"):
        assert nodecay.share_seen(ct.flat, bound) > 0.5   # the bound resolves the decay on most elements
        # where only the decay acts (rows no batch touched, the legacy padding row) the parameters moved
        decay_only = ~grad_seen & (p0 != 0)
        assert bool((eng.p32[decay_only] != p0[decay_only]).all())
        if kind in ("legacy_sasrec", "tisasrec"):
            key = "_model.item_embedder.item_emb.weight"
            row0, rowf, rowt = (m.state_dict()[key][N_ITEMS] for m in (_build(kind, opt, True)[0], mf, mt))
            assert bool((row0 != 0).all()) and bool((rowf != row0).all()) and bool((rowt != row0).all())
    saved = {}
    mf.on_save_checkpoint(saved)
    ref = topt.state_dict()
    got = saved["optimizer_states"][0]
    assert got["param_groups"] == ref["param_groups"]
    assert set(got["state"]) == set(ref["state"]) and set(got["state"].get(0, {})) == set(ref["state"].get(0, {}))
    for name, v in ref["state"].get(0, {}).items():
        if name == "step":
            assert float(got["state"][0][name]) == float(v) == 5.0
        else:
            assert got["state"][0][name].device.type == "cpu"
            assert float((got["state"][0][name].cuda() - v).norm()) <= 1e-5 * float(v.norm()), name


def _flat_steps(core, opt, grads):
    eng = core.engine
    for g in grads:
        eng.g32.copy_(g)
        eng.optimizer_step(opt=opt)


@pytest.mark.parametrize("opt", list(OPTS))
def test_graph_replay_equals_eager_bitwise(cuda, opt):
    """The optimizer launch captured in a CUDA graph and replayed gives the eager steps' bits (same gradients)."""
    (m1, c1), (m2, c2) = _build("sasrec", opt, True), _build("sasrec", opt, True)
    m2.load_state_dict(m1.state_dict())
    for c in (c1, c2):
        c.ensure_engine(B, L, with_grad=True)
        c.engine.lr.fill_(OPTS[opt].get("learning_rate", 1e-3))
    gen = torch.Generator().manual_seed(1)
    grads = [torch.randn(c1.engine.n_flat, generator=gen).cuda() for _ in range(4)]
    _flat_steps(c1, c1.optimizer, grads)
    _flat_steps(c2, c2.optimizer, grads[:1])   # first step eager: a kind switch may reset state outside the capture
    gbuf = torch.zeros_like(c2.engine.g32)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        c2.engine.optimizer_step(opt=c2.optimizer)
    for g in grads[1:]:
        gbuf.copy_(g)
        c2.engine.g32.copy_(gbuf)
        graph.replay()
    torch.cuda.synchronize()
    for name in ("p32", "p16", "adam_m", "adam_v", "step_count"):
        a, b = getattr(c1.engine, name), getattr(c2.engine, name)
        assert torch.equal(a.view(torch.uint8) if a.is_floating_point() else a,
                           b.view(torch.uint8) if b.is_floating_point() else b), name


def test_factory_change_drops_the_graph_and_resets_the_state(cuda):
    from replay_b200.nn.lightning import OptimizerFactory

    torch.manual_seed(0)
    m, core = _module("legacy_sasrec", OptimizerFactory())
    for s in range(4):   # two eager warm-up steps, then the captured step
        m.training_step(_batch("legacy_sasrec", s), s)
    tr, eng = core._trainer, core.engine
    assert tr._g_fb is not None and int(eng.step_count.item()) == 4 and eng.opt_kind == "adam"
    m.optimizer_factory = OptimizerFactory(optimizer="sgd", sgd_momentum=0.9, learning_rate=1e-2)
    m.training_step(_batch("legacy_sasrec", 4), 4)
    assert tr.opt.kind == "sgd" and tr._warm == 1 and tr._g_fb is None   # re-warming before a new capture
    assert eng.opt_kind == "sgd" and int(eng.step_count.item()) == 1 and float(eng.adam_v.abs().max()) == 0.0
    for s in range(5, 9):
        m.training_step(_batch("legacy_sasrec", s), s)
    assert tr._g_fb is not None and int(eng.step_count.item()) == 5
    m.optimizer_factory = OptimizerFactory(optimizer="rmsprop")
    before = eng.p32.clone()
    with pytest.raises(ValueError, match="Unexpected optimizer"):
        m.training_step(_batch("legacy_sasrec", 9), 9)
    assert torch.equal(before, eng.p32) and float(eng.g32.abs().max()) == 0.0


@pytest.mark.parametrize("opt", ["adam_wd", "sgd_mom_wd"])
def test_checkpoint_resume_is_bitwise(cuda, opt):
    """3 steps, save through the hooks, load into a new module, 3 more steps == 6 uninterrupted steps, bit for bit (the
    same gradients each step); the checkpoint also resumes a fused_optimizer=False module with the same state."""
    gen = torch.Generator().manual_seed(5)
    (ma, ca), (mb, cb), (mc, cc) = (_build("legacy_sasrec", opt, True) for _ in range(3))
    for c in (ca, cb, cc):
        c.ensure_engine(B, L, with_grad=True)
    n = ca.engine.n_flat
    grads = [torch.randn(n, generator=gen).cuda() * 1e-2 for _ in range(6)]
    _flat_steps(ca, ca.optimizer, grads)
    _flat_steps(cb, cb.optimizer, grads[:3])
    ckpt = {"state_dict": mb.state_dict()}
    mb.on_save_checkpoint(ckpt)
    ckpt = copy.deepcopy(ckpt)
    mc.load_state_dict(ckpt["state_dict"])
    mc.on_load_checkpoint(ckpt)
    _flat_steps(cc, cc.optimizer, grads[3:])
    torch.cuda.synchronize()
    for name in ("p32", "p16", "adam_m", "adam_v"):
        assert torch.equal(getattr(ca.engine, name), getattr(cc.engine, name)), name
    # the same checkpoint in a module that steps with torch.optim
    mt, ct = _build("legacy_sasrec", opt, False)
    mt.load_state_dict(ckpt["state_dict"])
    topt = mt.configure_optimizers()
    topt.load_state_dict(ckpt["optimizer_states"][0])
    st = topt.state[ct.flat]
    if opt == "adam_wd":
        assert float(st["step"]) == 3.0 and torch.equal(st["exp_avg"], cb.engine.adam_m)
        assert torch.equal(st["exp_avg_sq"], cb.engine.adam_v)
    else:
        assert torch.equal(st["momentum_buffer"], cb.engine.adam_m)
    # and back: the torch optimizer's checkpoint resumes the fused step
    md, cd = _build("legacy_sasrec", opt, True)
    md.on_load_checkpoint({"optimizer_states": [topt.state_dict()]})
    cd.ensure_engine(B, L, with_grad=True)
    assert torch.equal(cd.engine.adam_m, cb.engine.adam_m) and cd.engine.opt_kind == cb.engine.opt_kind
    assert int(cd.engine.step_count.item()) == (3 if opt == "adam_wd" else 1)


def test_padded_feature_slots_stay_zero(cuda):
    """hidden 50 runs in 64-wide slots: weight decay and momentum leave the padded entries exactly zero."""
    from replay_b200.models.nn.sequential import SasRec
    from replay_b200.nn.lightning import OptimizerFactory

    torch.manual_seed(0)
    m = SasRec(_schema(), block_count=1, head_count=1, hidden_size=50, max_seq_len=L, dropout_rate=0.0,
               optimizer_factory=OptimizerFactory(optimizer="sgd", sgd_momentum=0.9, weight_decay=1e-2, learning_rate=0.1))
    core = m._model.core
    sd = m.state_dict()
    m.load_state_dict({k: torch.ones_like(v) for k, v in sd.items()})
    pad = core.engine.p32 == 0
    m.load_state_dict(sd)
    assert pad.any()
    for s in range(4):
        m.training_step(_batch("legacy_sasrec", s), s)
    assert float(core.engine.p32[pad].abs().max()) == 0.0 and float(core.engine.adam_m[pad].abs().max()) == 0.0


@pytest.mark.parametrize("opt", list(OPTS))
@pytest.mark.parametrize("variant", ["new", "legacy"])
def test_fused_step_matches_oracle(cuda, variant, opt):
    """Five lock-step updates against the oracle: its fp32 autograd gradient (padding row frozen) steps the factory's
    torch optimizer on the oracle's parameters, and the same gradient, imported into the engine's flat layout, steps the
    fused module's optimizer.  Every parameter, the padding row included, agrees to the rounding of the update."""
    from oracle import sasrec as osr
    from replay_b200.nn.lightning import OptimizerFactory

    kind = "sasrec" if variant == "new" else "legacy_sasrec"
    m, core = _build(kind, opt, True)
    from_sd = osr.params_from_new_state_dict if variant == "new" else osr.params_from_legacy_state_dict
    prefix = "model." if variant == "new" else "_model."
    P = from_sd({k[len(prefix):]: v.cpu() for k, v in m.state_dict().items() if k.startswith(prefix)})
    params = [t.requires_grad_() for t in osr.flat_param_list(P)]
    lr = OPTS[opt].get("learning_rate", 1e-3)
    topt = OptimizerFactory(**OPTS[opt]).create(params)
    eng = core.ensure_engine(B, L, with_grad=True)
    eng.lr.fill_(lr)
    flat0 = torch.cat([t.detach().flatten() for t in params])
    bound, nodecay = _Bound(opt, lr, flat0), _WithoutDecay(opt, flat0)
    for s in range(5):
        b = _batch(kind, s)
        if variant == "new":
            ids, pm, lab, tm = (b["feature_tensors"]["item_id"], b["padding_mask"], b["positive_labels"][..., 0],
                                b["target_padding_mask"][..., 0])
        else:
            ids, pm, lab, tm = (b["feature_tensor"]["item_id"], b["padding_mask"], b["positive_labels"],
                                b["target_padding_mask"])
        _, G = osr.loss_and_grads({k: v for k, v in P.items()}, ids.cpu(), pm.cpu(), lab.cpu(), tm.cpu(), 1, variant)
        for name in eng.layout:
            blk, _, leaf = name.partition(".")
            eng.import_named(name, G["blocks"][int(blk[1:])][leaf] if leaf else G[name], dst=eng.grads)
        eng.optimizer_step(opt=core.optimizer)
        before = torch.cat([t.detach().flatten() for t in params])
        for t, gr in zip(params, osr.flat_param_list(G)):
            t.grad = gr
        nodecay.step(torch.cat([gr.flatten() for gr in osr.flat_param_list(G)]))
        with torch.no_grad():
            topt.step()
        bound.step(before, torch.cat([t.detach().flatten() for t in params]))
    torch.cuda.synchronize()
    got = torch.cat([t.flatten() for t in osr.flat_param_list(eng.export_canonical())])
    bound.check(got, torch.cat([t.detach().flatten() for t in params]), "parameters")
    if OPTS[opt].get("weight_decay"):
        assert nodecay.share_seen(torch.cat([t.detach().flatten() for t in params]), bound) > 0.5
        if variant == "legacy":   # its padding row is initialised and has a zero gradient: only the decay moved it
            pad0, padf = flat0[:P["item_emb"].numel()].view_as(P["item_emb"])[-1], P["item_emb"][-1]
            assert bool((pad0 != 0).all()) and bool((padf.detach() != pad0).all())
