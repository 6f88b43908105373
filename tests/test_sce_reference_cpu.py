"""Pins the float64 SCE-head reference of the kernel-level GPU test (tests/sce_reference.py) against the restatement
oracle/sce.py and its autograd, on random data and on the reference's golden cases; its counted-row and tie rules on
hand-built cases; the Philox port (tests/philox_stream.py) and the source lines the GPU test restates; and the shape
errors of rp_sce_head_fwd / rp_sce_head_bwd.  CPU only: no kernel is launched."""
import ctypes
import importlib.util
import os
import re

import numpy as np
import pytest
import torch

import philox_stream as ps
import sce_reference as ref
from oracle import sasrec as osr
from oracle import sce as osce

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "replay_b200", "csrc", "rp_sce_head.cu")
CASES = ["nomix", "mix", "bigx", "overlap", "fullcollide", "r111", "r221"]


def _oracle(x, y, w, pm, top_x, top_y):
    """oracle.sce.sce_loss with the given selections: loss and d_x (fp64 autograd)."""
    xg = x.detach().clone().requires_grad_(True)
    loss, _, _ = osce.sce_loss(xg, y, w, pm, torch.zeros(1, x.shape[1], dtype=x.dtype), top_x.shape[1], top_y.shape[1],
                               top_x=top_x, top_y=top_y)
    if torch.isfinite(loss):
        loss.backward()
    return loss.detach(), (xg.grad if xg.grad is not None else torch.zeros_like(xg))


def _score_x(x, buckets, pm, top_x):
    s = (buckets.double() @ x.double().T).masked_fill(~pm.view(1, -1), float("-inf"))
    return s.gather(1, top_x).float()


def _compare(x, y, w, pm, buckets, top_x, top_y):
    lo, dx = _oracle(x, y, w, pm, top_x, top_y)
    r = ref.reference(x, w, y, pm, x.shape[0], top_x, _score_x(x, buckets, pm, top_x), top_y, chunk=3)
    assert r["n_ambiguous"] == 0 and r["near_tie"] == 0
    torch.testing.assert_close(r["loss"], lo, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(r["d_hc"], dx, rtol=1e-10, atol=1e-13)
    return r


@pytest.mark.parametrize("mix", [False, True])
def test_reference_matches_oracle_random(mix):
    """Valid labels, the oracle's own selections (pad rows at -inf, bs_x above the real rows in one bucket set)."""
    g = torch.Generator().manual_seed(3 + mix)
    T, d, I, nb, bsx, bsy = 90, 16, 40, 5, 70, 12
    x = torch.randn(T, d, generator=g, dtype=torch.float64)
    w = torch.randn(I, d, generator=g, dtype=torch.float64) * 0.8
    y = torch.randint(0, I, (T,), generator=g)
    pm = torch.rand(T, generator=g) < 0.7
    draw = torch.randn(T, nb, generator=g, dtype=torch.float64) if mix else torch.randn(nb, d, generator=g, dtype=torch.float64)
    b = osce.buckets_of(x, draw, mix)
    tx, ty = osce.select(x, w, pm, b, bsx, bsy)
    y[tx[0, :5]] = ty[0, 0]                                        # collisions with the bucket's items
    r = _compare(x, y, w, pm, b, tx, ty)
    assert r["n_counted"] > 0 and (r["d_hc"][~pm] == 0).all()


@pytest.mark.parametrize("case", CASES)
def test_reference_matches_oracle_golden(golden_dir, case):
    """The golden cases' hidden states (oracle body), labels and the reference's own selections: the new reference equals
    oracle/sce.py to fp64 rounding, and the real reference's fp32 loss to 1e-5."""
    z = np.load(os.path.join(golden_dir, "sasrec_legacy_tiny.npz"))
    sd = {k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd::")}
    zs = np.load(os.path.join(golden_dir, "sce_losses.npz"))
    P = osr.params_to(osr.params_from_legacy_state_dict(sd), torch.float64)
    ids, pm = torch.from_numpy(z["ids"]), torch.from_numpy(z["pad_mask"])
    x = osr.sasrec_body(P, ids, pm, int(z["H"]), "legacy").detach()
    x = x.reshape(-1, x.shape[-1])
    w = P["item_emb"][:-1]
    n_b, bsx, bsy, mix = (int(v) for v in zs[f"{case}_params"])
    pmf = pm.reshape(-1)
    b = osce.buckets_of(x, torch.from_numpy(zs[f"{case}_draw"]).double(), bool(mix))
    tx, ty = torch.from_numpy(zs[f"{case}_top_x"]), torch.from_numpy(zs[f"{case}_top_y"])
    r = _compare(x, torch.from_numpy(zs[f"{case}_labels"]).reshape(-1), w, pmf, b, tx, ty)
    assert abs(float(r["loss"]) - float(zs[f"{case}_loss"])) <= 1e-5 * abs(float(zs[f"{case}_loss"]))


def _tiny():
    """Six rows, d 4, five items (item 4 = all ones)."""
    x = torch.tensor([[1.0, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0], [1, 1, 0, 0], [0, 0, 0, 1], [1, 0, 1, 0]],
                     dtype=torch.float64)
    w = torch.tensor([[2.0, 0, 0, 0], [0, 2, 0, 0], [0, 0, 2, 0], [0, 0, 0, 2], [1, 1, 1, 1]], dtype=torch.float64)
    return x, w, torch.ones(6, dtype=torch.bool)


def test_counted_row_rules():
    """Full collision (CE exactly 0), CE ~ 1e-12 (below the ambiguous band: treated as 0), CE ~ 1e-7 (in the band)."""
    x, w, pm = _tiny()
    y = torch.tensor([0, 1, 2, 3, 4, 0])
    top_x = torch.tensor([[0, 1], [2, 3], [4, 5]])
    top_y = torch.tensor([[0], [3], [0]])
    score_x = torch.tensor([[0.0, 0.0], [0.0, float("-inf")], [0.0, float("-inf")]])   # rows 3 and 5 are not selected
    # bucket 0: row 0's label is the bucket's only item (CE exactly 0); row 1: c = 2, z = 0 -> CE = log(1 + e^-2)
    # bucket 1: row 2, c = 2, z = 2a with 2a - 2 = log(1e-12) -> CE ~ 1e-12
    # bucket 2: row 4, c = 0.1, z = -16 -> CE = log(1 + e^-16.1) ~ 1e-7, inside [AMBIG_MIN, COUNT_MIN]
    x[2] = torch.tensor([0.0, 0, 1, (2 + np.log(1e-12)) / 2])
    x[4] = torch.tensor([-8.0, 0, 0, 8.1])
    r = ref.reference(x, w, y, pm, 6, top_x, score_x, top_y)
    assert float(r["row_max"][0]) == 0.0
    assert 0 < float(r["row_max"][2]) < ref.AMBIG_MIN and not r["ambiguous"][2]
    assert ref.AMBIG_MIN < float(r["row_max"][4]) < ref.COUNT_MIN and r["ambiguous"][4] and not r["checked"][4]
    assert r["counted"].tolist() == [False, True, False, False, False, False]
    assert r["n_counted"] == 1 and r["n_ambiguous"] == 1 and float(r["ce_sum_ambiguous"]) == float(r["row_max"][4])
    assert float(r["loss"]) == float(r["row_max"][1]) == pytest.approx(np.log1p(np.exp(-2.0)), rel=1e-14)
    # row 1 is the only counted row: its gradient is its slot's CE gradient (autograd of oracle/sce.py row_losses)
    xg = x.clone().requires_grad_(True)
    osce.row_losses(xg, y, w, top_x[:1], top_y[:1])[0, 1].backward()
    torch.testing.assert_close(r["d_hc"][1], xg.grad[1], rtol=1e-14, atol=1e-16)
    assert (r["d_hc"][[0, 2, 3, 4, 5]] == 0).all()


def test_exact_tie_splits_evenly_and_near_tie_is_excluded():
    x, w, pm = _tiny()
    y = torch.tensor([1, 0, 3, 4, 2, 1])
    # buckets 0 and 1 are duplicates (same rows, same items): rows 0 and 1 tie exactly between them
    top_x = torch.tensor([[0, 1], [0, 1], [2, 5]])
    top_y = torch.tensor([[2, 3], [2, 3], [0, 4]])
    score_x = torch.zeros(3, 2)
    r = ref.reference(x, w, y, pm, 6, top_x, score_x, top_y)
    assert r["winners"][[0, 1]].tolist() == [2, 2] and r["near_tie"] == 0 and bool(r["checked"].all())
    lo, dx = _oracle(x, y, w, pm, top_x, top_y)
    torch.testing.assert_close(r["loss"], lo, rtol=1e-14, atol=0)
    torch.testing.assert_close(r["d_hc"], dx, rtol=1e-12, atol=1e-15)
    # a near tie: bucket 1 holds item 4 in place of item 3, at row 0's logit + 1e-9 but in another direction
    w2 = w.clone()
    w2[4] = torch.tensor([1e-9, 3, 0, 0])
    top_y2 = torch.tensor([[2, 3], [2, 4], [0, 4]])
    r2 = ref.reference(x, w2, y, pm, 6, top_x, score_x, top_y2)
    assert r2["winners"][0] == 1 and r2["near_tie"] >= 1 and not r2["checked"][0] and r2["checked"][1]


def test_philox_port_known_answers():
    """philox4x32 (csrc/rp_philox.cuh): Random123's Philox4x32-10 known answer at key 0, counter 0, and two values of the
    header's host path."""
    for (seed, ctr), want in (((0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
                              ((0x123456789ABCDEF0, ps.SCE_SITE + 7), (0xB025C1A1, 0x04CF7BFB, 0x1D1519CF, 0x029F62AC)),
                              ((0xFFFFFFFFFFFFFFFF, 0xFEDCBA9876543210), (0x481ACE3B, 0xB3BAE32F, 0xC436714D, 0xEDC1FD47))):
        got = ps.philox4x32(seed, np.array([ctr], dtype=np.uint64))
        assert tuple(int(v[0]) for v in got) == want
    z = ps.sce_normals(5, 7, 200_001)
    assert z.shape == (200_001,) and np.isfinite(z).all()
    assert abs(z.mean()) < 0.02 and abs(z.var() - 1) < 0.02
    u1, _ = ps.sce_uniforms(12, 1000)
    assert u1.dtype == np.float32 and (u1 > 0).all() and (u1 <= 1).all()


def test_source_pins():
    src = open(SRC).read()
    hdr = open(os.path.join(ROOT, "replay_b200", "csrc", "rp_philox.cuh")).read()
    # the Philox constants and the draw the port restates
    for name, v in (("M0", 0xD2511F53), ("M1", 0xCD9E8D57), ("W0", 0x9E3779B9), ("W1", 0xBB67AE85)):
        assert re.search(rf"\b{name} = 0x{v:08X}u", hdr), name
    assert "constexpr unsigned long long kSceSite = 0x5CEull << 40;" in src and ps.SCE_SITE == 0x5CE << 40
    draw = src[src.index("__global__ void sce_draw_kernel("):]
    draw = draw[:draw.index("\n}\n")]
    for line in ("const unsigned long long seed = a.seed + *a.rng_counter;",
                 "const uint4 r = philox4x32(seed, kSceSite + (unsigned long long)p);",
                 "const float u1 = ((float)r.x + 1.f) * 2.3283064365386963e-10f;",
                 "const float u2 = (float)r.y * 2.3283064365386963e-10f;",
                 "const float rad = sqrtf(-2.f * logf(u1));", "sincospif(2.f * u2, &s, &c);",
                 "a.draw[2 * p] = rad * c;", "if (2 * p + 1 < n_elems) a.draw[2 * p + 1] = rad * s;"):
        assert line in draw, line
    assert "const float scale = 1.f / sqrtf(sqrtf((float)a.d_true));" in src
    # the bucket matrix is the first workspace region, omega (mix_x) the second, each 256-byte aligned
    lay = src[src.index("static size_t sce_layout("):]
    lay = lay[:lay.index("\n}\n")]
    takes = re.findall(r"const size_t (o_\w+) = (.*?take\(.*?\))( : 0)?;", lay)
    assert takes[0] == ("o_buck", "take(nb * d * 2)", "")
    assert takes[1] == ("o_omega", "s->mix_x ? take(ru(cap, 64) * nbp * 2)", " : 0")
    assert "auto take = [&](size_t bytes) { const size_t o = off; off = ru(off + bytes, 256); return o; };" in lay
    # the chunk of buckets: the formula the GPU test restates
    assert "constexpr size_t kSceChunkBytes = 256ull << 20;" in src
    assert 'const char* env = getenv("RP_SCE_CHUNK_BYTES");' in lay
    assert "const size_t budget = env ? (size_t)atoll(env) : kSceChunkBytes;" in lay
    assert "size_t chunk = budget / per_bucket;" in lay
    assert "chunk = chunk < 1 ? 1 : (chunk > nb ? nb : chunk);" in lay
    per = re.search(r"const size_t per_bucket = (.*?);", lay).group(1)
    gpu = _gpu_module()
    for d, bsx, bsy, nb in ((512, 1024, 1024, 43), (128, 256, 256, 64), (64, 1, 1, 600), (256, 65, 1000, 3)):
        bsxp, bsyp = -(-bsx // 64) * 64, -(-bsy // 64) * 64
        want = min(max((256 << 20) // eval(per, {}, dict(bsxp=bsxp, bsyp=bsyp, d=d)), 1), nb)
        assert gpu.buckets_per_chunk(d, bsx, bsy, nb) == want
    assert gpu.buckets_per_chunk(512, 1024, 1024, 43) == 42


def _gpu_module():
    spec = importlib.util.spec_from_file_location("sce_head_cases", os.path.join(ROOT, "tests", "test_gpu_sce_head.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("d,d_true,hd_valid", [(128, 128, 129), (64, 64, 200), (64, 50, 100), (256, 191, 96), (128, 96, 0),
                                               (128, 101, 50), (256, 200, 48), (512, 400, -1)])
def test_shape_errors(d, d_true, hd_valid):
    """hd_valid > 128, d not a multiple of the slot, d_true != the layout's real features: RP_ESHAPE before any memory is
    touched (non-NULL dummy pointers)."""
    from replay_b200._lib import SCE_ALL, SceDesc, lib
    L = lib()
    buf = ctypes.create_string_buffer(64)
    p = ctypes.cast(buf, ctypes.c_void_p).value
    s = SceDesc()
    for f in ("hc", "table", "labels", "pad_mask", "n_rows", "rng_counter", "draw", "top_x", "score_x", "top_y",
              "loss_out", "workspace"):
        setattr(s, f, p)
    s.capacity, s.n_items, s.d, s.d_true, s.hd_valid = 300, 500, d, d_true, hd_valid
    s.n_buckets, s.bucket_size_x, s.bucket_size_y, s.workspace_bytes = 4, 16, 16, 1 << 40
    assert L.rp_sce_head_fwd(ctypes.byref(s), SCE_ALL, None) == -2
    assert L.rp_sce_head_bwd(ctypes.byref(s), p, None) == -2
