"""A DiffTransformer training step is bitwise reproducible.  The kernels themselves are tested against float64 in
test_gpu_diff_fp64.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda")


def _pad_mask(B, L, kind, g):
    if kind == "full":
        return torch.ones(B, L, dtype=torch.bool)
    if kind == "one":
        pm = torch.zeros(B, L, dtype=torch.bool)
        pm[:, -1] = True
        return pm
    lens = torch.randint(1, L + 1, (B,), generator=g)
    return torch.arange(L).unsqueeze(0) >= (L - lens).unsqueeze(1)


def test_training_step_is_deterministic(cuda):
    from replay_b200.engine_diff import DiffConfig, DiffEngine

    cfg = DiffConfig(n_items=300, d=128, n_heads=2, n_blocks=2, max_len=100, out_norm="rmsnorm")
    g = torch.Generator().manual_seed(1)
    pm = _pad_mask(8, 100, "random", g)
    ids = torch.where(pm, torch.randint(0, 300, (8, 100), generator=g), torch.full((8, 100), 300))
    labels = torch.randint(0, 300, (8, 100), generator=g)
    out = []
    for _ in range(2):
        eng = DiffEngine(cfg, 8, 100, cuda, seed=3)
        eng.set_batch(ids.to(cuda), pm.to(cuda), labels.to(cuda), pm.to(cuda))
        eng.g32.zero_()
        loss = eng.forward_train().clone()
        eng.backward()
        torch.cuda.synchronize()
        # the embedding backward and the bias column sums are SASRec's kernels, which accumulate with fp32 atomics
        shared = ("item_emb", "pos_emb", ".ff_bg", ".ff_b1", ".ff_b2")
        grads = {k: v.clone().cpu() for k, v in eng.grads.items() if not k.endswith(shared)}
        out.append((loss.cpu(), eng.x[-1].clone().cpu(), grads))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])
    for k in out[0][2]:
        assert torch.equal(out[0][2][k], out[1][2][k]), k
