"""Full-catalog BCE head against the CE head and against materialised torch (CUDA events, median of 10), plus config-2
training throughput with each loss.  Prints one JSON object with the card's name and power limit.

    python tools/bench_bce_head.py [--no-train]"""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from replay_b200 import ops  # noqa: E402


def timeit(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(iters + 1)]
    ev[0].record()
    for i in range(iters):
        fn()
        ev[i + 1].record()
    torch.cuda.synchronize()
    ts = sorted(ev[i].elapsed_time(ev[i + 1]) for i in range(iters))
    return ts[len(ts) // 2]


def head_case(T, I, d, bias):
    g = torch.Generator(device="cuda").manual_seed(0)
    hc = (torch.randn(T, d, device="cuda", generator=g) * 0.5).bfloat16()
    table = (torch.randn(I, d, device="cuda", generator=g) * 0.3).bfloat16()
    b = torch.randn((I + 127) // 128 * 128, device="cuda", generator=g) * 0.1 if bias else None
    labels = torch.randint(0, I, (T,), device="cuda", generator=g).int()
    nv = torch.tensor([T], dtype=torch.int32, device="cuda")
    st = ops.CEHeadState(T, I, d, "cuda")
    d_hc = torch.zeros(T, d, device="cuda", dtype=torch.bfloat16)
    d_tab = torch.zeros(I, d, device="cuda")
    d_b = torch.zeros(I, device="cuda") if bias else None

    def ce():
        ops.ce_head_fwd(st, hc, table, labels, nv, bias=b, d_hc=d_hc, n_valid_hint=T)
        ops.ce_head_bwd(st, hc, table, labels, nv, d_hc, d_tab, bias=b, d_bias=d_b, n_valid_hint=T)

    def bce():
        ops.bce_head_fwd(st, hc, table, labels, nv, bias=b, d_hc=d_hc, n_valid_hint=T)
        ops.bce_head_bwd(st, hc, table, labels, nv, d_hc, d_tab, bias=b, d_bias=d_b, n_valid_hint=T)

    out = dict(T=T, I=I, d=d, bias=bias, ce_ms=timeit(ce), bce_ms=timeit(bce))
    if T * I * 4 * 3 < 8e9:   # materialised torch: logits fp32 + grad + target
        hr = hc.float().requires_grad_()
        Wr = table.float().requires_grad_()
        br = b[:I].clone().requires_grad_() if bias else None
        tgt = torch.zeros(T, I, device="cuda")
        tgt[torch.arange(T, device="cuda"), labels.long()] = 1.0

        def torch_bce():
            x = torch.nn.functional.linear(hr, Wr, br)
            loss = torch.nn.functional.binary_cross_entropy_with_logits(x, tgt, reduction="sum") / T
            loss.backward()

        out["torch_materialised_ms"] = timeit(torch_bce, iters=5, warm=2)
    return out


def train_rate(loss_name, steps=30, warm=5):
    from replay_b200.nn.loss import BCE, CE
    from replay_b200.nn.sequential import SasRec
    from replay_b200.schema import TensorFeatureInfo, TensorSchema
    from replay_b200.synthetic import make_sequences

    n_items, d, L, B = 50_000, 128, 200, 512    # config 2
    model = SasRec.from_params(TensorSchema(TensorFeatureInfo("item_id", n_items, n_items, d)), embedding_dim=d, num_heads=2,
                               num_blocks=2, max_sequence_length=L, dropout=0.2, seed=0)
    model.loss = BCE() if loss_name == "bce" else CE()
    model.train()
    ids, pm, lab, tm = (t.cuda() for t in make_sequences(B, n_items, L, seed=1))
    for _ in range(warm):
        model.core.fused_step(ids, pm, lab, tm, lr=1e-3)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        loss = model.core.fused_step(ids, pm, lab, tm, lr=1e-3)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    return dict(seq_per_s=B * steps / dt, ms_per_step=dt / steps * 1e3, last_loss=float(loss))


def main():
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    res = dict(card=card, heads=[])
    for T, I, d, bias in ((51200, 50_000, 128, False), (4096, 50_000, 128, False), (4096, 100_000, 256, True),
                          (28672, 100_000, 256, True)):
        res["heads"].append(head_case(T, I, d, bias))
    if "--no-train" not in sys.argv:
        res["train_config2"] = [dict(loss=k, **train_rate(k)) for k in ("ce", "bce", "ce", "bce")]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
