"""Attention forward and SASRec training at long windows with 128-wide heads, against 64-wide heads of equal FLOPs.

    python tools/bench_attn_long.py [--iters 50] [--warmup 5] [--steps 20]

fwd   rp_attn_fwd, causal with pad keys masked, every token real, B = 32 sequences of d = 512 columns: head_dim 128 x 4
      heads next to head_dim 64 x 8 heads at L in {256, 384, 512}.  At L = 256 head_dim 128 runs the resident kernel
      (attn_fwd_kernel<128, 1>), above it the kernel that streams V (<128, 2>); head_dim 64 is resident throughout.  Timed
      in training mode (row statistics and p_save written, as the un-fused backward needs) and at inference (no saves).
      TFLOP/s counts the causal-useful work only: 2 GEMMs x 2 x head_dim x L (L + 1) / 2 per (sequence, head).
step  one CUDA-graph training step (forward + backward + Adam) of the legacy SasRec body, hidden 128, 2 blocks,
      L = 512, dropout 0.2, |I| = 50 K, batch 128: head_count 1 (one 128-wide head) against head_count 2 (two 64-wide).
Prints the card name and power limit it read, then one JSON line per measurement."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

B_FWD, D_FWD = 32, 512
N_ITEMS, B_STEP, L_STEP = 50_000, 128, 512


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        out = ""
    return out or torch.cuda.get_device_name(0) + ", power limit unknown"


def elapsed_ms(fn, n, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def bench_fwd(L, hd, iters, warmup):
    from replay_b200._lib import AttnDesc, check, lib

    H, T, d = D_FWD // hd, B_FWD * L, D_FWD
    Lp = (L + 63) // 64 * 64
    g = torch.Generator(device="cuda").manual_seed(L + hd)
    q = torch.randn(T, d, device="cuda", generator=g).to(torch.bfloat16)
    kv = torch.randn(T, 2 * d, device="cuda", generator=g).to(torch.bfloat16)
    pad = torch.ones(T, dtype=torch.uint8, device="cuda")
    out = torch.empty(T, d, device="cuda", dtype=torch.bfloat16)
    p_save = torch.zeros(B_FWD * H, Lp, Lp, device="cuda", dtype=torch.bfloat16)
    inv = torch.empty(B_FWD * H, Lp, device="cuda")
    m = torch.empty(B_FWD * H, Lp, device="cuda")
    ad = AttnDesc()
    ad.q, ad.q_rows, ad.q_cols, ad.ldq, ad.q_c0 = q.data_ptr(), T, d, d, 0
    ad.k, ad.k_rows, ad.k_cols, ad.ldk, ad.k_c0 = kv.data_ptr(), T, 2 * d, 2 * d, 0
    ad.v, ad.v_rows, ad.v_cols, ad.ldv, ad.v_c0 = kv.data_ptr(), T, 2 * d, 2 * d, d
    ad.B, ad.H, ad.L, ad.head_dim = B_FWD, H, L, hd
    ad.causal, ad.mask_pad_keys, ad.scale = 1, 1, 0.0
    ad.pad_mask, ad.out, ad.ldo = pad.data_ptr(), out.data_ptr(), d
    stream = torch.cuda.current_stream().cuda_stream
    flop = 2 * 2 * hd * L * (L + 1) / 2 * B_FWD * H
    res = {}
    for mode in ("train", "infer"):
        train = mode == "train"
        ad.p_save, ad.inv_sum, ad.m_save = ((p_save.data_ptr(), inv.data_ptr(), m.data_ptr()) if train else (None, None, None))
        ms = elapsed_ms(lambda: check(lib().rp_attn_fwd(ctypes.byref(ad), stream), "rp_attn_fwd"), iters, warmup)
        res[mode] = dict(ms=round(ms, 4), tflops=round(flop / ms / 1e9, 1))
    return dict(kind="fwd", L=L, head_dim=hd, heads=H, batch=B_FWD, causal_useful_gflop=round(flop / 1e9, 2), **res)


def bench_step(heads, steps, warmup):
    from replay_b200.engine import EncoderConfig, SasRecEngine
    from replay_b200.synthetic import make_sequences
    from replay_b200.trainer import Trainer

    cfg = EncoderConfig(n_items=N_ITEMS, d=128, n_heads=heads, n_blocks=2, max_len=L_STEP, dropout=0.2, variant="legacy")
    eng = SasRecEngine(cfg, B_STEP, L_STEP, "cuda", seed=1)
    ids, pm, lab, tm = (t.cuda() for t in make_sequences(B_STEP, N_ITEMS, L_STEP, seed=3))
    tr = Trainer(eng)
    ms = elapsed_ms(lambda: tr.step(ids, pm, lab, tm), steps, warmup)
    loss = float(tr.step(ids, pm, lab, tm)[0])
    return dict(kind="step", model="legacy SasRec", hidden=128, heads=heads, head_slot=cfg.head_slot, L=L_STEP, batch=B_STEP,
                n_items=N_ITEMS, real_tokens=int(pm.sum()), ms_per_step=round(ms, 3), train_seq_per_s=round(B_STEP / ms * 1e3, 1),
                loss=round(loss, 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_attn_long.py needs a GPU")
    print("card:", card(), flush=True)
    for L in (256, 384, 512):
        for hd in (128, 64):
            print(json.dumps(bench_fwd(L, hd, args.iters, args.warmup)), flush=True)
    for heads in (1, 2):
        print(json.dumps(bench_step(heads, args.steps, args.warmup)), flush=True)


if __name__ == "__main__":
    main()
