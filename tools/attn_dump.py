"""Dump the outputs of the fused attention kernels (rp_attn_fwd: O, m_save, inv_sum; rp_attn_bwd: dQ, dK, dV) on fixed
seeds, or compare two dumps bit for bit.

    python tools/attn_dump.py --out A.pt          # (RP_B200_LIB=<other build> selects the library to dump)
    python tools/attn_dump.py --compare A.pt B.pt # "identical", or every differing tensor with its largest difference

Cases (head_dim 64, L 200, the masks of bench.make_batches at seed 1234):
- c2_packed / c2_packed_drop: the config-2 training body's operands, 512 sequences, 2 heads, on the packed rows of
  rp_row_plan (causal, pad keys masked), without and with dropout 0.2;
- c3_bert: config-3 BERT4Rec, 256 sequences, 4 heads, padded rows, key-padding mask only, dropout 0.1;
- legacy: the legacy SASRec's causal mask without a pad-key mask, 64 sequences, 2 heads, padded rows, dropout 0.2.
"""
import argparse
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

SEED, OFF, CTR = 77, 3, 5


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _row_plan(pad, labels, tmask, n_items):
    """rp_row_plan -> (seq_first, seq_off, packed row count, token of every packed row)."""
    from replay_b200._lib import check, lib

    B, L = pad.shape
    T = B * L
    dev = "cuda"
    sel = tmask & (labels >= 0) & (labels < n_items)
    vi = torch.zeros(T, dtype=torch.int32)
    idx = sel.reshape(-1).nonzero()[:, 0].to(torch.int32)
    vi[: idx.numel()] = idx
    vi, nv = vi.to(dev), torch.tensor([idx.numel()], dtype=torch.int32, device=dev)
    first, off = torch.zeros(B, dtype=torch.int32, device=dev), torch.zeros(B, dtype=torch.int32, device=dev)
    n_rows, row_tok, valid_rows = (torch.zeros(1, dtype=torch.int32, device=dev), torch.zeros(T, dtype=torch.int32, device=dev),
                                   torch.zeros(T, dtype=torch.int32, device=dev))
    pad_d, lab_d, tm_d = pad.to(dev).contiguous(), labels.to(dev).contiguous(), tmask.to(dev).contiguous()
    check(lib().rp_row_plan(pad_d.data_ptr(), lab_d.data_ptr(), tm_d.data_ptr(), B, L, n_items, vi.data_ptr(), nv.data_ptr(),
                            first.data_ptr(), off.data_ptr(), n_rows.data_ptr(), row_tok.data_ptr(), valid_rows.data_ptr(),
                            _stream()), "rp_row_plan")
    torch.cuda.synchronize()
    return first, off, int(n_rows[0]), row_tok


def _run(pad, H, causal, mpk, drop, seed, plan=None):
    from replay_b200._lib import AttnBwdDesc, AttnDesc, check, lib

    B, L = pad.shape
    d, Lp = H * 64, (L + 63) // 64 * 64
    T = B * L
    rows = T if plan is None else plan[2]
    g = torch.Generator().manual_seed(seed)
    q = torch.zeros(T, d, dtype=torch.bfloat16)
    kv = torch.zeros(T, 2 * d, dtype=torch.bfloat16)
    d_o = torch.zeros(T, d, dtype=torch.bfloat16)
    q[:rows] = torch.randn(rows, d, generator=g).to(torch.bfloat16)
    kv[:rows] = torch.randn(rows, 2 * d, generator=g).to(torch.bfloat16)
    d_o[:rows] = torch.randn(rows, d, generator=g).to(torch.bfloat16)
    q, kv, d_o, pad_d = q.cuda(), kv.cuda(), d_o.cuda(), pad.cuda().contiguous()
    ctr = torch.tensor([CTR], dtype=torch.int64, device="cuda")
    out = torch.zeros(T, d, dtype=torch.bfloat16, device="cuda")
    inv = torch.zeros(B * H, Lp, device="cuda")
    m = torch.zeros(B * H, Lp, device="cuda")
    dq = torch.zeros(T, d, dtype=torch.bfloat16, device="cuda")
    dkv = torch.zeros(T, 2 * d, dtype=torch.bfloat16, device="cuda")

    def common(x):
        x.q, x.q_rows, x.q_cols, x.ldq, x.q_c0 = q.data_ptr(), T, d, d, 0
        x.k, x.k_rows, x.k_cols, x.ldk, x.k_c0 = kv.data_ptr(), T, 2 * d, 2 * d, 0
        x.v, x.v_rows, x.v_cols, x.ldv, x.v_c0 = kv.data_ptr(), T, 2 * d, 2 * d, d
        x.B, x.H, x.L, x.head_dim = B, H, L, 64
        x.causal, x.mask_pad_keys, x.scale, x.pad_mask = causal, mpk, 0.0, pad_d.data_ptr()
        x.drop_p, x.seed, x.drop_off, x.seed_ptr = drop, SEED, OFF, ctr.data_ptr()
        if plan is not None:
            x.seq_first, x.seq_off = plan[0].data_ptr(), plan[1].data_ptr()
        return x

    ad = common(AttnDesc())
    ad.out, ad.ldo, ad.p_save, ad.inv_sum, ad.m_save = out.data_ptr(), d, None, inv.data_ptr(), m.data_ptr()
    check(lib().rp_attn_fwd(ctypes.byref(ad), _stream()), "rp_attn_fwd")
    bd = common(AttnBwdDesc())
    bd.d_out, bd.do_rows, bd.do_cols, bd.ld_do = d_o.data_ptr(), T, d, d
    bd.out, bd.ldo = out.data_ptr(), d
    bd.m_save, bd.inv_sum = m.data_ptr(), inv.data_ptr()
    bd.dq, bd.ld_dq, bd.dq_c0 = dq.data_ptr(), d, 0
    bd.dk, bd.ld_dk, bd.dk_c0 = dkv.data_ptr(), 2 * d, 0
    bd.dv, bd.ld_dv, bd.dv_c0 = dkv.data_ptr(), 2 * d, d
    check(lib().rp_attn_bwd(ctypes.byref(bd), _stream()), "rp_attn_bwd")
    torch.cuda.synchronize()
    res = dict(O=out[:rows], m_save=m, inv_sum=inv, dQ=dq[:rows], dK=dkv[:rows, :d], dV=dkv[:rows, d:])
    return {k: v.cpu() for k, v in res.items()}


def dump(path):
    import bench

    c2, c3 = bench.CONFIGS[2], bench.CONFIGS[3]
    ids, pm, labels, tmask = bench.make_batches(c2, 512, seed=1234)
    plan = _row_plan(pm, labels, tmask, c2["n_items"])
    pm3 = bench.make_batches(c3, 256, seed=1234)[1]
    cases = {
        "c2_packed": lambda: _run(pm, 2, 1, 1, 0.0, 1, plan),
        "c2_packed_drop": lambda: _run(pm, 2, 1, 1, 0.2, 2, plan),
        "c3_bert": lambda: _run(pm3, 4, 0, 1, 0.1, 3),
        "legacy": lambda: _run(pm[:64], 2, 1, 0, 0.2, 4),
    }
    res = {}
    for case, fn in cases.items():
        for k, v in fn().items():
            res[f"{case}/{k}"] = v
    torch.save(res, path)
    print(f"{len(res)} tensors -> {path}")


def _bits(t):
    return t.contiguous().view(torch.uint8)


def compare(a_path, b_path):
    a, b = torch.load(a_path), torch.load(b_path)
    if sorted(a) != sorted(b):
        print("different tensor sets:", sorted(set(a) ^ set(b)))
        return 1
    n_diff = 0
    for k in a:
        if a[k].shape != b[k].shape or not torch.equal(_bits(a[k]), _bits(b[k])):
            n_diff += 1
            diff = (a[k].double() - b[k].double()).abs().nan_to_num(0)
            rel = diff.max() / a[k].double().abs().max().clamp_min(1e-30)
            n = int((a[k] != b[k]).sum()) if a[k].shape == b[k].shape else -1
            print(f"{k}: {n} of {a[k].numel()} elements differ, max |diff| {diff.max().item():.3e} "
                  f"({rel.item():.3e} of max |value|)")
    print("identical" if n_diff == 0 else f"{n_diff} of {len(a)} tensors differ", f"({len(a)} tensors)")
    return 1 if n_diff else 0


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--compare", nargs=2)
    args = ap.parse_args()
    if args.compare:
        sys.exit(compare(*args.compare))
    dump(args.out)
