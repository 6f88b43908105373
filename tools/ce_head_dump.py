"""Dump every output of the full-catalog CE and BCE heads on fixed seeds, or compare two dumps bit for bit.

    python tools/ce_head_dump.py --out A.pt          # (RP_B200_LIB=<other build> selects the library to dump)
    python tools/ce_head_dump.py --compare A.pt B.pt # bitwise equal tensors counted; per differing tensor its max |diff|,
                                                     # max relative diff and max |A|

Labels are unique (a permutation of the catalog), so the dE pass's one-hot scatter has no order-dependent fp32 atomics and
two builds that run the same floating-point operations in the same order must agree exactly.  Cases, each with and
without bias:
- d = 64 / 128 / 256: the fused pass with one column split ("P1": as many row tiles as SMs) and with several ("Pn": one
  row tile); the two-pass path (no d_hc in the forward); the fused pass behind the two-pass forward (large logits fail the
  bound) at both shapes; the BCE head's fused token pass (P1 and Pn) and its un-fused forward; and the per-row CE
  variants (row_weight, and loss_kind 1 = LogInCE) on the fused, two-pass and behind paths.
- d = 512: the materialised-G backward of CE, its per-row variants and BCE, in one G chunk and in 128-row chunks.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch


def _inputs(T, n_valid, I, d, bias, scale_h, scale_e, seed):
    g = torch.Generator().manual_seed(seed)
    hc = (torch.randn(T, d, generator=g) * scale_h).to(torch.bfloat16)
    hc[n_valid:] = 0
    table = (torch.randn(I, d, generator=g) * scale_e).to(torch.bfloat16)
    b = (torch.randn(I, generator=g) * 0.5).float().cuda() if bias else None
    labels = torch.randperm(I, generator=g)[:T].int()
    nv = torch.tensor([n_valid], dtype=torch.int32, device="cuda")
    row_weight = (torch.rand(T, generator=g) * 2).cuda()
    return hc.cuda(), table.cuda(), b, labels.cuda(), nv, row_weight


def _run(ops, kind, path, T, n_valid, I, d, bias, seed):
    """kind: "ce", "ce_w" (row_weight), "login" (LogInCE) or "bce"; path: "fused", "twopass" (no d_hc) or "behind"."""
    scale_h, scale_e = (2.0, 1.0) if path == "behind" else (0.5, 0.3)
    hc, table, b, labels, nv, roww = _inputs(T, n_valid, I, d, bias, scale_h, scale_e, seed)
    st = ops.CEHeadState(T, I, d, "cuda")
    d_hc = torch.zeros(T, d, device="cuda", dtype=torch.bfloat16)
    d_tab = torch.zeros(I + 1, d, device="cuda")
    d_b = torch.zeros(I + 1, device="cuda") if bias else None
    fwd, bwd = (ops.bce_head_fwd, ops.bce_head_bwd) if kind == "bce" else (ops.ce_head_fwd, ops.ce_head_bwd)
    row = {"ce_w": dict(row_weight=roww), "login": dict(loss_kind=1, log_eps=1e-6, clamp=10.0)}.get(kind, {})
    loss = fwd(st, hc, table, labels, nv, bias=b, d_hc=None if path == "twopass" else d_hc, n_valid_hint=T, **row).clone()
    if kind != "bce" and path != "twopass" and d <= 256:
        assert ops.ce_head_fused_taken(st) == (path != "behind"), path
    bwd(st, hc, table, labels, nv, d_hc, d_tab, bias=b, d_bias=d_b)
    torch.cuda.synchronize()
    out = dict(loss=loss, d_hc=d_hc, d_table=d_tab)
    if kind != "bce":
        out.update(lse=st.lse, cvec=st.cvec)
    if bias:
        out["d_bias"] = d_b
    return {k: v.cpu() for k, v in out.items()}


def dump(path):
    from replay_b200 import ops
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    shapes = {"P1": (sms * 128, sms * 128 - 37, sms * 128 + 3011), "Pn": (1024, 999, 20011)}
    narrow = [("ce", "fused", "P1"), ("ce", "fused", "Pn"), ("ce", "twopass", "Pn"), ("ce", "behind", "Pn"), ("ce", "behind", "P1"),
              ("bce", "fused", "P1"), ("bce", "fused", "Pn"), ("bce", "twopass", "Pn")]
    narrow += [(k, p, s) for k in ("ce_w", "login") for p, s in (("fused", "P1"), ("fused", "Pn"), ("twopass", "Pn"),
                                                                 ("behind", "P1"), ("behind", "Pn"))]
    wide = [(k, "twopass", "Pn") for k in ("ce", "ce_w", "login", "bce")]
    res = {}
    for d in (64, 128, 256, 512):
        for chunks in (("one",) if d <= 256 else ("one", "several")):
            if chunks == "several":
                os.environ["RP_CE_WIDE_G_BYTES"] = "1"   # the smallest budget: 128-row G chunks (read on every call)
            for bias in (False, True):
                for i, (kind, p, s) in enumerate(narrow if d <= 256 else wide):
                    T, nv, I = shapes[s]
                    case = f"{kind}_{p}_{s}_d{d}_{'bias' if bias else 'nobias'}" + (f"_{chunks}" if d > 256 else "")
                    for k, v in _run(ops, kind, p, T, nv, I, d, bias, seed=1000 * d + 10 * i + bias).items():
                        res[f"{case}/{k}"] = v
            os.environ.pop("RP_CE_WIDE_G_BYTES", None)
    torch.save(res, path)
    print(f"{len(res)} tensors -> {path}")


def _bits(t):
    return t.contiguous().view(torch.uint8)


def compare(a_path, b_path):
    """Exit status 0 only if every tensor is bitwise equal.  Builds that round differently (e.g. a different exp2 on some
    logits) are judged from the per-tensor lines: max |B - A|, max |B - A| / |A| over the elements with A != 0 (inf where
    A = 0 but B != 0), and the largest finite |A| for scale."""
    a, b = torch.load(a_path), torch.load(b_path)
    if sorted(a) != sorted(b):
        print("different tensor sets:", sorted(set(a) ^ set(b)))
        return 1
    n_diff = 0
    for k in sorted(a):
        if a[k].shape != b[k].shape:
            print(f"{k}: shape {tuple(a[k].shape)} vs {tuple(b[k].shape)}")
            n_diff += 1
            continue
        if torch.equal(_bits(a[k]), _bits(b[k])):
            continue
        n_diff += 1
        x, y = a[k].double(), b[k].double()
        diff = torch.where(x == y, 0.0, (y - x).abs()).nan_to_num(float("inf"))   # equal infinities differ by 0
        nz = x != 0
        rel = (diff[nz] / x[nz].abs()).max().item() if nz.any() else 0.0
        if ((~nz) & (diff != 0)).any():
            rel = float("inf")
        n = int((_bits(a[k]) != _bits(b[k])).sum())
        print(f"{k}: {n} bytes differ, max |diff| {diff.max().item():.3e}, max rel {rel:.3e}, max |A| {x[x.isfinite()].abs().max().item():.3e}")
    print(f"{len(a) - n_diff} of {len(a)} tensors identical" if n_diff else f"identical ({len(a)} tensors)")
    return 1 if n_diff else 0


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--compare", nargs=2)
    args = ap.parse_args()
    if args.compare:
        sys.exit(compare(*args.compare))
    dump(args.out)
