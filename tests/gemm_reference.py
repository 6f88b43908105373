"""float64 model of rp_gemm's contract (csrc/rp_gemm.cu, include/rp_b200.h) on CPU tensors.

``gemm`` takes the keyword arguments of replay_b200.ops.gemm (seed_ptr, m_limit and k_limit as one-element tensors rather
than device pointers) and returns what the kernel must leave in C (and C2) from C's first element to the end of its
storage - including every element it must not touch:

- operands are read from the stored 2-D arrays (the views passed as A / B): batch element bz = outer*inner + in starts at
  row r0 + outer*ro + in*ri and column c0 + outer*co + in*ci; the contraction runs over ceil(K_eff / 64) * 64 elements
  (K_eff = clamp(*k_limit - k_limit_base, 0, K)), elements inside the stored array read as they are (the next batch
  element's data in the K tail), elements past it as 0; K split s covers chunks [kc*s/S, kc*(s+1)/S);
- the epilogue in the header's order: alpha, bias, C2 capture, act, dropout, gate, residual, post-residual dropout,
  rowmask[rowmask_off0 + outer*rowmask_oo + m]; dropout keeps come from tests/dropout_stream.py (row bz*M + m, column n);
- out_mode 0 / 2 store, 1 / 4 add to the previous contents, 3 stores split s's partial at C + s*c_split_stride; rows of
  128-row tiles that m_limit skips, rows >= M, columns >= N and the pitch padding keep their previous contents.

Each written element also gets a tolerance ``atol``: an fp32 accumulation slack of ACC_SLACK x |alpha| x sum_k |a_k b_k|
carried through the epilogue (the larger deviation of the epilogue at acc +- slack), plus a few fp32 ulps for every
epilogue stage.  ``err`` measures a result in units of that tolerance, plus one bf16 rounding for bf16 outputs.
``mistake`` selects a deliberately wrong model (tests/test_gemm_reference_cpu.py shows the tolerance rejects each).
"""
import math

import numpy as np
import torch

from dropout_stream import keep_draws

CHUNK = 64
TILE_M = 128
ACC_SLACK = 1e-5          # fp32 accumulation error of the contraction, relative to |alpha| sum_k |a_k b_k|
EPI_REL = 2.0 ** -20      # fp32 (fast-math) error of one epilogue stage, relative to the magnitudes it combines
LOG2E = 1.4426950408889634

MISTAKES = ("bias_after_act", "c2_after_act", "drop_before_act", "residual_before_drop", "post_drop_before_residual",
            "gelu_tanh", "gelu_tanh_grad", "drop_col_plus_one", "drop_row_m", "rowmask_by_inner", "k_tail_zero",
            "bias_per_split")


def flat_from(t):
    """1-D view of ``t``'s storage from its first element to the end of the storage (what rp_gemm can address)."""
    n = t.untyped_storage().nbytes() // t.element_size() - t.storage_offset()
    return torch.as_strided(t, (n,), (1,), t.storage_offset())


def gelu_erf(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def gelu_tanh(x):
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3)))


def gelu_erf_grad(z):
    return 0.5 * (1.0 + torch.erf(z / math.sqrt(2.0))) + z * torch.exp(-0.5 * z * z) / math.sqrt(2.0 * math.pi)


def gelu_tanh_grad(z):
    z = z.detach().clone().requires_grad_(True)
    gelu_tanh(z).sum().backward()
    return z.grad


def _padded(X, rows, cols):
    """float64 copy of the stored array X grown with zeros to at least [rows, cols]."""
    R, Cn = X.shape
    P = torch.zeros(max(R, rows), max(Cn, cols), dtype=torch.float64)
    P[:R, :Cn] = X.double()
    return P


def _limit(t):
    return None if t is None else int(torch.as_tensor(t).reshape(-1)[0])


def contraction(A, B, M, N, K, *, a_mn=False, b_mn=False, batch=1, inner=1, a_off=(0,) * 6, b_off=(0,) * 6, split_k=1,
                k_limit=None, k_limit_base=0, mistake=None):
    """(acc, mag): float64 [split_k, batch, M, N] partial sums of each K split and their sum_k |a_k b_k|."""
    k_eff = K
    if k_limit is not None:
        k_eff = max(0, min(K, _limit(k_limit) - k_limit_base))
    kc = -(-k_eff // CHUNK)
    klen = kc * CHUNK
    if mistake == "k_tail_zero":
        klen = k_eff
    ends = [(kc * s // split_k * CHUNK, kc * (s + 1) // split_k * CHUNK) for s in range(split_k)]

    def starts(off, b):
        outer, i = divmod(b, inner)
        return off[0] + outer * off[1] + i * off[2], off[3] + outer * off[4] + i * off[5]

    def rows_needed(off, mn, n_out):
        r_max = max(starts(off, b)[0] for b in range(batch))
        c_max = max(starts(off, b)[1] for b in range(batch))
        return (r_max + klen, c_max + n_out) if mn else (r_max + n_out, c_max + klen)

    PA, PB = _padded(A, *rows_needed(a_off, a_mn, M)), _padded(B, *rows_needed(b_off, b_mn, N))

    def fetch(P, mn, r, c, n_out):
        return P[r:r + klen, c:c + n_out].T if mn else P[r:r + n_out, c:c + klen]

    acc = torch.zeros(split_k, batch, M, N, dtype=torch.float64)
    mag = torch.zeros_like(acc)
    for b in range(batch):
        a = fetch(PA, a_mn, *starts(a_off, b), M)
        w = fetch(PB, b_mn, *starts(b_off, b), N)
        for s, (k0, k1) in enumerate(ends):
            k1 = min(k1, klen)
            acc[s, b] = a[:, k0:k1] @ w[:, k0:k1].T
            mag[s, b] = a[:, k0:k1].abs() @ w[:, k0:k1].abs().T
    return acc, mag


def _keep(seed_eff, off, p, batch, M, N, mistake):
    rows = np.arange(batch)[:, None] * M + np.arange(M)[None, :]
    if mistake == "drop_row_m":
        rows = np.broadcast_to(np.arange(M)[None, :], (batch, M))
    cols = N + 1 if mistake == "drop_col_plus_one" else N
    k = keep_draws(seed_eff, off, p, rows.reshape(-1), cols).view(batch, M, cols)
    return k[..., 1:] if mistake == "drop_col_plus_one" else k


def _geom(C, c_geom):
    if c_geom is None:
        return C.stride(0), 0, 0, 0
    return c_geom


def _index(M, N, batch, inner, geom):
    """int64 [batch, M, N]: element offset of (bz, m, n) in C's flat storage."""
    ldc, off0, oo, oi = geom
    bz = torch.arange(batch)
    base = off0 + (bz // inner) * oo + (bz % inner) * oi
    return base[:, None, None] + torch.arange(M)[None, :, None] * ldc + torch.arange(N)[None, None, :]


def _at(t, idx):
    """Values of a same-geometry operand (gate, residual) at C's element offsets."""
    return flat_from(t)[idx].double()


ORDER = ("bias", "c2", "act", "drop", "gate", "residual", "post_drop", "rowmask")
# mistake -> (stage, the stage it is wrongly placed after)
_MOVED = {"bias_after_act": ("bias", "act"), "c2_after_act": ("c2", "act"), "drop_before_act": ("drop", "c2"),
          "residual_before_drop": ("residual", "act"), "post_drop_before_residual": ("post_drop", "gate")}


def _order(mistake):
    """Epilogue stage order of the header, or the misplaced order of a mistake."""
    if mistake not in _MOVED:
        return ORDER
    st, after = _MOVED[mistake]
    order = [s for s in ORDER if s != st]
    order.insert(order.index(after) + 1, st)
    return tuple(order)


def gemm(A, B, C, M, N, K, *, a_mn=False, b_mn=False, bias=None, act=0, residual=None, rowmask=None, drop_p=0.0,
         drop_offset=0, seed=0, seed_ptr=None, out_mode=0, split_k=1, gate=None, gate_scale=1.0, gate_mode=0, alpha=1.0,
         batch=1, inner=1, a_off=(0,) * 6, b_off=(0,) * 6, c_geom=None, rowmask_oo=0, C2=None, post_drop_p=0.0,
         post_drop_offset=0, c_split_stride=0, row_exp2_offset=None, m_limit=None, m_limit_base=0, k_limit=None,
         k_limit_base=0, mistake=None):
    """Expected contents of C (and C2) after rp_gemm: dict with, for "C" and "C2" (None without C2):
    out float64 [n] (from the tensor's first element to the end of its storage), written bool [n], atol float64 [n]."""
    assert mistake is None or mistake in MISTAKES, mistake
    acc, mag = contraction(A, B, M, N, K, a_mn=a_mn, b_mn=b_mn, batch=batch, inner=inner, a_off=a_off, b_off=b_off,
                           split_k=split_k, k_limit=k_limit, k_limit_base=k_limit_base, mistake=mistake)
    geom = _geom(C, c_geom)
    idx = _index(M, N, batch, inner, geom)
    # rows that are computed: 128-row tiles below the dynamic limit
    m = torch.arange(M)
    live = torch.ones(M, dtype=torch.bool)
    if m_limit is not None:
        live = (m // TILE_M * TILE_M + m_limit_base) < _limit(m_limit)
    live = live[None, :, None].expand(batch, M, N)

    seed_eff = seed + (0 if seed_ptr is None else int(torch.as_tensor(seed_ptr).reshape(-1)[0]))
    ks = 1.0 / (1.0 - float(np.float32(drop_p))) if drop_p > 0 else 1.0
    ks2 = 1.0 / (1.0 - float(np.float32(post_drop_p))) if post_drop_p > 0 else 1.0
    b = torch.zeros(N, dtype=torch.float64) if bias is None else bias.double()
    off = None if row_exp2_offset is None else row_exp2_offset.double()[:M][None, :, None]
    keep1 = _keep(seed_eff, drop_offset, drop_p, batch, M, N, mistake).double() * ks if drop_p > 0 else None
    keep2 = _keep(seed_eff, post_drop_offset, post_drop_p, batch, M, N, mistake).double() * ks2 if post_drop_p > 0 else None
    res = None if residual is None else _at(residual, idx)
    g = None if gate is None else _at(gate, idx)
    rm = None
    if rowmask is not None:
        sel = torch.arange(batch) % inner if mistake == "rowmask_by_inner" else torch.arange(batch) // inner
        rm = (rowmask[(sel * rowmask_oo)[:, None] + m[None, :]] != 0).double()[..., None]
    gate_f = None
    if g is not None:
        if gate_mode == 0:
            gate_f = (g != 0).double() * gate_scale
        else:
            gate_f = (gelu_tanh_grad(g) if mistake == "gelu_tanh_grad" else gelu_erf_grad(g)) * gate_scale

    def activation(x):
        if act == 1:
            return torch.relu(x)
        if act == 2:
            return gelu_tanh(x) if mistake == "gelu_tanh" else gelu_erf(x)
        if act == 3:
            return torch.exp2(x * LOG2E + off)
        if act == 4:
            return torch.sigmoid(x) * torch.exp2(off)
        return x

    order = _order(mistake)
    bias_times = split_k if mistake == "bias_per_split" else 1

    def epilogue(x):
        """Stages after alpha on x = alpha * acc: (value, C2 value, product of the factors applied after the act,
        magnitude of the residual add carried to the output)."""
        y, c2, gain, term = x, None, torch.ones_like(x), torch.zeros_like(x)
        gate_in, after_gate = torch.zeros_like(x), torch.ones_like(x)
        for st in order:
            if st == "bias":
                y = y + b * bias_times
            elif st == "c2":
                c2 = y
            elif st == "act":
                y, gain = activation(y), torch.ones_like(y)
            elif st == "residual":
                if res is not None:
                    y, term = y + res, y.abs() + res.abs()
            else:
                f = {"drop": keep1, "gate": gate_f, "post_drop": keep2, "rowmask": rm}[st]
                if f is not None:
                    # after_gate: the factors applied after the gate (which carry the error of the gate factor itself)
                    gate_in, after_gate = (y.abs(), torch.ones_like(y)) if st == "gate" else (gate_in, after_gate * f)
                    y, gain, term = y * f, gain * f, term * f
        return y, c2, gain, term, gate_in, after_gate

    total = acc.sum(0)
    parts, mags = (acc, mag) if out_mode == 3 else (total[None], mag.sum(0)[None])
    vals, atols = [], []
    for s in range(parts.shape[0]):
        x = parts[s] * alpha
        delta = ACC_SLACK * abs(alpha) * mags[s] + EPI_REL * b.abs()
        y0, c2, gain, term, gate_in, after_gate = epilogue(x)
        prop = torch.maximum((epilogue(x + delta)[0] - y0).abs(), (epilogue(x - delta)[0] - y0).abs())
        pre = x + b
        y_act = activation(pre).abs()
        act_err = torch.zeros_like(pre)
        if act in (1, 2):
            act_err = EPI_REL * (pre.abs() + y_act)
        elif act in (3, 4):     # ex2.approx, and the rounding of its argument
            arg = pre.abs() * LOG2E + (off.abs() if act == 3 else 0.0)
            act_err = y_act * (EPI_REL + 2.0 ** -22 * torch.nan_to_num(arg, posinf=0.0))

        vals.append(y0)
        atol = prop + gain.abs() * act_err + EPI_REL * (term + y0.abs())
        if gate_f is not None and gate_mode == 1:   # gelu'(gate) in fp32 with a fast exp: an absolute error of the factor
            atol = atol + EPI_REL * (1.0 + g.abs()) * abs(gate_scale) * gate_in * after_gate.abs()
        atols.append(atol)
        if s == 0:
            c2v, c2a = c2, delta.expand_as(c2)
    prev = flat_from(C).double()
    out, written, atol = prev.clone(), torch.zeros(prev.shape, dtype=torch.bool), torch.zeros_like(prev)
    for s, (y, a) in enumerate(zip(vals, atols)):
        sel = (idx + (s * c_split_stride if out_mode == 3 else 0))[live]
        out[sel] = y[live]
        atol[sel] = a[live]
        if out_mode in (1, 4):   # fp32 adds onto the previous contents (one per K split for the atomics)
            out[sel] += prev[sel]
            atol[sel] += EPI_REL * split_k * (prev[sel].abs() + abs(alpha) * mag.sum(0)[live])
        written[sel] = True
    result = {"C": dict(out=out, written=written, atol=atol), "C2": None}
    if C2 is not None:
        prev2 = flat_from(C2).double()
        out2, w2, a2 = prev2.clone(), torch.zeros(prev2.shape, dtype=torch.bool), torch.zeros_like(prev2)
        sel = idx[live]
        out2[sel], w2[sel], a2[sel] = c2v[live], True, c2a[live]
        result["C2"] = dict(out=out2, written=w2, atol=a2)
    return result


def reduce_splits(src, n_splits, stride, n, dst, accumulate):
    """rp_reduce_splits: dst[i] (+)= sum_s src[s * stride + i], i < n; returns (out, written, atol) over dst's flat storage."""
    s = flat_from(src).double()
    prev = flat_from(dst).double()
    parts = torch.stack([s[k * stride:k * stride + n] for k in range(n_splits)])
    out, written, atol = prev.clone(), torch.zeros(prev.shape, dtype=torch.bool), torch.zeros_like(prev)
    base = prev[:n] if accumulate else torch.zeros(n, dtype=torch.float64)
    out[:n] = base + parts.sum(0)
    written[:n] = True
    atol[:n] = 2.0 ** -23 * (n_splits + 1) * (base.abs() + parts.abs().sum(0))
    return dict(out=out, written=written, atol=atol)


def _errors(got, exp, bf16):
    w = exp["written"]
    ref = exp["out"][w]
    g = got.double()[w.to(got.device)].cpu()
    r = ref.abs()
    if bf16:
        rnd = torch.exp2(torch.floor(torch.log2(r.clamp_min(1e-300))) - 7)     # one bf16 ulp of the reference
    else:
        rnd = torch.exp2(torch.floor(torch.log2(r.clamp_min(1e-300))) - 22)    # two fp32 ulps of the reference
    return (g - ref).abs() / (exp["atol"][w] + rnd), w


def worst(got, exp, bf16):
    """Flat index of the written element with the largest error."""
    e, w = _errors(got, exp, bf16)
    return torch.nonzero(w)[int(e.argmax())][0]


def err(got, exp, bf16):
    """Largest |got - out| over the written elements in units of (atol + one rounding of the output type): a correct
    kernel stays below 1.  ``got`` is the flat storage (flat_from) of the kernel's buffer."""
    e, _ = _errors(got, exp, bf16)
    return float(e.max()) if e.numel() else 0.0


def untouched(got, exp):
    """Number of elements the kernel must leave alone whose bits changed."""
    keep = ~exp["written"]
    prev = exp["out"][keep]
    g = got[keep.to(got.device)].cpu().double()
    return int((g != prev).sum())
