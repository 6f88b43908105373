"""SASRec with the DiffTransformer encoder on the H100 engine (replay/nn/sequential/sasrec/diff_transformer.py,
replay/nn/attention.py:67-157, replay/nn/ffn.py:60-99; arXiv 2410.05258).  Per block, post-norm:

    QKV = x [W_q; W_k; W_v]^T                      one GEMM (the three weights are adjacent in the flat buffer)
    O   = per-head RMSNorm(A . V) * rms_scale * (1 - lambda_init),  A = softmax(Q1 K1^T s) - lambda softmax(Q2 K2^T s)
    y   = RMSNorm_attn(O W_o^T + x)
    x'  = RMSNorm_ff(W2 (silu(WG y + bg) * (W1 y + b1)) + b2 + y)

The embedding and the loss heads are SASRec's; the output normalization is LayerNorm or RMSNorm.  The attention backward
runs through the saved exponentials: dA = dO . V^T, the row-wise softmax backward, then batched GEMMs for dQ, dK and dV."""
from __future__ import annotations

import ctypes
import math
from dataclasses import dataclass

import torch

from ._lib import DiffAttnDesc, DiffLambda, check
from .engine import BaseConfig, SasRecEngine, _ru
from .engine_swiglu import RMS_EPS, SwiGLUOps

_QK_SLOT = 64   # each of q1 / q2 / k1 / k2 occupies a 64-wide slot per head
_DIFF_BLOCK = ("wq", "wk", "wv", "wo", "lambda_q1", "lambda_k1", "lambda_q2", "lambda_k2", "rms_scale", "attn_norm",
               "ff_norm", "ff_wg", "ff_w1", "ff_bg", "ff_b1", "ff_w2", "ff_b2")


def lambda_init(block: int) -> float:
    """replay/nn/sequential/sasrec/diff_transformer.py: 0.8 - 0.6 exp(-0.3 block_index)"""
    return 0.8 - 0.6 * math.exp(-0.3 * block)


@dataclass
class DiffConfig(BaseConfig):
    out_norm: str = "layernorm"    # the body's output_normalization: "layernorm" or "rmsnorm"
    lnf_eps: float | None = None
    variant: str = "diff"

    def __post_init__(self):
        if self.d % self.n_heads:
            raise ValueError("embedding_dim must be divisible by num_heads")
        if self.d // self.n_heads > 64:
            raise ValueError(f"DiffTransformer supports head width <= 64 (embedding_dim / num_heads = {self.d // self.n_heads})")
        super().__post_init__()
        if self.dp > 256:
            raise ValueError(f"DiffTransformer supports at most 256 padded model columns ({self.n_heads} heads x 64 = {self.dp})")
        if self.max_len > 256:
            raise ValueError(f"DiffTransformer supports max_sequence_length <= 256, got {self.max_len}")
        if self.out_norm not in ("layernorm", "rmsnorm"):
            raise ValueError(f"output normalization must be LayerNorm or RMSNorm, got {self.out_norm!r}")
        if self.lnf_eps is None:
            self.lnf_eps = 1e-5 if self.out_norm == "layernorm" else RMS_EPS

    @property
    def pad_id(self) -> int:
        return self.n_items

    @property
    def v_slot(self) -> int:
        """columns of one head's value / attention output (true width 2 * head_dim)"""
        return 64 if self.head_dim <= 32 else 128

    @property
    def ffn_p(self) -> int:
        """SwiGLU hidden width (2d) as the kernels see it"""
        return _ru(2 * self.d, 128)

    @property
    def n_qkv(self) -> int:
        return self.n_heads * (4 * _QK_SLOT + self.v_slot)

    def axis_sizes(self) -> dict:
        """pad kinds of BaseConfig plus 'q' = the query / key rows (per head [q1 | q2], each in a 64-wide slot), 'v' = the
        value rows (per head 2 * head_dim in a v_slot-wide slot), 'r' = rms_scale, 'i' = the SwiGLU hidden axis (true
        entries first)"""
        return {**super().axis_sizes(), "q": 2 * self.d, "v": 2 * self.d, "r": 2 * self.head_dim, "i": 2 * self.d}

    def param_layout(self) -> list:
        d, H, hd, F = self.dp, self.n_heads, self.head_dim, self.ffn_p
        qk, v, vec = H * 2 * _QK_SLOT, H * self.v_slot, ("f", None)
        out = [("item_emb", (self.n_items + 1, d), (None, "f")), ("pos_emb", (self.max_len, d), (None, "f"))]
        for i in range(self.n_blocks):
            shapes = ((qk, d), (qk, d), (v, d), (d, v), (H, hd), (H, hd), (H, hd), (H, hd), (self.v_slot,), (d,), (d,),
                      (F, d), (F, d), (F,), (F,), (d, F), (d,))
            kinds = (("q", "f"), ("q", "f"), ("v", "f"), ("f", "v"), (None, None), (None, None), (None, None), (None, None),
                     ("r", None), vec, vec, ("i", "f"), ("i", "f"), ("i", None), ("i", None), ("f", "i"), vec)
            out += [(f"b{i}.{k}", s, pk) for k, s, pk in zip(_DIFF_BLOCK, shapes, kinds)]
        out.append(("lnf_w", (d,), vec))
        if self.out_norm == "layernorm":
            out.append(("lnf_b", (d,), vec))
        return out


class DiffEngine(SwiGLUOps, SasRecEngine):
    def _check_geometry(self, seq_len: int):
        if seq_len > self.cfg.max_len:
            raise ValueError(f"sequence length {seq_len} exceeds max_len {self.cfg.max_len}")

    # ------------------------------------------------------------------------------------------------ parameters
    def _axis_index(self, kind):
        cfg = self.cfg
        hd = cfg.head_dim
        k = torch.arange(2 * cfg.d, device=self.dev)
        if kind == "q":
            return (k // (2 * hd)) * 2 * _QK_SLOT + ((k % (2 * hd)) // hd) * _QK_SLOT + k % hd
        if kind == "v":
            return (k // (2 * hd)) * cfg.v_slot + k % (2 * hd)
        return super()._axis_index(kind)

    def init_parameters(self, seed: int = 0):
        """DiffTransformerLayer.reset_parameters: xavier_normal_ on every >= 2-D parameter (lambda_* included), RMSNorm
        weights and rms_scale at one, the SwiGLU biases at torch.nn.Linear's U(+-1/sqrt(fan_in)); the pad row of the item
        table zero, the output LayerNorm at (1, 0)."""
        g = torch.Generator(device="cpu").manual_seed(seed)
        with torch.no_grad():
            for name in self.layout:
                shp = self.true_shape(name)
                leaf = name.partition(".")[2] or name
                if len(shp) == 2:
                    v = torch.randn(shp, generator=g) * math.sqrt(2.0 / (shp[0] + shp[1]))
                    if name == "item_emb":
                        v[self.cfg.pad_id].zero_()
                elif leaf in ("rms_scale", "attn_norm", "ff_norm", "lnf_w"):
                    v = torch.ones(shp)
                elif leaf in ("ff_bg", "ff_b1", "ff_b2"):
                    fan_in = self.true_shape(name[:-2] + "w2")[1] if leaf == "ff_b2" else self.cfg.d
                    v = (torch.rand(shp, generator=g) * 2 - 1) / math.sqrt(fan_in)
                else:
                    v = torch.zeros(shp)
                self.import_named(name, v)
        self.refresh_shadow()

    # ------------------------------------------------------------------------------------------------ workspace
    def _alloc_body(self):
        cfg, T, d, dev = self.cfg, self.T, self.cfg.dp, self.dev
        H, vs, F, Lp = cfg.n_heads, cfg.v_slot, cfg.ffn_p, self.Lp
        BH = self.B * H
        bf = dict(device=dev, dtype=torch.bfloat16)
        f32 = dict(device=dev, dtype=torch.float32)
        for a in self.act:
            a.clear()
            a.update(QKV=torch.zeros(T, cfg.n_qkv, **bf), On=torch.zeros(T, H * vs, **bf), h=torch.zeros(T, d, **bf),
                     y=torch.zeros(T, d, **bf), GL=torch.zeros(T, 2 * F, **bf), U=torch.zeros(T, F, **bf),
                     z=torch.zeros(T, d, **bf))
            if self.with_grad:
                a.update(Opre=torch.zeros(T, H * vs, **bf), O32=torch.zeros(T, H * vs, **f32), O2=torch.zeros(T, H * vs, **f32), e1=torch.zeros(BH, Lp, Lp, **bf), e2=torch.zeros(BH, Lp, Lp, **bf),
                         inv1=torch.zeros(BH, Lp, **f32), inv2=torch.zeros(BH, Lp, **f32))
        self.meanf = torch.zeros(T, **f32)
        self.rstdf = torch.zeros(T, **f32)
        if self.with_grad:
            for k in ("d_o", "dpd"):
                self.s.pop(k, None)
            self.s.update(dz=torch.zeros(T, d, **bf), dU=torch.zeros(T, F, **bf), dGL=torch.zeros(T, 2 * F, **bf),
                          dy=torch.zeros(T, d, **bf), dh=torch.zeros(T, d, **bf), dOn=torch.zeros(T, H * vs, **bf),
                          dOpre=torch.zeros(T, H * vs, **bf), dQKV=torch.zeros(T, cfg.n_qkv, **bf),
                          dA=torch.zeros(BH, Lp, Lp, **bf), dS1=torch.zeros(BH, Lp, Lp, **bf), dS2=torch.zeros(BH, Lp, Lp, **bf),
                          dlam=torch.zeros(BH, Lp, **f32))
            need = max(self.lib.rp_rmsnorm_bwd_workspace(g) for g in {d, vs})
            self.rms_ws = torch.zeros(need, device=dev, dtype=torch.uint8)

    # ------------------------------------------------------------------------------------------------ kernel helpers
    def _lambda(self, i: int) -> DiffLambda:
        prm = self.params
        lam = DiffLambda()
        lam.q1, lam.k1, lam.q2, lam.k2 = (prm[f"b{i}.lambda_{k}"].data_ptr() for k in ("q1", "k1", "q2", "k2"))
        lam.head_dim, lam.lambda_init = self.cfg.head_dim, lambda_init(i)
        return lam

    def _final_norm_fwd(self, x, out, n_rows, gather=None, n_rows_dev=None):
        cfg = self.cfg
        if cfg.out_norm == "layernorm":
            return super()._final_norm_fwd(x, out, n_rows, gather, n_rows_dev)
        self._rms_fwd(x, self.params["lnf_w"], cfg.lnf_eps, out, n_rows, cfg.dp, cfg.d, gather=gather, n_rows_dev=n_rows_dev)

    def _final_norm_bwd(self, dy, x, dx, n_rows, gather=None, n_rows_dev=None):
        cfg = self.cfg
        if cfg.out_norm == "layernorm":
            return super()._final_norm_bwd(dy, x, dx, n_rows, gather, n_rows_dev)
        self._rms_bwd(dy, x, self.params["lnf_w"], cfg.lnf_eps, dx, self.grads["lnf_w"], n_rows, cfg.dp, cfg.d, gather=gather,
                      n_rows_dev=n_rows_dev)

    # ------------------------------------------------------------------------------------------------ forward
    def _attention_forward(self, i: int, save: bool):
        cfg, a = self.cfg, self.act[i]
        H = cfg.n_heads
        ad = DiffAttnDesc()
        ad.qk, ad.ld_qk, ad.q_c0, ad.k_c0 = a["QKV"].data_ptr(), cfg.n_qkv, 0, H * 2 * _QK_SLOT
        ad.v, ad.ldv, ad.v_c0 = a["QKV"].data_ptr(), cfg.n_qkv, H * 4 * _QK_SLOT
        ad.pad_mask = self.in_pad.data_ptr()
        ad.B, ad.H, ad.L, ad.head_dim, ad.v_slot = self.B, H, self.L, cfg.head_dim, cfg.v_slot
        ad.scale, ad.eps = 1.0 / math.sqrt(cfg.head_dim), 1e-5
        ad.lam = self._lambda(i)
        ad.rms_scale = self.params[f"b{i}.rms_scale"].data_ptr()
        ad.out, ad.ldo = a["On"].data_ptr(), H * cfg.v_slot
        if save:
            ad.o_pre, ad.e1_save, ad.e2_save = a["Opre"].data_ptr(), a["e1"].data_ptr(), a["e2"].data_ptr()
            ad.inv1, ad.inv2 = a["inv1"].data_ptr(), a["inv2"].data_ptr()
            ad.o32_save, ad.o2_save = a["O32"].data_ptr(), a["O2"].data_ptr()
        check(self.lib.rp_diff_attn_fwd(ctypes.byref(ad), self._stream()), "rp_diff_attn_fwd")

    def _body_forward(self, training: bool, last_only: bool = False):
        cfg, T, d, L = self.cfg, self.T, self.cfg.dp, self.L
        p16, prm = self.params16, self.params
        F = cfg.ffn_p
        drop = cfg.dropout if training else 0.0
        check(self.lib.rp_embed_fwd(p16["item_emb"].data_ptr(), prm["pos_emb"].data_ptr(), self.ids32.data_ptr(),
                                    self.in_pad.data_ptr(), T, L, d, cfg.max_len - L, math.sqrt(cfg.d), 0, drop, self.seed, 0,
                                    self.rng_counter.data_ptr(), self.x[0].data_ptr(), self._stream()), "rp_embed_fwd")
        for i in range(cfg.n_blocks):
            a, x = self.act[i], self.x[i]
            w = lambda k: p16[f"b{i}.{k}"]  # noqa: E731
            f = lambda k: prm[f"b{i}.{k}"]  # noqa: E731
            self._gemm(x, self._span(p16, f"b{i}.wq", f"b{i}.wv", cfg.n_qkv), a["QKV"], T, cfg.n_qkv, d)
            self._attention_forward(i, training and self.with_grad)
            self._gemm(a["On"], w("wo"), a["h"], T, d, cfg.n_heads * cfg.v_slot, residual=x)
            self._rms_fwd(a["h"], f("attn_norm"), RMS_EPS, a["y"], T, d, cfg.d)
            self._swiglu_block_fwd(f"b{i}.ff_", a["y"], a["GL"], a["U"], a["z"], self.x[i + 1], T, F)

    # ------------------------------------------------------------------------------------------------ backward
    def _attention_backward(self, i: int):
        """dQ1, dQ2, dK1, dK2, dV of block ``i`` into s["dQKV"] from s["dOpre"] and the forward's saves; the lambda chain
        into the lambda_* gradients."""
        cfg, L, Lp, a, s = self.cfg, self.L, self.Lp, self.act[i], self.s
        H, vs, n = cfg.n_heads, cfg.v_slot, cfg.n_qkv
        BH = self.B * H
        QKV, dQKV = a["QKV"], s["dQKV"]
        kc, vc = H * 2 * _QK_SLOT, H * 4 * _QK_SLOT
        heads = dict(batch=BH, inner=H, a_off=(0, H * Lp, Lp, 0, 0, 0))
        out = lambda c0, width: (n, c0, L * n, width)  # noqa: E731  per-head [L, width] blocks of dQKV
        # dA = dO_pre . V^T
        self._gemm(s["dOpre"], QKV, s["dA"], L, L, vs, batch=BH, inner=H, a_off=(0, L, 0, 0, 0, vs), b_off=(0, L, 0, vc, 0, vs),
                   c_geom=(Lp, 0, H * Lp * Lp, Lp * Lp))
        lam = self._lambda(i)
        check(self.lib.rp_diff_attn_softmax_bwd(a["e1"].data_ptr(), a["e2"].data_ptr(), a["inv1"].data_ptr(), a["inv2"].data_ptr(),
                                                s["dA"].data_ptr(), s["dS1"].data_ptr(), s["dS2"].data_ptr(), s["dA"].data_ptr(),
                                                s["dlam"].data_ptr(), BH, H, L, 1.0 / math.sqrt(cfg.head_dim),
                                                ctypes.byref(lam), s["dOn"].data_ptr(), a["O32"].data_ptr(), a["O2"].data_ptr(),
                                                self.params[f"b{i}.rms_scale"].data_ptr(), 1e-5, H * vs, vs, self._stream()),
              "rp_diff_attn_softmax_bwd")
        G = self.grads
        check(self.lib.rp_diff_lambda_bwd(s["dlam"].data_ptr(), self.B, H, L, ctypes.byref(lam),
                                          *(G[f"b{i}.lambda_{k}"].data_ptr() for k in ("q1", "k1", "q2", "k2")), self._stream()),
              "rp_diff_lambda_bwd")
        for half, dS in ((0, s["dS1"]), (_QK_SLOT, s["dS2"])):
            dSv = dS.view(BH * Lp, Lp)
            # dQ = dS . K   ;   dK = dS^T . Q
            self._gemm(dSv, QKV, dQKV, L, _QK_SLOT, L, b_mn=True, b_off=(0, L, 0, kc + half, 0, 2 * _QK_SLOT),
                       c_geom=out(half, 2 * _QK_SLOT), **heads)
            self._gemm(dSv, QKV, dQKV, L, _QK_SLOT, L, a_mn=True, b_mn=True, b_off=(0, L, 0, half, 0, 2 * _QK_SLOT),
                       c_geom=out(kc + half, 2 * _QK_SLOT), **heads)
        # dV = A^T . dO_pre   (A was written over dA)
        self._gemm(s["dA"].view(BH * Lp, Lp), s["dOpre"], dQKV, L, vs, L, a_mn=True, b_mn=True, b_off=(0, L, 0, 0, 0, vs),
                   c_geom=out(vc, vs), **heads)

    def backward(self):
        cfg, T, d, L = self.cfg, self.T, self.cfg.dp, self.L
        p16, prm, G, s = self.params16, self.params, self.grads, self.s
        H, vs, F = cfg.n_heads, cfg.v_slot, cfg.ffn_p
        dx = self._head_backward()
        other = s["dxb"]
        for i in reversed(range(cfg.n_blocks)):
            a, x = self.act[i], self.x[i]
            w = lambda k: p16[f"b{i}.{k}"]  # noqa: E731
            f = lambda k: prm[f"b{i}.{k}"]  # noqa: E731
            g = lambda k: G[f"b{i}.{k}"]  # noqa: E731
            self._swiglu_block_bwd(f"b{i}.ff_", dx, a["y"], a["GL"], a["U"], a["z"], s["dz"], s["dU"], s["dGL"], s["dy"], T, F)
            self._rms_bwd(s["dy"], a["h"], f("attn_norm"), RMS_EPS, s["dh"], g("attn_norm"), T, d, cfg.d)
            self._gemm(s["dh"], w("wo"), s["dOn"], T, H * vs, d, b_mn=True)
            self._rms_bwd(s["dOn"], a["Opre"], f("rms_scale"), 1e-5, s["dOpre"], g("rms_scale"), T, vs, 2 * cfg.head_dim,
                          alpha=1.0 - lambda_init(i))
            self._attention_backward(i)
            self._gemm(s["dQKV"], self._span(p16, f"b{i}.wq", f"b{i}.wv", cfg.n_qkv), other, T, d, cfg.n_qkv, b_mn=True,
                       residual=s["dh"])
            self._wgrad(s["dh"], a["On"], g("wo"), d, H * vs)
            self._wgrad(s["dQKV"], x, self._span(G, f"b{i}.wq", f"b{i}.wv", cfg.n_qkv), cfg.n_qkv, d)
            dx, other = other, dx
        check(self.lib.rp_embed_bwd(dx.data_ptr(), self.ids32.data_ptr(), self.in_pad.data_ptr(), self.B, L, d, cfg.pad_id,
                                    cfg.max_len - L, math.sqrt(cfg.d), 0, cfg.dropout, self.seed, 0, self.rng_counter.data_ptr(),
                                    G["item_emb"].data_ptr(), G["pos_emb"].data_ptr(), self._stream()), "rp_embed_bwd")

    # ------------------------------------------------------------------------------------------------ inference
    def forward_last_hidden(self):
        """Eval body over the whole window -> output normalization of the LAST row of every sequence -> self.hq bf16 [B, dp]."""
        self._prepare(False)
        self._body_forward(False)
        self._final_norm_fwd(self.x[-1], self.hq, self.B, gather=self.last_idx)
        return self.hq

    def forward_hidden_all(self):
        self._prepare(False)
        self._body_forward(False)
        out = torch.empty(self.T, self.cfg.dp, device=self.dev, dtype=torch.bfloat16)
        self._final_norm_fwd(self.x[-1], out, self.T)
        return out
