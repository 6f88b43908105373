"""TiSASRec (the legacy ``SasRecModel(ti_modification=True)``, replay/models/nn/sequential/sasrec/model.py:532-800) on the
H100 engine.  Per block, with the embedder's dropped positional and time terms shared by every block:

    q_in = LN1(x),  Q = q_in Wq^T + bq,  [K | V] = x [Wk; Wv]^T + [bk; bv]     rp_ln_qkv_fused (the three weights are adjacent)
    K' = K + dropout(pos_k),  V' = V + dropout(pos_v)                            rp_ti_pos_add
    S = Q K'^T                                                                   rp_gemm, per (sequence, head)
    A, Ad, hpre = q_in + Ad . TVm                                                rp_ti_attn_fwd (time terms from the timestamps)
    h = Ad V' + hpre                                                             rp_gemm (no output projection)
    x' = (LN2(h) + dropout(W2 dropout(relu(W1 LN2(h) + b1)) + b2)) * pad        rp_layernorm_fwd + two rp_gemm

The input is dropout(E[ids] sqrt(d)) * pad without a positional add (rp_embed_fwd without positions).  The legacy padded
layout is kept: pad keys are live, so there is no packed body."""
from __future__ import annotations

import ctypes
import math
from dataclasses import dataclass

import torch

from ._lib import TI_MAX_COLS, TI_MAX_SPAN, TiAttnDesc, check
from .core import SasRecCore
from .engine import BaseConfig, SasRecEngine
from .engine_swiglu import SwiGLUOps

_TI_BLOCK = ("ln1_w", "ln1_b", "qw", "kw", "vw", "qb", "kb", "vb", "ln2_w", "ln2_b", "w1", "b1", "w2", "b2")
# dropout sites of the embedder's terms, shared by every block of a step (block sites are 1 + 8 * block + k)
_SITE_POS_K, _SITE_POS_V, _SITE_TIME_K, _SITE_TIME_V = 4000, 4001, 4002, 4003
# timestamp dtypes the kernels compute intervals in (rp_ti_attn_desc.times_dtype)
_TIMES_DTYPE = {torch.int64: 0, torch.float32: 1, torch.float64: 2}


@dataclass
class TiConfig(BaseConfig):
    time_span: int = 256
    variant: str = "legacy"
    lnf_eps: float = 1e-8   # SasRecNormalizer

    def __post_init__(self):
        if self.d % self.n_heads:
            raise ValueError("hidden_size must be divisible by num_heads")
        if self.d // self.n_heads > 64:
            raise ValueError(f"TiSASRec supports head width <= 64 (hidden_size / num_heads = {self.d // self.n_heads})")
        super().__post_init__()
        if self.dp > TI_MAX_COLS:
            raise ValueError(f"TiSASRec supports at most {TI_MAX_COLS} padded columns ({self.n_heads} heads x 64 = {self.dp})")
        if self.max_len > 256:
            raise ValueError(f"TiSASRec supports max_seq_len <= 256, got {self.max_len}")
        if not 1 <= self.time_span <= TI_MAX_SPAN:
            raise ValueError(f"TiSASRec supports 1 <= time_span <= {TI_MAX_SPAN}, got {self.time_span}")

    @property
    def pad_id(self) -> int:
        return self.n_items

    def param_layout(self) -> list:
        d, emb, vec, mat = self.dp, (None, "f"), ("f", None), ("f", "f")
        out = [("item_emb", (self.n_items + 1, d), emb), ("pos_k", (self.max_len, d), emb), ("pos_v", (self.max_len, d), emb),
               ("time_k", (self.time_span + 1, d), emb), ("time_v", (self.time_span + 1, d), emb)]
        shapes = ((d,), (d,), (d, d), (d, d), (d, d), (d,), (d,), (d,), (d,), (d,), (d, d), (d,), (d, d), (d,))
        kinds = (vec, vec, mat, mat, mat, vec, vec, vec, vec, vec, mat, vec, mat, vec)
        for i in range(self.n_blocks):
            out += [(f"b{i}.{k}", s, pk) for k, s, pk in zip(_TI_BLOCK, shapes, kinds)]
        out += [("lnf_w", (d,), vec), ("lnf_b", (d,), vec)]
        return out


class TiSasRecEngine(SwiGLUOps, SasRecEngine):
    # ------------------------------------------------------------------------------------------------ parameters
    def init_parameters(self, seed: int = 0):
        """SasRecModel._init: xavier_normal_ on every >= 2-D parameter (the item table's padding row included); LayerNorms at
        (1, 0); the Linear / Conv1d biases at torch's U(+-1/sqrt(fan_in))."""
        g = torch.Generator(device="cpu").manual_seed(seed)
        with torch.no_grad():
            for name in self.layout:
                shp = self.true_shape(name)
                leaf = name.partition(".")[2] or name
                if len(shp) == 2:
                    v = torch.randn(shp, generator=g) * math.sqrt(2.0 / (shp[0] + shp[1]))
                elif leaf in ("qb", "kb", "vb", "b1", "b2"):
                    v = (torch.rand(shp, generator=g) * 2 - 1) / math.sqrt(self.cfg.d)
                elif leaf.endswith("_w"):
                    v = torch.ones(shp)
                else:
                    v = torch.zeros(shp)
                self.import_named(name, v)
        self.refresh_shadow()

    # ------------------------------------------------------------------------------------------------ workspace
    def _alloc_body(self):
        cfg, T, d, dev, Lp = self.cfg, self.T, self.cfg.dp, self.dev, self.Lp
        BH = self.B * cfg.n_heads
        bf = dict(device=dev, dtype=torch.bfloat16)
        for a in self.act:
            a.update({k: torch.zeros(T, d, **bf) for k in ("q_in", "Q", "h", "y", "u")})
            a["KV"] = torch.zeros(T, 2 * d, **bf)
            if self.with_grad:
                a["A"] = torch.zeros(BH, Lp, Lp, **bf)   # softmax probabilities, saved for the backward
        self.S = torch.zeros(BH, Lp, Lp, device=dev, dtype=torch.float32)
        self.Ad = torch.zeros(BH, Lp, Lp, **bf)          # dropped probabilities (eval: the probabilities themselves)
        self.hpre = torch.zeros(T, d, **bf)
        self.meanf = torch.zeros(T, device=dev, dtype=torch.float32)
        self.rstdf = torch.zeros(T, device=dev, dtype=torch.float32)
        # timestamps of the staged batch, 8 bytes per token: int64, or float32 / float64 in the same storage
        self.times = torch.zeros(T, device=dev, dtype=torch.int64)
        self.times_dtype = getattr(self, "times_dtype", 0)
        if self.with_grad:
            for k in ("d_o", "dpd"):
                self.s.pop(k, None)
            self.s.update({k: torch.zeros(T, d, **bf) for k in ("d_t", "du", "dy", "dh", "dQ", "dq_in", "tmp", "dqt")})
            self.s["dKV"] = torch.zeros(T, 2 * d, **bf)
            self.dS = torch.zeros(BH, Lp, Lp, **bf)
            n = self.lib.rp_ti_attn_bwd_workspace(self.B, cfg.n_heads, cfg.time_span)
            self.ti_ws = torch.zeros(n, device=dev, dtype=torch.uint8)
            self._wgrad_ws = None

    def set_times(self, times: torch.Tensor) -> bool:
        """Stage the [B, L] timestamps of the current batch (after set_batch's geometry checks).  int64 and the other integer
        dtypes give exact intervals; float32 / float64 intervals are computed (and floored) in that dtype, as the reference
        does.  Returns True when the dtype differs from the last batch's: a captured graph holds the old one."""
        if times.dim() != 2 or times.shape[1] != self.L or times.shape[0] > self.B:
            raise ValueError(f"timestamps {tuple(times.shape)} do not fit the engine ({self.B}, {self.L})")
        if not times.dtype.is_floating_point and times.dtype is not torch.bool:
            times = times.to(torch.int64)
        code = _TIMES_DTYPE.get(times.dtype)
        if code is None:
            raise ValueError(f"timestamps of dtype {times.dtype} are not supported (int64, float32 or float64)")
        n = times.numel()
        buf = {0: self.times, 1: self.times.view(torch.float32), 2: self.times.view(torch.float64)}[code]
        buf[:n].copy_(times.reshape(-1), non_blocking=True)
        moved = code != self.times_dtype
        self.times_dtype = code
        return moved

    # ------------------------------------------------------------------------------------------------ kernel helpers
    def _ti_desc(self, i: int, drop: float) -> TiAttnDesc:
        cfg, d = self.cfg, self.cfg.dp
        p = TiAttnDesc()
        p.q, p.ldq, p.pad_mask = self.act[i]["Q"].data_ptr(), d, self.in_pad.data_ptr()
        p.times, p.times_dtype = self.times.data_ptr(), self.times_dtype
        p.time_k, p.time_v, p.ld_t = self.params16["time_k"].data_ptr(), self.params16["time_v"].data_ptr(), d
        p.B, p.H, p.L, p.head_dim, p.time_span = self.B, cfg.n_heads, self.L, cfg.head_dim, cfg.time_span
        p.scale = 1.0 / math.sqrt(cfg.head_dim)
        p.drop_p, p.seed, p.seed_ptr = drop, self.seed, self.rng_counter.data_ptr()
        p.att_off, p.tk_off, p.tv_off = self._site(i, 0) << 40, _SITE_TIME_K << 40, _SITE_TIME_V << 40
        return p

    def _heads(self):
        """rp_gemm geometry of the per-(sequence, head) products over a [B*H*Lp, Lp] probability-shaped A operand"""
        H, Lp = self.cfg.n_heads, self.Lp
        return dict(batch=self.B * H, inner=H, a_off=(0, H * Lp, Lp, 0, 0, 0))

    def _scores_geom(self):
        """(a_off, c_geom) of a per-(sequence, head) [L, L] product of two [T, *] arrays into a [B*H, Lp, Lp] buffer"""
        H, Lp = self.cfg.n_heads, self.Lp
        return (0, self.L, 0, 0, 0, 64), (Lp, 0, H * Lp * Lp, Lp * Lp)

    # ------------------------------------------------------------------------------------------------ forward
    def _ti_attention_forward(self, i: int, save: bool, drop: float):
        """act[i]["h"] = Ad . V' + q_in + Ad . TVm: the block's attention and its residual."""
        cfg, L, d, a = self.cfg, self.L, self.cfg.dp, self.act[i]
        a_off, c_geom = self._scores_geom()
        BH, Lp = self.B * cfg.n_heads, self.Lp
        self._gemm(a["Q"], a["KV"], self.S, L, L, 64, batch=BH, inner=cfg.n_heads, a_off=a_off, b_off=a_off, c_geom=c_geom,
                   out_mode=2)
        a_save = a["A"] if save else self.Ad
        ad = self.Ad if drop > 0 else a_save
        check(self.lib.rp_ti_attn_fwd(ctypes.byref(self._ti_desc(i, drop)), self.S.data_ptr(), a["q_in"].data_ptr(),
                                      a_save.data_ptr(), ad.data_ptr(), self.hpre.data_ptr(), self._stream()), "rp_ti_attn_fwd")
        self._gemm(ad.view(BH * Lp, Lp), a["KV"], a["h"], L, 64, L, b_mn=True, b_off=(0, L, 0, d, 0, 64),
                   c_geom=(d, 0, L * d, 64), residual=self.hpre, **self._heads())

    def _body_forward(self, training: bool, last_only: bool = False):
        cfg, T, d, L = self.cfg, self.T, self.cfg.dp, self.L
        p16, prm, pad, hdv = self.params16, self.params, self.in_pad, cfg.hd_valid
        drop = cfg.dropout if training else 0.0
        check(self.lib.rp_embed_fwd(p16["item_emb"].data_ptr(), None, self.ids32.data_ptr(), pad.data_ptr(), T, L, d, 0,
                                    math.sqrt(cfg.d), 1, drop, self.seed, 0, self.rng_counter.data_ptr(), self.x[0].data_ptr(),
                                    self._stream()), "rp_embed_fwd")
        for i in range(cfg.n_blocks):
            a, x = self.act[i], self.x[i]
            w = lambda k: p16[f"b{i}.{k}"]  # noqa: E731
            f = lambda k: prm[f"b{i}.{k}"]  # noqa: E731
            in_w, in_b = self._span(p16, f"b{i}.qw", f"b{i}.vw", 3 * d), self._span(prm, f"b{i}.qb", f"b{i}.vb", 1).view(-1)
            if self.fused_pre_attn:
                check(self.lib.rp_ln_qkv_fused(x.data_ptr(), f("ln1_w").data_ptr(), f("ln1_b").data_ptr(), 1e-8,
                                               in_w.data_ptr(), in_b.data_ptr(), T, d, a["q_in"].data_ptr(), a["Q"].data_ptr(),
                                               a["KV"].data_ptr(), a["mean1"].data_ptr(), a["rstd1"].data_ptr(), hdv,
                                               self._stream()), "rp_ln_qkv_fused")
            else:
                self._ln_fwd(x, f("ln1_w"), f("ln1_b"), 1e-8, a["q_in"], a["mean1"], a["rstd1"], T)
                self._gemm(a["q_in"], in_w[:d], a["Q"], T, d, d, bias=in_b[:d])
                self._gemm(x, in_w[d:], a["KV"], T, 2 * d, d, bias=in_b[d:])
            check(self.lib.rp_ti_pos_add(a["KV"].data_ptr(), 2 * d, prm["pos_k"].data_ptr(), prm["pos_v"].data_ptr(), T, L, d,
                                         drop, self.seed, self.rng_counter.data_ptr(), _SITE_POS_K << 40, _SITE_POS_V << 40,
                                         self._stream()), "rp_ti_pos_add")
            self._ti_attention_forward(i, training and self.with_grad, drop)
            self._ln_fwd(a["h"], f("ln2_w"), f("ln2_b"), 1e-8, a["y"], a["mean2"], a["rstd2"], T)
            self._gemm(a["y"], w("w1"), a["u"], T, d, d, bias=f("b1"), act=1, drop_p=drop, drop_site=self._site(i, 1))
            self._gemm(a["u"], w("w2"), self.x[i + 1], T, d, d, bias=f("b2"), drop_p=drop, drop_site=self._site(i, 2),
                       residual=a["y"], rowmask=pad)

    # ------------------------------------------------------------------------------------------------ backward
    def _ti_attention_backward(self, i: int, drop: float):
        """dQ into s["dQ"], dK' | dV' into s["dKV"] and the time tables' gradients, from dO = s["dh"]."""
        cfg, L, d, a, s = self.cfg, self.L, self.cfg.dp, self.act[i], self.s
        BH, Lp, G = self.B * cfg.n_heads, self.Lp, self.grads
        a_off, c_geom = self._scores_geom()
        # dAd = dO . V'^T
        self._gemm(s["dh"], a["KV"], self.dS, L, L, 64, batch=BH, inner=cfg.n_heads, a_off=a_off, b_off=(0, L, 0, d, 0, 64),
                   c_geom=c_geom)
        ad = self.Ad if drop > 0 else a["A"]
        check(self.lib.rp_ti_attn_bwd(ctypes.byref(self._ti_desc(i, drop)), a["A"].data_ptr(), self.dS.data_ptr(),
                                      ad.data_ptr(), s["dh"].data_ptr(), s["dqt"].data_ptr(), self.ti_ws.data_ptr(),
                                      self.ti_ws.numel(), G["time_k"].data_ptr(), G["time_v"].data_ptr(), self._stream()),
              "rp_ti_attn_bwd")
        dS, heads = self.dS.view(BH * Lp, Lp), self._heads()
        out = lambda t, c0: (t.stride(0), c0, L * t.stride(0), 64)  # noqa: E731  per-head [L, 64] blocks of a [T, *] array
        # dQ = dS . K' + dS . TKm ;  dK' = dS^T . Q ;  dV' = Ad^T . dO
        self._gemm(dS, a["KV"], s["dQ"], L, 64, L, b_mn=True, b_off=(0, L, 0, 0, 0, 64), c_geom=out(s["dQ"], 0),
                   residual=s["dqt"], **heads)
        self._gemm(dS, a["Q"], s["dKV"], L, 64, L, a_mn=True, b_mn=True, b_off=(0, L, 0, 0, 0, 64), c_geom=out(s["dKV"], 0),
                   **heads)
        self._gemm(ad.view(BH * Lp, Lp), s["dh"], s["dKV"], L, 64, L, a_mn=True, b_mn=True, b_off=(0, L, 0, 0, 0, 64),
                   c_geom=out(s["dKV"], d), **heads)

    def backward(self):
        cfg, T, d, L = self.cfg, self.T, self.cfg.dp, self.L
        p16, prm, G, s, st = self.params16, self.params, self.grads, self.s, self._stream
        hdv, drop = cfg.hd_valid, cfg.dropout
        ks = 1.0 / (1.0 - drop) if drop > 0 else 1.0
        dx = self._head_backward()
        other = s["dxb"]
        for i in reversed(range(cfg.n_blocks)):
            a, x = self.act[i], self.x[i]
            w = lambda k: p16[f"b{i}.{k}"]  # noqa: E731
            f = lambda k: prm[f"b{i}.{k}"]  # noqa: E731
            g = lambda k: G[f"b{i}.{k}"]  # noqa: E731
            dz = dx
            check(self.lib.rp_dropout_bwd(dz.data_ptr(), dz.data_ptr(), T, d, self.in_pad.data_ptr(), 0.0, 0, 0, None, st()),
                  "rp_dropout_bwd")   # x' = (...) * pad
            d_t = dz
            if drop > 0:
                check(self.lib.rp_dropout_bwd(dz.data_ptr(), s["d_t"].data_ptr(), T, d, None, drop, self.seed,
                                              self._site(i, 2) << 40, self.rng_counter.data_ptr(), st()), "rp_dropout_bwd")
                d_t = s["d_t"]
            self._gemm(d_t, w("w2"), s["du"], T, d, d, b_mn=True, gate=a["u"], gate_scale=ks)
            self._gemm(s["du"], w("w1"), s["dy"], T, d, d, b_mn=True, residual=dz)
            self._ln_bwd(s["dy"], a["h"], f("ln2_w"), a["mean2"], a["rstd2"], s["dh"], g("ln2_w"), g("ln2_b"), T)
            self._ti_attention_backward(i, drop)
            in_w = self._span(p16, f"b{i}.qw", f"b{i}.vw", 3 * d)
            if self.fused_pre_attn:
                check(self.lib.rp_pre_attn_bwd(s["dQ"].data_ptr(), s["dKV"].data_ptr(), s["dh"].data_ptr(), x.data_ptr(),
                                               a["mean1"].data_ptr(), a["rstd1"].data_ptr(), f("ln1_w").data_ptr(),
                                               in_w.data_ptr(), T, d, other.data_ptr(), g("ln1_w").data_ptr(),
                                               g("ln1_b").data_ptr(), hdv, st()), "rp_pre_attn_bwd")
            else:
                self._gemm(s["dQ"], in_w[:d], s["dq_in"], T, d, d, b_mn=True, residual=s["dh"])
                self._ln_bwd(s["dq_in"], x, f("ln1_w"), a["mean1"], a["rstd1"], s["tmp"], g("ln1_w"), g("ln1_b"), T)
                self._gemm(s["dKV"], in_w[d:], other, T, d, 2 * d, b_mn=True, residual=s["tmp"])
            check(self.lib.rp_ti_pos_bwd(s["dKV"].data_ptr(), 2 * d, self.B, L, d, cfg.head_dim, drop, self.seed,
                                         self.rng_counter.data_ptr(), _SITE_POS_K << 40, _SITE_POS_V << 40,
                                         G["pos_k"].data_ptr(), G["pos_v"].data_ptr(), st()), "rp_ti_pos_bwd")
            g_w, g_b = self._span(G, f"b{i}.qw", f"b{i}.vw", 3 * d), self._span(G, f"b{i}.qb", f"b{i}.vb", 1).view(-1)
            pairs = [(d_t, a["u"], g("w2"), g("b2")), (s["du"], a["y"], g("w1"), g("b1")),
                     (s["dQ"], a["q_in"], g_w[:d], g_b[:d]), (s["dKV"], x, g_w[d:], g_b[d:])]
            if self.fused_wgrad:
                self._wgrad_group(pairs)
            else:
                for dY, X, dW, _ in pairs:
                    self._wgrad(dY, X, dW, *dW.shape)
                self._colsum_multi([(dY, db) for dY, _, _, db in pairs])
            dx, other = other, dx
        check(self.lib.rp_embed_bwd(dx.data_ptr(), self.ids32.data_ptr(), self.in_pad.data_ptr(), self.B, L, d, cfg.pad_id, 0,
                                    math.sqrt(cfg.d), 1, drop, self.seed, 0, self.rng_counter.data_ptr(),
                                    G["item_emb"].data_ptr(), None, st()), "rp_embed_bwd")

    # ------------------------------------------------------------------------------------------------ inference
    def forward_last_hidden(self):
        """Eval body over the whole window -> final LayerNorm of the LAST row of every sequence -> self.hq bf16 [B, dp]."""
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


_TI_LEAF = {"ln1_w": "attention_layernorms.{i}.weight", "ln1_b": "attention_layernorms.{i}.bias",
            "qw": "attention_layers.{i}.query_w.weight", "qb": "attention_layers.{i}.query_w.bias",
            "kw": "attention_layers.{i}.key_w.weight", "kb": "attention_layers.{i}.key_w.bias",
            "vw": "attention_layers.{i}.value_w.weight", "vb": "attention_layers.{i}.value_w.bias",
            "ln2_w": "forward_layernorms.{i}.weight", "ln2_b": "forward_layernorms.{i}.bias",
            "w1": "forward_layers.{i}.conv1.weight", "b1": "forward_layers.{i}.conv1.bias",
            "w2": "forward_layers.{i}.conv2.weight", "b2": "forward_layers.{i}.conv2.bias"}
_TI_EMBED = {"item_emb": "item_emb.weight", "pos_k": "abs_pos_k_emb.pe.weight", "pos_v": "abs_pos_v_emb.pe.weight",
             "time_k": "time_matrix_k_emb.weight", "time_v": "time_matrix_v_emb.weight"}


def ti_reference_key_map(n_blocks: int) -> dict:
    """engine parameter name -> key of a reference SasRecModel(ti_modification=True) state_dict"""
    m = {k: "item_embedder." + v for k, v in _TI_EMBED.items()}
    m.update({"lnf_w": "output_normalization.last_layernorm.weight", "lnf_b": "output_normalization.last_layernorm.bias"})
    for i in range(n_blocks):
        m.update({f"b{i}.{k}": "sasrec_layers." + v.format(i=i) for k, v in _TI_LEAF.items()})
    return m


class TiSasRecCore(SasRecCore):
    """SasRecCore over TiSasRecEngine: the reference's TiSASRec state_dict keys, and the batch's timestamps staged from the
    feature tensors under ``timestamp_feature``."""

    def __init__(self, cfg: TiConfig, item_feature: str, timestamp_feature: str, device=None, seed: int = 0):
        self.timestamp_feature = timestamp_feature
        super().__init__(cfg, item_feature=item_feature, device=device, seed=seed)

    def _init_args(self) -> dict:
        return {**super()._init_args(), "timestamp_feature": self.timestamp_feature}

    def _key_map(self) -> dict:
        return ti_reference_key_map(self.cfg.n_blocks)

    def _make_engine(self, batch: int, seq_len: int, with_grad: bool):
        return TiSasRecEngine(self.cfg, batch, seq_len, self._device, seed=self._seed, with_grad=with_grad)

    def _stage_features(self, eng, feats):
        if not feats or self.timestamp_feature not in feats:
            raise ValueError(f"TiSASRec needs the timestamps of the batch (feature {self.timestamp_feature!r})")
        if eng.set_times(feats[self.timestamp_feature]):
            self._drop_graphs()   # captured launches carry the timestamps' dtype

    def state_dict(self, *args, destination=None, prefix="", keep_vars=False):  # noqa: D102
        out = super().state_dict(destination=destination, prefix=prefix)
        for k in _TI_EMBED.values():   # the tied head registers the embedder again
            if prefix + "item_embedder." + k in out:
                out[prefix + "_head._item_embedder." + k] = out[prefix + "item_embedder." + k]
        return out
