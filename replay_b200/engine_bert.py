"""BERT4Rec on the H100 engine (replay/models/nn/sequential/bert4rec/model.py:10-527, lightning.py:332-351):
pre-LN transformer blocks with exact-erf GELU 4d FFN, a single <MASK> embedding, key-padding-only attention, no final
LayerNorm, and an untied ``Linear(d, |I|)`` head with bias (default) or the tied item table + ``out_bias``.  The loss is the
full-catalog CE over the positions that are real AND masked.  Same kernels as SASRec (rp_gemm / rp_attn_fwd / fused CE head),
driven by a different block program."""
from __future__ import annotations

from dataclasses import dataclass

import torch

from ._lib import check
from .engine import BaseConfig, SasRecEngine, _check_side_features, _ru


@dataclass
class BertConfig(BaseConfig):
    tying: bool = False
    pad_id: int = 0  # TensorFeatureInfo.padding_value: a VALID row for BERT4Rec (the table has |I| rows, no pad row)
    variant: str = "bert4rec"
    lnf_eps: float = 1e-5
    # num_passes_over_block: block i runs `passes` times in a row with its own weights (bert4rec/model.py:139-141); 0 applies
    # no block at all, as the reference's range(0) does
    passes: int = 1
    positional: bool = True   # enable_positional_embedding: the learned position table pos_emb [max_len, d]
    # side features summed into the item embedding (BertEmbedding, bert4rec/model.py:173-296): kinds "cat" (an Embedding of
    # cardinality rows, no padding row) and "ident" (tensor_dim == d, the values themselves); empty: item-only
    features: tuple = ()
    side_pad_rows = False

    def __post_init__(self):
        if int(self.passes) != self.passes or self.passes < 0:
            raise ValueError(f"num_passes_over_block must be a non-negative integer, got {self.passes}")
        super().__post_init__()
        if 1 + 8 * self.n_apps >= 1 << 24:   # a dropout site's offset is site << 40 in a 64-bit counter
            raise ValueError(f"{self.n_blocks} blocks x {self.passes} passes exceed the dropout sites' numbering")
        self.features = tuple(self.features)
        _check_side_features(self.features, self.d, ("cat", "ident"))

    @property
    def n_apps(self) -> int:
        """block applications of one body pass: application a runs block a // passes"""
        return self.n_blocks * self.passes

    def block_of(self, app: int) -> int:
        return app // self.passes

    # ---- the feature slots of BaseConfig; the FFN's inner axis (4d) has no head structure: its true units take the leading
    # columns and the width is rounded up to whole 128-column tiles.  The reference tutorial's hidden 300 / 4 heads
    # (head_dim 75) -> 4 slots of 128 = 512 columns, FFN 1200 -> 1280.
    @property
    def ffn(self) -> int:
        """true width of the FFN's inner axis (bert4rec/model.py:521-527: Linear(d, 4d))"""
        return 4 * self.d

    @property
    def ffn_p(self) -> int:
        """inner-axis columns as the kernels see them"""
        return _ru(self.ffn, 128)

    def axis_sizes(self) -> dict:
        """pad kinds of BaseConfig, plus 'i' = the FFN's inner axis and 'b' = the head bias (true items first, zero up to the
        128-padded length)"""
        return {**super().axis_sizes(), "i": self.ffn, "b": self.n_items}

    def param_layout(self) -> list:
        d, I, emb = self.dp, self.n_items, (None, "f")
        out = [("item_emb", (I, d), emb), ("mask_emb", (1, d), emb)]
        if self.positional:
            out.append(("pos_emb", (self.max_len, d), emb))
        for i in range(self.n_blocks):
            out += self._block_layout(i, self.ffn_p, "i")
        if not self.tying:
            out.append(("head_w", (I, d), emb))
        out.append(("head_b", (_ru(I, 128),), ("b", None)))  # padded: the kernels read the bias in 128-entry tiles
        # after every item-only parameter: an item-only model keeps its layout and seeded init
        return out + [(f"feat.{f.name}", (f.cardinality, d), emb) for f in self.features if f.kind == "cat"]


class Bert4RecEngine(SasRecEngine):
    def __init__(self, cfg: BertConfig, max_batch: int, seq_len: int, device="cuda", seed: int = 0, with_grad: bool = True):
        self.I128 = _ru(cfg.n_items, 128)
        super().__init__(cfg, max_batch, seq_len, device, seed, with_grad)

    # ------------------------------------------------------------------------------------------------ workspace
    def _check_geometry(self, seq_len: int):
        if seq_len != self.cfg.max_len:
            raise ValueError("BERT4Rec needs seq_len == max_len (bert4rec/model.py:276)")
        super()._check_geometry(seq_len)

    def _alloc_body(self):
        """BERT4Rec's block buffers: the <MASK> flags, LN outputs, packed QKV, the FFN's inner activations at its padded
        width and the backward's scratch."""
        T, d, F, dev = self.T, self.cfg.dp, self.cfg.ffn_p, self.dev
        bf = dict(device=dev, dtype=torch.bfloat16)
        self.in_tok = torch.zeros(T, device=dev, dtype=torch.bool)
        for a in self.act:
            a.update({k: torch.zeros(T, d, **bf) for k in ("xn", "y", "yn")})
            a["QKV"] = torch.zeros(T, 3 * d, **bf)
            a["pre"] = torch.zeros(T, F, **bf)
            a["u"] = torch.zeros(T, F, **bf)
        if self.with_grad:
            self.s.update({k: torch.zeros(T, d, **bf) for k in ("dz", "d_t", "dyn", "dy", "d_ao", "dxn")})
            self.s["du"] = torch.zeros(T, F, **bf)
            self.s["dQKV"] = torch.zeros(T, 3 * d, **bf)

    # ------------------------------------------------------------------------------------------------ batch
    def set_batch(self, ids, pad_mask, token_mask, labels=None):
        """[B, L] int64 ids, bool pad_mask (True = real), bool token_mask (False = <MASK>; pads are False too)."""
        B, L = ids.shape
        if L != self.L or B > self.B:
            raise ValueError(f"batch shape {tuple(ids.shape)} does not fit engine ({self.B}, {self.L})")
        n = B * L
        self.in_ids[:n].copy_(ids.reshape(-1), non_blocking=True)
        self.in_pad[:n].copy_(pad_mask.reshape(-1), non_blocking=True)
        self.in_tok[:n].copy_(token_mask.reshape(-1), non_blocking=True)
        if n < self.T:
            self.in_pad[n:].zero_()
            self.in_tok[n:].zero_()
        if labels is not None:
            self.in_labels[:n].copy_(labels.reshape(-1), non_blocking=True)
        # loss positions: real AND masked  (bert4rec/lightning.py:344-348)
        torch.logical_and(self.in_pad, torch.logical_not(self.in_tok), out=self.in_tmask)

    # ------------------------------------------------------------------------------------------------ forward
    def _body_forward(self, training: bool):
        cfg, T, d, F, L = self.cfg, self.T, self.cfg.dp, self.cfg.ffn_p, self.L
        p16, prm = self.params16, self.params
        drop = cfg.dropout if training else 0.0
        rng = self.rng_counter.data_ptr()
        pos = prm["pos_emb"].data_ptr() if cfg.positional else None
        if self.features:
            fa = self._feature_descs(False)
            check(self.lib.rp_bert_feature_embed_fwd(p16["item_emb"].data_ptr(), p16["mask_emb"].data_ptr(), pos,
                                                     self.ids32.data_ptr(), self.in_tok.data_ptr(), fa, len(fa), T, L, d,
                                                     cfg.hd_valid, drop, self.seed, 0, rng, self.x[0].data_ptr(),
                                                     self._stream()), "rp_bert_feature_embed_fwd")
        else:
            check(self.lib.rp_bert_embed_fwd(p16["item_emb"].data_ptr(), p16["mask_emb"].data_ptr(), pos,
                                             self.ids32.data_ptr(), self.in_tok.data_ptr(), T, L, d, drop, self.seed, 0, rng,
                                             self.x[0].data_ptr(), self._stream()), "rp_bert_embed_fwd")
        # application i runs block cfg.block_of(i): activations, saved statistics and dropout sites are per application,
        # weights per block
        for i in range(cfg.n_apps):
            a, x, blk = self.act[i], self.x[i], cfg.block_of(i)
            w = lambda k: p16[f"b{blk}.{k}"]  # noqa: E731
            f = lambda k: prm[f"b{blk}.{k}"]  # noqa: E731
            self._ln_fwd(x, f("ln1_w"), f("ln1_b"), 1e-5, a["xn"], a["mean1"], a["rstd1"], T)
            self._gemm(a["xn"], w("in_w"), a["QKV"], T, 3 * d, d, bias=f("in_b"))
            QKV = a["QKV"]
            self._attention_forward(i, training, (QKV, 0), (QKV, d), (QKV, 2 * d), causal=False, mask_pad_keys=True)
            # y = x + drop(O Wo^T + bo)
            self._gemm(a["O"], w("out_w"), a["y"], T, d, d, bias=f("out_b"), drop_p=drop, drop_site=self._site(i, 1), residual=x)
            self._ln_fwd(a["y"], f("ln2_w"), f("ln2_b"), 1e-5, a["yn"], a["mean2"], a["rstd2"], T)
            # u = drop(gelu(yn W1^T + b1)) ; the pre-activation is kept for gelu'
            self._gemm(a["yn"], w("w1"), a["u"], T, F, d, bias=f("b1"), act=2, drop_p=drop, drop_site=self._site(i, 2),
                       C2=a["pre"] if (training and self.with_grad) else None)
            # x_next = drop( y + drop(u W2^T + b2) )
            self._gemm(a["u"], w("w2"), self.x[i + 1], T, d, F, bias=f("b2"), drop_p=drop, drop_site=self._site(i, 3),
                       residual=a["y"], post_drop_p=drop, post_drop_site=self._site(i, 4))

    def _colsum(self, dY, db):
        """rp_colsum takes at most 1024 columns: wider bias gradients (the FFN's inner axis at d >= 300) in slices"""
        for c in range(0, dY.shape[1], 1024):
            super()._colsum(dY[:, c:c + 1024], db[c:c + 1024])

    def _head(self):
        cfg = self.cfg
        W16 = self.params16["item_emb"] if cfg.tying else self.params16["head_w"]
        return W16, self.params["head_b"]

    def set_loss(self, kind: str = "ce", **kw):
        """``"ce"`` (bert4rec/lightning.py:332-351) or ``"bce"`` (:273-305), both over the whole catalog through the biased /
        tied head.  The sampled kinds stage SASRec's buffers and are not built here."""
        if kind not in ("ce", "bce"):
            raise NotImplementedError(f"Not supported loss_type {kind!r} for BERT4Rec")
        self._loss_args = (kind, {})
        self.sampled, self.bce = None, kind == "bce"

    def forward_train(self):
        self._prepare(True)
        self._body_forward(True)
        check(self.lib.rp_gather_rows(self.x[-1].data_ptr(), self.valid_idx.data_ptr(), self.T, self.n_valid.data_ptr(),
                                      self.cfg.dp, self.hc.data_ptr(), 0, self._stream()), "rp_gather_rows")
        W16, bias = self._head()
        return self._catalog_head_fwd(W16, bias)

    # ------------------------------------------------------------------------------------------------ backward
    def backward(self):
        cfg, T, d, F, L = self.cfg, self.T, self.cfg.dp, self.cfg.ffn_p, self.L
        p16, prm, G, s = self.params16, self.params, self.grads, self.s
        drop = cfg.dropout
        st, rng = self._stream, self.rng_counter.data_ptr()
        W16, bias = self._head()
        dW = G["item_emb"] if cfg.tying else G["head_w"]
        # balanced over the whole capacity: the hint picks the split counts, and so the fp32 summation order, of the d = 512
        # and un-fused BCE gradient passes
        self._catalog_head_bwd(W16, dW, bias, G["head_b"], n_valid_hint=0)
        dx = s["dxa"]
        dx.zero_()
        check(self.lib.rp_gather_rows(s["dhc"].data_ptr(), self.valid_idx.data_ptr(), T, self.n_valid.data_ptr(), d,
                                      dx.data_ptr(), 1, st()), "rp_gather_rows")
        other = s["dxb"]

        def dbwd(src, dst, site):
            if drop > 0:
                check(self.lib.rp_dropout_bwd(src.data_ptr(), dst.data_ptr(), T, d, None, drop, self.seed, site << 40, rng, st()),
                      "rp_dropout_bwd")
                return dst
            return src

        # applications in reverse; each one ADDS its weight, bias and LayerNorm gradients into its block's (_wgrad reduces
        # into dW with +=, rp_colsum and rp_layernorm_bwd accumulate into db / dw), so a repeated block gets the sum over
        # its passes
        for i in reversed(range(cfg.n_apps)):
            a, x, blk = self.act[i], self.x[i], cfg.block_of(i)
            w = lambda k: p16[f"b{blk}.{k}"]  # noqa: E731
            f = lambda k: prm[f"b{blk}.{k}"]  # noqa: E731
            g = lambda k: G[f"b{blk}.{k}"]  # noqa: E731
            dz = dbwd(dx, s["dz"], self._site(i, 4))          # x_next = drop(z)
            d_t = dbwd(dz, s["d_t"], self._site(i, 3))        # z = y + drop(u W2^T + b2)
            self._wgrad(d_t, a["u"], g("w2"), d, F)
            self._colsum(d_t, g("b2"))
            # du_pre = (d_t W2) * dropmask/keep * gelu'(pre)
            self._gemm(d_t, w("w2"), s["du"], T, F, d, b_mn=True, drop_p=drop, drop_site=self._site(i, 2), gate=a["pre"],
                       gate_mode=1, gate_scale=1.0)
            self._wgrad(s["du"], a["yn"], g("w1"), F, d)
            self._colsum(s["du"], g("b1"))
            self._gemm(s["du"], w("w1"), s["dyn"], T, d, F, b_mn=True)
            # dy = dz (residual) + LN2'(dyn)
            self._ln_bwd(s["dyn"], a["y"], f("ln2_w"), a["mean2"], a["rstd2"], s["dy"], g("ln2_w"), g("ln2_b"), T, add_to=dz)
            d_ao = dbwd(s["dy"], s["d_ao"], self._site(i, 1))  # y = x + drop(O Wo^T + bo)
            self._wgrad(d_ao, a["O"], g("out_w"), d, d)
            self._colsum(d_ao, g("out_b"))
            self._gemm(d_ao, w("out_w"), s["d_o"], T, d, d, b_mn=True)
            # ---- attention backward, Q/K/V and dQ/dK/dV are column slices of QKV / dQKV
            QKV, dq = a["QKV"], s["dQKV"]
            self._attention_backward(i, (QKV, 0), (QKV, d), (QKV, 2 * d), (dq, 0), (dq, d), (dq, 2 * d), causal=False,
                                     mask_pad_keys=True)
            self._gemm(dq, w("in_w"), s["dxn"], T, d, 3 * d, b_mn=True)
            self._wgrad(dq, a["xn"], g("in_w"), 3 * d, d)
            self._colsum(dq, g("in_b"))
            # dx = dy (residual) + LN1'(dxn)
            self._ln_bwd(s["dxn"], x, f("ln1_w"), a["mean1"], a["rstd1"], other, g("ln1_w"), g("ln1_b"), T, add_to=s["dy"])
            dx, other = other, dx
        check(self.lib.rp_bert_embed_bwd(dx.data_ptr(), self.ids32.data_ptr(), self.in_pad.data_ptr(), self.in_tok.data_ptr(),
                                         self.B, L, d, drop, self.seed, 0, rng, G["item_emb"].data_ptr(),
                                         G["mask_emb"].data_ptr(), G["pos_emb"].data_ptr() if cfg.positional else None, st()),
              "rp_bert_embed_bwd")
        if self.features:
            fa = self._feature_descs(True)
            check(self.lib.rp_bert_feature_embed_bwd(dx.data_ptr(), self.in_pad.data_ptr(), self.in_tok.data_ptr(), fa, len(fa),
                                                     T, d, cfg.hd_valid, drop, self.seed, 0, rng, st()),
                  "rp_bert_feature_embed_bwd")

    # ------------------------------------------------------------------------------------------------ inference
    def forward_last_hidden(self):
        """Eval body -> hidden state of the LAST position (the caller has already shifted the window and put <MASK> there,
        bert4rec/dataset.py:322-345) -> self.hq bf16 [B, dp] (padded width; ``unpad_features`` gives the true d)."""
        self._prepare(False)
        self._body_forward(False)
        check(self.lib.rp_gather_rows(self.x[-1].data_ptr(), self.last_idx.data_ptr(), self.B, None, self.cfg.dp,
                                      self.hq.data_ptr(), 0, self._stream()), "rp_gather_rows")
        return self.hq

    def forward_hidden_all(self):
        """Eval-mode hidden states of every position, bf16 [T, dp] (padded width)."""
        self._prepare(False)
        self._body_forward(False)
        return self.x[-1]

    def head_for_scoring(self):
        """(W bf16 [I, dp], bias fp32 [I128]) for rp_score_topk (pairs with the padded-width hq)."""
        return self._head()
