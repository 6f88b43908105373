"""TwoTower on the H100 engine (replay/nn/sequential/twotower/model.py).  The query tower is the new-path SASRec body
(SasRecEngine: embedding, SasRecTransformerLayer blocks, output LayerNorm, packed live rows); the item tower is
SwiGLUEncoder(d, 2d) (replay/nn/ffn.py:102-135) over rows of the item table both towers share:

    X1 = RMSNorm1(SwiGLU1(X0) + X0),   Y = RMSNorm2(SwiGLU2(X1) + X1)

and the head is the dot product of the query rows with Y (EmbeddingTyingHead against the tower's output).

* Full-catalog losses: X0 = E[0:|I|]; the catalog head reads Y as its table, its fp32 d_table is dY; the tower's dX0 is added
  into the item table's gradient, on top of which the query tower's embedding backward accumulates.
* Sampled losses: as the reference's get_logits(h, candidates) -> item_tower(candidates), the tower runs on the step's
  distinct candidates only (rp_tower_compact: X0 = their rows in ascending item id, labels and negatives as slot ids); the
  sampled head scores the slots, and dX0 is scattered back to the items' gradient rows.
* Inference: Y over the catalog, computed once and reused until the parameters change (``tower_table``)."""
from __future__ import annotations

import ctypes
import math
from dataclasses import dataclass

import torch

from ._lib import check
from .engine import EncoderConfig, SasRecEngine, _ru
from .engine_swiglu import SwiGLUOps

TOWER_LAYERS = ("tw0.", "tw1.")   # SwiGLUEncoder.sw1 / norm1 and sw2 / norm2
_TOWER_PARAMS = ("wg", "w1", "bg", "b1", "w2", "b2", "norm")


@dataclass
class TwoTowerConfig(EncoderConfig):
    @property
    def ffn_p(self) -> int:
        """SwiGLU hidden width (2d) as the kernels see it"""
        return _ru(2 * self.d, 128)

    def axis_sizes(self) -> dict:
        """pad kinds of EncoderConfig plus 'i' = the item tower's SwiGLU hidden axis (true entries first)"""
        return {**super().axis_sizes(), "i": 2 * self.d}

    def param_layout(self) -> list:
        d, F, vec = self.dp, self.ffn_p, ("f", None)
        shapes = ((F, d), (F, d), (F,), (F,), (d, F), (d,), (d,))
        kinds = (("i", "f"), ("i", "f"), ("i", None), ("i", None), ("f", "i"), vec, vec)
        out = super().param_layout()
        for p in TOWER_LAYERS:
            out += [(p + k, s, pk) for k, s, pk in zip(_TOWER_PARAMS, shapes, kinds)]
        return out


class TwoTowerEngine(SwiGLUOps, SasRecEngine):
    MULTI_POSITIVE_KINDS = ()   # the candidate compaction (rp_tower_compact) takes one label per position
    _KINDS = ("ce", "ce_weighted", "login_ce", "bce", "ce_sampled", "bce_sampled", "login_ce_sampled", "ce_sampled_weighted")

    def __init__(self, cfg: TwoTowerConfig, *args, **kwargs):
        self.tw = None
        self.rms_ws = None
        self.tower_valid = False   # tw["cache"] holds the tower over the catalog for the current parameters
        super().__init__(cfg, *args, **kwargs)

    def init_parameters(self, seed: int = 0):
        """SasRec's initialisation for the query tower (xavier-normal matrices of the tower too); the tower's WG / W1 biases
        at torch.nn.Linear's U(+-1/sqrt(fan_in)) (W2's bias is drawn so by the base) and its RMSNorm weights at one, as
        SwiGLUEncoder.reset_parameters leaves them."""
        super().init_parameters(seed)
        g = torch.Generator(device="cpu").manual_seed(seed + 1)
        with torch.no_grad():
            for p in TOWER_LAYERS:
                self.import_named(p + "norm", torch.ones(self.true_shape(p + "norm")))
                self.import_named(p + "bg", (torch.rand(self.true_shape(p + "bg"), generator=g) * 2 - 1) / math.sqrt(self.cfg.d))
        self.refresh_shadow()
        self.tower_valid = False

    # ------------------------------------------------------------------------------------------------ workspace
    INFER_ROWS = 65536   # rows per pass of the tower over the catalog on an engine without gradients

    def _tower_rows(self) -> int:
        """Rows of the tower's working buffers: the catalog for a full-catalog loss (its backward needs every row's
        activations), the compacted candidates' capacity for a sampled loss, a bounded chunk without gradients.  The
        catalog cache is computed in passes of this many rows."""
        n = self.cfg.n_items
        if not self.with_grad:
            return min(n, self.INFER_ROWS)
        return self.sampled["cap"] if self.sampled is not None else n

    def _alloc_tower(self) -> dict:
        """The catalog cache tw["cache"] (bf16 [|I|, dp], allocated once) and the working buffers of _tower_rows() rows,
        (re-)allocated on first use after that changes, so that selecting a sampled loss never holds catalog-sized
        buffers; the cache keeps its content.  Without gradients both layers share their scratch."""
        cfg, dev = self.cfg, self.dev
        n, d, F = cfg.n_items, cfg.dp, cfg.ffn_p
        R = self._tower_rows()
        sampled = self.with_grad and self.sampled is not None
        key = (R, self.with_grad, sampled)
        if self.tw is not None and self.tw["key"] == key:
            return self.tw
        bf = dict(device=dev, dtype=torch.bfloat16)
        cache = self.tw["cache"] if self.tw is not None else torch.zeros(n, d, **bf)
        self.tw = None   # release the old working buffers first
        layer = lambda: dict(GL=torch.zeros(R, 2 * F, **bf), U=torch.zeros(R, F, **bf), z=torch.zeros(R, d, **bf))  # noqa: E731
        first = layer()
        tw = dict(key=key, cache=cache, layers=[first, layer() if self.with_grad else first], x1=torch.zeros(R, d, **bf))
        if self.with_grad:
            tw.update(dY32=torch.zeros(R, d, device=dev, dtype=torch.float32), dY=torch.zeros(R, d, **bf),
                      dz=torch.zeros(R, d, **bf), dU=torch.zeros(R, F, **bf), dGL=torch.zeros(R, 2 * F, **bf),
                      dxa=torch.zeros(R, d, **bf), dxb=torch.zeros(R, d, **bf))
        if sampled:   # the tower's output over the slots and the compaction's buffers
            tw.update(out=torch.zeros(R, d, **bf), x0=torch.zeros(R, d, **bf),
                      n_slots=torch.zeros(1, device=dev, dtype=torch.int32),
                      item_of_slot=torch.zeros(R, device=dev, dtype=torch.int32),
                      compact_ws=torch.zeros(self.lib.rp_tower_compact_workspace(n), device=dev, dtype=torch.uint8))
        self.tw = tw
        if self.rms_ws is None:
            self.rms_ws = torch.zeros(self.lib.rp_rmsnorm_bwd_workspace(d), device=dev, dtype=torch.uint8)
        return tw

    # ------------------------------------------------------------------------------------------------ loss selection
    def set_loss(self, kind: str = "ce", **kw):
        if kind not in self._KINDS:
            raise ValueError(f"TwoTower has no {kind!r} head (supported: {', '.join(self._KINDS)})")
        super().set_loss(kind, **kw)
        sp = self.sampled
        if sp is None:
            return
        entries = {0: 1, 1: self.T, 2: self.B}[sp["mode"]] * sp["n_neg"]
        sp["cap"] = min(self.cfg.n_items, self.T + entries)
        sp["labels_r"] = torch.zeros(self.T, device=self.dev, dtype=torch.int32)
        sp["neg_r"] = torch.zeros_like(sp["neg"])

    def _sampled_desc(self):
        """The sampled head over the compacted candidates: table = the tower's output slots, ids = slot ids."""
        sp = self.sampled
        sd = super()._sampled_desc()
        sd.table, sd.labels, sd.negatives = self.tw["out"].data_ptr(), sp["labels_r"].data_ptr(), sp["neg_r"].data_ptr()
        sd.n_items = sp["cap"]
        sd.ignore_index = sp["cap"] if sp["ignore_index"] >= 0 else sp["ignore_index"]
        return sd

    def _compact(self):
        sp, tw, cfg = self.sampled, self.tw, self.cfg
        check(self.lib.rp_tower_compact(self.labels_c.data_ptr(), self.n_valid.data_ptr(), self.T, sp["neg"].data_ptr(),
                                        sp["n_neg"], sp["mode"], sp["neg"].shape[0], self.valid_idx.data_ptr(), self.L,
                                        sp["ignore_index"], cfg.n_items, self.params16["item_emb"].data_ptr(), cfg.dp,
                                        sp["cap"], tw["n_slots"].data_ptr(), tw["item_of_slot"].data_ptr(),
                                        sp["labels_r"].data_ptr(), sp["neg_r"].data_ptr(), tw["x0"].data_ptr(),
                                        tw["compact_ws"].data_ptr(), tw["compact_ws"].numel(), self._stream()),
              "rp_tower_compact")

    # ------------------------------------------------------------------------------------------------ item tower
    def tower_forward(self, x0, rows: int, out, n_rows_dev=None):
        """out[:rows] = SwiGLUEncoder(x0[:rows]) (bf16 [rows, dp]); rows <= _tower_rows().  With ``n_rows_dev`` (the
        compacted slot count) the work past that row is skipped where the backward does not need it: the GEMMs and norms
        of the forward.  The backward still covers every row: there d(out) is zero past the slots, so every row's
        gradient is exactly zero whatever finite values the skipped activations hold."""
        tw, F = self.tw, self.cfg.ffn_p
        (l0, l1), x1 = tw["layers"], tw["x1"]
        self._swiglu_block_fwd(TOWER_LAYERS[0], x0[:rows], l0["GL"], l0["U"], l0["z"], x1, rows, F, n_rows_dev)
        self._swiglu_block_fwd(TOWER_LAYERS[1], x1, l1["GL"], l1["U"], l1["z"], out, rows, F, n_rows_dev)

    def tower_backward(self, x0, rows: int):
        """From tw["dY32"][:rows] (fp32 d(out)): the tower's parameter gradients (+=) and dX0 in tw["dxb"][:rows]."""
        tw, F = self.tw, self.cfg.ffn_p
        (l0, l1), d = tw["layers"], self.cfg.dp
        check(self.lib.rp_cast_bf16(tw["dY32"].data_ptr(), tw["dY"].data_ptr(), rows * d, self._stream()), "rp_cast_bf16")
        self._swiglu_block_bwd(TOWER_LAYERS[1], tw["dY"], tw["x1"], l1["GL"], l1["U"], l1["z"], tw["dz"], tw["dU"], tw["dGL"],
                               tw["dxa"], rows, F)
        self._swiglu_block_bwd(TOWER_LAYERS[0], tw["dxa"], x0[:rows], l0["GL"], l0["U"], l0["z"], tw["dz"], tw["dU"], tw["dGL"],
                               tw["dxb"], rows, F)

    def tower_table(self) -> torch.Tensor:
        """The tower over the whole catalog, bf16 [|I|, dp]: computed (in passes of _tower_rows() rows) on the first call
        after the parameters changed.  Whoever changes the parameters clears ``tower_valid``: forward_train does, and so
        must a caller that replays a captured training step (TwoTowerCore)."""
        n, cache = self.cfg.n_items, self._alloc_tower()["cache"]
        if not self.tower_valid:
            R, x0 = self._tower_rows(), self.params16["item_emb"]
            for r0 in range(0, n, R):
                rows = min(R, n - r0)
                self.tower_forward(x0[r0:r0 + rows], rows, cache[r0:r0 + rows])
            self.tower_valid = True
        return cache

    # ------------------------------------------------------------------------------------------------ training
    def forward_train(self):
        cfg, T = self.cfg, self.T
        self.tower_valid = False
        self._alloc_tower()
        self._prepare(True)
        self._body_forward(True)
        self._final_norm_fwd(self.x[-1], self.hc, T, gather=self._target_rows(), n_rows_dev=self.n_valid)
        if self.sampled is not None:
            if self.sampled["kind"] == self.SAMPLED_KINDS["ce_sampled_weighted"]:   # weights in the head's compacted order
                torch.index_select(self.in_roww, 0, self.valid_idx, out=self.roww_c)
            self._compact()
            self.tower_forward(self.tw["x0"], self.sampled["cap"], self.tw["out"], self.tw["n_slots"])
            check(self.lib.rp_sampled_head_fwd(ctypes.byref(self._sampled_desc()), self._stream()), "rp_sampled_head_fwd")
            return self.ce.loss
        self.tower_forward(self.params16["item_emb"], cfg.n_items, self.tw["cache"])
        return self._catalog_head_fwd(self.tw["cache"])

    def _head_backward(self):
        """Loss head -> item tower -> the item table's gradient (overwritten here; the query tower's embedding backward
        accumulates on top), then the output normalization: returns d(last block's output)."""
        cfg, T, G, s, tw = self.cfg, self.T, self.grads, self.s, self.tw
        n, d = cfg.n_items, cfg.dp
        G["item_emb"].zero_()
        if self.sampled is not None:
            rows = self.sampled["cap"]
            tw["dY32"][:rows].zero_()   # the sampled head accumulates into the slots it reads
            check(self.lib.rp_sampled_head_bwd(ctypes.byref(self._sampled_desc()), s["dhc"].data_ptr(), tw["dY32"].data_ptr(),
                                               self._stream()), "rp_sampled_head_bwd")
            self.tower_backward(tw["x0"], rows)
            check(self.lib.rp_tower_scatter_rows(tw["dxb"].data_ptr(), tw["item_of_slot"].data_ptr(), tw["n_slots"].data_ptr(),
                                                 rows, d, G["item_emb"].data_ptr(), self._stream()), "rp_tower_scatter_rows")
        else:
            self._catalog_head_bwd(tw["cache"], tw["dY32"])
            self.tower_backward(self.params16["item_emb"], n)
            check(self.lib.rp_tower_scatter_rows(tw["dxb"].data_ptr(), None, None, n, d, G["item_emb"].data_ptr(),
                                                 self._stream()), "rp_tower_scatter_rows")
        dx = s["dxa"]
        dx.zero_()
        self._final_norm_bwd(s["dhc"], self.x[-1], dx, T, gather=self._target_rows(), n_rows_dev=self.n_valid)
        return dx
