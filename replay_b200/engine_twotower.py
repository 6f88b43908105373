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
* Inference: Y over the catalog, computed once and reused until the parameters change (``tower_table``).
* Item features (``TwoTowerConfig.item_features``): X0 = E[i] + the sum of the reader's feature terms of item i
  (rp_item_feature_embed_fwd, over the same side tables as the query tower's), in place of the plain item rows.  Their
  backward runs right after the tower's (rp_item_feature_embed_bwd), before the query tower's embedding backward adds its
  own share into the same tables.  Over the whole catalog the categorical rows are reduced in a fixed order (bitwise
  reproducible); the sampled losses' few candidate rows use fp32 atomics, as the query tower's tables always do."""
from __future__ import annotations

import ctypes
import math
from dataclasses import dataclass

import torch

from ._lib import FEAT_MAX_NUM_COLS, ItemFeaturePlan, RpFeature, WgradPair, check
from .engine import _FEAT_KINDS, EncoderConfig, SasRecEngine, _ru
from .engine_swiglu import SwiGLUOps

TOWER_LAYERS = ("tw0.", "tw1.")   # SwiGLUEncoder.sw1 / norm1 and sw2 / norm2
_TOWER_PARAMS = ("wg", "w1", "bg", "b1", "w2", "b2", "norm")


@dataclass
class TwoTowerConfig(EncoderConfig):
    # names of the side ``features`` the item tower reads from the item features reader (ItemTower.feature_names less the
    # item id), in ``features`` order; the query tower reads every one of ``features`` from the batch
    item_features: tuple = ()

    def __post_init__(self):
        super().__post_init__()
        self.item_features = tuple(self.item_features)
        known = [f.name for f in self.features]
        unknown = [n for n in self.item_features if n not in known]
        if unknown:
            raise ValueError(f"Feature names found that embedder does not support {unknown}")
        self.item_features = tuple(n for n in known if n in self.item_features)

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
        side = [e for e in out if e[0].startswith("feat.")]   # the side tables after every item-only parameter
        out = [e for e in out if not e[0].startswith("feat.")]
        for p in TOWER_LAYERS:
            out += [(p + k, s, pk) for k, s, pk in zip(_TOWER_PARAMS, shapes, kinds)]
        return out + side


class TwoTowerEngine(SwiGLUOps, SasRecEngine):
    MULTI_POSITIVE_KINDS = ()   # the candidate compaction (rp_tower_compact) takes one label per position
    _KINDS = ("ce", "ce_weighted", "login_ce", "bce", "ce_sampled", "bce_sampled", "login_ce_sampled", "ce_sampled_weighted")

    ITEM_PLAN_CHUNK = 32   # entries per chunk of the fixed-order table-gradient reduction over the catalog

    def __init__(self, cfg: TwoTowerConfig, *args, item_values: dict | None = None, **kwargs):
        self.tw = None
        self.rms_ws = None
        self.tower_valid = False   # tw["cache"] holds the tower over the catalog for the current parameters
        self.item_in, self.item_plan = {}, None
        self.item_feats = tuple(f for f in cfg.features if f.name in cfg.item_features)
        super().__init__(cfg, *args, **kwargs)
        if self.item_feats:
            self._set_item_values(item_values or {})

    # ------------------------------------------------------------------------------------------------ item features
    def _set_item_values(self, values: dict):
        """The item features reader's columns on the device, indexed by item id (int32 ids, fp32 values, one row per
        item), and the fixed-order reduction plan of the categorical tables over the catalog, built here from the host
        columns so that no training step copies anything back to the host."""
        n, dev = self.cfg.n_items, self.dev
        host = {}
        for f in self.item_feats:
            if f.name not in values:
                raise ValueError(f"the item features reader lacks {f.name!r}")
            v = torch.as_tensor(values[f.name])
            if v.shape[0] != n or v.dim() > 2:
                raise ValueError(f"item feature {f.name!r}: expected [{n}] or [{n}, K], got {tuple(v.shape)}")
            v = v.reshape(n, -1)
            if f.kind == "cat" and v.shape[1] != 1 or not f.categorical and v.shape[1] != f.width:
                raise ValueError(f"item feature {f.name!r}: {v.shape[1]} columns per item, expected "
                                 f"{1 if f.kind == 'cat' else f.width}")
            host[f.name] = v.to(torch.int32 if f.categorical else torch.float32).cpu().contiguous()
            self.item_in[f.name] = host[f.name].to(dev)
        self.item_plan = self._build_item_plan(host)

    def _build_item_plan(self, host: dict):
        """rp_item_feature_plan of the categorical item features: every live (feature, table row, item) entry, grouped by
        table row and split into chunks of ITEM_PLAN_CHUNK entries, in ascending (feature, row, item) order (an empty plan
        without categorical features).  The reader is fixed for the model's life, so this is built once.  ``host``: the
        reader's categorical columns, int32 [n_items, K] on the host."""
        import numpy as np

        feat, row, item, w = [], [], [], []
        for k, f in enumerate(self.item_feats):
            if not f.categorical:
                continue
            v = host[f.name].numpy()
            live = (v != f.padding_value) & (v >= 0) & (v <= f.cardinality)
            cnt = live.sum(1, keepdims=True).astype(np.float32)
            wt = np.broadcast_to(np.float32(1) / np.maximum(cnt, 1) if f.kind == "bag_mean" else np.float32(1), v.shape)
            it = np.broadcast_to(np.arange(v.shape[0], dtype=np.int64)[:, None], v.shape)
            feat.append(np.full(int(live.sum()), k, np.int64))
            row.append(v[live].astype(np.int64))
            item.append(it[live])
            w.append(wt[live].astype(np.float32))
        if not feat:
            feat, row, item, w = (np.zeros(0, np.int64),) * 3 + (np.zeros(0, np.float32),)
        feat, row, item, w = (np.concatenate(a) if isinstance(a, list) else a for a in (feat, row, item, w))
        order = np.lexsort((item, row, feat))
        feat, row, item, w = feat[order], row[order], item[order], w[order]
        key = feat * (1 << 32) + row
        starts = np.flatnonzero(np.r_[True, key[1:] != key[:-1]]) if key.size else np.zeros(0, np.int64)
        ends = np.r_[starts[1:], key.size]
        chunk_off, grp_chunk = [], [0]
        for a, b in zip(starts.tolist(), ends.tolist()):
            chunk_off += list(range(a, b, self.ITEM_PLAN_CHUNK))
            grp_chunk.append(len(chunk_off))
        chunk_off.append(int(key.size))
        i32 = dict(device=self.dev, dtype=torch.int32)
        p = dict(ent_item=torch.as_tensor(item, **i32), ent_w=torch.as_tensor(w, device=self.dev),
                 chunk_off=torch.tensor(chunk_off, **i32), grp_chunk=torch.tensor(grp_chunk, **i32),
                 grp_feat=torch.as_tensor(feat[starts], **i32), grp_row=torch.as_tensor(row[starts], **i32),
                 partial=torch.zeros(max(len(chunk_off) - 1, 1), self.cfg.dp, device=self.dev))
        desc = ItemFeaturePlan()
        for k in ("ent_item", "ent_w", "chunk_off", "grp_chunk", "grp_feat", "grp_row", "partial"):
            setattr(desc, k, p[k].data_ptr())
        desc.n_chunks, desc.n_groups = len(chunk_off) - 1, len(starts)
        p["desc"] = desc
        return p

    def _item_descs(self, with_grad: bool):
        """ctypes array of rp_feature for the item tower's features (values: the reader's columns on the device)."""
        arr = (RpFeature * len(self.item_feats))()
        col = 0
        for k, f in enumerate(self.item_feats):
            a, buf = arr[k], self.item_in[f.name]
            a.kind, a.width, a.values = _FEAT_KINDS[f.kind], buf.shape[1], buf.data_ptr()
            if f.categorical:
                a.n_rows, a.padding_value = f.cardinality + 1, f.padding_value
                a.table = self.params16[f"feat.{f.name}"].data_ptr()
                a.d_table = self.grads[f"feat.{f.name}"].data_ptr() if with_grad else None
            elif f.kind == "num":
                a.table, a.bias = self.params[f"feat.{f.name}.w"].data_ptr(), self.params[f"feat.{f.name}.b"].data_ptr()
                a.val_col = col
                col += f.width
        return arr

    def _item_x0(self, out, rows: int, item0: int = 0, item_of_slot=None, n_slots=None):
        """out[:rows] = the item tower's input: item rows plus their feature terms (rp_item_feature_embed_fwd)."""
        fa = self._item_descs(False)
        check(self.lib.rp_item_feature_embed_fwd(self.params16["item_emb"].data_ptr(), fa, len(fa),
                                                 None if item_of_slot is None else item_of_slot.data_ptr(),
                                                 None if n_slots is None else n_slots.data_ptr(), rows, item0, self.cfg.dp,
                                                 self.cfg.hd_valid, out.data_ptr(), self._stream()), "rp_item_feature_embed_fwd")

    def _item_feature_bwd(self, rows: int, item_of_slot=None, n_slots=None):
        """The item tower's share of the side-feature gradients, from its dX0 (tw["dxb"][:rows]): categorical table rows by
        rp_item_feature_embed_bwd, the numerical Linears' dW = dX0^T . V by rp_wgrad_group and db = column sums of dX0."""
        tw, G, d = self.tw, self.grads, self.cfg.dp
        fa = self._item_descs(True)
        nums = [f for f in self.item_feats if f.kind == "num"]
        if nums and item_of_slot is not None:
            tw["fv"].zero_()   # rows past the slots stay zero (their dX0 is zero too)
        plan = ctypes.byref(self.item_plan["desc"]) if item_of_slot is None else None
        stage = nums and item_of_slot is not None   # the catalog's values are staged once (_alloc_tower)
        check(self.lib.rp_item_feature_embed_bwd(tw["dxb"].data_ptr(), fa, len(fa),
                                                 None if item_of_slot is None else item_of_slot.data_ptr(),
                                                 None if n_slots is None else n_slots.data_ptr(), rows, d, self.cfg.hd_valid,
                                                 plan, tw["fv"].data_ptr() if stage else None, FEAT_MAX_NUM_COLS,
                                                 self._stream()), "rp_item_feature_embed_bwd")
        if not nums:
            return
        self._wgrad_rows([(tw["dxb"], tw["fv"], tw["fdw"], tw["fdb"])], rows)
        col = 0
        for f in nums:
            G[f"feat.{f.name}.w"].add_(tw["fdw"][:, col:col + f.width])
            G[f"feat.{f.name}.b"].add_(tw["fdb"])
            col += f.width

    def _wgrad_rows(self, pairs, rows: int):
        """rp_wgrad_group over ``rows`` rows, overwriting (dW, db) (the tower's row count is not the engine's T)"""
        arr = (WgradPair * len(pairs))()
        for k, (dY, X, dW, db) in enumerate(pairs):
            arr[k].dY, arr[k].dy_ld, arr[k].n_out = dY.data_ptr(), dY.stride(0), dW.shape[0]
            arr[k].X, arr[k].x_ld, arr[k].n_in = X.data_ptr(), X.stride(0), dW.shape[1]
            arr[k].dW, arr[k].dw_ld, arr[k].db = dW.data_ptr(), dW.stride(0), db.data_ptr()
        need = self.lib.rp_wgrad_group_workspace(arr, len(pairs))
        if self._wgrad_ws is None or self._wgrad_ws.numel() < need:
            self._wgrad_ws = torch.zeros(need, device=self.dev, dtype=torch.uint8)
        check(self.lib.rp_wgrad_group(arr, len(pairs), rows, 0, self._wgrad_ws.data_ptr(), self._wgrad_ws.numel(),
                                      self._stream()), "rp_wgrad_group")

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
        if self.item_feats:   # the tower's input rows (item rows plus features) and the numerical features' staging
            tw["x0"] = torch.zeros(R, d, **bf)
            nums = [f for f in self.item_feats if f.kind == "num"]
            if self.with_grad and nums:
                tw.update(fv=torch.zeros(R, FEAT_MAX_NUM_COLS, **bf),
                          fdw=torch.zeros(d, FEAT_MAX_NUM_COLS, device=dev, dtype=torch.float32),
                          fdb=torch.zeros(d, device=dev, dtype=torch.float32))
                if not sampled:   # the catalog's numerical values never change: staged once for dW = dX0^T . V
                    col = 0
                    for f in nums:
                        tw["fv"][:, col:col + f.width] = self.item_in[f.name].to(torch.bfloat16)
                        col += f.width
        if sampled:   # the tower's output over the slots and the compaction's buffers
            tw.update(out=torch.zeros(R, d, **bf), x0=tw.get("x0", torch.zeros(R, d, **bf)),
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
                                        sp["labels_r"].data_ptr(), sp["neg_r"].data_ptr(),
                                        None if self.item_feats else tw["x0"].data_ptr(),
                                        tw["compact_ws"].data_ptr(), tw["compact_ws"].numel(), self._stream()),
              "rp_tower_compact")
        if self.item_feats:   # the slots' rows with their features (the compaction gathered no rows)
            self._item_x0(tw["x0"], sp["cap"], item_of_slot=tw["item_of_slot"], n_slots=tw["n_slots"])

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
                if self.item_feats:
                    self._item_x0(self.tw["x0"], rows, item0=r0)
                self.tower_forward(self.tw["x0"] if self.item_feats else x0[r0:r0 + rows], rows, cache[r0:r0 + rows])
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
        self.tower_forward(self._catalog_x0(), cfg.n_items, self.tw["cache"])
        return self._catalog_head_fwd(self.tw["cache"])

    def _catalog_x0(self):
        """the tower's input over the whole catalog: the item table itself, or (item features) its rows with the features
        summed in, rebuilt on every training forward"""
        if not self.item_feats:
            return self.params16["item_emb"]
        self._item_x0(self.tw["x0"], self.cfg.n_items)
        return self.tw["x0"]

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
            if self.item_feats:
                self._item_feature_bwd(rows, tw["item_of_slot"], tw["n_slots"])
        else:
            self._catalog_head_bwd(tw["cache"], tw["dY32"])
            self.tower_backward(tw["x0"] if self.item_feats else self.params16["item_emb"], n)
            check(self.lib.rp_tower_scatter_rows(tw["dxb"].data_ptr(), None, None, n, d, G["item_emb"].data_ptr(),
                                                 self._stream()), "rp_tower_scatter_rows")
            if self.item_feats:
                self._item_feature_bwd(n)
        dx = s["dxa"]
        dx.zero_()
        self._final_norm_bwd(s["dhc"], self.x[-1], dx, T, gather=self._target_rows(), n_rows_dev=self.n_valid)
        return dx
