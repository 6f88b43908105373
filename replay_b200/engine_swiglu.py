"""The SwiGLU feed-forward sub-block both the DiffTransformer body (engine_diff.py) and the TwoTower item tower
(engine_twotower.py) run, with its RMSNorm helpers (replay/nn/ffn.py:60-135):

    x' = RMSNorm(W2 (silu(WG x + bg) * (W1 x + b1)) + b2 + x)

One sub-block's parameters are named ``<prefix>wg``, ``w1``, ``bg``, ``b1``, ``w2``, ``b2`` and ``norm`` in the engine's flat
layout, with [WG; W1] and [bg; b1] adjacent so that each pair is one GEMM operand.  The hidden axis (2 * d) is padded to
``F`` columns, true entries first; the model axis is the engine's padded width ``dp``."""
from __future__ import annotations

import torch

from ._lib import check

RMS_EPS = float(torch.finfo(torch.float32).eps)   # torch.nn.RMSNorm(d) with eps=None on fp32 activations


class SwiGLUOps:
    """Mixin for SasRecEngine subclasses.  ``self.rms_ws`` is the RMSNorm backward's workspace (the subclass sizes it)."""

    def _span(self, bufs: dict, first: str, last: str, rows: int) -> torch.Tensor:
        """[rows, cols] view over the adjacent parameters ``first`` .. ``last`` of one flat buffer (the packed QKV weight,
        [WG; W1] and [bg; b1])"""
        t0, t1 = bufs[first], bufs[last]
        n = t1.data_ptr() - t0.data_ptr() + t1.numel() * t1.element_size()
        flat = t0.view(-1).as_strided((n // t0.element_size(),), (1,))
        return flat.view(rows, -1)

    def _rms_fwd(self, x, w, eps, y, n_rows, group, n_true, alpha=1.0, gather=None, n_rows_dev=None):
        check(self.lib.rp_rmsnorm_fwd(x.data_ptr(), w.data_ptr(), eps, alpha, n_rows, x.shape[1], group, n_true,
                                      None if n_rows_dev is None else n_rows_dev.data_ptr(),
                                      None if gather is None else gather.data_ptr(), y.data_ptr(), self._stream()),
              "rp_rmsnorm_fwd")

    def _rms_bwd(self, dy, x, w, eps, dx, dw, n_rows, group, n_true, alpha=1.0, gather=None, n_rows_dev=None):
        check(self.lib.rp_rmsnorm_bwd(dy.data_ptr(), x.data_ptr(), w.data_ptr(), eps, alpha, n_rows, x.shape[1], group, n_true,
                                      None if n_rows_dev is None else n_rows_dev.data_ptr(),
                                      None if gather is None else gather.data_ptr(), dx.data_ptr(), dw.data_ptr(),
                                      self.rms_ws.data_ptr(), self.rms_ws.numel(), self._stream()), "rp_rmsnorm_bwd")

    def _swiglu_block_fwd(self, p: str, x, GL, U, z, out, rows: int, F: int, n_rows_dev=None):
        """``out`` = the sub-block ``p`` applied to ``rows`` rows of ``x``; GL = [WG x + bg | W1 x + b1], U = the gate and
        z = the pre-norm sum are kept for the backward.  ``n_rows_dev`` (device int32): only the rows before it are needed;
        the GEMMs skip the 128-row tiles past it and the norm the rows past it, which keep finite values of an earlier pass."""
        p16, prm, d = self.params16, self.params, self.cfg.dp
        self._gemm(x, self._span(p16, p + "wg", p + "w1", 2 * F), GL, rows, 2 * F, d,
                   bias=self._span(prm, p + "bg", p + "b1", 1)[0], m_limit=n_rows_dev)
        check(self.lib.rp_swiglu_fwd(GL.data_ptr(), rows, F, U.data_ptr(), self._stream()), "rp_swiglu_fwd")
        self._gemm(U, p16[p + "w2"], z, rows, d, F, bias=prm[p + "b2"], residual=x, m_limit=n_rows_dev)
        self._rms_fwd(z, prm[p + "norm"], RMS_EPS, out, rows, d, self.cfg.d, n_rows_dev=n_rows_dev)

    def _swiglu_block_bwd(self, p: str, dout, x, GL, U, z, dz, dU, dGL, dx, rows: int, F: int):
        """Backward of ``_swiglu_block_fwd`` from d(out) ``dout``: ``dx`` = d(x); the sub-block's weight, bias and norm
        gradients accumulate (+=).  dz, dU and dGL are scratch."""
        p16, prm, G, d = self.params16, self.params, self.grads, self.cfg.dp
        self._rms_bwd(dout, z, prm[p + "norm"], RMS_EPS, dz, G[p + "norm"], rows, d, self.cfg.d)
        self._gemm(dz, p16[p + "w2"], dU, rows, F, d, b_mn=True)
        check(self.lib.rp_swiglu_bwd(dU.data_ptr(), GL.data_ptr(), rows, F, dGL.data_ptr(), self._stream()), "rp_swiglu_bwd")
        self._gemm(dGL, self._span(p16, p + "wg", p + "w1", 2 * F), dx, rows, d, 2 * F, b_mn=True, residual=dz)
        self._wgrad(dz, U, G[p + "w2"], d, F, rows=rows)
        self._wgrad(dGL, x, self._span(G, p + "wg", p + "w1", 2 * F), 2 * F, d, rows=rows)
        if 2 * F <= 1024:   # rp_colsum_multi sums at most 1024 columns per pair
            gates = [(dGL[:rows], self._span(G, p + "bg", p + "b1", 1)[0])]
        else:
            gates = [(dGL[:rows, :F], G[p + "bg"]), (dGL[:rows, F:], G[p + "b1"])]
        self._colsum_multi([(dz[:rows], G[p + "b2"])] + gates)
