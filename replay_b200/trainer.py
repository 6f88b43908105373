"""Data-parallel training driver for the engine: one process per GPU, CUDA-graph captured step, NCCL gradient all-reduce.

Mirrors what ``lightning.Trainer(strategy="ddp")`` does around the reference's ``training_step`` (SURVEY.md §5, §8e):
every rank runs forward/backward on its own shard of the batch, the flat fp32 gradient is sum-reduced over NVLink with
one ``ncclAllReduce`` and the optimizer step applies it scaled by 1/world_size on every rank."""
from __future__ import annotations

import os

import torch
import torch.distributed as dist

from .engine import OptimizerConfig, SasRecEngine


class Trainer:
    def __init__(self, engine: SasRecEngine, use_graph: bool = True, opt: OptimizerConfig = OptimizerConfig(),
                 one_graph: bool | None = None):
        self.engine = engine
        self.world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        self.use_graph = use_graph
        # RP_DDP_ONE_GRAPH=1 (experimental, off): capture ncclAllReduce inside the step graph.  With torch 2.11 / NCCL 2.28 the
        # capture has been seen to hang (also in "thread_local" capture-error mode), so the NCCL path runs graph (forward +
        # backward), eager all-reduce, graph (Adam).
        self.one_graph = (os.environ.get("RP_DDP_ONE_GRAPH", "0") != "0") if one_graph is None else one_graph
        if self.world > 1 and dist.get_backend() != "nccl":
            self.one_graph = False   # gloo stages CUDA tensors through the host: not capturable
        # the engine's gradient sits in a symmetric allocation: the exchange is rp_peer_allreduce, a kernel of the step graph
        self.peer = getattr(engine, "peer", None) if self.world > 1 else None
        self.opt = opt
        # the step reads only the loss and the gradients, so the body runs on packed rows where that is exact
        # (SasRecEngine.packed_eligible); RP_PACKED_BODY=0 keeps the padded rows for A/B runs
        engine.packed_body = os.environ.get("RP_PACKED_BODY", "1") != "0"
        self.launches_per_step = None
        self.invalidate()

    def invalidate(self):
        """Drop the captured graphs (the engine's workspace was re-allocated, the loss head or the optimizer changed)."""
        self._g_fb = None
        self._g_opt = None
        self._warm = 0

    # gradient exchange: one flat fp32 bucket (the CE backward finishes the big item-table gradient first)
    def _all_reduce(self):
        if self.peer is not None:
            self.peer.all_reduce(self.engine._stream())
            self.engine.lib.count += 1
        elif self.world > 1:
            dist.all_reduce(self.engine.g32, op=dist.ReduceOp.SUM)
        return 1.0 / self.world

    def _fwd_bwd(self):
        e = self.engine
        e.tick_rng()
        e.forward_train()
        e.backward()

    def _opt(self, scale):
        self.engine.optimizer_step(grad_scale=scale, opt=self.opt)

    def step(self, *batch):
        """One optimisation step on this rank's shard; ``batch`` is what the engine's ``set_batch`` takes (SASRec: ids,
        pad_mask, labels, target_mask; BERT4Rec: ids, pad_mask, token_mask, labels).  Returns the device loss tensor fp32 [2]
        (mean CE, 1/n_valid)."""
        self.engine.set_batch(*batch)
        return self.run()

    def run(self):
        """The step on the batch already staged in the engine's static input buffers (``set_batch`` / ``set_negatives``)."""
        e = self.engine
        self.opt.validate()   # before the backward accumulates a gradient that no step would consume
        if not self.use_graph:
            c0 = e.lib.count
            self._fwd_bwd()
            self._opt(self._all_reduce())
            self.launches_per_step = e.lib.count - c0
            return e.ce.loss
        if self._g_fb is None:
            if self._warm < 2:  # eager warm-up (lazy module load, func attributes, workspaces) before capture
                self._warm += 1
                c0 = e.lib.count
                self._fwd_bwd()
                self._opt(self._all_reduce())
                self.launches_per_step = e.lib.count - c0
                return e.ce.loss
            torch.cuda.synchronize()
            self._g_fb = torch.cuda.CUDAGraph()
            if self.peer is not None:   # forward / backward, the peer all-reduce kernel and Adam: one graph, one launch
                with torch.cuda.graph(self._g_fb):
                    self._fwd_bwd()
                    self._opt(self._all_reduce())
                self._g_opt = None
            elif self.world > 1 and self.one_graph:
                with torch.cuda.graph(self._g_fb, capture_error_mode="thread_local"):
                    self._fwd_bwd()
                    dist.all_reduce(e.g32, op=dist.ReduceOp.SUM)
                    self._opt(1.0 / self.world)
                self._g_opt = None
            else:
                with torch.cuda.graph(self._g_fb):
                    self._fwd_bwd()
                self._g_opt = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self._g_opt):
                    self._opt(1.0 / self.world)
            # capture does not execute: run the captured work once so this call is a real step
        self._g_fb.replay()
        if self._g_opt is not None:
            self._all_reduce()
            self._g_opt.replay()
        return e.ce.loss


def user_shard(n_users: int, rank: int, world: int) -> tuple[int, int]:
    """Contiguous, exact (no wrap-around duplicates) shard of the users for predict(): SURVEY.md §8e.  The reference's
    own DP sharding pads by wrap-around (replay/data/nn/parquet/info/partitioning.py:102-122) and can emit duplicated
    users at the tail; here every user is scored exactly once."""
    base, rem = divmod(n_users, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)
