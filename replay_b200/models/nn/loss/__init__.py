"""Loss parameters of the legacy modules with the reference's names (replay/models/nn/loss/sce.py).  They carry no
computation: ``SasRec(loss_type="SCE", sce_params=...)`` selects the fused CUDA head rp_sce_head_*."""
from __future__ import annotations

from dataclasses import dataclass


@dataclass(frozen=True)
class SCEParams:
    """Parameters of the scalable cross-entropy loss (arXiv 2409.18721), as ``replay.models.nn.loss.SCEParams``.

    :param n_buckets: number of buckets the rows and items are distributed into.
    :param bucket_size_x: hidden rows per bucket (at most 1024 and at most B * L of a batch).
    :param bucket_size_y: items per bucket (at most 1024 and at most the catalog size).
    :param mix_x: draw the buckets as a random mix of the batch's hidden rows instead of directly.
    """

    n_buckets: int
    bucket_size_x: int
    bucket_size_y: int
    mix_x: bool = False

    def _get_not_none_params(self):
        return [self.n_buckets, self.bucket_size_x, self.bucket_size_y]


def check_sce_params(sce_params: SCEParams) -> None:
    """The reference's check in ScalableCrossEntropyLoss.__init__ (sce.py:35-37)."""
    assert all(param is not None for param in sce_params._get_not_none_params()), (
        "You should define ``n_buckets``, ``bucket_size_x``, ``bucket_size_y`` when using SCE loss function.")


__all__ = ["SCEParams"]
