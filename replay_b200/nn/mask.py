"""Mirror of ``replay.nn.mask`` (config only: the attention kernels derive the mask from the padding mask)."""
from __future__ import annotations


class DefaultAttentionMask:
    """replay/nn/mask.py:29-51,58-80: causal mask where key j is visible to query i iff j <= i and (j is real or j == i)."""

    def __init__(self, reference_feature_name: str, num_heads: int) -> None:
        self.reference_feature_name = reference_feature_name
        self.num_heads = num_heads
